"""Test helpers for interleaved pairs on the text path (--interleaved_in, --stdin, --stdout): the C port (oracle/fastp_oracle_interleaved.c),
the reference's own FastqReaderPair through the harness, the reference CLI runs both test files use, and what their outputs must hold."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np

import fp_merge as M
import fp_outs as O
from fastp_b200 import capi
from fp_testlib import ORACLE_DIR, REF_CLI, ROOT, oracle, oracle_dup_flags, oracle_fastq_encode, run_cpu

IL_SO = os.path.join(ORACLE_DIR, "libfastp_oracle_interleaved.so")
_il_lib = None


def il_oracle():
    """oracle/libfastp_oracle_interleaved.so (built by __graft_entry__.build(); built here when it is missing)."""
    global _il_lib
    if _il_lib is None:
        oracle()                                                   # libfastp_oracle.so, which the port links
        if not os.path.exists(IL_SO):
            subprocess.run(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", ORACLE_DIR,
                            os.path.join(ORACLE_DIR, "fastp_oracle_interleaved.c"), "-o", IL_SO, "-L", ORACLE_DIR, "-lfastp_oracle",
                            "-Wl,-rpath,$ORIGIN"], check=True)
        lib = C.CDLL(IL_SO)
        lib.fp_oracle_fastq_decode_interleaved.restype = C.c_int
        lib.fp_oracle_fastq_decode_interleaved.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8 + [
            C.c_int64, C.POINTER(capi.FastqInfo)]
        lib.fp_oracle_fastq_encode_interleaved.restype = C.c_int64
        lib.fp_oracle_fastq_encode_interleaved.argtypes = [C.c_void_p] * 10 + [C.c_int, C.c_int64, C.c_void_p, C.c_int64]
        _il_lib = lib
    return _il_lib


def oracle_decode_il(text, final=1, phred64=0, stride=160, capacity=None):
    """C port of fp_fastq_decode_interleaved -> {"sides": [dict(seq, qual, len, recs)] * 2, "info": dict}; capacity counts pairs."""
    cap = capacity if capacity is not None else text.count(b"@") // 2 + 2
    c1 = max(cap, 1)
    buf = np.frombuffer(text, np.uint8).copy() if len(text) else np.zeros(1, np.uint8)
    sides = [dict(seq=np.zeros((c1, stride), np.uint8), qual=np.zeros((c1, stride), np.uint8), len=np.zeros(c1, np.uint16),
                  recs=np.zeros(c1, capi.FASTQ_REC_DTYPE)) for _ in range(2)]
    info = capi.FastqInfo()
    ptrs = [sides[s][k].ctypes.data for s in range(2) for k in ("seq", "qual", "len", "recs")]
    rc = il_oracle().fp_oracle_fastq_decode_interleaved(buf.ctypes.data, len(text), final, phred64, stride, *ptrs, cap, C.byref(info))
    assert rc == 0
    n = int(info.n_records)
    return {"sides": [{k: v[:n] for k, v in sd.items()} for sd in sides], "info": {k: int(getattr(info, k)) for k, _ in capi.FastqInfo._fields_}}


def oracle_encode_il(text1, recs1, text2, recs2, res1, res2, seq1, qual1, seq2, qual2, stride, out_cap=None):
    """C port of fp_fastq_encode_interleaved -> (bytes, total)."""
    fn = il_oracle().fp_oracle_fastq_encode_interleaved
    keep = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in (text1, text2)]
    keep += [np.ascontiguousarray(x) for x in (recs1, recs2, res1, res2, seq1, qual1, seq2, qual2)]
    t1, t2, r1, r2, e1, e2, s1, q1, s2, q2 = [k.ctypes.data for k in keep]
    n = len(recs1)
    total = int(fn(t1, r1, t2, r2, e1, e2, s1, q1, s2, q2, stride, n, None, 0))
    cap = total if out_cap is None else out_cap
    out = np.zeros(max(cap, 1), np.uint8)
    assert fn(t1, r1, t2, r2, e1, e2, s1, q1, s2, q2, stride, n, out.ctypes.data, cap) == total
    return out[:min(cap, total) if out_cap is None else cap].tobytes(), total


REF_IL_SO = os.path.join(ORACLE_DIR, "_ref", "libfastp_ref_interleaved.so")
_ref_il = None


def have_ref_interleaved():
    """oracle/_ref/libfastp_ref_interleaved.so (oracle/ref_build/ref_harness_interleaved.cpp) was built."""
    return os.path.exists(REF_IL_SO)


def ref_read_interleaved(path, phred64=0):
    """The reference's FastqReaderPair(path, interleaved = true): list of pairs of (name, seq, strand, qual) byte strings."""
    global _ref_il
    if _ref_il is None:
        _ref_il = C.CDLL(REF_IL_SO)
    lib = _ref_il
    lib.fp_ref_fastq_read_interleaved.restype = C.c_int64
    lib.fp_ref_fastq_read_interleaved.argtypes = [C.c_char_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
    cap = os.path.getsize(path) * 2 + 4096
    out = np.zeros(cap, np.uint8); used = C.c_int64()
    n = lib.fp_ref_fastq_read_interleaved(str(path).encode(), phred64, out.ctypes.data, cap, C.byref(used))
    assert used.value <= cap
    pairs, o = [], 0
    for _ in range(n):
        pair = []
        for _m in range(2):
            h = out[o:o + 16].view(np.int32); o += 16
            f = []
            for k in range(4):
                f.append(out[o:o + int(h[k])].tobytes()); o += int(h[k])
            pair.append(tuple(f))
        pairs.append(tuple(pair))
    return pairs


def il_fields(text, d):
    """[(mate 1 fields, mate 2 fields)] of a decode result, comparable with ref_read_interleaved."""
    out = []
    for i in range(len(d["sides"][0]["recs"])):
        pair = []
        for sd in d["sides"]:
            r = sd["recs"][i]; n = int(sd["len"][i])
            pair.append((text[int(r["name_off"]):int(r["name_off"]) + int(r["name_len"])], sd["seq"][i, :n].tobytes(),
                         text[int(r["strand_off"]):int(r["strand_off"]) + int(r["strand_len"])], sd["qual"][i, :n].tobytes()))
        out.append(tuple(pair))
    return out


def records(text):
    """Records of a text that holds exactly four lines per record."""
    lines = text.split(b"\n")
    return [b"\n".join(lines[k:k + 4]) + b"\n" for k in range(0, len(lines) - 1, 4)]


def interleave(t1, t2):
    """Two texts of four-line records -> one text, record by record (the shorter one decides)."""
    return b"".join(a + b for a, b in zip(records(t1), records(t2)))


# ---------------- CLI runs ----------------
# run name -> (fp_outs case, input mode, output mode, writer set of fp_outs.WRITER_SETS or None)
#   input:  "files" (-i / -I), "il" (--interleaved_in file), "stdin_il" (--stdin --interleaved_in, text through a pipe), "stdin" (SE --stdin)
#   output: "files" (-o / -O / --merged_out), "stdout", "stdout_merged_out" (-m --stdout --merged_out: stdout empty), "o1_merged" (0.19.8)
RUNS = {
    "filters_se/stdout": ("filters_se", "files", "stdout", None),
    "filters_se/stdin_stdout": ("filters_se", "stdin", "stdout", None),
    "filters_pe/stdout": ("filters_pe", "files", "stdout", None),
    "filters_pe/il": ("filters_pe", "il", "files", None),
    "filters_pe/il_stdout": ("filters_pe", "il", "stdout", None),
    "filters_pe/stdin_il_stdout": ("filters_pe", "stdin_il", "stdout", None),
    "filters_pe/stdout_u1u2f": ("filters_pe", "files", "stdout", "u1u2f"),
    "filters_pe/il_stdout_f": ("filters_pe", "il", "stdout", "f"),
    "dedup_pe/il_stdout": ("dedup_pe", "il", "stdout", None),
    "merge_pe/il": ("merge_pe", "il", "files", None),
    "merge_pe/stdout": ("merge_pe", "files", "stdout", None),
    "merge_pe/il_stdout": ("merge_pe", "il", "stdout", None),
    "merge_pe/stdout_merged_out": ("merge_pe", "files", "stdout_merged_out", None),
    "merge_pe/o1_merged": ("merge_pe", "files", "o1_merged", None),
    "merge_pe/il_o1_merged": ("merge_pe", "il", "o1_merged", None),
    "merge_iu_pe/il_stdout": ("merge_iu_pe", "il", "stdout", None),
    "edge48_pe/il_stdout": ("edge48_pe", "il", "stdout", None),
    "edge160_pe/stdin_il_stdout": ("edge160_pe", "stdin_il", "stdout", None),
    "edge256_pe/il": ("edge256_pe", "il", "files", None),
}
FILES = ("stdout", "o1.fq", "o2.fq", "m.fq", "u1.fq", "u2.fq", "f.fq")


def run_inputs(run):
    """(texts of the input files / pipe, paired) of a run: text 1, text 2 (b"" when interleaved or single-end)."""
    name, inp = RUNS[run][:2]
    _, _, paired, t1, t2 = O.fastq_outs_cases()[name][:5]
    if inp in ("il", "stdin_il"):
        return interleave(t1, t2), b"", paired
    return t1, t2, paired


def cli_args(d, run, input_paths):
    """Arguments of a run (reference CLI or mirror) after the program name, reading from input_paths (None = through --stdin)."""
    name, inp, outm, wset = RUNS[run]
    flags, _, paired = O.fastq_outs_cases()[name][:3]
    args = []
    if inp in ("stdin", "stdin_il"):
        args += ["--stdin"]
    else:
        args += ["-i", input_paths[0]] + (["-I", input_paths[1]] if inp == "files" and paired else [])
    if inp in ("il", "stdin_il"):
        args += ["--interleaved_in"]
    args += flags
    iu = "--include_unmerged" in flags
    if outm == "files":
        args += ([] if iu else ["-o", str(d / "o1.fq")] + (["-O", str(d / "o2.fq")] if paired else [])) + (["--merged_out", str(d / "m.fq")] if "-m" in flags else [])
    elif outm == "stdout":
        args += ["--stdout"]
    elif outm == "stdout_merged_out":
        args += ["--stdout", "--merged_out", str(d / "m.fq")]
    elif outm == "o1_merged":
        args += ["-o", str(d / "o1.fq")]
    if wset:
        u1, u2, f = O.WRITER_SETS[wset]
        args += (["--unpaired1", str(d / "u1.fq")] if u1 else []) + (["--unpaired2", str(d / "u2.fq")] if u2 else []) + (["--failed_out", str(d / "f.fq")] if f else [])
    return args


def run_cli(exe, tmp_path, run, extra=()):
    """One CLI (the reference's or the mirror) on a run -> (seven outputs as bytes: stdout then FILES[1:], b"" when absent; stderr)."""
    name, inp = RUNS[run][:2]
    flags = O.fastq_outs_cases()[name][0]
    t1, t2, paired = run_inputs(run)
    (tmp_path / "r1.fq").write_bytes(t1)
    paths = [str(tmp_path / "r1.fq")]
    if t2:
        (tmp_path / "r2.fq").write_bytes(t2)
        paths.append(str(tmp_path / "r2.fq"))
    cmd = [exe] + cli_args(tmp_path, run, paths) + list(extra)
    if "-D" not in flags:
        cmd.append("--dont_eval_duplication")
    r = subprocess.run(cmd, input=t1 if inp.startswith("stdin") else None, capture_output=True, cwd=tmp_path, timeout=600)
    assert r.returncode == 0, r.stderr[-600:]
    return (r.stdout,) + tuple((tmp_path / f).read_bytes() if (tmp_path / f).exists() else b"" for f in FILES[1:]), r.stderr


def run_ref_cli(tmp_path, run):
    return run_cli(REF_CLI, tmp_path, run, ["-w", "1", "-j", str(tmp_path / "t.json"), "-h", str(tmp_path / "t.html")])


@functools.lru_cache(maxsize=None)
def port_streams(run):
    """C-port text path of a run from its own input: interleaved inputs through the interleaved decode port; every stream the run's
    options produce, plus "stdout_il" (the interleaved encode port of the pairs)."""
    name, inp, outm, wset = RUNS[run]
    flags, kw, paired, _, _, S, dedup = O.fastq_outs_cases()[name]
    p = O.case_params(name)
    t1, t2, _ = run_inputs(run)
    if inp in ("il", "stdin_il"):
        d = oracle_decode_il(t1, stride=S)
        sd1, sd2 = d["sides"]
        text1 = text2 = t1
    else:
        from fp_testlib import oracle_fastq_decode
        sd1 = oracle_fastq_decode(t1, stride=S)
        sd2 = oracle_fastq_decode(t2, stride=S) if paired else None
        text1, text2 = t1, t2
    n = min(len(sd1["recs"]), len(sd2["recs"])) if paired else len(sd1["recs"])
    arrs = {"seq1": sd1["seq"][:n].copy(), "qual1": sd1["qual"][:n].copy(), "len1": sd1["len"][:n].copy()}
    if paired:
        arrs.update(seq2=sd2["seq"][:n].copy(), qual2=sd2["qual"][:n].copy(), len2=sd2["len"][:n].copy())
    is_dup = oracle_dup_flags([arrs], paired, 3)[0][0] if dedup else None
    merging = bool(paired and p.merge_enabled)
    res = run_cpu("oracle", p, arrs, 2 * S if merging else S, is_dup=is_dup)
    a = res["arrs"]
    got = {"n": n}
    writers = O.port_writers(name, wset) if wset else 0
    side2 = dict(text2=text2, recs2=sd2["recs"][:n], res2=res["out2"], seq2=a["seq2"], qual2=a["qual2"], len2=sd2["len"][:n]) if paired else {}
    for key, which in O.REJECTS:
        got[key] = b"" if (which != O.FAILED and not paired) else O.oracle_fastq_encode_rejects(
            which, writers, p, text1, sd1["recs"][:n], res["out1"], a["seq1"], a["qual1"], sd1["len"][:n], stride=S, **side2)[0]
    if merging:
        for key, which in (("merged", M.FQ_OUT_MERGED), ("out1", M.FQ_OUT_R1), ("out2", M.FQ_OUT_R2)):
            got[key] = M.oracle_fastq_encode_merge(which, p.merge_include_unmerged, text1, sd1["recs"][:n], text2, sd2["recs"][:n], res["out1"],
                                                   res["out2"], res["ov"], a["seq1"], a["qual1"], a["seq2"], a["qual2"], S)[0]
        got["stdout_il"] = None
    else:
        got["merged"] = b""
        got["out1"] = oracle_fastq_encode(text1, sd1["recs"][:n], res["out1"], a["seq1"], a["qual1"], S)
        got["out2"] = oracle_fastq_encode(text2, sd2["recs"][:n], res["out2"], a["seq2"], a["qual2"], S) if paired else b""
        got["stdout_il"] = oracle_encode_il(text1, sd1["recs"][:n], text2, sd2["recs"][:n], res["out1"], res["out2"], a["seq1"], a["qual1"],
                                            a["seq2"], a["qual2"], S)[0] if paired else None
    return got


def expected_outputs(run):
    """What a CLI run's stdout and six files hold, from the port (b"" for an output that is not written)."""
    name, inp, outm, wset = RUNS[run]
    flags, _, paired = O.fastq_outs_cases()[name][:3]
    g = port_streams(run)
    merging = "-m" in flags
    iu = "--include_unmerged" in flags
    stdout = o1 = o2 = m = b""
    if outm == "files":
        o1, o2 = (b"", b"") if iu else (g["out1"], g["out2"])
        m = g["merged"]
    elif outm == "stdout":
        stdout = g["merged"] if merging else (g["stdout_il"] if paired else g["out1"])
    elif outm == "stdout_merged_out":
        m = g["merged"]
    elif outm == "o1_merged":
        o1 = g["merged"]
    u1 = u2 = f = b""
    if wset:
        wu1, wu2, wf = O.WRITER_SETS[wset]
        ignored = not paired or iu
        u1 = g["unpaired1"] if wu1 and not ignored else b""
        u2 = g["unpaired2"] if wu1 and wu2 and not ignored else b""
        f = g["failed"] if wf else b""
    return (stdout, o1, o2, m, u1, u2, f)
