"""Test helpers for --overlapped_out on the text path: the C port of the stream (oracle/fastp_oracle_overlapped.c), the cases both test
files run, the reference CLI runner and the device-side callers."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np

import fp_testlib as T
from fastp_b200 import capi
from fp_testlib import (ORACLE_DIR, REF_CLI, ROOT, TRUSEQ_R1, TRUSEQ_R2, fastq_text, oracle, oracle_dup_flags, oracle_fastq_decode, run_cpu,
                        synth_host)

OV_SO = os.path.join(ORACLE_DIR, "libfastp_oracle_overlapped.so")
# fp_overlapped_result: the analysis of --overlapped_out and read 1's length when it ran
OVX_DTYPE = np.dtype([("overlapped", "u1"), ("_pad", "u1"), ("offset", "<i2"), ("overlap_len", "<i2"), ("r1_len", "<u2")])
_ov_lib = None


def ov_oracle():
    """oracle/libfastp_oracle_overlapped.so (built by __graft_entry__.build(); built here when it is missing)."""
    global _ov_lib
    if _ov_lib is None:
        if not os.path.exists(OV_SO):
            oracle()
            subprocess.run(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", ORACLE_DIR,
                            os.path.join(ORACLE_DIR, "fastp_oracle_overlapped.c"), "-o", OV_SO, "-L", ORACLE_DIR, "-lfastp_oracle",
                            "-Wl,-rpath,$ORIGIN"], check=True)
        lib = C.CDLL(OV_SO)
        lib.fp_oracle_overlapped_analyze.restype = C.c_int
        lib.fp_oracle_overlapped_analyze.argtypes = [C.POINTER(capi.Params), C.POINTER(capi.CounterLayout), C.POINTER(capi.Batch), C.c_void_p]
        lib.fp_oracle_fastq_encode_overlapped.restype = C.c_int64
        lib.fp_oracle_fastq_encode_overlapped.argtypes = [C.c_void_p] * 7 + [C.c_int, C.c_int64, C.c_void_p, C.c_int64]
        _ov_lib = lib
    return _ov_lib


def port_analyze(p, arrs, cycles):
    """fp_oracle_overlapped_analyze over a COPY of arrs -> ovx (OVX_DTYPE[n])."""
    a = T.copy_arrays(arrs)
    b = capi.batch_from_arrays(a)
    L = capi.make_layout(oracle(), True, cycles, p.insert_size_max, p)
    ovx = np.zeros(max(b.n, 1), OVX_DTYPE)
    assert ov_oracle().fp_oracle_overlapped_analyze(C.byref(p), C.byref(L), C.byref(b), ovx.ctypes.data) == 0
    return ovx[:b.n]


def oracle_encode_overlapped(text1, recs1, res1, res2, ovx, seq1, qual1, stride, out_cap=None):
    """C port of the stream -> (bytes written region, total); out_cap None = all."""
    fn = ov_oracle().fp_oracle_fastq_encode_overlapped
    n = len(recs1)
    keep = [np.frombuffer(text1, np.uint8).copy() if len(text1) else np.zeros(1, np.uint8)]
    keep += [np.ascontiguousarray(x) if n else np.zeros(16, np.uint8) for x in (recs1, res1, res2, ovx, seq1, qual1)]
    args = tuple(k.ctypes.data for k in keep) + (stride, n)
    total = fn(*args, None, 0)
    cap = int(total) if out_cap is None else out_cap
    out = np.zeros(max(cap, 1), np.uint8)
    assert fn(*args, out.ctypes.data, cap) == total
    return (out[:total].tobytes(), total) if out_cap is None else (out[:cap].tobytes(), total)


def port_text_path(p, t1, t2, stride, dedup=0):
    """C-port text path: decode, (-D: duplicate filter at level 3,) chain, the analysis, the stream -> dict(overlapped, ovx, res, arrs, dec, n)."""
    d1 = oracle_fastq_decode(t1, stride=stride); d2 = oracle_fastq_decode(t2, stride=stride)
    n = min(len(d1["recs"]), len(d2["recs"]))
    arrs = {"seq1": d1["seq"][:n].copy(), "qual1": d1["qual"][:n].copy(), "len1": d1["len"][:n].copy(),
            "seq2": d2["seq"][:n].copy(), "qual2": d2["qual"][:n].copy(), "len2": d2["len"][:n].copy()}
    is_dup = oracle_dup_flags([arrs], 1, 3)[0][0] if dedup else None       # -D: accuracy level 3 (main.cpp:203-209)
    cycles = 2 * stride if p.merge_enabled else stride
    res = run_cpu("oracle", p, arrs, cycles, is_dup=is_dup)
    ovx = port_analyze(p, arrs, cycles)
    a = res["arrs"]
    text = oracle_encode_overlapped(t1, d1["recs"][:n], res["out1"], res["out2"], ovx, a["seq1"], a["qual1"], stride)[0]
    return {"overlapped": text, "ovx": ovx, "res": res, "arrs": arrs, "dec": (d1, d2), "n": n}


# ---------------- cases ----------------
def _fasta(path):
    seqs = [TRUSEQ_R1, "CTGTCTCTTATACACATCT", TRUSEQ_R2[:20], "AAAAAAAAAAAA", "GGGGGGGGGG"]
    path.write_text("".join(f">adapter{i:02d}\n{s}\n" for i, s in enumerate(seqs)))
    return ["--adapter_fasta", str(path), "-a", TRUSEQ_R1[:12]]


# reference CLI flags of the option sets of fp_testlib.config_params (the base names; gap_ / merge_ / mergeu_ add their flags)
BASE_FLAGS = {
    "default": [], "cfg2_cut_right_polyg": ["--cut_right", "-g", "-A"], "cfg3_overlap_correction": ["-c"],
    "cfg4_full": ["--cut_right", "-g", "-x", "-c", "-a", TRUSEQ_R1, "--adapter_sequence_r2", TRUSEQ_R2],
    "cut_front_tail": ["-5", "-3", "--cut_front_window_size", "4", "--cut_front_mean_quality", "20", "--cut_tail_window_size", "5",
                       "--cut_tail_mean_quality", "18"],
    "trim_fixed": ["-f", "3", "-t", "2", "-F", "5", "-T", "1", "-b", "100", "-B", "90"],
    "all_cuts": ["-5", "-r", "-3", "-f", "2", "-T", "3", "--cut_right_window_size", "6", "--cut_right_mean_quality", "25", "-x", "-g",
                 "--poly_x_min_len", "8", "--poly_g_min_len", "12", "-a", TRUSEQ_R1, "--adapter_sequence_r2", TRUSEQ_R2],
    "filters": ["-y", "-Y", "30", "-e", "25", "-l", "40", "--length_limit", "148", "-n", "2", "-u", "20", "-q", "20"],
    "no_filters": ["-Q", "-L", "-A"], "fasta_adapters": "fasta",
    # the CLI runs one worker, thread 0; the port runs the option set as a worker other than thread 0 would: the stream is the same
    "tid_nonzero": ["-A"], "short_adapter": ["-a", "AGATCGGAAG", "--adapter_sequence_r2", "AGATCGG", "-x"],
    "tight_overlap": ["-c", "--allow_gap_overlap_trimming", "--overlap_len_require", "20", "--overlap_diff_limit", "3",
                      "--overlap_diff_percent_limit", "10", "-a", TRUSEQ_R1, "--adapter_sequence_r2", TRUSEQ_R2],
}


def config_flags(name):
    if name.startswith("gap_"):
        return config_flags(name[4:]) + ["--allow_gap_overlap_trimming"]
    if name.startswith("merge_") or name.startswith("mergeu_"):
        return config_flags(name.split("_", 1)[1]) + ["-m"] + (["--include_unmerged"] if name.startswith("mergeu_") else [])
    return list(BASE_FLAGS[name]) if BASE_FLAGS[name] != "fasta" else ["fasta"]


def _revcomp(s):
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


def planted_pairs(seed=31, L=150):
    """Pairs built from a fragment F (read 1 = F + pad, read 2 = revcomp(F) + pad, both cut to L) for each rule of the stream:
      kind 0  |F| = 2L - 31 / 2L - 30: an overlap of overlap_require + 1 bases (found) and of exactly overlap_require (not looked at)
      kind 1  a mismatch 10 bases into the overlap (rejected: limit 0 on the first 50), or 60 bases in (accepted all the same)
      kind 2  |F| < L, = L, > L: negative, zero and positive offsets
      kind 3  a mismatch 10 bases in whose read-1 base has quality 2 and read-2 base 40: -c corrects it, and the overlap becomes exact
      kind 4  read 2 of 3 bases: -F 4 drops it, so the pair writes nothing
      kind 5  bytes outside A/C/G/T/N in read 1 before the overlap (the byte path of the analysis)
    -> (text1, text2, kinds)."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    rnd = lambda k: bytes(rng.choice(acgt, k))          # noqa: E731
    o1, o2, kinds = [], [], []
    for i in range(1200):
        kind = i % 6
        q1 = bytearray(b"I" * L); q2 = bytearray(b"I" * L)
        if kind == 0:
            f = rnd(2 * L - 31 - (i // 6) % 2)
        elif kind == 2:
            f = rnd(int(rng.integers(60, 2 * L - 40)) if (i // 6) % 3 else L)
        else:
            f = rnd(int(rng.integers(L + 10, 2 * L - 80)))
        r1 = bytearray((f + rnd(L))[:L]); r2 = bytearray((_revcomp(f) + rnd(L))[:L])
        off = max(len(f) - L, 0)                          # where the overlap starts in read 1 (offset >= 0)
        if kind == 1 or kind == 3:
            k = off + (10 if kind == 3 or (i // 6) % 2 else 60)
            if k < min(len(f), L):
                r1[k] = b"ACGT"[(b"ACGT".index(r1[k]) + 1) % 4]
                if kind == 3:
                    q1[k] = ord("#")
        if kind == 4:
            r2 = r2[:3]; q2 = q2[:3]
        if kind == 5 and off >= 3:
            r1[0:3] = b"xRn"
        o1.append(b"@P:%d 1:N:0\n%s\n+\n%s\n" % (i, bytes(r1), bytes(q1)))
        o2.append(b"@P:%d 2:N:0\n%s\n+\n%s\n" % (i, bytes(r2), bytes(q2)))
        kinds.append(kind)
    return b"".join(o1), b"".join(o2), np.array(kinds)


def _texts(arrs, strand="+"):
    return (fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0", strand=strand),
            fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0", strand=strand))


@functools.lru_cache(maxsize=None)
def overlapped_cases():
    """name -> (reference CLI flags, fp_params, text 1, text 2, row stride, -D): what tests/test_oracle_fastq_overlapped.py pins to the
    unmodified CLI and tests/test_gpu_fastq_overlapped.py runs on the device."""
    import edge_inputs as E
    cases = {}
    for k, name in enumerate(T.CONFIG_NAMES + T.MERGE_CONFIG_NAMES + T.GAP_CONFIG_NAMES):
        if "all_cuts" in name:            # BASE_FLAGS has no CLI spelling that reproduces all_cuts' parameters; trim_cut below covers -5 / -3 / -f / -t
            continue
        profile = 2 if "gap" in name or name == "tight_overlap" else 1
        _, arrs = synth_host(1200, 160, 1, 0, 40 + k, profile, 150)
        cases["cfg_" + name] = (config_flags(name), T.config_params(name, 1), *_texts(arrs), 160, 0)
    t1, t2, _ = planted_pairs()
    P = lambda **kw: capi.default_params(1, lib=oracle(), seq_len1=150, seq_len2=150, **kw)    # noqa: E731
    cases["planted"] = (["-A"], P(adapter_enabled=0), t1, t2, 160, 0)
    cases["planted_c"] = (["-A", "-c"], P(adapter_enabled=0, correction_enabled=1), t1, t2, 160, 0)
    cases["planted_drop"] = (["-F", "4"], P(trim_front2=4), t1, t2, 160, 0)
    cases["planted_gap"] = (["--allow_gap_overlap_trimming", "-c"], P(allow_gap_overlap_trimming=1, correction_enabled=1), t1, t2, 160, 0)
    for req in (2, 31, 149):
        cases[f"planted_req{req}"] = (["--overlap_len_require", str(req)], P(overlap_require=req), t1, t2, 160, 0)
    # failing pairs, adapter dimers and a quality filter that fails most pairs: all written
    t1, t2 = _dimer_pairs(900, 32)
    cases["dimer_filters"] = (["-a", TRUSEQ_R1, "--adapter_sequence_r2", TRUSEQ_R2, "-q", "30", "-u", "10"],
                              P(adapter_seq_r1=TRUSEQ_R1, adapter_seq_r2=TRUSEQ_R2, qualified_qual=33 + 30, unqualified_percent_limit=10), t1, t2, 160, 0)
    # -D: every third pair of the first 600 again at the end
    _, arrs = synth_host(1200, 160, 1, 0, 33, 1, 150)
    rows = np.concatenate([np.arange(1200), np.arange(0, 600, 3)])
    t1, t2 = _texts({k: v[rows] for k, v in arrs.items()})
    cases["dedup"] = (["-D", "-c"], P(correction_enabled=1), t1, t2, 160, 1)
    cases["max_len_polyx"] = (["-b", "100", "-B", "90", "-x"], P(max_len1=100, max_len2=90, polyx_enabled=1), t1, t2, 160, 0)
    cases["merge_dedup"] = (["-m", "-D"], P(merge_enabled=1, correction_enabled=1), t1, t2, 160, 1)
    cases["trim_cut"] = (["-f", "6", "-t", "4", "-F", "3", "-T", "5", "-5", "-3"],
                         P(trim_front1=6, trim_tail1=4, trim_front2=3, trim_tail2=5, cut_front=1, cut_tail=1), t1, t2, 160, 0)
    for S in (48, 160, 256):
        eb = E.edge_batch(3 * S + 500, S, 1, 34 + S, capi.default_params(1, lib=oracle()))
        t1, t2 = _texts(eb, strand="+again")
        cases[f"edge{S}"] = (["-c"], capi.default_params(1, lib=oracle(), seq_len1=S, seq_len2=S, correction_enabled=1), t1, t2, S, 0)
    _, arrs = synth_host(1000, 256, 1, 0, 35, 1, 250)
    cases["pe250"] = (["-c"], capi.default_params(1, lib=oracle(), seq_len1=250, seq_len2=250, correction_enabled=1), *_texts(arrs), 256, 0)
    return cases


def _dimer_pairs(n, seed):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    o1, o2 = [], []
    for i in range(n):
        ins = bytes(rng.choice(acgt, (i // 3) % 3 if i % 3 == 0 else int(rng.integers(20, 150))))
        r1 = (ins + TRUSEQ_R1.encode() + bytes(rng.choice(acgt, 150)))[:150]
        r2 = (_revcomp(ins) + TRUSEQ_R2.encode() + bytes(rng.choice(acgt, 150)))[:150]
        q1 = bytes(rng.integers(33 + 10, 33 + 41, len(r1)).astype(np.uint8)); q2 = bytes(rng.integers(33 + 10, 33 + 41, len(r2)).astype(np.uint8))
        o1.append(b"@D:%d 1:N:0\n%s\n+\n%s\n" % (i, r1, q1)); o2.append(b"@D:%d 2:N:0\n%s\n+\n%s\n" % (i, r2, q2))
    return b"".join(o1), b"".join(o2)


def interleave(t1, t2):
    a, b = t1.split(b"\n"), t2.split(b"\n")
    out = []
    for k in range(0, len(a) - 1, 4):
        out += a[k:k + 4] + b[k:k + 4]
    return b"\n".join(out) + b"\n"


def run_ref_cli(tmp_path, flags, t1, t2, interleaved=False, gz=False):
    """The unmodified reference CLI with --overlapped_out -> bytes of that file (decompressed for gz)."""
    import gzip
    flags = list(flags)
    if flags == ["fasta"] or "fasta" in flags:
        flags = [f for f in flags if f != "fasta"] + _fasta(tmp_path / "ad.fa")
    cmd = [REF_CLI, "-w", "1", "-j", str(tmp_path / "t.json"), "-h", str(tmp_path / "t.html")]
    if interleaved:
        (tmp_path / "il.fq").write_bytes(interleave(t1, t2))
        cmd += ["-i", str(tmp_path / "il.fq"), "--interleaved_in"]
    else:
        (tmp_path / "r1.fq").write_bytes(t1); (tmp_path / "r2.fq").write_bytes(t2)
        cmd += ["-i", str(tmp_path / "r1.fq"), "-I", str(tmp_path / "r2.fq")]
    ov = tmp_path / ("ov.fq.gz" if gz else "ov.fq")
    cmd += ["--overlapped_out", str(ov)] + flags
    if "-D" not in flags:
        cmd.append("--dont_eval_duplication")
    if "-m" in flags:
        cmd += ["--merged_out", str(tmp_path / "m.fq")]
    if "--include_unmerged" not in flags:
        cmd += ["-o", str(tmp_path / "o1.fq"), "-O", str(tmp_path / "o2.fq")]
    subprocess.run(cmd, check=True, capture_output=True, cwd=tmp_path)
    data = ov.read_bytes()
    return gzip.decompress(data) if gz and data else data


def case_params(name):
    """fp_params of a case (the fasta option set keeps its adapters in the params; the CLI gets them from a file)."""
    return overlapped_cases()[name][1]
