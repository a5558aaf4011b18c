"""Test helpers for --unpaired1 / --unpaired2 / --failed_out on the text path: the C port of the three streams
(oracle/fastp_oracle_outs.c), the cases both test files run, the reference CLI runner, and what the CLI's files must hold."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np

import edge_inputs as E
import fp_merge as M
from fastp_b200 import capi
from fp_testlib import (ORACLE_DIR, REF_CLI, ROOT, TRUSEQ_R1, TRUSEQ_R2, fastq_text, oracle, oracle_dup_flags, oracle_fastq_decode,
                        oracle_fastq_encode, run_cpu, synth_host)

OUTS_SO = os.path.join(ORACLE_DIR, "libfastp_oracle_outs.so")
_outs_lib = None
U1, U2, FAILED = capi.FP_FQ_OUT_UNPAIRED1, capi.FP_FQ_OUT_UNPAIRED2, capi.FP_FQ_OUT_FAILED
REJECTS = (("unpaired1", U1), ("unpaired2", U2), ("failed", FAILED))
# writer sets: which of --unpaired1 / --unpaired2 / --failed_out a run names
WRITER_SETS = {"f": (0, 0, 1), "u1": (1, 0, 0), "u2": (0, 1, 0), "u1u2": (1, 1, 0), "u1f": (1, 0, 1), "u2f": (0, 1, 1), "u1u2f": (1, 1, 1)}
TAGS = (b"failed_too_many_n_bases", b"failed_too_short", b"failed_too_long", b"failed_quality_filter", b"failed_low_complexity",
        b"failed_adapter_dimer", b"paired_read_is_failing")


def outs_oracle():
    """oracle/libfastp_oracle_outs.so (built by __graft_entry__.build(); built here when it is missing)."""
    global _outs_lib
    if _outs_lib is None:
        if not os.path.exists(OUTS_SO):
            subprocess.run(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", ORACLE_DIR,
                            os.path.join(ORACLE_DIR, "fastp_oracle_outs.c"), "-o", OUTS_SO], check=True)
        lib = C.CDLL(OUTS_SO)
        lib.fp_oracle_fastq_encode_rejects.restype = C.c_int64
        lib.fp_oracle_fastq_encode_rejects.argtypes = [C.c_int] * 5 + [C.c_void_p] * 12 + [C.c_int, C.c_int64, C.c_void_p, C.c_int64]
        _outs_lib = lib
    return _outs_lib


def writers_mask(u1, u2):
    return (capi.FP_FQ_W_UNPAIRED1 if u1 else 0) | (capi.FP_FQ_W_UNPAIRED2 if u2 else 0)


def oracle_fastq_encode_rejects(which, writers, p, text1, recs1, res1, seq1, qual1, len1, text2=b"", recs2=None, res2=None, seq2=None, qual2=None,
                                len2=None, stride=160, out_cap=None):
    """C port of one reject stream -> (bytes written region, total); out_cap None = all."""
    fn = outs_oracle().fp_oracle_fastq_encode_rejects
    n = len(recs1)
    paired = int(p.paired)
    side2 = (recs2, res2, seq2, qual2, len2) if paired else (np.zeros(1, np.uint8),) * 5
    keep = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in (text1, text2 if paired else b"")]
    keep += [np.ascontiguousarray(x) for x in (recs1, side2[0], res1, side2[1], seq1, qual1, len1, side2[2], side2[3], side2[4])]
    # fp_oracle_fastq_encode_rejects: text1, recs1, text2, recs2, res1, res2, seq1, qual1, len1, seq2, qual2, len2
    t1, t2, r1, r2, e1, e2, s1, q1, l1, s2, q2, l2 = [k.ctypes.data for k in keep]
    args = (which, writers, paired, int(bool(paired and p.merge_enabled)), int(p.merge_include_unmerged), t1, r1, t2, r2, e1, e2, s1, q1, l1,
            s2, q2, l2, stride, n)
    total = fn(*args, None, 0)
    assert total >= 0
    cap = int(total) if out_cap is None else out_cap
    out = np.zeros(max(cap, 1), np.uint8)
    assert fn(*args, out.ctypes.data, cap) == total
    return (out[:total].tobytes(), total) if out_cap is None else (out[:cap].tobytes(), total)


# ---------------- cases ----------------
FILTERS = (["-n", "2", "-q", "20", "-u", "20", "-l", "40", "--length_limit", "140", "-y"],
           dict(n_base_limit=2, qualified_qual=33 + 20, unqualified_percent_limit=20, length_required=40, length_limit=140, complexity_filter_enabled=1))
ADAPTERS = (["-a", TRUSEQ_R1, "--adapter_sequence_r2", TRUSEQ_R2], dict(adapter_seq_r1=TRUSEQ_R1, adapter_seq_r2=TRUSEQ_R2))


def _revcomp(s):
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


def _texts(arrs, paired, strand="+"):
    t1 = fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0", strand=strand)
    return t1, fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0", strand=strand) if paired else b""


def _filter_arrs(n, S, paired, seed):
    """Ragged lengths 0..S, quality extremes, 1 % N (edge_inputs.edge_batch), and every 13th read 1 / 17th read 2 made of runs of
    eight A and one C, which the low-complexity filter fails (2 base changes in 9 < 30 %)."""
    arrs = E.edge_batch(n, S, paired, seed, capi.default_params(paired, lib=oracle(), **FILTERS[1]))
    for sd, k in (("1", 13), ("2", 17))[: 2 if paired else 1]:
        rows = np.arange(0, n, k)
        arrs["seq" + sd][rows] = np.where(np.arange(S) % 9 == 8, ord("C"), ord("A")).astype(np.uint8)[None, :]
        E._zero_padding(arrs)
    return arrs


def _dimer_texts(n, paired, seed):
    """Every third unit an adapter dimer (0..2 insert bases, then the adapter: trimmed to <= dimer_max_len bases), the rest ordinary
    reads with the adapter at a random position or none."""
    rng = np.random.default_rng(seed)
    o1, o2 = [], []
    for i in range(n):
        ins = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), (i // 3) % 3 if i % 3 == 0 else int(rng.integers(20, 150))))
        pad1 = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), 150))
        pad2 = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), 150))
        r1 = (ins + TRUSEQ_R1.encode() + pad1)[:150]
        r2 = (_revcomp(ins) + TRUSEQ_R2.encode() + pad2)[:150]
        q1 = bytes(rng.integers(33 + 20, 33 + 41, len(r1)).astype(np.uint8)); q2 = bytes(rng.integers(33 + 20, 33 + 41, len(r2)).astype(np.uint8))
        o1.append(b"@D:%d 1:N:0\n%s\n+\n%s\n" % (i, r1, q1)); o2.append(b"@D:%d 2:N:0\n%s\n+\n%s\n" % (i, r2, q2))
    return b"".join(o1), b"".join(o2) if paired else b""


@functools.lru_cache(maxsize=None)
def fastq_outs_cases():
    """name -> (reference CLI flags, fp_params keywords, paired, text 1, text 2, row stride, -D): the cases that
    tests/test_oracle_fastq_outs.py pins to the unmodified CLI and tests/test_gpu_fastq_outs.py runs on the device."""
    cases = {}
    for paired in (1, 0):
        tag = "pe" if paired else "se"
        noad = ([], {}) if paired else (["-A"], dict(adapter_enabled=0))     # SE: no adapter detection from the data
        fl = _filter_arrs(3000, 160, paired, 21)
        t1, t2 = _texts(fl, paired)
        cases[f"filters_{tag}"] = (FILTERS[0] + noad[0], dict(FILTERS[1], **noad[1]), paired, t1, t2, 160, 0)
        d1, d2 = _dimer_texts(1500, paired, 22)
        ad = ADAPTERS if paired else (ADAPTERS[0][:2], dict(adapter_seq_r1=TRUSEQ_R1))
        cases[f"dimer_{tag}"] = (ad[0], ad[1], paired, d1, d2, 160, 0)
        # trimAndCut returns NULL for reads this short: they are written whole, as read
        tn = _filter_arrs(1500, 48, paired, 23)
        t1, t2 = _texts(tn, paired)
        cut = ["-f", "5", "-t", "7", "-F", "5", "-T", "7", "-5", "-3", "-r"]
        cases[f"trim_null_{tag}"] = (cut + noad[0], dict(trim_front1=5, trim_tail1=7, trim_front2=5, trim_tail2=7, cut_front=1, cut_tail=1,
                                                         cut_right=1, **noad[1]), paired, t1, t2, 48, 0)
        for S in (48, 160, 256):
            eb = E.edge_batch(3 * S + 500, S, paired, 24 + S, capi.default_params(paired, lib=oracle()))
            t1, t2 = _texts(eb, paired, strand="+again")
            cases[f"edge{S}_{tag}"] = (noad[0], dict(noad[1]), paired, t1, t2, S, 0)
    # -c: overlapping pairs with planted mismatches; -T 20 -l 135 fails read 2 after its bases were corrected
    rng = np.random.default_rng(25)
    cp = E.dense_correction_pairs(2000, 150, 160, 4, rng)
    t1, t2 = _texts(cp, 1)
    cases["correction_pe"] = (["-c", "-T", "20", "-l", "135"], dict(correction_enabled=1, trim_tail2=20, length_required=135), 1, t1, t2, 160, 0)
    # -D: every third pair of the first 900 again at the end
    rows = np.concatenate([np.arange(3000), np.arange(0, 900, 3)])
    fl_pe = _filter_arrs(3000, 160, 1, 21)
    dup = {k: v[rows] for k, v in fl_pe.items()}
    t1, t2 = _texts(dup, 1)
    cases["dedup_pe"] = (["-D"] + FILTERS[0], dict(FILTERS[1]), 1, t1, t2, 160, 1)
    # merging mode: only pairs that neither merged nor were taken by --include_unmerged write here
    t1, t2 = cases["filters_pe"][3:5]
    cases["merge_pe"] = (["-m"] + FILTERS[0], dict(FILTERS[1], merge_enabled=1, correction_enabled=1), 1, t1, t2, 160, 0)
    # with --include_unmerged only pairs with a dropped read are left: -f/-t on reads of 0..160 bases drop the shortest
    cut = ["-f", "3", "-t", "3", "-F", "3", "-T", "3"]
    cases["merge_iu_pe"] = (["-m", "--include_unmerged"] + cut + FILTERS[0], dict(FILTERS[1], merge_enabled=1, correction_enabled=1, merge_include_unmerged=1,
                                                                                  trim_front1=3, trim_tail1=3, trim_front2=3, trim_tail2=3), 1, t1, t2, 160, 0)
    return cases


def case_writer_sets(name):
    """Writer sets a case runs: every one for paired runs; single-end and --include_unmerged runs, where the reference ignores the unpaired
    options, --failed_out alone and all three."""
    flags, _, paired = fastq_outs_cases()[name][:3]
    if not paired or "--include_unmerged" in flags:
        return ["f", "u1u2f"]
    return list(WRITER_SETS)


def case_params(name):
    flags, kw, paired, t1, t2, S = fastq_outs_cases()[name][:6]
    L = min(150, S) if "edge" not in name else S
    return capi.default_params(paired, lib=oracle(), seq_len1=L, seq_len2=L, **kw)


def port_writers(name, wset):
    """The library's writer mask for a case's writer set: none where the reference ignores the unpaired options."""
    flags, _, paired = fastq_outs_cases()[name][:3]
    u1, u2, _ = WRITER_SETS[wset]
    if not paired or "--include_unmerged" in flags:
        return 0
    return writers_mask(u1, u2)


@functools.lru_cache(maxsize=None)
def port_text_path(name, writers):
    """C-port text path of a case: decode, (duplicate filter,) chain, then every stream -> dict."""
    flags, kw, paired, t1, t2, S, dedup = fastq_outs_cases()[name]
    p = case_params(name)
    d1 = oracle_fastq_decode(t1, stride=S)
    d2 = oracle_fastq_decode(t2, stride=S) if paired else None
    n = min(len(d1["recs"]), len(d2["recs"])) if paired else len(d1["recs"])
    arrs = {"seq1": d1["seq"][:n].copy(), "qual1": d1["qual"][:n].copy(), "len1": d1["len"][:n].copy()}
    if paired:
        arrs.update(seq2=d2["seq"][:n].copy(), qual2=d2["qual"][:n].copy(), len2=d2["len"][:n].copy())
    is_dup = oracle_dup_flags([arrs], paired, 3)[0][0] if dedup else None      # -D: accuracy level 3 (main.cpp:203-209)
    merging = bool(paired and p.merge_enabled)
    res = run_cpu("oracle", p, arrs, 2 * S if merging else S, is_dup=is_dup)
    a = res["arrs"]
    got = {"n": n, "res": res, "dec": (d1, d2), "counters": res["counters"]}
    side2 = dict(text2=t2, recs2=d2["recs"][:n], res2=res["out2"], seq2=a["seq2"], qual2=a["qual2"], len2=d2["len"][:n]) if paired else {}
    for key, which in REJECTS:
        if which != FAILED and not paired:
            got[key] = b""
            continue
        got[key] = oracle_fastq_encode_rejects(which, writers, p, t1, d1["recs"][:n], res["out1"], a["seq1"], a["qual1"], d1["len"][:n],
                                               stride=S, **side2)[0]
    if merging:
        for key, which in (("merged", M.FQ_OUT_MERGED), ("out1", M.FQ_OUT_R1), ("out2", M.FQ_OUT_R2)):
            got[key] = M.oracle_fastq_encode_merge(which, p.merge_include_unmerged, t1, d1["recs"][:n], t2, d2["recs"][:n], res["out1"], res["out2"],
                                                   res["ov"], a["seq1"], a["qual1"], a["seq2"], a["qual2"], S)[0]
    else:
        got["merged"] = b""
        got["out1"] = oracle_fastq_encode(t1, d1["recs"][:n], res["out1"], a["seq1"], a["qual1"], S)
        got["out2"] = oracle_fastq_encode(t2, d2["recs"][:n], res["out2"], a["seq2"], a["qual2"], S) if paired else b""
    return got


FILES = ("o1.fq", "o2.fq", "m.fq", "u1.fq", "u2.fq", "f.fq")


def expected_files(name, wset):
    """What the reference CLI's six files hold for a case and writer set, from the port: b"" for a file that is not written.  --unpaired2
    alone creates its file but leaves it empty (the hand-off of src/peprocessor.cpp:681-686 needs both writers)."""
    flags, _, paired = fastq_outs_cases()[name][:3]
    u1, u2, f = WRITER_SETS[wset]
    ignored = not paired or "--include_unmerged" in flags
    got = port_text_path(name, port_writers(name, wset))
    return (got["out1"], got["out2"], got["merged"], got["unpaired1"] if u1 and not ignored else b"",
            got["unpaired2"] if u1 and u2 and not ignored else b"", got["failed"] if f else b"")


def cli_output_args(d, flags, paired, wset, mname="m.fq"):
    """Output arguments of a run (reference CLI or mirror) into directory d; file names from FILES."""
    u1, u2, f = WRITER_SETS[wset]
    args = []
    if "--include_unmerged" not in flags:
        args += ["-o", str(d / "o1.fq")] + (["-O", str(d / "o2.fq")] if paired else [])
    if "-m" in flags:
        args += ["--merged_out", str(d / mname)]
    if u1:
        args += ["--unpaired1", str(d / "u1.fq")]
    if u2:
        args += ["--unpaired2", str(d / "u2.fq")]
    if f:
        args += ["--failed_out", str(d / "f.fq")]
    return args


def run_ref_cli_outs(tmp_path, name, wset):
    """The unmodified reference CLI on a case -> (six files as bytes, b"" when absent; set of files that exist; stderr)."""
    flags, _, paired, t1, t2 = fastq_outs_cases()[name][:5]
    (tmp_path / "r1.fq").write_bytes(t1)
    cmd = [REF_CLI, "-i", str(tmp_path / "r1.fq"), "-w", "1", "-j", str(tmp_path / "t.json"), "-h", str(tmp_path / "t.html")]
    if paired:
        (tmp_path / "r2.fq").write_bytes(t2)
        cmd += ["-I", str(tmp_path / "r2.fq")]
    if "-D" not in flags:
        cmd.append("--dont_eval_duplication")
    cmd += flags + cli_output_args(tmp_path, flags, paired, wset)
    r = subprocess.run(cmd, check=True, capture_output=True, cwd=tmp_path)
    files = tuple((tmp_path / f).read_bytes() if (tmp_path / f).exists() else b"" for f in FILES)
    return files, {f for f in FILES if (tmp_path / f).exists()}, r.stderr
