"""Test helpers for the index filter (--filter_by_index1 / --filter_by_index2) on the text path: the C port (oracle/fastp_oracle_index.c),
the cases both test files run, the reference CLI runner and the port's text path."""
import ctypes as C
import functools
import gzip
import json
import os
import subprocess

import numpy as np

import fp_merge as M
import fp_outs as O
import fp_overlapped as V
import fp_testlib as T
from fastp_b200 import capi
from fp_testlib import ORACLE_DIR, REF_CLI, ROOT, oracle, oracle_dup_flags, oracle_fastq_decode, oracle_fastq_encode

IX_SO = os.path.join(ORACLE_DIR, "libfastp_oracle_index.so")
F2_INDEX_FILTERED = 0x01          # FP_F2_INDEX_FILTERED, in the record's last field (READ_RESULT_DTYPE "reserved")
_ix_lib = None


def ix_oracle():
    """oracle/libfastp_oracle_index.so (built by __graft_entry__.build(); built here when it is missing)."""
    global _ix_lib
    if _ix_lib is None:
        if not os.path.exists(IX_SO):
            oracle()
            subprocess.run(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", ORACLE_DIR,
                            os.path.join(ORACLE_DIR, "fastp_oracle_index.c"), "-o", IX_SO, "-L", ORACLE_DIR, "-lfastp_oracle",
                            "-Wl,-rpath,$ORIGIN"], check=True)
        lib = C.CDLL(IX_SO)
        lib.fp_oracle_index_of.restype = C.c_int64
        lib.fp_oracle_index_of.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.POINTER(C.c_int64)]
        lib.fp_oracle_index_match.restype = C.c_int
        lib.fp_oracle_index_match.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int]
        lib.fp_oracle_index_load.restype = C.c_int64
        lib.fp_oracle_index_load.argtypes = [C.c_char_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        lib.fp_oracle_index_flags.restype = None
        lib.fp_oracle_index_flags.argtypes = [C.c_void_p] * 4 + [C.c_int64, C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int, C.c_void_p]
        lib.fp_oracle_process_index.restype = C.c_int
        lib.fp_oracle_process_index.argtypes = [C.POINTER(capi.Params), C.POINTER(capi.CounterLayout), C.POINTER(capi.Batch)] + [C.c_void_p] * 6
        _ix_lib = lib
    return _ix_lib


def index_of(name, first):
    """Read::firstIndex (first) / lastIndex of a name line (bytes, '@' included)."""
    s = C.c_int64()
    n = ix_oracle().fp_oracle_index_of(name, len(name), int(first), C.byref(s))
    return name[s.value: s.value + n]


def _blob(barcodes):
    return b"".join(b + b"\0" for b in barcodes) or b"\0"


def match(barcodes, index, threshold):
    return bool(ix_oracle().fp_oracle_index_match(_blob(barcodes), len(barcodes), index, len(index), threshold))


def load_list(data):
    """Options::makeListFromFileByLine over a file's bytes -> list of barcodes (bytes), or None where the reference stops with an error."""
    lib = ix_oracle()
    need = C.c_int64()
    n = lib.fp_oracle_index_load(data, len(data), None, 0, C.byref(need))
    if n < 0:
        return None
    out = C.create_string_buffer(max(need.value, 1))
    assert lib.fp_oracle_index_load(data, len(data), out, need.value, C.byref(need)) == n
    return out.raw[:need.value].split(b"\0")[:n]


def port_flags(text1, recs1, text2, recs2, list1, list2, threshold):
    """Filter::filterByIndex for decoded records (recs2 None: single-end) -> uint8[n]."""
    n = len(recs1)
    flags = np.zeros(max(n, 1), np.uint8)
    t1 = np.frombuffer(text1 + b"\0", np.uint8).copy()
    r1 = np.ascontiguousarray(recs1) if n else np.zeros(1, capi.FASTQ_REC_DTYPE)
    if recs2 is not None:
        t2 = np.frombuffer(text2 + b"\0", np.uint8).copy(); r2 = np.ascontiguousarray(recs2) if n else np.zeros(1, capi.FASTQ_REC_DTYPE)
        a2 = (t2.ctypes.data, r2.ctypes.data)
    else:
        a2 = (None, None)
    ix_oracle().fp_oracle_index_flags(t1.ctypes.data, r1.ctypes.data, *a2, n, _blob(list1), len(list1), _blob(list2), len(list2), threshold,
                                      flags.ctypes.data)
    return flags[:n]


def port_process(p, arrs, cycles, is_dup, ix):
    """fp_oracle_process_index over a COPY of arrs -> dict like fp_testlib.run_cpu."""
    a = T.copy_arrays(arrs)
    b = capi.batch_from_arrays(a)
    paired = bool(p.paired)
    L = capi.make_layout(oracle(), paired, cycles, p.insert_size_max, p)
    n = b.n
    out1 = np.zeros(max(n, 1), capi.READ_RESULT_DTYPE); out2 = np.zeros(max(n, 1), capi.READ_RESULT_DTYPE); ov = np.zeros(max(n, 1), capi.OV_RESULT_DTYPE)
    cnt = np.zeros(L.total, np.int64)
    ixf = np.ascontiguousarray(ix, np.uint8) if n else np.zeros(1, np.uint8)
    dup = np.ascontiguousarray(is_dup, np.uint8) if is_dup is not None else None
    rc = ix_oracle().fp_oracle_process_index(C.byref(p), C.byref(L), C.byref(b), dup.ctypes.data if dup is not None else None, ixf.ctypes.data,
                                             out1.ctypes.data, out2.ctypes.data if paired else None, ov.ctypes.data if paired else None,
                                             cnt.ctypes.data)
    assert rc == 0, rc
    return {"out1": out1[:n], "out2": out2[:n], "ov": ov[:n], "counters": capi.CounterView(L, cnt), "arrs": a, "layout": L}


# ---------------- names and lists ----------------
I7 = [b"ACGTACGT", b"TTGGCCAA", b"GATTACAG", b"CCCCGGGG", b"ATATATAT", b"GGTCCCGA", b"TATAGCCT", b"CAGTCAGT"]


def _name(rng, i, side):
    """One name line of an assorted shape (see the issue's name cases); side 1 or 2."""
    k = int(rng.integers(0, 14))
    i7, i5 = I7[int(rng.integers(0, len(I7)))], I7[int(rng.integers(0, len(I7)))]
    if int(rng.integers(0, 4)) == 0:                                 # one base changed: within threshold 1
        j = int(rng.integers(0, 8)); i7 = i7[:j] + b"ACGT"[(b"ACGT".index(i7[j:j + 1]) + 1) % 4:][:1] + i7[j + 1:]
    if k <= 3:
        return b"@M:1:FC:1:%d:%d %d:N:0:%s+%s" % (i, i % 97, side, i7, i5)            # Illumina dual index
    if k <= 5:
        return b"@M:1:FC:1:%d %d:N:0:%s" % (i, side, i7)                             # single index
    if k == 6:
        return b"@M:%d %d:N:0:%sN%s+%s" % (i, side, i7[:3], i7[4:].lower(), i5)       # N and lower case
    if k == 7:
        return b"@SRR1.%d %d length=150" % (i, i)                                     # no ':' : firstIndex ""
    if k == 8:
        return [b"@", b"@a", b"@a:", b"@a:b", b"@a:bc", b"@a+b:c"][i % 6]              # 1 .. 6 bytes
    if k == 9:
        return b"@M:%d %d:N:0:%s:+" % (i, side, i7) if i % 2 else b"@M%d+A:" % i     # separators in the last two bytes
    if k == 10:
        return b"@M:%d:%s+%s+%s" % (i, i7[:4], i5[:3], i7[:2])                        # several '+' after the last ':'
    if k == 11:
        return b"@M:%d %d:N:0:%s%s" % (i, side, i7, i5)                               # index longer than the barcodes
    if k == 12:
        return b"@M:%d %d:N:0:%s" % (i, side, i7[:5])                                 # shorter
    return b"@M:%d %d:N:0:+%s" % (i, side, i5)                                        # '+' right after the ':'


def named_texts(n, seed, paired, read_len=150, eol=b"\n"):
    """FASTQ text(s) of n units of random reads with assorted names."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGTN", np.uint8)
    out = [[], []]
    for i in range(n):
        for sd in range(2 if paired else 1):
            L = int(rng.integers(read_len - 40, read_len + 1))
            s = bytes(rng.choice(acgt, L, p=[0.2475, 0.2475, 0.2475, 0.2475, 0.01]))
            q = bytes(rng.integers(33 + 2, 33 + 41, L).astype(np.uint8))
            out[sd].append(_name(rng, i, sd + 1) + eol + s + eol + b"+" + eol + q + eol)
    return b"".join(out[0]), b"".join(out[1])


def barcode_list(n, seed, lens=(8,)):
    """n barcodes: the first three from I7 cut to the given lengths, the rest random."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        L = lens[k % len(lens)]
        out.append(I7[k][:L] if k < 3 else bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), L)))
    return out


def list_file(barcodes, eol=b"\n", final_eol=True):
    return eol.join(barcodes) + (eol if final_eol and barcodes else b"")


@functools.lru_cache(maxsize=None)
def index_cases():
    """name -> (reference CLI flags, fp_params keywords, paired, text 1, text 2, row stride, -D, list file 1, list file 2, threshold); list
    files are bytes or None (option not given).  What tests/test_oracle_fastq_index.py pins to the unmodified CLI and
    tests/test_gpu_fastq_index.py runs on the device."""
    cases = {}
    one = list_file([b"ACGTACGT"]); l96 = list_file(barcode_list(96, 3, lens=(8, 6, 10, 8)))
    mixed = list_file([b"TTGGCCAA", b"GATTAC", b"", b"CCCCGGGGAA", b"TTGGCCAA", b"ATAT"])      # an empty line and a duplicate
    crlf = list_file([b"ACGTACGT", b"GATTACAG", b"CAGTCAGT"], eol=b"\r\n")
    for paired in (1, 0):
        tag = "pe" if paired else "se"
        t1, t2 = named_texts(1500, 7 + paired, paired)
        noad = ([], {}) if paired else (["-A"], dict(adapter_enabled=0))
        for thr in (-1, 0, 1, 2):
            cases[f"l96_t{thr}_{tag}"] = (noad[0], noad[1], paired, t1, t2, 160, 0, l96, l96 if paired else None, thr)
        cases[f"one_{tag}"] = (noad[0], noad[1], paired, t1, t2, 160, 0, one, None, 0)
        cases[f"mixed1_{tag}"] = (noad[0], noad[1], paired, t1, t2, 160, 0, mixed, None, 1)
        cases[f"only2_{tag}"] = (noad[0], noad[1], paired, t1, t2, 160, 0, None, crlf, 0)           # SE: on, and nothing filtered
        cases[f"empty_{tag}"] = (noad[0], noad[1], paired, t1, t2, 160, 0, b"", b"", 0)             # filter off
        cases[f"failed_{tag}"] = (noad[0] + O.FILTERS[0], dict(O.FILTERS[1], **noad[1]), paired, t1, t2, 160, 0, l96, None, 0)
        c1, c2 = named_texts(800, 11 + paired, paired, eol=b"\r\n")
        cases[f"crlf_{tag}"] = (noad[0], noad[1], paired, c1, c2, 160, 0, crlf, crlf if paired else None, 1)
    t1, t2 = named_texts(1500, 8, 1)
    cases["cfg4_full_pe"] = (V.config_flags("cfg4_full"), "cfg4_full", 1, t1, t2, 160, 0, l96, crlf, 0)
    cases["merge_pe"] = (["-m", "-c"], dict(merge_enabled=1, correction_enabled=1), 1, t1, t2, 160, 0, l96, None, 1)
    cases["mergeu_pe"] = (["-m", "--include_unmerged"], dict(merge_enabled=1, correction_enabled=1, merge_include_unmerged=1), 1, t1, t2, 160, 0,
                          l96, None, 1)
    # -D: a filtered pair and, later, its copy under another index that the filter keeps -- a duplicate all the same
    rows1, rows2 = t1.split(b"\n"), t2.split(b"\n")
    tail1, tail2 = [], []
    for u in range(0, 600, 3):
        tail1 += [b"@DUP:%d 1:N:0:GGGGAAAA+TTTTCCCC" % u] + rows1[4 * u + 1: 4 * u + 4]
        tail2 += [b"@DUP:%d 2:N:0:GGGGAAAA+TTTTCCCC" % u] + rows2[4 * u + 1: 4 * u + 4]
    d1 = t1 + b"\n".join(tail1) + b"\n"; d2 = t2 + b"\n".join(tail2) + b"\n"
    cases["dedup_pe"] = (["-D"], {}, 1, d1, d2, 160, 1, l96, l96, 0)
    s1 = t1 + b"\n".join(tail1) + b"\n"
    cases["dedup_se"] = (["-D", "-A"], dict(adapter_enabled=0), 0, s1, b"", 160, 1, l96, None, 0)
    for S, L in ((48, 40), (256, 250)):
        a1, a2 = named_texts(900, 20 + S, 1, read_len=L)
        cases[f"stride{S}_pe"] = (["-c"], dict(correction_enabled=1, seq_len1=L, seq_len2=L), 1, a1, a2, S, 0, l96, l96, 1)
    a1, _ = named_texts(900, 21, 0, read_len=500)
    cases["stride512_se"] = (["-A"], dict(adapter_enabled=0, seq_len1=500), 0, a1, b"", 512, 0, l96, None, 1)
    return cases


def case_params(name):
    """fp_params of a case: keywords over the defaults, or an option set of fp_testlib.config_params by name."""
    flags, kw, paired, t1, t2, S = index_cases()[name][:6]
    if isinstance(kw, str):
        return T.config_params(kw, paired)
    kw = dict(kw)
    kw.setdefault("seq_len1", min(150, S)); kw.setdefault("seq_len2", min(150, S))
    return capi.default_params(paired, lib=oracle(), **kw)


def case_lists(name):
    """The two barcode lists of a case as the reference loads them (None: a list file it stops on)."""
    f1, f2 = index_cases()[name][7:9]
    return (load_list(f1) if f1 else []), (load_list(f2) if f2 else [])


STREAMS = ("out1", "out2", "merged", "unpaired1", "unpaired2", "failed", "overlapped")


@functools.lru_cache(maxsize=None)
def port_text_path(name, writers=O.writers_mask(1, 1), overlapped=True):
    """C-port text path of a case: decode, duplicate filter, index flags, chain, then every stream from the units the filter kept -> dict."""
    flags, kw, paired, t1, t2, S, dedup, f1, f2, thr = index_cases()[name]
    p = case_params(name)
    l1, l2 = case_lists(name)
    d1 = oracle_fastq_decode(t1, stride=S)
    d2 = oracle_fastq_decode(t2, stride=S) if paired else None
    n = min(len(d1["recs"]), len(d2["recs"])) if paired else len(d1["recs"])
    arrs = {"seq1": d1["seq"][:n].copy(), "qual1": d1["qual"][:n].copy(), "len1": d1["len"][:n].copy()}
    if paired:
        arrs.update(seq2=d2["seq"][:n].copy(), qual2=d2["qual"][:n].copy(), len2=d2["len"][:n].copy())
    is_dup = oracle_dup_flags([arrs], paired, 3)[0][0] if dedup else None
    on = bool(l1) or bool(l2)
    ix = port_flags(t1, d1["recs"][:n], t2, d2["recs"][:n] if paired else None, l1, l2, thr) if on else np.zeros(n, np.uint8)
    merging = bool(paired and p.merge_enabled)
    cycles = 2 * S if merging else S
    res = port_process(p, arrs, cycles, is_dup, ix)
    a = res["arrs"]
    keep = np.nonzero(ix == 0)[0]
    r1, e1, s1, q1, n1 = d1["recs"][:n][keep], res["out1"][keep], a["seq1"][keep], a["qual1"][keep], d1["len"][:n][keep]
    got = {"n": n, "ix": ix, "res": res, "is_dup": is_dup, "arrs": arrs}
    if paired:
        r2, e2, s2, q2, n2 = d2["recs"][:n][keep], res["out2"][keep], a["seq2"][keep], a["qual2"][keep], d2["len"][:n][keep]
        side2 = dict(text2=t2, recs2=r2, res2=e2, seq2=s2, qual2=q2, len2=n2)
    else:
        side2 = {}
    for key, which in O.REJECTS:
        got[key] = b"" if (which != O.FAILED and not paired) else \
            O.oracle_fastq_encode_rejects(which, writers if paired else 0, p, t1, r1, e1, s1, q1, n1, stride=S, **side2)[0]
    if merging:
        for key, which in (("merged", M.FQ_OUT_MERGED), ("out1", M.FQ_OUT_R1), ("out2", M.FQ_OUT_R2)):
            got[key] = M.oracle_fastq_encode_merge(which, p.merge_include_unmerged, t1, r1, t2, r2, e1, e2, res["ov"][keep], s1, q1, s2, q2, S)[0]
    else:
        got["merged"] = b""
        got["out1"] = oracle_fastq_encode(t1, r1, e1, s1, q1, S)
        got["out2"] = oracle_fastq_encode(t2, r2, e2, s2, q2, S) if paired else b""
    got["overlapped"] = b""
    if paired and overlapped:
        sub = {k: v[keep] for k, v in arrs.items()}
        ovx = V.port_analyze(p, sub, cycles)
        got["overlapped"] = V.oracle_encode_overlapped(t1, r1, e1, e2, ovx, s1, q1, S)[0]
    return got


def summary_counts(cv, paired):
    """The -j figures the text path decides: before / after filtering reads and bases, the filtering_result counts."""
    pre = [cv.stats(T_S) for T_S in ((0, 2) if paired else (0,))]
    post = [cv.stats(T_S) for T_S in ((1, 3) if paired else (1,))]
    fr = cv.filter
    return {"before_reads": sum(s["reads"] for s in pre), "before_bases": sum(s["length_sum"] for s in pre),
            "after_reads": sum(s["reads"] for s in post), "after_bases": sum(s["length_sum"] for s in post),
            "passed": int(fr[0]), "low_quality": int(fr[20]), "too_many_N": int(fr[12]), "too_short": int(fr[16]), "too_long": int(fr[17]),
            "low_complexity": int(fr[24]), "adapter_dimer": int(fr[28])}


def json_counts(j):
    s, f = j["summary"], j["filtering_result"]
    return {"before_reads": s["before_filtering"]["total_reads"], "before_bases": s["before_filtering"]["total_bases"],
            "after_reads": s["after_filtering"]["total_reads"], "after_bases": s["after_filtering"]["total_bases"],
            "passed": f["passed_filter_reads"], "low_quality": f["low_quality_reads"], "too_many_N": f["too_many_N_reads"],
            "too_short": f["too_short_reads"], "too_long": f["too_long_reads"], "low_complexity": f.get("low_complexity_reads", 0),
            "adapter_dimer": f.get("adapter_dimer_reads", 0)}


FILES = {"out1": "o1.fq", "out2": "o2.fq", "merged": "m.fq", "unpaired1": "u1.fq", "unpaired2": "u2.fq", "failed": "f.fq", "overlapped": "ov.fq"}


def run_cli(exe, tmp_path, name, extra=(), gz=False, interleaved=False):
    """Reference CLI (exe = REF_CLI) or the mirror (exe = the mirror's path; --device_fastq added) on a case with every output stream ->
    (dict stream -> bytes, json dict or None, completed process)."""
    flags, kw, paired, t1, t2, S, dedup, f1, f2, thr = index_cases()[name]
    flags = list(flags)
    if "fasta" in flags:
        flags = [f for f in flags if f != "fasta"] + V._fasta(tmp_path / "ad.fa")
    z = ".gz" if gz else ""
    cmd = [exe, "-j", str(tmp_path / "t.json")]
    if exe == REF_CLI:
        cmd += ["-w", "1", "-h", str(tmp_path / "t.html")]
    else:
        cmd += ["--device_fastq"]
    if interleaved:
        (tmp_path / "il.fq").write_bytes(V.interleave(t1, t2))
        cmd += ["-i", str(tmp_path / "il.fq"), "--interleaved_in"]
    else:
        (tmp_path / "r1.fq").write_bytes(t1)
        cmd += ["-i", str(tmp_path / "r1.fq")]
        if paired:
            (tmp_path / "r2.fq").write_bytes(t2)
            cmd += ["-I", str(tmp_path / "r2.fq")]
    for k, f in ((1, f1), (2, f2)):
        if f is not None:
            (tmp_path / f"ix{k}.txt").write_bytes(f)
            cmd += [f"--filter_by_index{k}", str(tmp_path / f"ix{k}.txt")]
    cmd += ["--filter_by_index_threshold", str(thr)]
    if not dedup:
        cmd.append("--dont_eval_duplication")
    cmd += flags
    merging = "-m" in flags
    if "--include_unmerged" not in flags:
        cmd += ["-o", str(tmp_path / ("o1.fq" + z))] + (["-O", str(tmp_path / ("o2.fq" + z))] if paired else [])
    if merging:
        cmd += ["--merged_out", str(tmp_path / ("m.fq" + z))]
    if paired and "--include_unmerged" not in flags:
        cmd += ["--unpaired1", str(tmp_path / ("u1.fq" + z)), "--unpaired2", str(tmp_path / ("u2.fq" + z))]
    cmd += ["--failed_out", str(tmp_path / ("f.fq" + z))]
    if paired:
        cmd += ["--overlapped_out", str(tmp_path / ("ov.fq" + z))]
    cmd += list(extra)
    r = subprocess.run(cmd, capture_output=True, cwd=tmp_path)
    out = {}
    for key, f in FILES.items():
        pth = tmp_path / (f + z)
        data = pth.read_bytes() if pth.exists() else b""
        out[key] = gzip.decompress(data) if gz and data else data
    js = json.loads((tmp_path / "t.json").read_text()) if r.returncode == 0 and (tmp_path / "t.json").exists() else None
    return out, js, r


def expected_streams(name):
    """What a run with every stream writes, from the port: the unpaired writers only on paired runs without --include_unmerged."""
    flags, kw, paired = index_cases()[name][:3]
    got = port_text_path(name, O.writers_mask(1, 1) if paired and "--include_unmerged" not in flags else 0)
    return {k: got[k] for k in STREAMS}
