"""Test helpers for merging mode on the text path (--merge / --include_unmerged / --merged_out): the C port of the three output
streams (oracle/fastp_oracle_merge.c), the cases both test files run, the reference CLI runner, and the device-side callers."""
import ctypes as C
import os
import subprocess

import numpy as np

from fastp_b200 import capi
from fp_testlib import (ORACLE_DIR, REF_CLI, ROOT, TRUSEQ_R1, TRUSEQ_R2, fastq_text, oracle, oracle_dup_flags, oracle_fastq_decode, run_cpu,
                        synth_host)

MERGE_SO = os.path.join(ORACLE_DIR, "libfastp_oracle_merge.so")
_merge_lib = None


def build_merge_oracle():
    subprocess.run(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", ORACLE_DIR,
                    os.path.join(ORACLE_DIR, "fastp_oracle_merge.c"), "-o", MERGE_SO], check=True)


def merge_oracle():
    """oracle/libfastp_oracle_merge.so (built by __graft_entry__.build(); built here when it is missing)."""
    global _merge_lib
    if _merge_lib is None:
        if not os.path.exists(MERGE_SO):
            build_merge_oracle()
        lib = C.CDLL(MERGE_SO)
        lib.fp_oracle_fastq_encode_merge.restype = C.c_int64
        lib.fp_oracle_fastq_encode_merge.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_int64, C.c_void_p, C.c_int64]
        lib.fp_oracle_merge_complement.restype = C.c_uint8
        lib.fp_oracle_merge_complement.argtypes = [C.c_uint8]
        _merge_lib = lib
    return _merge_lib


# ---------------- merging mode on the text path (--merge / --include_unmerged / --merged_out) ----------------
FQ_OUT_MERGED, FQ_OUT_R1, FQ_OUT_R2 = 0, 1, 2               # fp_fastq_encode_merge `which`


def oracle_fastq_encode_merge(which, include_unmerged, text1, recs1, text2, recs2, res1, res2, ov, seq1, qual1, seq2, qual2, stride, out_cap=None):
    """C port of the three merging-mode output streams; out_cap: bytes the output may take (None = all) -> (bytes written region, total)."""
    fn = merge_oracle().fp_oracle_fastq_encode_merge
    n = len(recs1)
    keep = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in (text1, text2)]
    keep += [np.ascontiguousarray(x) for x in (recs1, recs2, res1, res2, ov, seq1, qual1, seq2, qual2)]
    t1, t2, r1, r2, o1, o2, ovv, s1, q1, s2, q2 = [k.ctypes.data for k in keep]
    args = (which, int(include_unmerged), t1, r1, t2, r2, o1, o2, ovv, s1, q1, s2, q2, stride, n)
    total = fn(*args, None, 0)
    assert total >= 0
    cap = int(total) if out_cap is None else out_cap
    out = np.zeros(max(cap, 1), np.uint8)
    assert fn(*args, out.ctypes.data, cap) == total
    return (out[:total].tobytes(), total) if out_cap is None else (out[:cap].tobytes(), total)


def oracle_merge_text_path(p, t1, t2, stride, dup_level=0, dedup=0):
    """C-port text path in merging mode: decode both texts, (duplicate filter,) chain, the three streams.
    -> dict(merged, out1, out2, counters, plus the intermediate arrays for callers that feed the device encoder)."""
    d1 = oracle_fastq_decode(t1, stride=stride); d2 = oracle_fastq_decode(t2, stride=stride)
    n = min(len(d1["recs"]), len(d2["recs"]))
    arrs = {"seq1": d1["seq"][:n].copy(), "qual1": d1["qual"][:n].copy(), "len1": d1["len"][:n].copy(),
            "seq2": d2["seq"][:n].copy(), "qual2": d2["qual"][:n].copy(), "len2": d2["len"][:n].copy()}
    is_dup = None
    if dup_level:
        flags = oracle_dup_flags([arrs], 1, dup_level)[0][0]
        is_dup = flags if dedup else None
    res = run_cpu("oracle", p, arrs, 2 * stride, is_dup=is_dup)
    a = res["arrs"]
    streams = {}
    for key, which in (("merged", FQ_OUT_MERGED), ("out1", FQ_OUT_R1), ("out2", FQ_OUT_R2)):
        streams[key] = oracle_fastq_encode_merge(which, p.merge_include_unmerged, t1, d1["recs"][:n], t2, d2["recs"][:n], res["out1"], res["out2"], res["ov"],
                                                 a["seq1"], a["qual1"], a["seq2"], a["qual2"], stride)[0]
    streams.update(counters=res["counters"], res=res, dec=(d1, d2), n=n)
    return streams


def _revcomp_text(s):
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


def merge_pairs_text(frags, L1, L2, seed, name=lambda i: f"@M:{i} 1:N:0", name2=lambda i: f"@M:{i} 2:N:0", strand=lambda i: "+", qlo=35, qhi=74):
    """Error-free pairs cut from random fragments: read 1 = the fragment's first L1 bases, read 2 = the reverse complement of its last
    L2 (each capped at the fragment), so the pair overlaps whenever L1 + L2 - len(fragment) reaches the required overlap; a fragment
    shorter than the reads gives offset <= 0 (len2 = 0)."""
    rng = np.random.default_rng(seed)
    o1, o2 = [], []
    for i, F in enumerate(frags):
        frag = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), F))
        a = frag[:min(L1(i), F)]; b = _revcomp_text(frag)[:min(L2(i), F)]
        q1 = bytes(rng.integers(qlo, qhi, len(a)).astype(np.uint8)); q2 = bytes(rng.integers(qlo, qhi, len(b)).astype(np.uint8))
        o1.append(name(i).encode() + b"\n" + a + b"\n" + strand(i).encode() + b"\n" + q1 + b"\n")
        o2.append(name2(i).encode() + b"\n" + b + b"\n" + strand(i).encode() + b"\n" + q2 + b"\n")
    return b"".join(o1), b"".join(o2)


def fastq_merge_cases():
    """name -> (reference CLI flags, fp_params keywords, text 1, text 2, row stride, -D): the merging-mode text-path cases that
    tests/test_oracle_fastq_merge.py pins to the unmodified CLI and tests/test_gpu_fastq_merge.py runs on the device."""
    full = (["--cut_right", "-g", "-x", "-c", "-a", TRUSEQ_R1, "--adapter_sequence_r2", TRUSEQ_R2],
            dict(cut_right=1, polyg_enabled=1, polyx_enabled=1, adapter_seq_r1=TRUSEQ_R1, adapter_seq_r2=TRUSEQ_R2))
    _, arrs = synth_host(3000, 160, 1, 0, 31, 1, 150)
    s1 = fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0"); s2 = fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0")
    cases = {
        "default": ([], {}, s1, s2, 160, 0),
        "full": (full[0], full[1], s1, s2, 160, 0),
        "include_unmerged": (["--include_unmerged"], dict(merge_include_unmerged=1), s1, s2, 160, 0),
        "include_unmerged_full": (["--include_unmerged"] + full[0], dict(merge_include_unmerged=1, **full[1]), s1, s2, 160, 0),
    }
    # -D: every third pair of the first 900 again at the end (merged duplicates are still written, unmerged ones are not)
    rows = np.concatenate([np.arange(3000), np.arange(0, 900, 3)])
    dup = {k: v[rows] for k, v in arrs.items()}
    d1 = fastq_text(dup["seq1"], dup["qual1"], dup["len1"], "1:N:0"); d2 = fastq_text(dup["seq2"], dup["qual2"], dup["len2"], "2:N:0")
    cases["dedup"] = (["-D"], {}, d1, d2, 160, 1)
    cases["dedup_include_unmerged"] = (["-D", "--include_unmerged"], dict(merge_include_unmerged=1), d1, d2, 160, 1)
    # len1 / len2 across 9|10 and 99|100, offset <= 0 (fragment shorter than the reads: len2 = 0), one- to three-digit suffixes
    n = 1200
    frags = [40 + (i * 7) % 161 for i in range(n)]
    e1, e2 = merge_pairs_text(frags, lambda i: 31 + (i * 13) % 121, lambda i: 31 + (i * 29) % 119, 5)
    cases["digit_borders"] = ([], {}, e1, e2, 160, 0)
    cases["digit_borders_include_unmerged"] = (["--include_unmerged"], dict(merge_include_unmerged=1), e1, e2, 160, 0)
    # read 1 covers the whole fragment but for 0..12 bases: len2 = 0..12; read 2 longer than read 1's remainder by design
    frags = [60 + i % 90 for i in range(600)]
    f1, f2 = merge_pairs_text(frags, lambda i: frags[i] - i % 13, lambda i: 35 + i % 100, 6)
    cases["short_tail"] = ([], {}, f1, f2, 160, 0)
    # names with a comment field, strand lines that repeat the name: the suffix goes on both lines
    g1, g2 = merge_pairs_text([50 + (i * 11) % 200 for i in range(500)], lambda i: 40 + (i * 3) % 110, lambda i: 40 + (i * 5) % 110, 7,
                              name=lambda i: f"@inst:7:FC:1:{i}:9 1:N:0:ACGT extra words", name2=lambda i: f"@inst:7:FC:1:{i}:9 2:N:0:ACGT",
                              strand=lambda i: "+" if i % 3 == 0 else f"+inst:7:FC:1:{i}:9" if i % 3 == 1 else "+ ")
    cases["named_strand"] = ([], {}, g1, g2, 160, 0)
    cases["named_strand_include_unmerged"] = (["--include_unmerged"], dict(merge_include_unmerged=1), g1, g2, 160, 0)
    # 2 x 250 at stride 256: merged reads up to 470 bases
    _, big = synth_host(1500, 256, 1, 0, 41, 1, 250)
    cases["pe250"] = ([], {}, fastq_text(big["seq1"], big["qual1"], big["len1"], "1:N:0"), fastq_text(big["seq2"], big["qual2"], big["len2"], "2:N:0"), 256, 0)
    return cases


def merge_case_params(kw, L):
    """fp_params of a merging-mode case: --merge forces correction (options.cpp:120-121)."""
    return capi.default_params(1, lib=oracle(), seq_len1=L, seq_len2=L, merge_enabled=1, correction_enabled=1, **kw)


def run_ref_cli_merge(tmp_path, flags, t1, t2):
    """The unmodified reference CLI in merging mode -> (merged, out1, out2, parsed JSON); out1 / out2 are b"" with --include_unmerged."""
    import json
    (tmp_path / "r1.fq").write_bytes(t1); (tmp_path / "r2.fq").write_bytes(t2)
    cmd = [REF_CLI, "-i", str(tmp_path / "r1.fq"), "-I", str(tmp_path / "r2.fq"), "-m", "--merged_out", str(tmp_path / "m.fq"), "-w", "1",
           "-j", str(tmp_path / "t.json"), "-h", str(tmp_path / "t.html")] + list(flags)
    if "-D" not in flags:
        cmd.append("--dont_eval_duplication")
    if "--include_unmerged" not in flags:
        cmd += ["-o", str(tmp_path / "o1.fq"), "-O", str(tmp_path / "o2.fq")]
    subprocess.run(cmd, check=True, capture_output=True, cwd=tmp_path)
    rd = lambda f: (tmp_path / f).read_bytes() if (tmp_path / f).exists() else b""     # noqa: E731
    return rd("m.fq"), rd("o1.fq"), rd("o2.fq"), json.load(open(tmp_path / "t.json"))


# ---------------- device side (needs cuda:0) ----------------
GUARD = 0xA5

def gpu_chain_on_decoded(ctx, dec1, dec2, n):
    """fp_process_pe over the rows two gpu_fastq_decode calls left on the device -> dict of device tensors (res1, res2, ov) and host
    copies of everything the merged-stream encoder reads (records, overlap results, rows after correction)."""
    import torch
    lib = ctx.lib
    (_, s1, q1, l1, _), (_, s2, q2, l2, _) = dec1["dev"], dec2["dev"]
    b = capi.Batch()
    b.n, b.stride = n, ctx.stride
    b.seq1, b.qual1, b.len1, b.seq2, b.qual2, b.len2 = s1.data_ptr(), q1.data_ptr(), l1.data_ptr(), s2.data_ptr(), q2.data_ptr(), l2.data_ptr()
    m = max(n, 1)
    d = {"res1": torch.zeros(m * 16, dtype=torch.uint8, device="cuda:0"), "res2": torch.zeros(m * 16, dtype=torch.uint8, device="cuda:0"),
         "ov": torch.zeros(m * 8, dtype=torch.uint8, device="cuda:0")}
    capi.check(lib.fp_process_pe(ctx.h, C.byref(b), d["res1"].data_ptr(), d["res2"].data_ptr(), d["ov"].data_ptr(), None, 0, None, None), lib)
    torch.cuda.synchronize()
    S = ctx.stride
    host = {"res1": d["res1"].cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy(), "res2": d["res2"].cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy(),
            "ov": d["ov"].cpu().numpy().view(capi.OV_RESULT_DTYPE)[:n].copy()}
    for k, t in (("seq1", s1), ("qual1", q1), ("seq2", s2), ("qual2", q2)):
        host[k] = t.cpu().numpy()[:m * S].reshape(m, S)[:n].copy()
    d["host"] = host
    return d


def gpu_fastq_encode_merge(ctx, which, dec1, dec2, chain, n, out_cap=None):
    """fp_fastq_encode_merge for one stream.  out_cap None: size query (NULL buffer, cap 0) then a buffer of exactly that size -> bytes.
    Otherwise -> (rc, first out_cap bytes, total, guard_ok) with 64 guard bytes behind the buffer."""
    import torch
    lib = ctx.lib
    (t1, s1, q1, _, r1), (t2, s2, q2, _, r2) = dec1["dev"], dec2["dev"]

    def call(buf, cap, total):
        return lib.fp_fastq_encode_merge(ctx.h, which, t1.data_ptr(), r1.data_ptr(), t2.data_ptr(), r2.data_ptr(), chain["res1"].data_ptr(), chain["res2"].data_ptr(),
                                         chain["ov"].data_ptr(), s1.data_ptr(), q1.data_ptr(), s2.data_ptr(), q2.data_ptr(), n, buf, cap, C.byref(total))
    if out_cap is None:
        total = C.c_int64()
        capi.check(call(None, 0, total), lib)
        out_cap = total.value
        exact = True
    else:
        exact = False
    d_out = torch.full((out_cap + 64,), GUARD, dtype=torch.uint8, device="cuda:0")
    t2v = C.c_int64()
    rc = call(d_out.data_ptr(), out_cap, t2v)
    h = d_out.cpu().numpy()
    guard_ok = bool((h[out_cap:] == GUARD).all())
    if exact:
        capi.check(rc, lib)
        assert t2v.value == out_cap and guard_ok
        return h[:out_cap].tobytes()
    return rc, h[:out_cap].tobytes(), t2v.value, guard_ok


def gpu_fastq_process_host_merge(ctx, text1, text2, final=1, phred64=0, out_cap=None, entry="fp_fastq_process_host_merge"):
    """fp_fastq_process_host_merge on host buffers -> dict(rc, out1, out2, merged, n, consumed, guard_ok).  out_cap = (cap1, cap2, capm).
    entry="fp_fastq_process_host" calls the two-stream entry point with the same buffers instead (for its refusal)."""
    lib = ctx.lib
    texts = [text1, text2]
    caps = list(out_cap) if out_cap is not None else [len(text1) + 64, len(text2) + 64, len(text1) + len(text2) + len(text1) // 4 + 256]
    bufs = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in texts]
    outs = [np.full(c + 64, GUARD, np.uint8) for c in caps]
    nout = [C.c_int64(), C.c_int64(), C.c_int64()]; cons = [C.c_int64(), C.c_int64()]; nu = C.c_int64()
    infos = [capi.FastqInfo(), capi.FastqInfo()]
    head = (ctx.h, bufs[0].ctypes.data, len(text1), bufs[1].ctypes.data, len(text2), final, phred64,
            outs[0].ctypes.data, caps[0], C.byref(nout[0]), outs[1].ctypes.data, caps[1], C.byref(nout[1]))
    tail = (C.byref(nu), C.byref(cons[0]), C.byref(cons[1]), C.byref(infos[0]), C.byref(infos[1]))
    if entry == "fp_fastq_process_host":
        rc = lib.fp_fastq_process_host(*head, *tail)
    else:
        rc = lib.fp_fastq_process_host_merge(*head, outs[2].ctypes.data, caps[2], C.byref(nout[2]), *tail)
    res = {"rc": rc, "n": nu.value, "consumed": (cons[0].value, cons[1].value),
           "guard_ok": all(bool((o[c:] == GUARD).all()) for o, c in zip(outs, caps)),
           "untouched": all(bool((o == GUARD).all()) for o in outs)}
    for key, o, c, nb in zip(("out1", "out2", "merged"), outs, caps, nout):
        res[key] = o[:min(nb.value, c)].tobytes() if rc == 0 else b""
    return res
