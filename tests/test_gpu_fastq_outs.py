"""-m gpu: --unpaired1 / --unpaired2 / --failed_out on the device text path.  fp_fastq_encode_rejects against its C port on the records
the device chain itself produced; fp_fastq_process_host_outs and fastp_gpu_cli --device_fastq against the port's whole text path, the
committed digests of the UNMODIFIED reference CLI's files (tests/golden/fastq_outs_cli_digests.json) and, where oracle/_ref/fastp_ref
travelled along, that CLI itself.  The port is pinned to the CLI on the CPU by tests/test_oracle_fastq_outs.py."""
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import fp_outs as O
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "fastp_b200", "host", "fastp_gpu_cli")
DIGESTS = os.path.join(ROOT, "tests", "golden", "fastq_outs_cli_digests.json")
CASES = O.fastq_outs_cases()
GUARD = 0xA5
STREAM_KEYS = ("merged", "out1", "out2", "unpaired1", "unpaired2", "failed")       # FP_FQ_OUT_* order


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def cycles_of(p, S):
    return 2 * S if (p.paired and p.merge_enabled) else S


def device_chain(gpu, ctx, t1, t2, n):
    """decode -> fp_process_se / _pe on the device -> dict with the decodes, device records and host copies of what the encoders read."""
    import torch
    lib, S, paired = ctx.lib, ctx.stride, bool(ctx.params.paired)
    d1 = gpu.gpu_fastq_decode(ctx, t1, capacity=n)
    d2 = gpu.gpu_fastq_decode(ctx, t2, capacity=n) if paired else None
    assert d1["info"]["n_records"] == n and (not paired or d2["info"]["n_records"] == n)
    m = max(n, 1)
    res = [torch.zeros(m * 16, dtype=torch.uint8, device="cuda:0") for _ in range(2)]
    b = capi.Batch()
    b.n, b.stride = n, S
    _, s1, q1, l1, _ = d1["dev"]
    b.seq1, b.qual1, b.len1 = s1.data_ptr(), q1.data_ptr(), l1.data_ptr()
    if paired:
        _, s2, q2, l2, _ = d2["dev"]
        b.seq2, b.qual2, b.len2 = s2.data_ptr(), q2.data_ptr(), l2.data_ptr()
        ov = torch.zeros(m * 8, dtype=torch.uint8, device="cuda:0")
        capi.check(lib.fp_process_pe(ctx.h, C.byref(b), res[0].data_ptr(), res[1].data_ptr(), ov.data_ptr(), None, 0, None, None), lib)
    else:
        capi.check(lib.fp_process_se(ctx.h, C.byref(b), res[0].data_ptr(), None), lib)
    torch.cuda.synchronize()
    host = {}
    for sd, d in (("1", d1), ("2", d2))[: 2 if paired else 1]:
        host["res" + sd] = res[int(sd) - 1].cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy()
        host["seq" + sd] = d["dev"][1].cpu().numpy()[:m * S].reshape(m, S)[:n].copy()
        host["qual" + sd] = d["dev"][2].cpu().numpy()[:m * S].reshape(m, S)[:n].copy()
    return {"d1": d1, "d2": d2, "res": res, "host": host, "n": n}


def gpu_encode_rejects(ctx, ch, which, writers, out_cap=None):
    """fp_fastq_encode_rejects for one stream.  out_cap None: size query, then a buffer of exactly that size -> bytes.
    Otherwise -> (rc, first out_cap bytes, total, guard_ok) with 64 guard bytes behind the buffer."""
    import torch
    lib, paired = ctx.lib, bool(ctx.params.paired)
    t1, s1, q1, l1, r1 = ch["d1"]["dev"]
    t2, s2, q2, l2, r2 = ch["d2"]["dev"] if paired else (None,) * 5
    ptr = lambda t: t.data_ptr() if t is not None else None          # noqa: E731

    def call(buf, cap, total):
        return lib.fp_fastq_encode_rejects(ctx.h, which, writers, ptr(t1), ptr(r1), ptr(t2), ptr(r2), ptr(ch["res"][0]), ptr(ch["res"][1]) if paired else None,
                                           ptr(s1), ptr(q1), ptr(l1), ptr(s2), ptr(q2), ptr(l2), ch["n"], buf, cap, C.byref(total))
    exact = out_cap is None
    if exact:
        total = C.c_int64()
        capi.check(call(None, 0, total), lib)
        out_cap = total.value
    d_out = torch.full((out_cap + 64,), GUARD, dtype=torch.uint8, device="cuda:0")
    tv = C.c_int64()
    rc = call(d_out.data_ptr(), out_cap, tv)
    h = d_out.cpu().numpy()
    guard_ok = bool((h[out_cap:] == GUARD).all())
    if exact:
        capi.check(rc, lib)
        assert tv.value == out_cap and guard_ok
        return h[:out_cap].tobytes()
    return rc, h[:out_cap].tobytes(), tv.value, guard_ok


def port_on_device_records(ctx, ch, t1, t2, which, writers, n=None):
    h, d1, d2 = ch["host"], ch["d1"], ch["d2"]
    n = ch["n"] if n is None else n
    side2 = dict(text2=t2, recs2=d2["recs"][:n], res2=h["res2"][:n], seq2=h["seq2"][:n], qual2=h["qual2"][:n], len2=d2["len"][:n]) if ctx.params.paired else {}
    return O.oracle_fastq_encode_rejects(which, writers, ctx.params, t1, d1["recs"][:n], h["res1"][:n], h["seq1"][:n], h["qual1"][:n], d1["len"][:n],
                                         stride=ctx.stride, **side2)[0]


def writer_masks(p):
    return [0, 1, 2, 3] if p.paired and not (p.merge_enabled and p.merge_include_unmerged) else [0]


def check_all_streams(ctx, ch, t1, t2, what):
    for which in (O.U1, O.U2, O.FAILED) if ctx.params.paired else (O.FAILED,):
        for w in writer_masks(ctx.params):
            got = gpu_encode_rejects(ctx, ch, which, w)
            want = port_on_device_records(ctx, ch, t1, t2, which, w)
            assert got == want, (what, which, w, len(got), len(want))


@pytest.mark.parametrize("name", list(CASES))
def test_encode_equals_port(gpu, name):
    """Every case, every stream x writer set: the device encoder equals the port on the device chain's own records."""
    flags, kw, paired, t1, t2, S, _ = CASES[name]
    p = O.case_params(name)
    n = O.port_text_path(name, 0)["n"]
    ctx = gpu.GpuCtx(p, n, S, cycles_of(p, S))
    ch = device_chain(gpu, ctx, t1, t2, n)
    check_all_streams(ctx, ch, t1, t2, name)
    ctx.close()


def test_encode_large_enriched(gpu):
    """60 K enriched pairs (profile 1, 2 x 150) under a filter set that fails a real share of reads."""
    n = 60000
    _, arrs = T.synth_host(n, 160, 1, 0, 99, 1, 150)
    t1 = T.fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0"); t2 = T.fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0")
    p = capi.default_params(1, lib=T.oracle(), seq_len1=150, seq_len2=150, qualified_qual=33 + 30, unqualified_percent_limit=10, length_required=120)
    ctx = gpu.GpuCtx(p, n, 160, 160)
    ch = device_chain(gpu, ctx, t1, t2, n)
    check_all_streams(ctx, ch, t1, t2, "60K")
    failed = gpu_encode_rejects(ctx, ch, O.FAILED, 0)
    ctx.close()
    assert failed.count(b" paired_read_is_failing\n") > 100


@pytest.mark.parametrize("n", [1, 7, 2047, 2048, 2049])
def test_encode_batch_sizes_around_one_block(gpu, n):
    """The encode block walks 2 048 units: one short, exact, one over; and tiny batches (filters case, both modes)."""
    for name in ("filters_pe", "filters_se"):
        flags, kw, paired, t1, t2, S, _ = CASES[name]
        cut = lambda t: b"\n".join(t.split(b"\n")[:4 * n]) + b"\n"            # noqa: E731
        a, b = cut(t1), cut(t2) if paired else b""
        p = O.case_params(name)
        ctx = gpu.GpuCtx(p, 4096, S, S)
        ch = device_chain(gpu, ctx, a, b, n)
        check_all_streams(ctx, ch, a, b, (name, n))
        ctx.close()


def test_encode_out_cap(gpu):
    """One byte short of the total: the last unit that writes is left out whole and nothing lands at or behind its offset."""
    flags, kw, paired, t1, t2, S, _ = CASES["filters_pe"]
    n = 600
    a = b"\n".join(t1.split(b"\n")[:4 * n]) + b"\n"; b = b"\n".join(t2.split(b"\n")[:4 * n]) + b"\n"
    ctx = gpu.GpuCtx(O.case_params("filters_pe"), n, S, S)
    ch = device_chain(gpu, ctx, a, b, n)
    for which, w in ((O.FAILED, 0), (O.U1, 1), (O.U2, 3)):
        full = port_on_device_records(ctx, ch, a, b, which, w)
        k = n
        while len(port_on_device_records(ctx, ch, a, b, which, w, k - 1)) == len(full):
            k -= 1
        head = port_on_device_records(ctx, ch, a, b, which, w, k - 1)
        rc, buf, tot, guard_ok = gpu_encode_rejects(ctx, ch, which, w, out_cap=len(full) - 1)
        assert rc == 0 and tot == len(full) and guard_ok
        assert buf[:len(head)] == head and set(buf[len(head):]) <= {GUARD}
    ctx.close()


def process_host_outs(ctx, t1, t2, want, caps=None):
    """fp_fastq_process_host_outs; want = set of FP_FQ_OUT_* to pass a buffer for -> dict(rc, streams by key, n, consumed, guard_ok, untouched)."""
    lib, paired = ctx.lib, bool(ctx.params.paired)
    if caps is None:
        big = 2 * (len(t1) + len(t2)) + 256
        caps = [big] * 6
    bufs = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in (t1, t2)]
    outs = [np.full(caps[s] + 64, GUARD, np.uint8) if s in want else None for s in range(6)]
    optr = (C.c_void_p * 6)(*[o.ctypes.data if o is not None else None for o in outs])
    ocap = (C.c_int64 * 6)(*[caps[s] if s in want else 0 for s in range(6)])
    ob = (C.c_int64 * 6)(*([-7] * 6))
    nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64()
    i1, i2 = capi.FastqInfo(), capi.FastqInfo()
    rc = lib.fp_fastq_process_host_outs(ctx.h, bufs[0].ctypes.data, len(t1), bufs[1].ctypes.data if paired else None, len(t2) if paired else 0, 1, 0,
                                        optr, ocap, ob, C.byref(nu), C.byref(c1), C.byref(c2) if paired else None, C.byref(i1), C.byref(i2) if paired else None)
    r = {"rc": rc, "n": nu.value, "consumed": (c1.value, c2.value), "ob": list(ob),
         "guard_ok": all(o is None or bool((o[caps[s]:] == GUARD).all()) for s, o in enumerate(outs)),
         "untouched": all(o is None or bool((o == GUARD).all()) for o in outs) and list(ob) == [-7] * 6}
    for s, key in enumerate(STREAM_KEYS):
        r[key] = outs[s][:min(ob[s], caps[s])].tobytes() if (rc == 0 and outs[s] is not None) else b""
    return r


def want_of(name, wset):
    flags, _, paired = CASES[name][:3]
    u1, u2, f = O.WRITER_SETS[wset]
    ignored = not paired or "--include_unmerged" in flags
    w = {capi.FP_FQ_OUT_R1} | ({capi.FP_FQ_OUT_R2} if paired else set()) | ({capi.FP_FQ_OUT_MERGED} if "-m" in flags else set())
    w |= ({O.U1} if u1 and not ignored else set()) | ({O.U2} if u2 and not ignored else set()) | ({O.FAILED} if f else set())
    return w


@pytest.mark.parametrize("name", list(CASES))
def test_text_path_equals_port_digests_and_reference_cli(gpu, tmp_path, name):
    """fp_fastq_process_host_outs over several rounds (max_batch 700) == C-port text path, for every writer set of the case; the files the
    reference CLI writes from those streams match the committed digests (and the CLI itself where it is present)."""
    flags, kw, paired, t1, t2, S, dedup = CASES[name]
    p = O.case_params(name)
    digests = json.load(open(DIGESTS))
    for wset in O.case_writer_sets(name):
        want = O.port_text_path(name, O.port_writers(name, wset))
        ctx = gpu.GpuCtx(p, 700, S, cycles_of(p, S))
        if dedup:
            capi.check(ctx.lib.fp_fastq_set_dedup(ctx.h, 3, 1), ctx.lib)
        got = process_host_outs(ctx, t1, t2, want_of(name, wset))
        ctx.close()
        assert got["rc"] == 0 and got["guard_ok"] and got["n"] == want["n"], (name, wset)
        assert got["consumed"][0] == len(t1) and (not paired or got["consumed"][1] == len(t2))
        w = want_of(name, wset)
        for s, key in enumerate(STREAM_KEYS):
            assert got[key] == (want[key] if s in w else b""), (name, wset, key)
        u1, u2, f = O.WRITER_SETS[wset]
        files = (got["out1"], got["out2"], got["merged"], got["unpaired1"], got["unpaired2"] if u1 else b"", got["failed"])
        assert [hashlib.md5(x).hexdigest() for x in files] == digests[f"{name}/{wset}"], (name, wset)
        if os.path.exists(T.REF_CLI):
            (tmp_path / wset).mkdir()
            assert O.run_ref_cli_outs(tmp_path / wset, name, wset)[0] == files


def test_text_path_too_small_and_refusals(gpu):
    flags, kw, paired, t1, t2, S, _ = CASES["filters_pe"]
    p = O.case_params("filters_pe")
    allw = {1, 2, 3, 4, 5}
    ctx = gpu.GpuCtx(p, 700, S, S)
    full = process_host_outs(ctx, t1, t2, allw)
    ctx.close()
    assert full["rc"] == 0 and len(full["failed"]) > 0
    for s in (O.U1, O.U2, O.FAILED):                                          # one byte short: FP_E_TOOLARGE, nothing written past the buffer
        caps = [len(full[k]) + 1 for k in STREAM_KEYS]
        caps[s] = len(full[STREAM_KEYS[s]]) - 1
        ctx = gpu.GpuCtx(p, 700, S, S)
        r = process_host_outs(ctx, t1, t2, allw, caps)
        ctx.close()
        assert r["rc"] == -4 and r["guard_ok"], s
    refusals = [(O.case_params("filters_se"), CASES["filters_se"], {1, O.U1}),                 # unpaired buffer on a single-end ctx
                (O.case_params("merge_iu_pe"), CASES["merge_iu_pe"], {0, O.U2, O.FAILED}),   # unpaired buffer with --include_unmerged
                (p, CASES["filters_pe"], {0, 1, 2})]                                        # merged buffer on a ctx that does not merge
    for pp, case, want in refusals:
        ctx = gpu.GpuCtx(pp, 700, case[5], cycles_of(pp, case[5]))
        r = process_host_outs(ctx, case[3], case[4], want)
        assert r["rc"] == -1 and r["untouched"], want
        ctx.close()
    ctx = gpu.GpuCtx(O.case_params("filters_se"), 700, S, S)
    total = C.c_int64(5)
    assert ctx.lib.fp_fastq_encode_rejects(ctx.h, O.U1, 0, *([None] * 12), 0, None, 0, C.byref(total)) == -1 and total.value == 0
    assert ctx.lib.fp_fastq_encode_rejects(ctx.h, capi.FP_FQ_OUT_R1, 0, *([None] * 12), 0, None, 0, C.byref(total)) == -1
    ctx.close()


MIRROR = [("filters_pe", "u1u2f", True), ("filters_pe", "u2", False), ("filters_se", "u1u2f", False), ("dedup_pe", "u1f", False),
          ("merge_pe", "u2f", True), ("merge_iu_pe", "u1u2f", False), ("trim_null_pe", "u1u2", False)]


@pytest.mark.parametrize("name,wset,gz", MIRROR)
def test_mirror_cli(gpu, tmp_path, name, wset, gz):
    """fastp_gpu_cli --device_fastq with --unpaired1 / --unpaired2 / --failed_out at two chunk sizes: files (gzip-decompressed) equal the
    committed digests of the reference CLI's files, --unpaired2 alone leaves its file empty, ignored options are reported."""
    assert os.path.exists(CLI), "build with __graft_entry__.build()"
    flags, kw, paired, t1, t2, S, dedup = CASES[name]
    digests = json.load(open(DIGESTS))[f"{name}/{wset}"]
    (tmp_path / "r1.fq").write_bytes(t1)
    if paired:
        (tmp_path / "r2.fq").write_bytes(t2)
    for chunk in (100003, 1 << 20):
        d = tmp_path / str(chunk); d.mkdir()
        cmd = [CLI, "-i", str(tmp_path / "r1.fq"), "--device_fastq", "--chunk_bytes", str(chunk), "--pack_size", "2048", "--max_read_len", str(S)]
        cmd += (["-I", str(tmp_path / "r2.fq")] if paired else []) + flags + (["--dont_eval_duplication"] if not dedup else [])
        out_args = O.cli_output_args(d, flags, paired, wset)
        if gz:
            out_args = [a + ".gz" if a.startswith(str(d)) else a for a in out_args]
        r = subprocess.run(cmd + out_args, capture_output=True, timeout=600)
        assert r.returncode == 0, r.stderr[-500:]
        files = []
        for f in O.FILES:
            path = d / (f + ".gz" if gz else f)
            x = path.read_bytes() if path.exists() else b""
            files.append(gzip.decompress(x) if gz and x else x)
        assert [hashlib.md5(x).hexdigest() for x in files] == digests, (name, wset, chunk)
        u1, u2, f = O.WRITER_SETS[wset]
        if paired and "--include_unmerged" not in flags:
            assert (d / ("u2.fq" + (".gz" if gz else ""))).exists() == bool(u2)
        else:
            assert not (d / "u1.fq").exists() and b"Ignoring argument --unpaired1" in r.stderr


def test_mirror_cli_argument_rules(gpu, tmp_path):
    (tmp_path / "r.fq").write_bytes(b"@a\nACGT\n+\nIIII\n")
    base = [CLI, "-i", str(tmp_path / "r.fq")]
    pe = ["-I", str(tmp_path / "r.fq"), "--device_fastq", "-o", str(tmp_path / "o1.fq"), "-O", str(tmp_path / "o2.fq")]
    for extra, msg in ((["--failed_out", str(tmp_path / "f.fq")], b"--device_fastq"),
                       (pe + ["--unpaired1", str(tmp_path / "o1.fq")], b"--unpaired1 and --out1 shouldn't have same file name"),
                       (pe + ["--unpaired2", str(tmp_path / "o2.fq")], b"--unpaired2 and --out2 shouldn't have same file name"),
                       (pe + ["--unpaired1", str(tmp_path / "u.fq"), "--failed_out", str(tmp_path / "u.fq")],
                        b"--failed_out and --unpaired1 shouldn't have same file name"),
                       (pe + ["--failed_out", str(tmp_path / "o2.fq")], b"--failed_out and --out2 shouldn't have same file name")):
        r = subprocess.run(base + extra, capture_output=True, timeout=120)
        assert r.returncode == 2 and msg in r.stderr, (extra, r.stderr)
    assert not (tmp_path / "f.fq").exists() and not (tmp_path / "u.fq").exists()
