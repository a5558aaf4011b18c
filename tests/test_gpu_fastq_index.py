"""-m gpu: the index filter on the device.  The matcher (fp_fastq_index_flags) against the C port over the name and list matrix, the chain
with fp_set_index_flags against fp_oracle_process_index, the text path (fp_fastq_set_index_filter) and the mirror CLI against the committed
digests of the UNMODIFIED reference CLI and, where oracle/_ref/fastp_ref travelled along, that CLI itself, and the refusals.  The port is
pinned to the CLI on the CPU by tests/test_oracle_fastq_index.py."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import fp_index as X
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.gpu
FP_E_INVAL = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "fastp_b200", "host", "fastp_gpu_cli")
DIGESTS = json.load(open(os.path.join(ROOT, "tests", "golden", "fastq_index_cli_digests.json")))
STREAM_KEYS = ("merged", "out1", "out2", "unpaired1", "unpaired2", "failed")          # FP_FQ_OUT_*


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def _set_lists(ctx, l1, l2, thr):
    a1 = (C.c_char_p * max(len(l1), 1))(*l1); a2 = (C.c_char_p * max(len(l2), 1))(*l2)
    return ctx.lib.fp_fastq_set_index_filter(ctx.h, a1, len(l1), a2, len(l2), thr)


def _device_flags(gpu, ctx, t1, recs1, t2, recs2):
    import torch
    n = len(recs1)
    dt1 = torch.from_numpy(np.frombuffer(t1 + b"\0", np.uint8).copy()).cuda(); dr1 = torch.from_numpy(np.ascontiguousarray(recs1).view(np.uint8).copy()).cuda()
    dt2 = dr2 = None
    if recs2 is not None:
        dt2 = torch.from_numpy(np.frombuffer(t2 + b"\0", np.uint8).copy()).cuda(); dr2 = torch.from_numpy(np.ascontiguousarray(recs2).view(np.uint8).copy()).cuda()
    df = torch.full((n + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")
    capi.check(ctx.lib.fp_fastq_index_flags(ctx.h, dt1.data_ptr(), dr1.data_ptr(), dt2.data_ptr() if dt2 is not None else None,
                                            dr2.data_ptr() if dr2 is not None else None, n, df.data_ptr()), ctx.lib)
    f = df.cpu().numpy()
    assert (f[n:] == 0xA5).all()
    return f[:n]


@pytest.mark.parametrize("paired", [1, 0])
@pytest.mark.parametrize("lst", ["one", "l96", "mixed", "n2048", "n20000", "long"])
@pytest.mark.parametrize("thr", [-1, 0, 1, 2])
def test_matcher_equals_port(gpu, paired, lst, thr):
    t1, t2 = X.named_texts(3000, 40 + paired, paired)
    d1 = T.oracle_fastq_decode(t1); d2 = T.oracle_fastq_decode(t2) if paired else None
    lists = {"one": [b"ACGTACGT"], "l96": X.barcode_list(96, 3, lens=(8, 6, 10, 8)), "mixed": [b"TTGGCCAA", b"GATTAC", b"", b"CCCCGGGGAA"],
             "n2048": X.barcode_list(2048, 5, lens=(8, 7, 9)), "n20000": X.barcode_list(20000, 6, lens=(8, 16)),
             "long": [b"ACGT" * 100, b"GATTACAG" * 40 + b"T", b"A" * 1024]}[lst]
    l2 = lists[::-1] if paired else []
    p = capi.default_params(paired, lib=T.oracle())
    ctx = gpu.GpuCtx(p, 4096, 160, 160)
    capi.check(_set_lists(ctx, lists, l2, thr), ctx.lib)
    got = _device_flags(gpu, ctx, t1, d1["recs"], t2, d2["recs"] if paired else None)
    want = X.port_flags(t1, d1["recs"], t2, d2["recs"] if paired else None, lists, l2, thr)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]
    ctx.close()


def _chain(gpu, ctx, p, arrs, ix, is_dup, bounds, ix_on=True):
    """fp_process_* in launches [bounds[k], bounds[k+1]) with the index flags (and dup flags) at each launch's first unit."""
    import torch
    paired = bool(p.paired)
    n, S = arrs["seq1"].shape
    lib = ctx.lib
    ctx.reset()
    b, t = gpu.device_batch(T.copy_arrays(arrs))
    d1 = torch.zeros(n * 16 + 16, dtype=torch.uint8, device="cuda:0"); d2 = torch.zeros(n * 16 + 16, dtype=torch.uint8, device="cuda:0")
    dov = torch.full((n * 8 + 8,), 0x5A, dtype=torch.uint8, device="cuda:0")
    dix = torch.from_numpy(np.concatenate([ix, [0]]).astype(np.uint8)).cuda()
    ddup = torch.from_numpy(np.concatenate([is_dup, [0]]).astype(np.uint8)).cuda() if is_dup is not None else None
    cap = 4 * n + 16
    dp = torch.zeros(cap * 12, dtype=torch.uint8, device="cuda:0"); dnp = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        if ix_on:
            capi.check(lib.fp_set_index_flags(ctx.h, dix.data_ptr() + lo), lib)
        if ddup is not None:
            capi.check(lib.fp_set_dup_flags(ctx.h, ddup.data_ptr() + lo), lib)
        sb = capi.Batch(); sb.n, sb.stride = hi - lo, S
        for k, v in t.items():
            setattr(sb, k, v.data_ptr() + lo * (2 if k.startswith("len") else S))
        if paired:
            capi.check(lib.fp_process_pe(ctx.h, C.byref(sb), d1.data_ptr() + lo * 16, d2.data_ptr() + lo * 16, dov.data_ptr() + lo * 8,
                                         dp.data_ptr(), cap, dnp.data_ptr(), None), lib)
        else:
            capi.check(lib.fp_process_se(ctx.h, C.byref(sb), d1.data_ptr() + lo * 16, None), lib)
    torch.cuda.synchronize()
    capi.check(lib.fp_set_index_flags(ctx.h, None), lib); capi.check(lib.fp_set_dup_flags(ctx.h, None), lib)
    out = {"out1": d1.cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy(), "out2": d2.cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy(),
           "ov": dov.cpu().numpy().view(capi.OV_RESULT_DTYPE)[:n].copy(), "counters": ctx.counters(), "layout": ctx.L,
           "arrs": {k: v.cpu().numpy() for k, v in t.items()}}
    return out


def _pattern(kind, n, tile, rng):
    ix = np.zeros(n, np.uint8)
    if kind == "all":
        ix[:] = 1
    elif kind == "random":
        ix[:] = rng.random(n) < 0.3
    elif kind == "alternating":
        ix[::2] = 1
    elif kind == "tile_ends":
        ix[::tile] = 1; ix[tile - 1::tile] = 1
    return ix


def _compare(got, want, paired, what):
    T.assert_results_equal(got, want, paired, what=what)
    for k in ("out1", "out2") if paired else ("out1",):
        assert np.array_equal(got[k]["reserved"], want[k]["reserved"]), what


@pytest.mark.parametrize("paired", [1, 0])
@pytest.mark.parametrize("kind", ["none", "all", "random", "alternating", "tile_ends"])
@pytest.mark.parametrize("cfg", ["cfg4_full", "default"])
def test_chain_equals_port(gpu, paired, kind, cfg):
    rng = np.random.default_rng([paired, len(kind), len(cfg)])
    _, arrs = T.synth_host(3000, 160, paired, 0, 61 + paired, 1, 150)
    p = T.config_params(cfg, paired)
    ctx = gpu.GpuCtx(p, 3000, 160, 160)
    ix = _pattern(kind, 3000, 128, rng)                       # 128 units per tile at stride 160
    is_dup = (rng.random(3000) < 0.2).astype(np.uint8)
    got = _chain(gpu, ctx, p, arrs, ix, is_dup, [0, 3000])
    want = X.port_process(p, arrs, 160, is_dup, ix)
    _compare(got, want, paired, f"{cfg} {kind}")
    ctx.close()


@pytest.mark.parametrize("paired", [1, 0])
@pytest.mark.parametrize("sampling", [1, 7, 20])
def test_chain_overrep_equals_port(gpu, paired, sampling):
    rng = np.random.default_rng(sampling)
    _, arrs = T.synth_host(2500, 160, paired, 0, 71, 1, 150)
    p = T.overrep_params("cfg4_full", paired, arrs, 150, sampling=sampling)
    ctx = gpu.GpuCtx(p, 2500, 160, 160)
    ix = (rng.random(2500) < 0.4).astype(np.uint8)
    got = _chain(gpu, ctx, p, arrs, ix, None, [0, 700, 2500])
    want = X.port_process(p, arrs, 160, None, ix)
    _compare(got, want, paired, f"overrep {sampling}")
    ctx.close()


def test_chain_merging_small_batches_and_null_pointer(gpu):
    rng = np.random.default_rng(5)
    _, arrs = T.synth_host(1200, 160, 1, 0, 81, 1, 150)
    p = T.config_params("merge_cfg4_full", 1)
    ctx = gpu.GpuCtx(p, 1200, 160, 320)
    ix = (rng.random(1200) < 0.35).astype(np.uint8)
    bounds = [0]
    while bounds[-1] < 1200:                                   # batches of 1-7 units, then the rest in three launches
        bounds.append(min(1200, bounds[-1] + (int(rng.integers(1, 8)) if bounds[-1] < 200 else 400)))
    got = _chain(gpu, ctx, p, arrs, ix, None, bounds)
    want = X.port_process(p, arrs, 320, None, ix)
    _compare(got, want, 1, "merge")
    ctx.close()
    # the pointer off, and all-zero flags: byte-identical to a ctx that never set it
    p = T.config_params("cfg4_full", 1)
    zero = np.zeros(1200, np.uint8)
    fresh = gpu.run_gpu(p, arrs, 160, mode="device")
    ctx = gpu.GpuCtx(p, 1200, 160, 160)
    for on in (True, False):
        got = _chain(gpu, ctx, p, arrs, zero, None, [0, 1200], ix_on=on)
        T.assert_results_equal(got, fresh, 1, what=f"zero flags on={on}")
        assert (got["out1"]["reserved"] == 0).all() and (got["out2"]["reserved"] == 0).all()
    ctx.close()


def _text_path(gpu, name, max_batch=300):
    flags, kw, paired, t1, t2, S, dedup, f1, f2, thr = X.index_cases()[name]
    p = X.case_params(name)
    merging = bool(paired and p.merge_enabled)
    ctx = gpu.GpuCtx(p, max_batch, S, 2 * S if merging else S)
    lib = ctx.lib
    l1, l2 = X.case_lists(name)
    capi.check(_set_lists(ctx, l1, l2, thr), lib)
    if dedup:
        capi.check(lib.fp_fastq_set_dedup(ctx.h, 3, 1), lib)
    iu = "--include_unmerged" in flags
    big = 2 * (len(t1) + len(t2)) + 4096
    want = {1, 2, 5} | ({0} if merging else set()) | ({3, 4} if paired and not iu else set())
    if iu:
        want -= {1, 2}
    if not paired:
        want -= {2}
    bufs = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in (t1, t2)]
    outs = [np.zeros(big, np.uint8) if s in want else None for s in range(6)]
    optr = (C.c_void_p * 6)(*[o.ctypes.data if o is not None else None for o in outs])
    ocap = (C.c_int64 * 6)(*[big if s in want else 0 for s in range(6)]); ob = (C.c_int64 * 6)()
    ovb = np.zeros(big, np.uint8); ovn = C.c_int64()
    if paired:
        capi.check(lib.fp_fastq_set_overlapped_out(ctx.h, ovb.ctypes.data, big, C.byref(ovn)), lib)
    nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64()
    capi.check(lib.fp_fastq_process_host_outs(ctx.h, bufs[0].ctypes.data, len(t1), bufs[1].ctypes.data if paired else None, len(t2) if paired else 0,
                                              1, 0, optr, ocap, ob, C.byref(nu), C.byref(c1), C.byref(c2) if paired else None, None, None), lib)
    got = {k: outs[s][:ob[s]].tobytes() if outs[s] is not None else b"" for s, k in enumerate(STREAM_KEYS)}
    got["overlapped"] = ovb[:ovn.value].tobytes() if paired else b""
    counts = X.summary_counts(ctx.counters(), paired)
    ctx.close()
    return got, counts


@pytest.mark.parametrize("name", sorted(X.index_cases()))
def test_text_path_equals_digests(gpu, name):
    got, counts = _text_path(gpu, name)
    d = DIGESTS[name]
    assert {k: hashlib.md5(got[k]).hexdigest() for k in X.STREAMS} == d["files"], name
    assert counts == d["counts"], name


def _mirror_counts(js, paired):
    b, a, f = js["before_filtering"], js["after_filtering"], js["filtering_result"]
    return {"before_reads": b["total_reads"], "before_bases": b["total_bases"], "after_reads": a["total_reads"], "after_bases": a["total_bases"],
            "passed": f["passed_filter_reads"], "low_quality": f["low_quality_reads"], "too_many_N": f["too_many_N_reads"],
            "too_short": f["too_short_reads"], "too_long": f["too_long_reads"], "low_complexity": f["low_complexity_reads"],
            "adapter_dimer": f["adapter_dimer_reads"]}


@pytest.mark.parametrize("name,gz,il", [("l96_t1_pe", False, False), ("dedup_pe", False, False), ("merge_pe", True, False), ("crlf_se", True, False),
                                        ("failed_pe", False, True), ("only2_se", False, False), ("stride48_pe", False, False)])
def test_mirror_cli_equals_digests(gpu, tmp_path, name, gz, il):
    out, js, r = X.run_cli(CLI, tmp_path, name, extra=["--chunk_bytes", "90000"], gz=gz, interleaved=il)
    assert r.returncode == 0, r.stderr[-2000:]
    d = DIGESTS[name]
    assert {k: hashlib.md5(out[k]).hexdigest() for k in X.STREAMS} == d["files"], name
    c = _mirror_counts(js, X.index_cases()[name][2])
    assert {k: v for k, v in c.items() if k in ("before_reads", "before_bases", "after_reads", "after_bases", "passed")} == \
        {k: v for k, v in d["counts"].items() if k in ("before_reads", "before_bases", "after_reads", "after_bases", "passed")}
    if os.path.exists(T.REF_CLI) and not gz:                 # the reference build here writes plain FASTQ only
        (tmp_path / "ref").mkdir()
        ref, _, rr = X.run_cli(T.REF_CLI, tmp_path / "ref", name, gz=gz, interleaved=il)
        assert rr.returncode == 0 and ref == out


def test_refusals(gpu, tmp_path):
    import torch
    _, arrs = T.synth_host(64, 160, 1, 0, 3, 1, 150)
    p = T.config_params("default", 1)
    ctx = gpu.GpuCtx(p, 64, 160, 160)
    lib = ctx.lib
    d = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    capi.check(lib.fp_set_index_flags(ctx.h, d.data_ptr()), lib)
    a = T.copy_arrays(arrs); b = capi.batch_from_arrays(a)
    o1 = np.zeros(64, capi.READ_RESULT_DTYPE); o2 = np.zeros(64, capi.READ_RESULT_DTYPE); ov = np.zeros(64, capi.OV_RESULT_DTYPE)
    assert lib.fp_process_pe_host(ctx.h, C.byref(b), o1.ctypes.data, o2.ctypes.data, ov.ctypes.data) == FP_E_INVAL
    t1, t2 = X.named_texts(10, 1, 1)
    b1 = np.frombuffer(t1, np.uint8).copy(); b2 = np.frombuffer(t2, np.uint8).copy()
    out = np.zeros(len(t1) * 2, np.uint8); n1, n2, nu, c1, c2 = (C.c_int64() for _ in range(5))
    assert lib.fp_fastq_process_host(ctx.h, b1.ctypes.data, len(t1), b2.ctypes.data, len(t2), 1, 0, out.ctypes.data, len(out), C.byref(n1),
                                     out.ctypes.data, len(out), C.byref(n2), C.byref(nu), C.byref(c1), C.byref(c2), None, None) == FP_E_INVAL
    capi.check(lib.fp_set_index_flags(ctx.h, None), lib)
    assert _set_lists(ctx, [b"ACGT", b"ACNT"], [], 0) == FP_E_INVAL
    assert _set_lists(ctx, [b"acgt"], [], 0) == FP_E_INVAL
    assert _set_lists(ctx, [b"A" * 1025], [], 0) == FP_E_INVAL
    ctx.close()
    (tmp_path / "r1.fq").write_bytes(t1); (tmp_path / "r2.fq").write_bytes(t2); (tmp_path / "ix.txt").write_bytes(b"ACGT\n")
    r = subprocess.run([CLI, "-i", str(tmp_path / "r1.fq"), "-I", str(tmp_path / "r2.fq"), "--filter_by_index1", str(tmp_path / "ix.txt")],
                       capture_output=True, text=True)
    assert r.returncode == 2 and "need --device_fastq" in r.stderr
    (tmp_path / "bad.txt").write_bytes(b"ACGT\nACNT\n")
    r = subprocess.run([CLI, "--device_fastq", "-i", str(tmp_path / "r1.fq"), "-o", str(tmp_path / "o.fq"), "--filter_by_index1", str(tmp_path / "bad.txt")],
                       capture_output=True, text=True)
    assert r.returncode == 255 and "each line should be one barcode, which can only contain A/T/C/G" in r.stderr
    r = subprocess.run([CLI, "--device_fastq", "-i", str(tmp_path / "r1.fq"), "-o", str(tmp_path / "o.fq"), "--filter_by_index2", str(tmp_path / "nope.txt")],
                       capture_output=True, text=True)
    assert r.returncode == 255 and "doesn't exist" in r.stderr
