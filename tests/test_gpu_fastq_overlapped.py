"""-m gpu: --overlapped_out on the device.  The chain's analysis (fp_set_overlapped_sink) against the C port's, the other outputs of the
chain with and without the sink, fp_fastq_encode_overlapped against the port on the device's own records, and the text path
(fp_fastq_process_host_outs with fp_fastq_set_overlapped_out, fastp_gpu_cli --device_fastq --overlapped_out) against the committed digests
of the UNMODIFIED reference CLI's file and, where oracle/_ref/fastp_ref travelled along, that CLI itself.  The port is pinned to the CLI
on the CPU by tests/test_oracle_fastq_overlapped.py."""
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import edge_inputs as E
import fp_overlapped as O
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.gpu
FP_E_INVAL, FP_E_TOOLARGE = -1, -4                            # include/fastp_b200.h
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "fastp_b200", "host", "fastp_gpu_cli")
DIGESTS = json.load(open(os.path.join(ROOT, "tests", "golden", "fastq_overlapped_cli_digests.json")))
CASES = O.overlapped_cases()
GPU_CASES = ["cfg_cfg4_full", "cfg_tid_nonzero", "cfg_merge_cfg4_full", "cfg_mergeu_gap_cfg4_full", "cfg_tight_overlap", "planted",
             "planted_c", "planted_drop", "planted_req2", "dimer_filters", "max_len_polyx", "edge48", "edge256", "pe250"]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def _ctx(gpu, p, n, stride):
    return gpu.GpuCtx(p, max(n, 1), stride, 2 * stride if p.merge_enabled else stride)


def _run_chain(gpu, ctx, arrs, sink_chunks=None):
    """fp_process_pe over arrs (device copy) in launches of the given sizes; with sink_chunks each launch gets the sink at its own offset of
    one array (the pointer moves between launches) -> dict of host results."""
    import torch
    n = arrs["seq1"].shape[0]
    b, t = gpu.device_batch(T.copy_arrays(arrs))
    lib = ctx.lib
    d1 = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0"); d2 = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0")
    dov = torch.zeros(n * 8, dtype=torch.uint8, device="cuda:0"); dx = torch.full((n * 8 + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")
    ev = torch.zeros(n * 64 * 16, dtype=torch.uint8, device="cuda:0"); evn = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    capi.check(lib.fp_set_event_sink(ctx.h, ev.data_ptr(), n * 64, evn.data_ptr()), lib)
    patch_cap = 4 * n + 1024
    dp = torch.zeros(patch_cap * 12, dtype=torch.uint8, device="cuda:0"); dnp = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    sizes = sink_chunks or [n]
    o = 0
    for sz in sizes:
        sb = capi.Batch()
        sb.n, sb.stride = sz, b.stride
        for k in ("seq1", "qual1", "seq2", "qual2"):
            setattr(sb, k, getattr(b, k) + o * b.stride)
        sb.len1, sb.len2 = b.len1 + 2 * o, b.len2 + 2 * o
        capi.check(lib.fp_set_overlapped_sink(ctx.h, dx.data_ptr() + 8 * o if sink_chunks else None), lib)
        capi.check(lib.fp_process_pe(ctx.h, C.byref(sb), d1.data_ptr() + 16 * o, d2.data_ptr() + 16 * o, dov.data_ptr() + 8 * o,
                                     dp.data_ptr(), patch_cap, dnp.data_ptr(), None), lib)
        torch.cuda.synchronize()
        o += sz
    capi.check(lib.fp_set_overlapped_sink(ctx.h, None), lib)
    capi.check(lib.fp_set_event_sink(ctx.h, None, 0, None), lib)
    ne = int(evn.cpu()[0])
    evs = np.sort(ev.cpu().numpy()[:min(ne, n * 64) * 16].reshape(-1, 16).view(np.uint8), axis=0) if ne else np.zeros((0, 16), np.uint8)
    npatch = int(dnp.cpu()[0])
    return {"res1": d1.cpu().numpy().view(capi.READ_RESULT_DTYPE).copy(), "res2": d2.cpu().numpy().view(capi.READ_RESULT_DTYPE).copy(),
            "ov": dov.cpu().numpy().copy(), "ovx": dx.cpu().numpy()[:n * 8].view(O.OVX_DTYPE).copy(), "guard": bytes(dx.cpu().numpy()[n * 8:]),
            "events": ne, "ev": evs, "patches": npatch, "counters": ctx.counters().data.copy(),
            "rows": {k: v.cpu().numpy().copy() for k, v in t.items()}}


def _decoded(name):
    flags, p, t1, t2, S, dedup = CASES[name]
    d = O.port_text_path(p, t1, t2, S, dedup)
    return p, d["arrs"], S, d


@pytest.mark.parametrize("name", GPU_CASES)
def test_sink_equals_port_and_changes_nothing_else(gpu, name):
    p, arrs, S, port = _decoded(name)
    n = arrs["seq1"].shape[0]
    ctx = _ctx(gpu, p, n, S)
    base = _run_chain(gpu, ctx, arrs)
    ctx.reset()
    with_sink = _run_chain(gpu, ctx, arrs, sink_chunks=[n])
    got = with_sink["ovx"]
    want = port["ovx"]
    for f in ("overlapped", "offset", "overlap_len"):
        assert (got[f] == want[f]).all(), (name, f, int(np.flatnonzero(got[f] != want[f])[0]))
    m = want["overlapped"] == 1
    assert (got["r1_len"][m] == want["r1_len"][m]).all(), name
    assert with_sink["guard"] == bytes([0xA5]) * 64
    for k in ("res1", "res2", "ov", "events", "patches", "counters"):
        assert np.array_equal(np.asarray(base[k]), np.asarray(with_sink[k])), (name, k)
    assert np.array_equal(base["ev"], with_sink["ev"])
    for k in base["rows"]:
        assert np.array_equal(base["rows"][k], with_sink["rows"][k]), (name, k)
    ctx.close()


def test_sink_small_batches_and_moved_pointer(gpu):
    """Launches of 1..7 units and of several tiles per CTA, the sink pointer moved to each launch's first unit."""
    p, arrs, S, port = _decoded("planted_c")
    n = arrs["seq1"].shape[0]
    ctx = _ctx(gpu, p, n, S)
    sizes = [1, 2, 3, 4, 5, 6, 7]
    sizes += [n - sum(sizes) - 700, 700]
    got = _run_chain(gpu, ctx, arrs, sink_chunks=sizes)["ovx"]
    for f in ("overlapped", "offset", "overlap_len"):
        assert (got[f] == port["ovx"][f]).all(), f
    ctx.close()


@pytest.mark.parametrize("S", [48, 160, 256])
def test_sink_edge_inputs(gpu, S):
    p = capi.default_params(1, lib=T.oracle(), correction_enabled=1, seq_len1=S, seq_len2=S)
    arrs = E.edge_batch(4 * S + 700, S, 1, 90 + S, p)
    want = O.port_analyze(p, arrs, S)
    ctx = _ctx(gpu, p, arrs["seq1"].shape[0], S)
    got = _run_chain(gpu, ctx, arrs, sink_chunks=[arrs["seq1"].shape[0] // 3, arrs["seq1"].shape[0] - arrs["seq1"].shape[0] // 3])["ovx"]
    for f in ("overlapped", "offset", "overlap_len"):
        assert (got[f] == want[f]).all(), (S, f)
    ctx.close()


def _process_host(ctx, t1, t2, caps=None, ov_cap=None):
    lib = ctx.lib
    b1 = np.frombuffer(t1, np.uint8).copy(); b2 = np.frombuffer(t2, np.uint8).copy()
    caps = caps or [0, len(t1) + 64, len(t2) + 64, 0, 0, 0]
    bufs = [np.zeros(max(c, 1), np.uint8) if c else None for c in caps]
    outs = (C.c_void_p * 6)(*[b.ctypes.data if b is not None else None for b in bufs])
    ocap = (C.c_int64 * 6)(*caps); ob = (C.c_int64 * 6)()
    ov_cap = len(t1) + 64 if ov_cap is None else ov_cap
    ovb = np.full(ov_cap + 64, 0xA5, np.uint8); ovn = C.c_int64()
    capi.check(lib.fp_fastq_set_overlapped_out(ctx.h, ovb.ctypes.data, ov_cap, C.byref(ovn)), lib)
    nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64()
    rc = lib.fp_fastq_process_host_outs(ctx.h, b1.ctypes.data, len(t1), b2.ctypes.data, len(t2), 1, 0, outs, ocap, ob, C.byref(nu),
                                        C.byref(c1), C.byref(c2), None, None)
    capi.check(lib.fp_fastq_set_overlapped_out(ctx.h, None, 0, None), lib)
    return rc, ovb[:min(ovn.value, ov_cap)].tobytes(), ovn.value, bool((ovb[ov_cap:] == 0xA5).all())


@pytest.mark.parametrize("name", ["cfg_cfg4_full", "cfg_merge_cfg4_full", "planted_c", "dedup", "edge160"])
def test_text_path_rounds_equal_digests(gpu, name):
    flags, p, t1, t2, S, dedup = CASES[name]
    ctx = _ctx(gpu, p, 300, S)                                    # several rounds of 300 pairs
    if dedup:
        capi.check(ctx.lib.fp_fastq_set_dedup(ctx.h, 3, 1), ctx.lib)
    caps = [len(t1) + len(t2) + 4096 if p.merge_enabled else 0, 0 if p.merge_include_unmerged else len(t1) + 64,
            0 if p.merge_include_unmerged else len(t2) + 64, 0, 0, 0]
    for call in range(2):                                        # a second call on the same ctx
        rc, got, total, guard = _process_host(ctx, t1, t2, caps)
        capi.check(rc, ctx.lib)
        assert guard and hashlib.md5(got).hexdigest() == DIGESTS[name], (name, call)
    rc, _, total2, guard = _process_host(ctx, t1, t2, caps, ov_cap=total - 1)  # one byte short
    assert rc == FP_E_TOOLARGE and guard
    ctx.close()


def test_device_encoder_equals_port_on_device_records(gpu):
    import torch
    p, arrs, S, port = _decoded("planted_c")
    flags, _, t1, t2, _, _ = CASES["planted_c"]
    ctx = _ctx(gpu, p, arrs["seq1"].shape[0], S)
    dec1 = gpu.gpu_fastq_decode(ctx, t1); dec2 = gpu.gpu_fastq_decode(ctx, t2)
    n = min(len(dec1["recs"]), len(dec2["recs"]))
    (dt1, s1, q1, l1, r1), (_, s2, q2, l2, _) = dec1["dev"], dec2["dev"]
    b = capi.Batch(); b.n, b.stride = n, S
    b.seq1, b.qual1, b.len1, b.seq2, b.qual2, b.len2 = s1.data_ptr(), q1.data_ptr(), l1.data_ptr(), s2.data_ptr(), q2.data_ptr(), l2.data_ptr()
    d1 = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0"); d2 = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0")
    dx = torch.zeros(n * 8, dtype=torch.uint8, device="cuda:0")
    lib = ctx.lib
    capi.check(lib.fp_set_overlapped_sink(ctx.h, dx.data_ptr()), lib)
    capi.check(lib.fp_process_pe(ctx.h, C.byref(b), d1.data_ptr(), d2.data_ptr(), None, None, 0, None, None), lib)
    capi.check(lib.fp_set_overlapped_sink(ctx.h, None), lib)
    torch.cuda.synchronize()
    total = C.c_int64()
    args = lambda buf, cap: (ctx.h, dt1.data_ptr(), r1.data_ptr(), d1.data_ptr(), d2.data_ptr(), dx.data_ptr(), s1.data_ptr(), q1.data_ptr(), n, buf, cap)  # noqa: E731
    capi.check(lib.fp_fastq_encode_overlapped(*args(None, 0), C.byref(total)), lib)
    out = torch.full((total.value + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")
    t2v = C.c_int64()
    capi.check(lib.fp_fastq_encode_overlapped(*args(out.data_ptr(), total.value), C.byref(t2v)), lib)
    h = out.cpu().numpy()
    host = {k: t.cpu().numpy()[:n * S].reshape(n, S) for k, t in (("seq1", s1), ("qual1", q1))}
    want = O.oracle_encode_overlapped(t1, dec1["recs"][:n], d1.cpu().numpy().view(capi.READ_RESULT_DTYPE), d2.cpu().numpy().view(capi.READ_RESULT_DTYPE),
                                      dx.cpu().numpy().view(O.OVX_DTYPE), host["seq1"], host["qual1"], S)[0]
    assert t2v.value == total.value == len(want) and h[:total.value].tobytes() == want and (h[total.value:] == 0xA5).all()
    assert hashlib.md5(want).hexdigest() == DIGESTS["planted_c"]
    ctx.close()


def test_refusals(gpu):
    import torch
    lib = capi.load()
    se = gpu.GpuCtx(capi.default_params(0, lib=T.oracle()), 64, 160, 160)
    dummy = torch.zeros(1024, dtype=torch.uint8, device="cuda:0")
    assert lib.fp_set_overlapped_sink(se.h, dummy.data_ptr()) == FP_E_INVAL
    buf = np.zeros(64, np.uint8); nb = C.c_int64()
    assert lib.fp_fastq_set_overlapped_out(se.h, buf.ctypes.data, 64, C.byref(nb)) == FP_E_INVAL
    se.close()
    p = capi.default_params(1, lib=T.oracle())
    ctx = gpu.GpuCtx(p, 64, 160, 160)
    _, arrs = T.synth_host(16, 160, 1, 0, 3, 1, 150)
    capi.check(lib.fp_set_overlapped_sink(ctx.h, dummy.data_ptr()), lib)
    b = capi.batch_from_arrays(T.copy_arrays(arrs))
    o1 = np.zeros(16, capi.READ_RESULT_DTYPE); o2 = np.zeros(16, capi.READ_RESULT_DTYPE)
    assert lib.fp_process_pe_host(ctx.h, C.byref(b), o1.ctypes.data, o2.ctypes.data, None) == FP_E_INVAL
    assert (o1.view(np.uint8) == 0).all()
    t = T.fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0")
    out = np.zeros(len(t) + 64, np.uint8); ob1, ob2, nu, c1, c2 = (C.c_int64() for _ in range(5))
    tb = np.frombuffer(t, np.uint8).copy()
    assert lib.fp_fastq_process_host(ctx.h, tb.ctypes.data, len(t), tb.ctypes.data, len(t), 1, 0, out.ctypes.data, len(out), C.byref(ob1),
                                     out.ctypes.data, len(out), C.byref(ob2), C.byref(nu), C.byref(c1), C.byref(c2), None, None) == FP_E_INVAL
    capi.check(lib.fp_set_overlapped_sink(ctx.h, None), lib)
    ctx.close()


def _mirror(tmp_path, name, extra=(), interleaved=False, gz=False):
    flags, p, t1, t2, S, dedup = CASES[name]
    flags = [f for f in flags]
    if "fasta" in flags:
        pytest.skip("the mirror CLI takes no --adapter_fasta")
    ov = tmp_path / ("ov.fq.gz" if gz else "ov.fq")
    cmd = [CLI, "--device_fastq", "--overlapped_out", str(ov), "-j", str(tmp_path / "s.json")]
    if interleaved:
        (tmp_path / "il.fq").write_bytes(O.interleave(t1, t2)); cmd += ["-i", str(tmp_path / "il.fq"), "--interleaved_in"]
    else:
        (tmp_path / "r1.fq").write_bytes(t1); (tmp_path / "r2.fq").write_bytes(t2)
        cmd += ["-i", str(tmp_path / "r1.fq"), "-I", str(tmp_path / "r2.fq")]
    if "-m" in flags:
        cmd += ["--merged_out", str(tmp_path / "m.fq")]
    if "--include_unmerged" not in flags:
        cmd += ["-o", str(tmp_path / "o1.fq"), "-O", str(tmp_path / "o2.fq")]
    if "-D" not in flags:
        cmd.append("--dont_eval_duplication")
    subprocess.run(cmd + flags + list(extra), check=True, capture_output=True)
    data = ov.read_bytes()
    return gzip.decompress(data) if gz and data else data


@pytest.mark.parametrize("name", ["cfg_cfg3_overlap_correction", "cfg_merge_cfg4_full", "dedup", "max_len_polyx", "planted_c", "planted_drop"])
def test_mirror_cli_equals_digests(tmp_path, name):
    got = _mirror(tmp_path, name, extra=["--chunk_bytes", "60000"])
    assert hashlib.md5(got).hexdigest() == DIGESTS[name], name
    if os.path.exists(T.REF_CLI):
        flags, p, t1, t2 = CASES[name][:4]
        assert got == O.run_ref_cli(tmp_path, flags, t1, t2)


def test_mirror_cli_interleaved_and_gz(tmp_path):
    assert hashlib.md5(_mirror(tmp_path, "cfg_cfg4_full", interleaved=True)).hexdigest() == DIGESTS["cfg_cfg4_full"]
    assert hashlib.md5(_mirror(tmp_path, "cfg_cfg4_full", gz=True)).hexdigest() == DIGESTS["cfg_cfg4_full"]


def test_mirror_cli_single_end_and_without_device_fastq(tmp_path):
    flags, p, t1, t2 = CASES["cfg_default"][:4]
    (tmp_path / "r1.fq").write_bytes(t1)
    r = subprocess.run([CLI, "--device_fastq", "-i", str(tmp_path / "r1.fq"), "-o", str(tmp_path / "o.fq"), "--overlapped_out", str(tmp_path / "ov.fq")],
                       capture_output=True, text=True)
    assert r.returncode == 0 and "Not paired-end mode. Ignoring argument --overlapped_out = " in r.stderr and not (tmp_path / "ov.fq").exists()
    r = subprocess.run([CLI, "-i", str(tmp_path / "r1.fq"), "-I", str(tmp_path / "r1.fq"), "--overlapped_out", str(tmp_path / "ov.fq")],
                       capture_output=True, text=True)
    assert r.returncode == 2 and "--overlapped_out needs --device_fastq" in r.stderr
