"""-m gpu: the CUDA path against the CPU oracle on the edge inputs of tests/edge_inputs.py, bit-exact (records, overlap records,
corrected rows, the whole counter block): quality bytes over all of [33, 126] and lengths up to the full stride at every tile
layout, batch shapes that leave ragged last tiles, and the documented capacity paths -- more corrections than a tile's work list
(FP_CORR_CAP) or a device patch list holds, more than a host chunk's patch list holds, and more adapter events per unit than four.
tests/test_oracle_edges.py pins the oracle to the reference's objects on the same generators."""
import ctypes as C

import numpy as np
import pytest

import edge_inputs as E
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.gpu

PE_STRIDES = [48, 64, 128, 160, 192, 256]        # 64 / 128 / 192: stride % 64 == 0 flips the item order
SE_STRIDES = [48, 160, 256, 304, 512]            # above 256 the SE tile holds fewer than 256 reads
FASTA = [T.TRUSEQ_R1, "CTGTCTCTTATACACATCT", T.TRUSEQ_R2[:20], "AAAAAAAAAAAA", "GGGGGGGGGG"]      # the fasta_adapters option set's list
INCOMPLETE = (1 << 63) - 1                        # *n_patches of a host call whose patch list could not be complete


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def grid_input(name, paired, S, n=1500, seed=None, max_len=None):
    p = T.config_params(name, paired)
    return p, E.edge_batch(n, S, paired, seed or S, p, read_len=min(150, S) if S <= 256 else S - 12, max_len=max_len)


def corrected_bases(before, after):
    return sum(int((after["seq" + s] != before["seq" + s]).sum()) for s in "12")


# ---------------- quality x length grid ----------------
@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", T.CONFIG_NAMES)
def test_quality_length_grid_pe(gpu, name, S):
    p, arrs = grid_input(name, 1, S)
    T.assert_results_equal(gpu.run_gpu(p, arrs, S), T.run_cpu("oracle", p, arrs, S), 1, what=f"{name}/PE/S{S}")


@pytest.mark.parametrize("S", SE_STRIDES)
@pytest.mark.parametrize("name", T.CONFIG_NAMES)
def test_quality_length_grid_se(gpu, name, S):
    p, arrs = grid_input(name, 0, S)
    T.assert_results_equal(gpu.run_gpu(p, arrs, S), T.run_cpu("oracle", p, arrs, S), 0, what=f"{name}/SE/S{S}")


@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", T.MERGE_CONFIG_NAMES)
def test_quality_length_grid_merge(gpu, name, S):
    p, arrs = grid_input(name, 1, S)
    T.assert_results_equal(gpu.run_gpu(p, arrs, 2 * S), T.run_cpu("oracle", p, arrs, 2 * S), 1, what=f"{name}/S{S}")


# ---------------- batch shapes ----------------
def multi_tile_n():
    """n = 5 (mod 8) above 2 * SMs * 256: every CTA of the persistent grid does at least two tiles and the last tile holds 5 units."""
    import torch
    m = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 256
    return m - m % 8 + 8 + 5


@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, "multi_tile"])
@pytest.mark.parametrize("name,paired,S", [("cfg4_full", 1, 160), ("cfg3_overlap_correction", 1, 256), ("cfg4_full", 0, 160),
                                           ("all_cuts", 0, 512), ("merge_cfg4_full", 1, 128)])
def test_batch_shapes(gpu, name, paired, S, n):
    n = multi_tile_n() if n == "multi_tile" else n
    p, arrs = grid_input(name, paired, S, n=n, seed=n % 1000 + 1)
    cycles = 2 * S if name.startswith("merge") else S
    T.assert_results_equal(gpu.run_gpu(p, arrs, cycles), T.run_cpu("oracle", p, arrs, cycles), paired, what=f"{name} n={n}")


@pytest.mark.parametrize("name,paired", [("all_cuts", 1), ("cfg4_full", 0)])
def test_counters_accumulate_over_three_launches(gpu, name, paired):
    n = multi_tile_n()
    p, arrs = grid_input(name, paired, 160, n=n, seed=3)
    T.assert_results_equal(gpu.run_gpu(p, arrs, 160, splits=3), T.run_cpu("oracle", p, arrs, 160), paired, what=f"{name} 3 launches")


# ---------------- host entry points ----------------
@pytest.mark.parametrize("mode,max_batch", [pytest.param(m, mb, id=m if mb is None else f"{m}-max_batch{mb}")
                                            for mb in (None, 1024) for m in ("host", "host_tight", "host_pack2bit", "packed")])
@pytest.mark.parametrize("name,paired", [("cfg4_full", 1), ("cfg3_overlap_correction", 1), ("all_cuts", 1), ("cfg4_full", 0), ("filters", 0)])
def test_host_entry_points(gpu, name, paired, mode, max_batch):
    """The same inputs through fp_process_*_host at the device pitch, at the tight pitch of the longest read (150 of 160),
    packed on the fly (FP_B_PACK2BIT) and packed by the caller (the rows hold A/C/G/T/N only).  max_batch 1024: a ctx whose host
    chunks hold 1024 units, so the 20000 units go through about 20 chunks (completion on the helper thread, the 'N' list sliced at
    every chunk's offset) instead of one."""
    p, arrs = grid_input(name, paired, 160, n=20000, seed=17, max_len=150 if mode == "host_tight" else None)
    if mode == "host_tight":
        assert arrs["len1"].max() == 150
    want = T.run_cpu("oracle", p, arrs, 160)
    ctx = gpu.GpuCtx(p, max_batch, 160, 160) if max_batch else None
    try:
        T.assert_results_equal(gpu.run_gpu(p, arrs, 160, mode=mode, ctx=ctx), want, paired, what=f"{mode} {name} max_batch {max_batch}")
    finally:
        if ctx:
            ctx.close()


# ---------------- correction overflow on the device ----------------
def run_pe_device(gpu, ctx, t, n, patch_cap):
    """One fp_process_pe pass over the resident rows `t` with a patch list of patch_cap entries."""
    import torch
    lib = ctx.lib
    b = capi.Batch()
    b.n, b.stride = n, t["seq1"].shape[1]
    for k, v in t.items():
        setattr(b, k, v.data_ptr())
    d = {"out1": torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0"), "out2": torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0"),
         "ov": torch.zeros(n * 8, dtype=torch.uint8, device="cuda:0"), "patches": torch.zeros(max(patch_cap, 1) * 12, dtype=torch.uint8, device="cuda:0"),
         "np": torch.zeros(1, dtype=torch.int32, device="cuda:0")}
    ctx.reset()
    capi.check(lib.fp_process_pe(ctx.h, C.byref(b), d["out1"].data_ptr(), d["out2"].data_ptr(), d["ov"].data_ptr(), d["patches"].data_ptr(),
                                 patch_cap, d["np"].data_ptr(), None), lib)
    torch.cuda.synchronize()
    npatch = int(d["np"].item())
    got = {"out1": d["out1"].cpu().numpy().view(capi.READ_RESULT_DTYPE), "out2": d["out2"].cpu().numpy().view(capi.READ_RESULT_DTYPE),
           "ov": d["ov"].cpu().numpy().view(capi.OV_RESULT_DTYPE), "counters": ctx.counters(), "arrs": {k: v.cpu().numpy() for k, v in t.items()},
           "layout": ctx.L, "n_patches": npatch, "patches": d["patches"].cpu().numpy().view(capi.PATCH_DTYPE)[:min(npatch, patch_cap)].copy()}
    return got, b, d


@pytest.mark.parametrize("limit", [5, 20])
def test_correction_overflow_device(gpu, limit):
    """More corrections than a tile's work list holds (FP_CORR_CAP = 1024 per 128 pairs): the rest of a pair is
    corrected by the sequential path after part of it went through the list.  Then a patch list of 16 entries: the rows and
    counters are the same and the count still covers every correction.  fp_patches_undo restores the pristine rows."""
    n = 4000
    p = T.config_params("cfg3_overlap_correction", 1)
    p.overlap_diff_limit = limit
    arrs = E.dense_correction_pairs(n, 150, 160, 12, np.random.default_rng(limit))
    want = T.run_cpu("oracle", p, arrs, 160)
    ncorr = corrected_bases(arrs, want["arrs"])
    assert ncorr > 1024 / 128 * n
    ctx = gpu.GpuCtx(p, n, 160, 160)
    _, t = gpu.device_batch({k: v.copy() for k, v in arrs.items()})
    cap = 16 * n
    got, b, d = run_pe_device(gpu, ctx, t, n, cap)
    T.assert_results_equal(got, want, 1, what=f"dense limit {limit}")
    assert got["n_patches"] == ncorr
    rebuilt = {k: v.copy() for k, v in arrs.items()}
    for pt in got["patches"]:
        side = "2" if pt["which"] else "1"
        assert arrs["seq" + side][pt["pair"], pt["pos"]] == pt["old_base"] and arrs["qual" + side][pt["pair"], pt["pos"]] == pt["old_qual"]
        rebuilt["seq" + side][pt["pair"], pt["pos"]] = pt["base"]
        rebuilt["qual" + side][pt["pair"], pt["pos"]] = pt["qual"]
    for k in ("seq1", "qual1", "seq2", "qual2"):
        assert (rebuilt[k] == got["arrs"][k]).all(), k
    full = {tuple(x) for x in got["patches"].tolist()}
    capi.check(ctx.lib.fp_patches_undo(ctx.h, C.byref(b), d["patches"].data_ptr(), d["np"].data_ptr(), cap, None), ctx.lib)
    import torch
    torch.cuda.synchronize()
    for k in ("seq1", "qual1", "seq2", "qual2"):
        assert (t[k].cpu().numpy() == arrs[k]).all(), f"undo {k}"
    small, _, _ = run_pe_device(gpu, ctx, t, n, 16)              # the pristine rows again, 16 listed
    T.assert_results_equal(small, want, 1, what=f"dense limit {limit}, patch_cap 16")
    assert small["n_patches"] == ncorr and len(small["patches"]) == 16
    assert {tuple(x) for x in small["patches"].tolist()} <= full
    ctx.close()


# ---------------- host patch overflow ----------------
@pytest.fixture(scope="module")
def dense_host():
    """300 000 correction-dense pairs: two host chunks, about 9.5 corrections per pair (a chunk lists 2 per pair + 1024)."""
    p = T.config_params("cfg3_overlap_correction", 1)
    arrs = E.dense_correction_pairs(300000, 150, 160, 12, np.random.default_rng(300))
    want = T.run_cpu("oracle", p, arrs, 160)
    assert corrected_bases(arrs, want["arrs"]) > 2 * 300000 + 2048
    return p, arrs, want


@pytest.mark.parametrize("mode", ["host", "host_tight", "host_pack2bit"])
def test_host_patch_overflow_writes_the_rows_back(gpu, dense_host, mode):
    """A chunk whose corrections overflow its patch list is copied back whole (re-pitched to the caller's pitch)."""
    p, arrs, want = dense_host
    T.assert_results_equal(gpu.run_gpu(p, arrs, 160, mode=mode), want, 1, what=f"dense {mode}")


def test_host_patch_list_reports_incomplete(gpu, dense_host):
    p, arrs, want = dense_host
    n = arrs["seq1"].shape[0]
    ctx = gpu.GpuCtx(p, n, 160, 160)
    a = {k: v.copy() for k, v in arrs.items()}
    b = capi.batch_from_arrays(a)
    out1, out2 = np.zeros(n, capi.READ_RESULT_DTYPE), np.zeros(n, capi.READ_RESULT_DTYPE)
    ov = np.zeros(n, capi.OV_RESULT_DTYPE)
    cap = 16 * n
    hp = np.zeros(cap, capi.PATCH_DTYPE); hn = C.c_uint64()
    capi.check(ctx.lib.fp_process_pe_host_patches(ctx.h, C.byref(b), out1.ctypes.data, out2.ctypes.data, ov.ctypes.data, hp.ctypes.data, cap,
                                                  C.byref(hn)), ctx.lib)
    assert hn.value >= INCOMPLETE
    got = {"out1": out1, "out2": out2, "ov": ov, "counters": ctx.counters(), "arrs": a, "layout": ctx.L}
    T.assert_results_equal(got, want, 1, what="dense host_patches")
    ctx.close()


def test_packed_patch_overflow_is_an_error(gpu, dense_host):
    """fp_process_pe_host_packed returns corrections through the patch list only: when a chunk's list overflows it must fail, not
    return FP_OK with corrections missing from the list."""
    p, arrs, want = dense_host
    with pytest.raises(RuntimeError, match="patch list"):
        gpu.run_gpu(p, arrs, 160, mode="packed")


# ---------------- adapter events past the old chunk buffer ----------------
def concatemer_params(paired):
    p = T.config_params("fasta_adapters", paired)
    capi.set_params(p, adapter_seq_r1=None)                 # its 12 bases also start TRUSEQ_R2[:20]: it would cut three adapters at once
    return p


def sorted_events(ev):
    return np.sort(ev, order=["unit", "key"])


@pytest.mark.parametrize("paired", [1, 0])
def test_host_event_sink_with_many_events_per_unit(gpu, paired):
    """Concatemers of the five fasta adapters: 10 events per pair / 5 per read, over two host chunks.  The host list equals the
    device list (the device sink counts every event, and lists a valid prefix when its capacity is small), and the maps replayed
    from it equal the reference's."""
    import torch
    n, S = (1 << 18) + 5, 160
    p = concatemer_params(paired)
    arrs = E.adapter_concatemers(n, S, FASTA, np.random.default_rng(7 + paired), paired)
    ctx = gpu.GpuCtx(p, n, S, S)
    lib = ctx.lib
    dcap = (2 + 2 * len(FASTA) if paired else 1 + len(FASTA)) * n          # the most events the chain can make
    d_ev = torch.zeros(dcap * 16, dtype=torch.uint8, device="cuda:0"); d_n = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    capi.check(lib.fp_set_event_sink(ctx.h, d_ev.data_ptr(), dcap, d_n.data_ptr()), lib)
    dev = gpu.run_gpu(p, arrs, S, mode="device", ctx=ctx)
    nd = int(d_n.item())
    assert nd > 4 * (1 << 18) + 1024                                      # more than a host chunk buffered before
    dev_ev = sorted_events(d_ev.cpu().numpy().view(capi.EVENT_DTYPE)[:nd].copy())
    small_cap = 1000
    d_n.zero_()
    capi.check(lib.fp_set_event_sink(ctx.h, d_ev.data_ptr(), small_cap, d_n.data_ptr()), lib)
    gpu.run_gpu(p, arrs, S, mode="device", ctx=ctx)
    assert int(d_n.item()) == nd
    prefix = d_ev.cpu().numpy().view(capi.EVENT_DTYPE)[:small_cap]
    ukey = lambda e: (e["unit"].astype(np.uint64) << np.uint64(16)) | e["key"]      # noqa: E731  (unit, key) names one call
    at = np.searchsorted(ukey(dev_ev), ukey(prefix))
    assert (at < nd).all() and (dev_ev[np.minimum(at, nd - 1)] == prefix).all()
    capi.check(lib.fp_set_event_sink(ctx.h, None, 0, None), lib)
    h_ev = np.zeros(nd + 1024, capi.EVENT_DTYPE); h_n = C.c_uint64()
    capi.check(lib.fp_set_host_event_sink(ctx.h, h_ev.ctypes.data, h_ev.size, C.byref(h_n)), lib)
    host = gpu.run_gpu(p, arrs, S, mode="host", ctx=ctx)
    assert h_n.value == nd
    assert (sorted_events(h_ev[:nd]) == dev_ev).all()
    T.assert_results_equal(host, dev, paired, what="host vs device")
    if T.have_ref():
        want, wcnt = T.ref_adapter_maps(p, arrs, S)
        adapters = ["", ""] + FASTA
        maps = T.rebuild_adapter_maps(h_ev[:nd], host["arrs"], adapters)
        assert maps[0] == want[0]
        assert maps[1] == want[1]
        T.assert_counters_equal(host["counters"], wcnt, what="counters")
    ctx.close()
