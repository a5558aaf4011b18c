"""-m gpu: the CUDA over-representation scan (fp_overrep_kernel and the post-filter rank kernels) against the CPU port on the edge
inputs of tests/overrep_edges.py, bit-exact over the whole counter block: every case and option set in one launch and in three, launches
of 1-7 units with sampling steps larger than a launch, indexed and unindexed batches, fp_counters_reset between runs, the four host
entry points over more than one host chunk, the text path, the deferred post-filter protocol on uneven shards, and candidate lists
empty for one mate.  tests/test_oracle_overrep_edges.py pins the port to the reference's objects on the same inputs."""
import ctypes as C

import numpy as np
import pytest

import fp_testlib as T
import overrep_edges as O
from fastp_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def what(case, config, paired, extra=""):
    return f"{case}/{config}/{'PE' if paired else 'SE'}{extra}"


# ---------------- every case, one launch and three ----------------
def check_device(gpu, case, config, paired, sampling=1):
    p, arrs = O.overrep_case(case, paired, config, sampling)
    S = arrs["seq1"].shape[1]
    want = T.run_cpu("oracle", p, arrs, S)
    T.assert_results_equal(gpu.run_gpu(p, arrs, S), want, paired, what=what(case, config, paired))
    if not (paired and p.correction_enabled):                 # patch indices are batch-local: one launch per pass with correction
        T.assert_results_equal(gpu.run_gpu(p, arrs, S, splits=3), want, paired, what=what(case, config, paired, " 3 launches"))


@pytest.mark.parametrize("case,config", O.case_ids(1))
def test_device_pe(gpu, case, config):
    check_device(gpu, case, config, 1)


@pytest.mark.parametrize("case,config", O.case_ids(0))
def test_device_se(gpu, case, config):
    check_device(gpu, case, config, 0)


# ---------------- launch shapes and the sampling state ----------------
def small_launches(n, rng):
    b = [0]
    while b[-1] < n:
        b.append(min(n, b[-1] + int(rng.integers(1, 8))))
    return b


@pytest.mark.parametrize("sampling", [1, 2, 7, 20])
@pytest.mark.parametrize("case,paired,config", [("read_lengths", 1, "all_cuts"), ("skip_rule", 0, "cfg4_full"), ("trimmed_windows", 0, "all_cuts"),
                                                ("k0_side2", 1, "no_filters")])
def test_launches_of_1_to_7_units(gpu, case, paired, config, sampling):
    """Launches of 1-7 units: with sampling 7 and 20 most launches sample nothing.  Unindexed launches continue the context's own read
    count; then every other launch is indexed (FP_B_INDEXED, its true first index), which must give the same counts."""
    p, arrs = O.overrep_case(case, paired, config, sampling, n=300)
    want = T.run_cpu("oracle", p, arrs, 160)
    bounds = small_launches(300, np.random.default_rng(sampling))
    T.assert_results_equal(gpu.run_gpu(p, arrs, 160, bounds=bounds), want, paired, what=what(case, config, paired, " small launches"))
    T.assert_results_equal(gpu.run_gpu(p, arrs, 160, bounds=bounds, first_index=0, indexed=range(0, len(bounds), 2)), want, paired,
                           what=what(case, config, paired, " small launches, every other indexed"))


@pytest.mark.parametrize("sampling", [7, 20])
@pytest.mark.parametrize("paired", [1, 0])
def test_indexed_batch_not_on_a_sampling_step(gpu, paired, sampling):
    """A batch whose first_read_index (5) is no multiple of the step: pre-filter sampling by the global index.  The port sees the same
    rows behind five empty reads, which fail the length filter and so leave the post-filter rank alone; their own counts are taken
    back out."""
    first = 5
    p, arrs = O.overrep_case("read_lengths", paired, "all_cuts", sampling, n=600)
    lead = {k: np.zeros((first,) + v.shape[1:], v.dtype) for k, v in arrs.items()}
    both = {k: np.concatenate([lead[k], v]) for k, v in arrs.items()}
    whole, head = T.run_cpu("oracle", p, both, 160), T.run_cpu("oracle", p, lead, 160)
    want = {k: v[first:] for k, v in whole.items() if k in ("out1", "out2", "ov")}
    want.update(arrs={k: v[first:] for k, v in whole["arrs"].items()},
                counters=capi.CounterView(whole["layout"], whole["counters"].data - head["counters"].data))
    for bounds in ([0, 600], [0, 3, 4, 250, 600]):
        T.assert_results_equal(gpu.run_gpu(p, arrs, 160, bounds=bounds, first_index=first), want, paired, what=f"first index {first}, {bounds}")


@pytest.mark.parametrize("paired", [1, 0])
def test_a_few_tiles_and_counters_reset(gpu, paired):
    """One batch of several tiles, run twice on one context: fp_counters_reset before the second run restarts the pre-filter read count
    and the post-filter rank, so both runs equal the port."""
    p, arrs = O.overrep_case("read_lengths", paired, "all_cuts", 7, n=3000)
    want = T.run_cpu("oracle", p, arrs, 160)
    ctx = gpu.GpuCtx(p, 3000, 160, 160)
    for rep in range(2):
        T.assert_results_equal(gpu.run_gpu(p, arrs, 160, ctx=ctx, splits=1 if p.correction_enabled and paired else 2), want, paired, what=f"run {rep}")
    ctx.close()


# ---------------- host entry points over more than one host chunk ----------------
HOST_N = (1 << 18) + 40000


@pytest.fixture(scope="module")
def host_inputs():
    """read_lengths and k0 rows repeated past one 262 144-unit host chunk, sampling 50; port results cached per case."""
    out = {}
    for case, paired in (("read_lengths", 1), ("k0_side2", 1), ("read_lengths", 0), ("k0_side1", 0)):
        p, arrs = O.overrep_case(case, paired, "cfg4_full", 50, n=700)
        big = {k: np.ascontiguousarray(np.resize(v, (HOST_N,) + v.shape[1:])) for k, v in arrs.items()}
        out[(case, paired)] = (p, big, T.run_cpu("oracle", p, big, 160))
    return out


@pytest.mark.parametrize("mode", ["host", "host_tight", "host_pack2bit", "packed"])
@pytest.mark.parametrize("case,paired", [("read_lengths", 1), ("k0_side2", 1), ("read_lengths", 0), ("k0_side1", 0)])
def test_host_entry_points(gpu, host_inputs, case, paired, mode):
    p, arrs, want = host_inputs[(case, paired)]
    assert sum(int(want["counters"].overrep(s)[0].sum()) for s in range(4 if paired else 2)) > 0 or case.startswith("k0")
    T.assert_results_equal(gpu.run_gpu(p, arrs, 160, mode=mode), want, paired, what=f"{case} {mode}")


# ---------------- the text path ----------------
def text_pipeline(p, texts):
    """Port decode -> port chain -> port encode of whole texts: (outputs, units, counters)."""
    dec = [T.oracle_fastq_decode(t, stride=160, capacity=t.count(b"\n") // 4 + 2) for t in texts]
    n = min(int(d["info"]["n_records"]) for d in dec)
    arrs = {}
    for k, d in enumerate(dec):
        sd = str(k + 1)
        arrs["seq" + sd], arrs["qual" + sd], arrs["len" + sd] = d["seq"][:n].copy(), d["qual"][:n].copy(), d["len"][:n].copy()
    r = T.run_cpu("oracle", p, arrs, 160)
    outs = [T.oracle_fastq_encode(t, d["recs"][:n], r["out" + str(k + 1)], r["arrs"]["seq" + str(k + 1)], r["arrs"]["qual" + str(k + 1)], 160)
            for k, (t, d) in enumerate(zip(texts, dec))]
    return outs, n, r["counters"]


@pytest.mark.parametrize("sampling", [1, 7])
@pytest.mark.parametrize("case,paired", [("read_lengths", 1), ("k0_side2", 1), ("skip_rule", 1), ("read_lengths", 0), ("k0_side1", 0),
                                         ("trimmed_windows", 0)])
def test_text_path(gpu, case, paired, sampling):
    """fp_fastq_process_host in rounds of 250 units: outputs and the counter block (over-representation regions included) equal the
    port's decode -> chain -> encode of the same text."""
    p, arrs = O.overrep_case(case, paired, "cfg4_full", sampling, n=1100)
    texts = [T.fastq_text(arrs["seq" + sd], arrs["qual" + sd], arrs["len" + sd], sd + ":N:0") for sd in ("1", "2")[: 2 if paired else 1]]
    outs, n, cnt = text_pipeline(p, texts)
    assert n == 1100
    ctx = gpu.GpuCtx(p, 250, 160, 160)
    got = gpu.gpu_fastq_process_host(ctx, *texts)
    assert got["n"] == n and got["guard_ok"]
    for k, o in enumerate(outs):
        assert got["out%d" % (k + 1)] == o, k
    T.assert_counters_equal(ctx.counters(), cnt, f"text {case}")
    ctx.close()


# ---------------- deferred post-filter scan on uneven shards ----------------
@pytest.mark.parametrize("sampling", [1, 7])
@pytest.mark.parametrize("case", ["read_lengths", "k0_side2", "dense_correction"])
def test_deferred_post_on_uneven_shards(gpu, case, sampling):
    """fp_overrep_defer_post / fp_pass_count / fp_overrep_post over shards of 1, 2 and the rest of the units (first_read_index
    indexed): the sum of the shards' counter blocks equals the port's block of the whole stream."""
    import torch
    p, arrs = O.overrep_case(case, 1, "cfg3_overlap_correction", sampling, n=500)
    S = arrs["seq1"].shape[1]
    want = T.run_cpu("oracle", p, arrs, S)
    n = arrs["seq1"].shape[0]
    bounds = [0, 1, 3, 4 + n // 3, n]
    total = None
    base = 0
    shards = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        ctx = gpu.GpuCtx(p, hi - lo, S, S)
        capi.check(ctx.lib.fp_overrep_defer_post(ctx.h, 1), ctx.lib)
        b, t = gpu.device_batch({k: np.ascontiguousarray(v[lo:hi]) for k, v in arrs.items()})
        b.flags, b.first_read_index = capi.FP_B_INDEXED, lo
        d = {k: torch.zeros((hi - lo) * w, dtype=torch.uint8, device="cuda:0") for k, w in (("out1", 16), ("out2", 16), ("ov", 8))}
        capi.check(ctx.lib.fp_process_pe(ctx.h, C.byref(b), d["out1"].data_ptr(), d["out2"].data_ptr(), d["ov"].data_ptr(), None, 0, None, None), ctx.lib)
        c = C.c_int64()
        capi.check(ctx.lib.fp_pass_count(ctx.h, d["out1"].data_ptr(), hi - lo, C.byref(c), None), ctx.lib)
        shards.append((ctx, b, t, d, c.value))
    for ctx, b, t, d, c in shards:
        capi.check(ctx.lib.fp_overrep_post(ctx.h, C.byref(b), d["out1"].data_ptr(), d["out2"].data_ptr(), base, None), ctx.lib)
        base += c
        blk = ctx.counters().data
        total = blk if total is None else total + blk
    assert base == int(want["counters"].stats(capi.STATS_POST1)["reads"])
    T.assert_counters_equal(capi.CounterView(shards[0][0].L, total), want["counters"], what=f"{case} shards, sampling {sampling}")
    for s in shards:
        s[0].close()
