"""-m gpu: the CUDA path against the CPU oracle on the option sets of tests/option_edges.py (every option at the ends of its accepted
range, each set named after the kernel branch it targets), bit-exact: records, overlap records, corrected rows, the whole counter
block.  Two inputs per set: the edge batch and reads that sit exactly on the set's thresholds.  Device mode at PE strides 48 / 160 /
256 and SE 160 / 512 (merging sets at 2·S cycles), the host entry point at the tight pitch for the threshold sets, and a batch of
several tiles per CTA for the insert-size sets, so that many CTAs add to the same insert-size bins.  tests/test_oracle_option_edges.py
pins the oracle to the reference's objects on the same sets and inputs."""
import pytest

import edge_inputs as E
import fp_testlib as T
import option_edges as O
from test_gpu_edges import multi_tile_n
from test_oracle_option_edges import PE_SETS, PE_STRIDES, SE_SETS, SE_STRIDES, assert_both_sides

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def check(gpu, name, paired, S, mode="device"):
    p = O.edge_params(name, paired, S)
    cycles = O.cycles_for(name, S)
    edge = E.edge_batch(600, S, paired, 5 + S, p, read_len=O.read_len(S))
    thr, labels = O.threshold_batch(p, S, paired, 7 + S)
    n = max(len(edge["len1"]), len(thr["len1"]))
    ctx = gpu.GpuCtx(p, n, S, cycles)
    try:
        for gen, arrs in (("edge", edge), ("threshold", thr)):
            if mode == "host_tight" and gen == "edge":
                continue
            want = T.run_cpu("oracle", p, arrs, cycles)
            got = gpu.run_gpu(p, arrs, cycles, mode=mode, ctx=ctx)
            T.assert_results_equal(got, want, paired, what=f"{name}/{gen}/S{S}/{mode}")
            if gen == "threshold" and O.threshold_checks(name, S):
                assert_both_sides(name, O.boundary_outcomes(labels, got, paired), S)
    finally:
        ctx.close()


@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", PE_SETS)
def test_option_edges_pe(gpu, name, S):
    check(gpu, name, 1, S)


@pytest.mark.parametrize("S", SE_STRIDES)
@pytest.mark.parametrize("name", SE_SETS)
def test_option_edges_se(gpu, name, S):
    check(gpu, name, 0, S)


@pytest.mark.parametrize("name,paired", [(k, pr) for pr in (1, 0) for k in sorted(O.THRESHOLD_CHECKS) if k in O.option_edge_sets(pr)])
def test_option_edges_host_tight(gpu, name, paired):
    """The threshold reads through fp_process_*_host at the pitch of the longest read."""
    check(gpu, name, paired, 160, mode="host_tight")


@pytest.mark.parametrize("name", [k for k in PE_SETS if k.startswith("isize.")])
def test_insert_size_sets_over_many_tiles(gpu, name):
    """insert_size_max on both sides of FP_MAX_ISIZE_SMEM (1025): below it the bins are counted in shared memory and flushed per CTA,
    from it on every insert size goes to the global bins directly; several tiles per CTA add to the same bins either way."""
    S = 160
    p = O.edge_params(name, 1, S)
    arrs = E.edge_batch(multi_tile_n(), S, 1, 41, p, read_len=O.read_len(S))
    T.assert_results_equal(gpu.run_gpu(p, arrs, S), T.run_cpu("oracle", p, arrs, S), 1, what=f"{name} multi-tile")
