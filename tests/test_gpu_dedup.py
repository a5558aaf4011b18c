"""-m gpu: --dedup in the chain kernel (fp_set_dup_flags -> FP_F_DUPLICATE) against the C port (fp_oracle_process_dedup, pinned to the
reference's objects by tests/test_oracle_dedup.py), bit-exact on records, overlap records, corrected rows and the whole counter
block; what the host entry points do with a set flag pointer; and the duplicate filter itself beyond one shape, one accuracy level
at a time in a child process (tests/_gpu_dup_cases_worker.py) so that its bit arrays are gone before the next one starts."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import fp_testlib as T
from fastp_b200 import capi
from test_gpu_edges import grid_input, multi_tile_n

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
FP_F_MERGED, FP_F_DUPLICATE, FP_FR_MERGED_PAIRS = 0x80, 0x40, 107
PATTERNS = ["none", "all", "random", "passing", "failing"]
GRID = ([(name, 1, 160) for name in T.CONFIG_NAMES] + [(name, 0, 160) for name in T.CONFIG_NAMES] +
        [(name, 1, S) for name in ("cfg4_full", "all_cuts") for S in (48, 256)] + [(name, 0, 512) for name in ("cfg4_full", "all_cuts")] +
        [(name, 1, 128) for name in T.MERGE_CONFIG_NAMES])


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def cycles_of(name, S):
    return 2 * S if name.startswith("merge") else S


def flag_pattern(kind, plain, seed):
    """Flags over the units of `plain` (the unflagged C-port result): none / all / 30 % at random / exactly the units whose pair
    verdict is PASS / exactly the others."""
    n = len(plain["out1"])
    ok = plain["out1"]["pair_verdict"] == 0
    if kind == "none":
        return np.zeros(n, np.uint8)
    if kind == "all":
        return np.ones(n, np.uint8)
    if kind == "random":
        return (np.random.default_rng(seed).random(n) < 0.3).astype(np.uint8)
    return (ok if kind == "passing" else ~ok).astype(np.uint8)


@pytest.mark.parametrize("name,paired,S", GRID)
def test_chain_with_duplicate_flags(gpu, name, paired, S):
    p, arrs = grid_input(name, paired, S)
    cyc = cycles_of(name, S)
    plain = T.run_cpu("oracle", p, arrs, cyc)
    assert 0 < (plain["out1"]["pair_verdict"] == 0).sum() < len(plain["out1"])
    ctx = gpu.GpuCtx(p, len(arrs["len1"]), S, cyc)
    for kind in PATTERNS:
        f = flag_pattern(kind, plain, S)
        want = T.run_cpu("oracle", p, arrs, cyc, is_dup=f)
        got = gpu.run_gpu(p, arrs, cyc, ctx=ctx, is_dup=f)
        T.assert_results_equal(got, want, paired, what=f"{name}/{'PE' if paired else 'SE'}/S{S}/{kind}")
        assert np.array_equal(got["out1"]["flags"] & FP_F_DUPLICATE != 0, f != 0)
    T.assert_results_equal(gpu.run_gpu(p, arrs, cyc, ctx=ctx), plain, paired, what=f"{name}: flags cleared")   # after fp_set_dup_flags(NULL)
    ctx.close()


@pytest.mark.parametrize("n", [1, 7, "multi_tile"])
@pytest.mark.parametrize("name,paired,S", [("cfg4_full", 1, 160), ("all_cuts", 0, 512), ("mergeu_all_cuts", 1, 128)])
def test_batch_shapes_with_flags(gpu, name, paired, S, n):
    n = multi_tile_n() if n == "multi_tile" else n
    p, arrs = grid_input(name, paired, S, n=n, seed=n % 1000 + 1)
    f = (np.random.default_rng(n).random(n) < 0.5).astype(np.uint8)
    f[0] = 1
    cyc = cycles_of(name, S)
    T.assert_results_equal(gpu.run_gpu(p, arrs, cyc, is_dup=f), T.run_cpu("oracle", p, arrs, cyc, is_dup=f), paired, what=f"{name} n={n}")


@pytest.mark.parametrize("name,paired", [("all_cuts", 1), ("cfg4_full", 0)])
def test_flags_follow_three_launches(gpu, name, paired):
    """Three launches into one counter block; the flag pointer is moved to each launch's first unit.  The thirds are flagged
    differently (none / all / every other unit), so flags read at the wrong offset change the answer."""
    n, S = multi_tile_n(), 160
    p, arrs = grid_input(name, paired, S, n=n, seed=3)
    f = np.zeros(n, np.uint8)
    f[n // 3: 2 * n // 3] = 1
    f[2 * n // 3::2] = 1
    cyc = cycles_of(name, S)
    T.assert_results_equal(gpu.run_gpu(p, arrs, cyc, splits=3, is_dup=f), T.run_cpu("oracle", p, arrs, cyc, is_dup=f), paired, what=f"{name} 3 launches")


def test_merged_duplicates_are_counted_and_unmerged_ones_are_not(gpu):
    """src/peprocessor.cpp:528-534 against :547 / :553, with every pair flagged."""
    p, arrs = grid_input("mergeu_cfg3_overlap_correction", 1, 128, n=4000)
    plain = T.run_cpu("oracle", p, arrs, 256)
    merged_ok = (plain["out1"]["flags"] & FP_F_MERGED != 0) & (plain["out1"]["pair_verdict"] == 0)
    unmerged = plain["out1"]["flags"] & FP_F_MERGED == 0
    unmerged_reads = int((unmerged & (plain["out1"]["verdict"] == 0)).sum() + (unmerged & (plain["out2"]["verdict"] == 0)).sum())
    assert merged_ok.sum() > 100 and unmerged_reads > 100        # the input holds both kinds
    assert plain["counters"].stats(1)["reads"] == int(merged_ok.sum()) + unmerged_reads
    f = np.ones(4000, np.uint8)
    got = gpu.run_gpu(p, arrs, 256, is_dup=f)
    T.assert_results_equal(got, T.run_cpu("oracle", p, arrs, 256, is_dup=f), 1, what="all flagged")
    assert got["counters"].stats(1)["reads"] == int(merged_ok.sum())          # every merged read still counted, no unmerged one
    assert got["counters"].filter[FP_FR_MERGED_PAIRS] == int(merged_ok.sum())
    assert np.array_equal(got["counters"].filter, plain["counters"].filter)   # FilterResult does not see the flags


@pytest.mark.parametrize("mode", ["host", "host_tight", "host_pack2bit", "packed"])
@pytest.mark.parametrize("paired", [1, 0])
def test_host_entry_points_refuse_a_set_flag_pointer(gpu, paired, mode):
    """include/fastp_b200.h: a flag array belongs to one launch; the host entry points return FP_E_INVAL while one is set, write
    nothing, and work again once it is cleared."""
    import torch
    p, arrs = grid_input("cfg4_full", paired, 160, n=3000, seed=5, max_len=150)
    ctx = gpu.GpuCtx(p, 3000, 160, 160)
    d = torch.ones(3000, dtype=torch.uint8, device="cuda:0")
    capi.check(ctx.lib.fp_set_dup_flags(ctx.h, d.data_ptr()), ctx.lib)
    with pytest.raises(RuntimeError, match="duplicate flags"):
        gpu.run_gpu(p, arrs, 160, mode=mode, ctx=ctx)
    assert not ctx.counters().data.any()
    if mode == "host":
        t = T.fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1")
        with pytest.raises(RuntimeError, match="duplicate flags"):
            gpu.gpu_fastq_process_host(ctx, t, t if paired else None)
    capi.check(ctx.lib.fp_set_dup_flags(ctx.h, None), ctx.lib)
    T.assert_results_equal(gpu.run_gpu(p, arrs, 160, mode=mode, ctx=ctx), T.run_cpu("oracle", p, arrs, 160), paired, what="cleared")
    ctx.close()


# ---------------- the duplicate filter, one accuracy level per child process ----------------
@pytest.mark.parametrize("level", [1, 2, 3])
def test_duplicate_filter_shapes(level):
    r = subprocess.run([sys.executable, os.path.join(HERE, "_gpu_dup_cases_worker.py"), str(level)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-2500:], r.stderr[-1500:])
    assert r.stdout.count("ok:") == 5, r.stdout[-2500:]
