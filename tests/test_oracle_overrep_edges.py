"""The over-representation scan of the plain-C port (oracle/fastp_oracle.c) on the edge inputs of tests/overrep_edges.py: against a
plain Python restatement of Stats::statRead's scan (src/stats.cpp:270-288) on the pre-filter stats, and against the reference's
own objects (oracle/_ref/libfastp_ref.so) on everything, counter block included.  tests/test_gpu_overrep_edges.py compares the CUDA
scan with the port on the same inputs, so this is what makes the port a valid comparator there."""
import numpy as np
import pytest

import fp_testlib as T
import overrep_edges as O
from fastp_b200 import capi

needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built (needs /root/reference)")


def py_scan(seq, lens, cands, seq_len, sampling, first=0):
    """Stats::statRead's scan over the rows of one side, read i sampled when (first + i) % sampling == 0: (count[K], dist[K][seq_len])."""
    index = {c: k for k, c in enumerate(cands)}
    K = len(cands)
    count = np.zeros(K, np.int64)
    dist = np.zeros((K, seq_len), np.int64)
    steps = (10, 20, 40, 100, min(150, seq_len - 2))
    for r in range(seq.shape[0]):
        if (first + r) % sampling:
            continue
        s = seq[r, :int(lens[r])].tobytes()
        for step in steps:
            i = 0
            while i < len(s) - step:
                k = index.get(s[i:i + step])
                if k is not None:
                    count[k] += 1
                    dist[k, i:min(i + step, seq_len)] += 1
                    i += step
                i += 1
    return count, dist


def check_pre_filter(x, arrs, p, paired):
    for k, sd in enumerate(("1", "2")[: 2 if paired else 1]):
        cands = [c for c in (p._overrep_keepalive["overrep_seqs" + sd][1] if ("overrep_seqs" + sd) in p._overrep_keepalive else [])]
        seq_len = p.seq_len2 if k else p.seq_len1
        c, d = py_scan(arrs["seq" + sd], arrs["len" + sd], cands, seq_len, p.overrep_sampling)
        xc, xd = x["counters"].overrep(2 * k)
        assert np.array_equal(xc, c), f"pre{sd} count"
        assert np.array_equal(xd, d), f"pre{sd} dist"
    return x


# ---------------- the port against the Python restatement (runs without the reference build) ----------------
@pytest.mark.parametrize("case,paired", [(c, pe) for c, (pe_only, _) in O.CASES.items() for pe in (1, 0) if pe or not pe_only])
def test_port_pre_filter_scan_equals_python(case, paired):
    cfg = O.CASES[case][1][0] if O.CASES[case][1] else "no_filters"
    p, arrs = O.overrep_case(case, paired, cfg)
    check_pre_filter(T.run_cpu("oracle", p, arrs, arrs["seq1"].shape[1]), arrs, p, paired)


def test_collision_pair_hashes_alike():
    """COLLISION_X != COLLISION_Y, one length, one scan hash (the table keeps both in one probe chain); reversed they hash apart, so
    the equality is the lattice's doing and not a hash that ignores byte order."""
    X, Y = O.COLLISION_X, O.COLLISION_Y
    assert X != Y and len(X) == len(Y) == 10
    assert O.scan_hash(X) == O.scan_hash(Y)
    assert O.scan_hash(X[::-1]) != O.scan_hash(Y[::-1])
    assert all(33 <= c <= 126 for c in X + Y) and not set(X + Y) <= set(b"ACGTN")


def test_collision_counts_each_string_under_its_own_index():
    for case, paired in (("collision_x_only", 0), ("collision_both", 1)):
        p, arrs = O.overrep_case(case, paired, "no_filters")
        x = check_pre_filter(T.run_cpu("oracle", p, arrs, 160), arrs, p, paired)
        cands = p._overrep_keepalive["overrep_seqs1"][1]
        cnt = x["counters"].overrep(capi.STATS_PRE1)[0]
        assert cnt[cands.index(O.COLLISION_X)] > 0
        if case == "collision_both":
            assert cnt[cands.index(O.COLLISION_Y)] > 0


def test_case_sizes_reach_the_table_branches():
    """K = 1 gets the smallest table; 2048 and 2049 reach the 32 768-slot cap of the occupancy bitmap, 8192 still fits in it and
    8193 folds it (slot & 32767); the K = 0 sides are empty."""
    assert O.table_size(1) == 64
    assert O.table_size(2048) == O.table_size(2049) == O.table_size(8192) == O.TABLE_BITMAP_BITS
    assert O.table_size(8193) > O.TABLE_BITMAP_BITS and O.table_size(20000) > O.TABLE_BITMAP_BITS
    for case, K in (("k1", 1), ("k2049", 2049), ("k8193", 8193), ("k20000", 20000)):
        _, cands, _ = O.overrep_inputs(case, 1)
        assert [len(c) for c in cands] == [K, K] and all(len(set(c)) == K for c in cands)
    _, cands, _ = O.overrep_inputs("k0_side2", 1)
    assert len(cands[0]) > 0 and cands[1] == []


def test_loop_bound_and_eval_len_clip():
    """A candidate that is exactly a read's last `step` bases is not counted (the loop is i < len - step); one base earlier it is.  With
    seq_len 60 on 150-base reads the dist stops at position 59."""
    rng = np.random.default_rng(9)
    reads = [rng.choice(O.E.ACGT, 150).tobytes() for _ in range(4)]
    c = reads[0][140:150]
    reads[1] = reads[1][:139] + c + reads[1][149:]
    reads[2] = reads[2][:55] + c + reads[2][65:]
    b, arrs = capi.batch_from_strings([(s, b"I" * len(s)) for s in reads], stride=160)
    p = O.with_overrep(T.config_params("no_filters", 0), [[c], []], (60, 60), 1, 0)
    for which in ("oracle", "ref") if T.have_ref() else ("oracle",):
        cnt, dist = T.run_cpu(which, p, arrs, 160)["counters"].overrep(capi.STATS_PRE1)
        assert cnt.tolist() == [2], which
        assert dist[0].tolist() == [0] * 55 + [1] * 5, which


# ---------------- the port against the reference's objects ----------------
def check_ref(case, config, paired, sampling=1):
    p, arrs = O.overrep_case(case, paired, config, sampling)
    S = arrs["seq1"].shape[1]
    x = T.run_cpu("oracle", p, arrs, S)
    y = T.run_cpu("ref", p, arrs, S)
    T.assert_results_equal(x, y, paired, skip=("adapter_pos",), what=f"{case}/{config}/{'PE' if paired else 'SE'}/sampling {sampling}")
    if case not in ("k0_side1", "k0_both"):                   # the planted candidates are found before and after the filters
        assert int(x["counters"].overrep(capi.STATS_PRE1)[0].sum()) > 0 and int(x["counters"].overrep(capi.STATS_POST1)[0].sum()) > 0
    return x


@needs_ref
@pytest.mark.reference
@pytest.mark.parametrize("case,config", O.case_ids(1))
def test_port_equals_reference_overrep_edges_pe(case, config):
    check_ref(case, config, 1)


@needs_ref
@pytest.mark.reference
@pytest.mark.parametrize("case,config", O.case_ids(0))
def test_port_equals_reference_overrep_edges_se(case, config):
    check_ref(case, config, 0)


@needs_ref
@pytest.mark.reference
@pytest.mark.parametrize("sampling", [2, 7, 20])
@pytest.mark.parametrize("case,paired", [("read_lengths", 1), ("skip_rule", 0), ("trimmed_windows", 1), ("k8193", 0)])
def test_port_equals_reference_overrep_sampling(case, paired, sampling):
    check_ref(case, "all_cuts", paired, sampling)


@needs_ref
@pytest.mark.reference
def test_dense_correction_pre_and_post_see_different_bases():
    """Around a corrected base, the pre-filter scan counts the original 20 bases and never the corrected ones; the post-filter scan the
    other way round."""
    arrs, cands, orig, corr = O.dense_correction_candidates(400, np.random.default_rng(O.hash_name("dense_correction") + 1))
    p = O.with_overrep(T.config_params("cfg3_overlap_correction", 1), cands, (150, 150), 1, 1)
    x = T.run_cpu("oracle", p, arrs, 160)
    T.assert_results_equal(x, T.run_cpu("ref", p, arrs, 160), 1, skip=("adapter_pos",), what="dense correction")
    for k in range(2):
        pre, post = x["counters"].overrep(2 * k)[0], x["counters"].overrep(2 * k + 1)[0]
        io = [cands[k].index(c) for c in orig[k]]
        ic = [cands[k].index(c) for c in corr[k]]
        assert pre[io].sum() > 0 and post[io].sum() == 0
        assert pre[ic].sum() == 0 and post[ic].sum() > 0
