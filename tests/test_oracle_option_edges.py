"""Pins the plain-C port (oracle/fastp_oracle.c) against the reference's own objects (oracle/_ref/libfastp_ref.so) on the option
sets of tests/option_edges.py -- every option at the ends of its accepted range -- over two inputs each: the edge batch of
tests/edge_inputs.py and reads that sit exactly on the set's thresholds.  PE at strides 48 / 160 / 256, SE at 160 / 512, merging
sets at 2·S cycles.  tests/test_gpu_option_edges.py compares the CUDA path with the port on the same sets and inputs, so this is
what makes the port a valid comparator there.  The threshold reads are also checked to land on both sides of each limit."""
import pytest

import edge_inputs as E
import fp_testlib as T
import option_edges as O

needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built (needs the reference sources)")

PE_STRIDES = [48, 160, 256]
SE_STRIDES = [160, 512]
PE_SETS = sorted(O.option_edge_sets(1))
SE_SETS = sorted(O.option_edge_sets(0))


def inputs(name, paired, S, n=600):
    p = O.edge_params(name, paired, S)
    yield p, "edge", E.edge_batch(n, S, paired, 5 + S, p, read_len=O.read_len(S))
    arrs, _ = O.threshold_batch(p, S, paired, 7 + S)
    yield p, "threshold", arrs


def check(name, paired, S):
    cycles = O.cycles_for(name, S)
    for p, gen, arrs in inputs(name, paired, S):
        x = T.run_cpu("oracle", p, arrs, cycles)
        y = T.run_cpu("ref", p, arrs, cycles)
        T.assert_results_equal(x, y, paired, skip=("adapter_pos",), what=f"{name}/{gen}/S{S}")


@pytest.mark.reference
@needs_ref
@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", PE_SETS)
def test_port_equals_reference_option_edges_pe(name, S):
    check(name, 1, S)


@pytest.mark.reference
@needs_ref
@pytest.mark.parametrize("S", SE_STRIDES)
@pytest.mark.parametrize("name", SE_SETS)
def test_port_equals_reference_option_edges_se(name, S):
    check(name, 0, S)


def assert_both_sides(name, oc, S):
    """Every predicate the set checks saw reads on its limit come out on the limit's side and reads one past it come out on the other;
    at least half of each group did (the rest met another operator first: a chance overlap, a trim of the mate)."""
    for kind in O.threshold_checks(name, S):
        assert kind in oc, f"{name}/S{S}: no {kind} threshold reads"
        on_ok, on_n, past_ok, past_n = oc[kind]
        assert on_ok >= 1 and past_ok >= 1, f"{name}/S{S} {kind}: on the limit {on_ok}/{on_n}, one past {past_ok}/{past_n}"
        assert 2 * on_ok >= on_n and 2 * past_ok >= past_n, f"{name}/S{S} {kind}: on the limit {on_ok}/{on_n}, one past {past_ok}/{past_n}"


@pytest.mark.parametrize("paired,S", [(1, 48), (1, 160), (1, 256), (0, 160), (0, 512)])
@pytest.mark.parametrize("name", sorted(O.THRESHOLD_CHECKS))
def test_threshold_reads_land_on_both_sides(name, paired, S):
    sets = O.option_edge_sets(paired)
    if name not in sets or not O.threshold_checks(name, S):
        pytest.skip("paired-end option set, or a limit that does not fit the stride")
    p = O.edge_params(name, paired, S)
    arrs, labels = O.threshold_batch(p, S, paired, 7 + S)
    x = T.run_cpu("oracle", p, arrs, O.cycles_for(name, S))
    assert_both_sides(name, O.boundary_outcomes(labels, x, paired), S)


def test_every_branch_and_range_end_has_a_set():
    """The set names cover each kernel branch the grid targets and both ends of every option's accepted range."""
    pe, se = O.option_edge_sets(1), O.option_edge_sets(0)
    names = " ".join(pe) + " " + " ".join(se)
    for tag in ("cut_right.plane4.", "cut_right.plane4_dp4a.", "cut_right.scalar.", "polyg.plane_off", "polyx.plane", "polyx.scan",
                "overlap.filter_req_le1", "overlap.filter_narrow", "overlap.filter_wide", "thr_gt32", "isize.global", "isize.smem",
                "merge.filter.", "mergeu.filter.", "merge.overlap.", "mergeu.overlap.", "tid1."):
        assert tag in names, tag
    vals = {}
    for kw in list(pe.values()) + list(se.values()):
        for k, v in O.resolve(kw, 160, 150).items():
            vals.setdefault(k, set()).add(v)
    ends = {"cut_front_window": (1, 1000), "cut_tail_window": (1, 1000), "cut_right_window": (1, 1000),
            "cut_front_quality": (1, 30), "cut_right_quality": (1, 30), "polyg_min_len": (0, 161), "polyx_min_len": (0, 161),
            "qualified_qual": (33, 33 + 93), "unqualified_percent_limit": (0, 100), "avg_qual_req": (1, 93), "n_base_limit": (0, 50),
            "complexity_threshold": (0.0, 1.0), "overlap_require": (0, 151), "overlap_diff_limit": (0, 1000),
            "overlap_diff_percent_limit": (0, 100), "trim_front1": (149, 160), "max_len1": (1, 160), "insert_size_max": (0, 4096),
            "length_required": (0, 161), "length_limit": (1, 160), "dimer_max_len": (0, 160)}
    for k, (lo, hi) in ends.items():
        assert lo in vals[k] and hi in vals[k], (k, sorted(vals[k]))
