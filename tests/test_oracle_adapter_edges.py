"""Pins the plain-C port (oracle/fastp_oracle.c) against the reference's own objects (oracle/_ref/libfastp_ref.so) on the adapter
shapes and lists of tests/adapter_edges.py: every adapter length, alphabet and list size the device trimmer branches on, with reads
planted on both sides of each limit of scan 1, its tail, and the one-gap scans 2 / 3.  SE at strides 160 / 512, PE at 160 / 256:
records, rows, the whole counter block and the reference's adapter-string maps.  tests/test_gpu_adapter_edges.py compares the CUDA
path with the port on the same inputs, so this is what makes the port a valid comparator there.  The planted reads are also checked
to land on both sides of each limit."""
import numpy as np
import pytest

import adapter_edges as A
import fp_testlib as T

needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built (needs the reference sources)")

SE_STRIDES = [160, 512]
PE_STRIDES = [160, 256]
SE_CASES = sorted(A.adapter_cases(0))
PE_CASES = sorted(A.adapter_cases(1))


def check(name, paired, S):
    p = A.case_params(name, paired)
    arrs, _ = A.case_batch(name, paired, S, 3 + S)
    x = T.run_cpu("oracle", p, arrs, S)
    y = T.run_cpu("ref", p, arrs, S)
    T.assert_results_equal(x, y, paired, skip=("adapter_pos",), what=f"{name}/S{S}")
    maps, cnt = T.ref_adapter_maps(p, arrs, S)
    T.assert_counters_equal(x["counters"], cnt, what=f"{name}/S{S} maps pass")
    if A.checked_kinds(name):
        assert all(maps[k] for k in range(1 + paired)), f"{name}/S{S}: no adapter string recorded"


@pytest.mark.reference
@needs_ref
@pytest.mark.parametrize("S", SE_STRIDES)
@pytest.mark.parametrize("name", SE_CASES)
def test_port_equals_reference_adapter_edges_se(name, S):
    check(name, 0, S)


@pytest.mark.reference
@needs_ref
@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", PE_CASES)
def test_port_equals_reference_adapter_edges_pe(name, S):
    check(name, 1, S)


@pytest.mark.reference
@needs_ref
def test_port_equals_reference_many_trims_per_read():
    """The 40-entry list of 6-mers whose concatemers trim about 40 times per read (the GPU test's many-events input)."""
    p, arrs = A.many_trims_input(600, T.oracle())
    x = T.run_cpu("oracle", p, arrs, 256)
    T.assert_results_equal(x, T.run_cpu("ref", p, arrs, 256), 1, skip=("adapter_pos",), what="many trims")
    maps, _ = T.ref_adapter_maps(p, arrs, 256)
    assert sum(sum(m.values()) for m in maps) > 62 * 600


def assert_both_sides(name, oc, what):
    """Every class the case checks saw reads on its limit trimmed to the planted length and reads one past it not trimmed there; at
    least half of each group (the rest met another position or adapter first by chance)."""
    for kind in A.checked_kinds(name):
        assert kind in oc, f"{what}: no {kind} reads planted"
        on_ok, on_n, past_ok, past_n = oc[kind]
        assert on_ok >= 1 and past_ok >= 1, f"{what} {kind}: on the limit {on_ok}/{on_n}, one past {past_ok}/{past_n}"
        assert 2 * on_ok >= on_n and 2 * past_ok >= past_n, f"{what} {kind}: on the limit {on_ok}/{on_n}, one past {past_ok}/{past_n}"


@pytest.mark.parametrize("paired,S", [(0, 160), (0, 512), (1, 160), (1, 256)])
def test_planted_reads_land_on_both_sides(paired, S):
    for name in sorted(A.adapter_cases(paired)):
        if not A.checked_kinds(name):
            continue
        p = A.case_params(name, paired)
        arrs, labels = A.case_batch(name, paired, S, 3 + S)
        x = T.run_cpu("oracle", p, arrs, S)
        assert_both_sides(name, A.boundary_outcomes(labels, x, paired), f"{name}/S{S}")


def test_every_shape_and_list_size_has_a_case():
    """The cases reach each branch of the trimmer: lengths below matchReq, every A-tail start, one to eight plane words, both sides
    of the 64-bit fields, the N plane, the byte path, and fasta lists on both sides of matchReq's two steps."""
    lens = {len(a) for a in A.SHAPES.values()}
    for L in A.LENGTHS:
        assert L in lens
    assert any(any(c not in "ACGTN" for c in a) for a in A.SHAPES.values())
    for pos in (0, 31, 32, 63, 64):
        assert any(len(a) > pos and a[pos] == "N" for a in A.SHAPES.values()), pos
    assert any(a.endswith("N") for a in A.SHAPES.values())
    sizes = {len(c["kw"]["fasta_adapters"]) for c in A.adapter_cases(1).values() if "fasta_adapters" in c["kw"]}
    for n in A.LIST_SIZES:
        assert n in sizes
    items = A.LISTS["list512"]
    assert len(set(items)) < len(items)                                  # a repeated entry
    a64 = A.SHAPES["rand64"]
    assert a64[63] != "A"
    arrs, labels = A.case_batch("seq.rand64", 0, 160, 163)
    gap = (labels["1"]["kind"] == A.K["gap2"])
    assert gap.any() and (arrs["seq1"][gap, 64] == ord(a64[63])).all()   # read[64] == adapter[63] on the insertion reads


def test_port_trims_the_64_base_one_gap_reads():
    """The case the device's one-gap quick reject got wrong at 64 bases (DESIGN §3): the port trims the insertion reads that hold
    exactly 64/8 - 1 mismatches to length 0."""
    arrs, labels = A.case_batch("seq.rand64", 0, 160, 163)
    x = T.run_cpu("oracle", A.case_params("seq.rand64", 0), arrs, 160)
    sel = (labels["1"]["kind"] == A.K["gap2"]) & (labels["1"]["at"] == 0) & (arrs["len1"] >= 65)
    assert sel.sum() >= 8
    assert (x["out1"]["len"][sel] == 0).mean() >= 0.5
    assert np.count_nonzero(x["out1"]["len"][sel] == 0) >= 8
