"""Pins the plain-C port (oracle/fastp_oracle.c) against the reference's own objects (oracle/_ref/libfastp_ref.so) on the
edge inputs of tests/edge_inputs.py: quality bytes over all of [33, 126], lengths up to the full row stride, correction-dense
pairs and adapter concatemers, at strides 48 to 512.  The GPU edge tests compare the CUDA path with the oracle on the same
generators, so this is what makes the oracle a valid comparator there."""
import numpy as np
import pytest

import edge_inputs as E
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.reference
needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built (needs /root/reference)")

PE_STRIDES = [48, 112, 160, 256]
SE_STRIDES = [48, 112, 160, 256, 512]
FASTA = [T.TRUSEQ_R1, "CTGTCTCTTATACACATCT", T.TRUSEQ_R2[:20], "AAAAAAAAAAAA", "GGGGGGGGGG"]      # the fasta_adapters option set's list


def make_input(gen, n, S, paired, seed, p):
    rng = np.random.default_rng(seed)
    if gen == "extremes":
        return E.edge_batch(n, S, paired, seed, p, read_len=min(150, S) if S <= 256 else S - 12)
    if gen == "dense":
        return E.dense_correction_pairs(n, min(150, S), S, min(12, S // 4), rng)
    return E.adapter_concatemers(n, S, FASTA, rng, paired)


def check(name, paired, gen, S, cycles, n=1200):
    p = T.config_params(name, paired)
    arrs = make_input(gen, n, S, paired, 11 + S, p)
    x = T.run_cpu("oracle", p, arrs, cycles)
    y = T.run_cpu("ref", p, arrs, cycles)
    T.assert_results_equal(x, y, paired, skip=("adapter_pos",), what=f"{gen}/{name}/S{S}")
    return x


@needs_ref
@pytest.mark.parametrize("gen", ["extremes", "dense", "concat"])
@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", T.CONFIG_NAMES)
def test_port_equals_reference_edges_pe(name, S, gen):
    check(name, 1, gen, S, S)


@needs_ref
@pytest.mark.parametrize("gen", ["extremes", "concat"])
@pytest.mark.parametrize("S", SE_STRIDES)
@pytest.mark.parametrize("name", T.CONFIG_NAMES)
def test_port_equals_reference_edges_se(name, S, gen):
    check(name, 0, gen, S, S)


@needs_ref
@pytest.mark.parametrize("gen", ["extremes", "dense"])
@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", T.MERGE_CONFIG_NAMES)
def test_port_equals_reference_edges_merge(name, S, gen):
    check(name, 1, gen, S, 2 * S)


@needs_ref
@pytest.mark.parametrize("limit", [5, 20])
def test_dense_pairs_overflow_the_tile_correction_list(limit):
    """The correction-dense generator really corrects more than FP_CORR_CAP (1024) bases per 128-pair tile, and more than the
    2 per pair a host chunk's patch list holds."""
    p = T.config_params("cfg3_overlap_correction", 1)
    p.overlap_diff_limit = limit
    arrs = E.dense_correction_pairs(1000, 150, 160, 12, np.random.default_rng(3))
    x = T.run_cpu("oracle", p, arrs, 160)
    y = T.run_cpu("ref", p, arrs, 160)
    T.assert_results_equal(x, y, 1, skip=("adapter_pos",), what=f"dense limit {limit}")
    corrected = sum(int((x["arrs"]["seq" + s] != arrs["seq" + s]).sum()) for s in "12")
    assert corrected > 1024 / 128 * 1000


@needs_ref
@pytest.mark.parametrize("paired", [1, 0])
def test_concatemers_trim_once_per_adapter(paired):
    """With the fasta list alone (no adapter_seq_r1, whose 12 bases also start TRUSEQ_R2[:20] and would cut three adapters at
    once) each adapter of the concatemer trims once: five addAdapterTrimmed calls per read, more than four per unit."""
    p = concatemer_params(paired)
    n = 2000
    arrs = E.adapter_concatemers(n, 160, FASTA, np.random.default_rng(5), paired)
    T.assert_results_equal(T.run_cpu("oracle", p, arrs, 160), T.run_cpu("ref", p, arrs, 160), paired, skip=("adapter_pos",), what="concatemers")
    maps, _ = T.ref_adapter_maps(p, arrs, 160)
    assert sum(sum(m.values()) for m in maps) == len(FASTA) * n * (2 if paired else 1)


def concatemer_params(paired):
    p = T.config_params("fasta_adapters", paired)
    capi.set_params(p, adapter_seq_r1=None)
    return p
