"""The C port's --dedup rule (fp_oracle_process_dedup), its duplicate filter beyond one shape and its FASTQ decoder on long dirty
texts, each against the reference's own objects (oracle/_ref).  The device tests (tests/test_gpu_dedup.py,
tests/test_gpu_fastq_blocks.py) compare with the C port on the same inputs."""
import ctypes as C

import numpy as np
import pytest

import edge_inputs as E
import fp_testlib as T
from fastp_b200 import capi
from test_duplicate_oracle import planted

pytestmark = pytest.mark.reference
needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref not built (needs the reference sources)")
needs_ref_dedup = pytest.mark.skipif(not T.have_ref_dedup(), reason="oracle/_ref/libfastp_ref.so is absent or was built from a harness "
                                     "without fp_ref_process_dedup (rebuild it: make -C oracle, needs the reference sources)")
PATTERNS = ["none", "all", "random"]
REF_SKIP = ("adapter_pos",)                                  # the reference keeps no trim position; the harness leaves it 0


def flags_for(kind, n, paired, seed):
    if kind == "none":
        return np.zeros(n, np.uint8)
    if kind == "all":
        return np.ones(n, np.uint8)
    if kind == "random":
        return (np.random.default_rng(seed).random(n) < 0.3).astype(np.uint8)
    raise KeyError(kind)


def check_configs(names, paired, S, cycles):
    for name in names:
        p = T.config_params(name, paired)
        arrs = E.edge_batch(600, S, paired, S + paired, p, read_len=min(150, S))
        for kind in PATTERNS:
            f = flags_for(kind, 600, paired, S)
            a, b = T.run_cpu("oracle", p, arrs, cycles, is_dup=f), T.run_cpu("ref", p, arrs, cycles, is_dup=f)
            T.assert_results_equal(a, b, paired, skip=REF_SKIP, what=f"{name}/{kind}")
            assert np.array_equal(a["out1"]["flags"] & 0x40 != 0, f != 0)
        T.assert_results_equal(T.run_cpu("oracle", p, arrs, cycles, is_dup=np.zeros(600, np.uint8)), T.run_cpu("oracle", p, arrs, cycles), paired,
                               what=f"{name}: no flags == fp_oracle_process")


@needs_ref_dedup
@pytest.mark.parametrize("paired", [1, 0])
def test_port_equals_reference_with_flags(paired):
    check_configs(T.CONFIG_NAMES, paired, 160, 160)


@needs_ref_dedup
def test_port_equals_reference_with_flags_merging():
    check_configs(T.MERGE_CONFIG_NAMES, 1, 128, 256)


@needs_ref_dedup
@pytest.mark.parametrize("name,paired", [("cfg4_full", 1), ("cfg4_full", 0), ("mergeu_cfg3_overlap_correction", 1)])
def test_port_equals_reference_with_the_filters_own_flags(name, paired):
    arrs = planted(paired)
    p = T.config_params(name, paired)
    f = T.oracle_dup_flags([arrs], paired, 3)[0][0]
    assert 1000 < f.sum() < len(f)
    cyc = 320 if name.startswith("merge") else 160
    T.assert_results_equal(T.run_cpu("oracle", p, arrs, cyc, is_dup=f), T.run_cpu("ref", p, arrs, cyc, is_dup=f), paired, skip=REF_SKIP, what=name)


def ref_dup_flags(batches, paired, level):
    r = T.ref()
    r.fp_ref_dup_create.restype = C.c_void_p; r.fp_ref_dup_create.argtypes = [C.c_int]
    r.fp_ref_dup_check.argtypes = [C.c_void_p, C.POINTER(capi.Batch), C.c_int, C.c_void_p]
    r.fp_ref_dup_destroy.argtypes = [C.c_void_p]
    d = r.fp_ref_dup_create(level)
    try:
        out = []
        for arrs in batches:
            a = {k: np.ascontiguousarray(v) for k, v in arrs.items()}
            f = np.zeros(len(a["len1"]), np.uint8)
            b = capi.batch_from_arrays(a)
            r.fp_ref_dup_check(d, C.byref(b), paired, f.ctypes.data)
            out.append(f)
        return out
    finally:
        r.fp_ref_dup_destroy(d)


@needs_ref
@pytest.mark.parametrize("level", [1, 2, 3])
@pytest.mark.parametrize("paired,S", [(1, 256), (1, 512), (0, 512)])
def test_duplicate_filter_port_equals_reference(level, paired, S):
    """Lengths 0, 1 and the full stride, read 1 empty with read 2 not, bytes outside A/C/G/T, and (pairs at stride 512) positions past
    the end of the prime arrays, where the index (q * bufNum + i) & mOffsetMask wraps."""
    from _gpu_dup_cases_worker import cut, units
    arrs = units(paired, S, seed=7 * level + S + paired, n0=3000)
    total_len = arrs["len1"].astype(int) + (arrs["len2"].astype(int) if paired else 0)
    buf_num = 4 if level == 3 else 2
    if paired and S == 512:
        assert (total_len.max() - 1) * buf_num > 512 * buf_num - 1                 # the prime index wraps
    assert total_len.min() == 0 and (arrs["len1"] == 1).any()
    if paired:
        assert ((arrs["len1"] == 0) & (arrs["len2"] > 0)).any()
    seen = set(np.unique(np.concatenate([arrs["seq1"][i, :arrs["len1"][i]] for i in range(len(total_len))])))
    assert {ord("N"), ord("a"), ord(".")} <= seen
    batches = cut(arrs, [1, 0, 7, 2000, len(total_len) - 2008])
    got, want = T.oracle_dup_flags(batches, paired, level)[0], ref_dup_flags(batches, paired, level)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert sum(int(w.sum()) for w in want) > 800


@needs_ref
@pytest.mark.parametrize("text", ["shifted", "fuzz", "fuzz_unbroken", "crlf", "cr", "two_bad"])
def test_decoder_port_equals_reference_reader_on_long_texts(tmp_path, text):
    if text == "shifted":
        t = T.fastq_shifted_text()
    elif text.startswith("fuzz"):
        t = T.fastq_fuzz_text(np.random.default_rng(11), nrec=5000, broken=0 if text.endswith("unbroken") else 0.04)
    elif text == "two_bad":
        t = T.fastq_shifted_text(at_quality_on_block_start=False)
        recs = T.oracle_fastq_decode(t, stride=160, capacity=12000)["recs"]
        t = T.fastq_break_record(T.fastq_break_record(t, recs, 9000, "strand"), recs, 5200, "length")
    else:
        t = T.fastq_eol_text("\r\n" if text == "crlf" else "\r")
    d = T.oracle_fastq_decode(t, stride=160)
    path = tmp_path / "t.fq"
    path.write_bytes(t)
    want = T.ref_fastq_read(path)
    assert len(want) == d["info"]["n_records"] > (0 if text == "fuzz" else 2500)
    assert T.decoded_fields(t, d) == want
