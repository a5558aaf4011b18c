"""The C port of --overlapped_out (oracle/fastp_oracle_overlapped.c: the analysis of src/peprocessor.cpp:488-495 and the record it
writes) against the UNMODIFIED reference CLI's file.  The device chain and encoder (tests/test_gpu_fastq_overlapped.py) are compared
with this port, so the port is pinned here first."""
import hashlib
import json
import os

import numpy as np
import pytest

import fp_overlapped as O
import fp_testlib as T

CASES = O.overlapped_cases()
DIGESTS = os.path.join(os.path.dirname(__file__), "golden", "fastq_overlapped_cli_digests.json")
needs_cli = pytest.mark.skipif(not os.path.exists(T.REF_CLI), reason="oracle/_ref/fastp_ref (the reference CLI) is not built")


def port(name):
    flags, p, t1, t2, stride, dedup = CASES[name]
    return O.port_text_path(p, t1, t2, stride, dedup)


@needs_cli
@pytest.mark.parametrize("name", list(CASES))
def test_port_equals_reference_cli(tmp_path, name):
    flags, p, t1, t2, stride, dedup = CASES[name]
    want = O.run_ref_cli(tmp_path, flags, t1, t2)
    assert port(name)["overlapped"] == want, name
    assert hashlib.md5(want).hexdigest() == json.load(open(DIGESTS))[name], "tests/golden/make_fastq_overlapped_digests.py is out of date"


@needs_cli
@pytest.mark.parametrize("name", ["cfg_cfg4_full", "planted_c", "dedup"])
def test_interleaved_input_equals_reference_cli(tmp_path, name):
    flags, p, t1, t2, stride, dedup = CASES[name]
    assert O.run_ref_cli(tmp_path, flags, t1, t2, interleaved=True) == port(name)["overlapped"]


def test_committed_digests_are_the_ports():
    """Runs without the reference binary too: the committed CLI digests equal the port's stream."""
    digests = json.load(open(DIGESTS))
    assert set(digests) == set(CASES)
    for name in CASES:
        assert hashlib.md5(port(name)["overlapped"]).hexdigest() == digests[name], name


def _records(text):
    lines = text.split(b"\n")
    return {lines[k].split(b" ")[0][1:]: lines[k + 1] for k in range(0, len(lines) - 1, 4)}


def test_planted_pairs_cover_every_rule():
    """Each kind of planted_pairs does what its docstring says, in the port's analysis and in the stream."""
    _, _, kinds = O.planted_pairs()
    plain, corr, drop = port("planted"), port("planted_c"), port("planted_drop")
    ov, ovc, ovd = plain["ovx"], corr["ovx"], drop["ovx"]
    k0 = np.flatnonzero(kinds == 0)
    found = ov["overlapped"][k0].astype(bool) & (ov["overlap_len"][k0] == 31)
    assert found.sum() > 50 and (ov["overlap_len"][k0][ov["overlapped"][k0] == 1] != 30).all()
    k1 = np.flatnonzero(kinds == 1)
    near, far = k1[(k1 // 6) % 2 == 1], k1[(k1 // 6) % 2 == 0]
    assert ov["overlapped"][near].mean() < 0.1 and ov["overlapped"][far].mean() > 0.9
    k2 = np.flatnonzero(kinds == 2)
    offs = ov["offset"][k2][ov["overlapped"][k2] == 1]
    assert (offs < 0).sum() > 20 and (offs == 0).sum() > 20 and (offs > 0).sum() > 20
    k3 = np.flatnonzero(kinds == 3)
    assert ov["overlapped"][k3].mean() < 0.1 and ovc["overlapped"][k3].mean() > 0.9
    k4 = np.flatnonzero(kinds == 4)
    assert (ovd["overlapped"][k4] == 0).all()
    k5 = np.flatnonzero(kinds == 5)
    assert ov["overlapped"][k5].mean() > 0.9
    # records: read 1 after the overlap -- empty for offsets >= 0 that reach read 1's end, the adapter part for negative offsets
    recs = _records(plain["overlapped"])
    assert len(recs) == int(ov["overlapped"].sum())
    assert any(len(v) == 0 for v in recs.values()) and any(len(v) > 0 for v in recs.values())


def test_failing_and_duplicate_pairs_are_written():
    """The filters and -D come after the analysis.  (An adapter dimer keeps at most dimer_max_len bases per read, fewer than overlap_require,
    so it never overlaps: the dimer pairs of the case show that they write nothing rather than being skipped by a rule.)"""
    d = port("dimer_filters")
    res1, ovx = d["res"]["out1"], d["ovx"]
    written = ovx["overlapped"] == 1
    assert (written & (res1["pair_verdict"] != 0)).sum() > 50
    assert ((res1["flags"] & 0x20) != 0).sum() > 100                              # FP_F_ADAPTER_DIMER
    dd = port("dedup")
    assert (dd["ovx"]["overlapped"].astype(bool) & ((dd["res"]["out1"]["flags"] & 0x40) != 0)).sum() > 20   # FP_F_DUPLICATE


def test_port_out_cap():
    d = port("planted")
    a, (d1, _) = d["res"]["arrs"], d["dec"]
    full, total = O.oracle_encode_overlapped(CASES["planted"][2], d1["recs"][:d["n"]], d["res"]["out1"], d["res"]["out2"], d["ovx"],
                                             a["seq1"], a["qual1"], 160)
    part, t2 = O.oracle_encode_overlapped(CASES["planted"][2], d1["recs"][:d["n"]], d["res"]["out1"], d["res"]["out2"], d["ovx"],
                                          a["seq1"], a["qual1"], 160, out_cap=total - 1)
    assert t2 == total and part[:len(full) - len(full.split(b"\n@")[-1]) - 1] == full[:len(full) - len(full.split(b"\n@")[-1]) - 1]
