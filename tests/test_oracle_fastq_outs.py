"""The C port of --unpaired1 / --unpaired2 / --failed_out (fp_oracle_fastq_encode_rejects: src/seprocessor.cpp:280-290,
src/peprocessor.cpp:575-620, records as Read::appendToStringWithTag writes them) against the UNMODIFIED reference CLI's files.
The device encoder (tests/test_gpu_fastq_outs.py) is compared with this port, so the port is pinned here first."""
import hashlib
import json
import os

import numpy as np
import pytest

import fp_outs as O
import fp_testlib as T

DIGESTS = os.path.join(os.path.dirname(__file__), "golden", "fastq_outs_cli_digests.json")
needs_cli = pytest.mark.skipif(not os.path.exists(T.REF_CLI), reason="oracle/_ref/fastp_ref (the reference CLI) is not built")
RUNS = [(name, ws) for name in O.fastq_outs_cases() for ws in O.case_writer_sets(name)]


@needs_cli
@pytest.mark.parametrize("name,wset", RUNS)
def test_port_equals_reference_cli(tmp_path, name, wset):
    files, exist, err = O.run_ref_cli_outs(tmp_path, name, wset)
    assert files == O.expected_files(name, wset), (name, wset)
    u1, u2, f = O.WRITER_SETS[wset]
    flags, _, paired = O.fastq_outs_cases()[name][:3]
    if paired and "--include_unmerged" not in flags:
        assert ("u1.fq" in exist) == bool(u1) and ("u2.fq" in exist) == bool(u2)      # --unpaired2 alone: created, left empty
    else:
        assert "u1.fq" not in exist and "u2.fq" not in exist
        why = b"Not paired-end mode" if not paired else b"You specified --include_unmerged in merging mode"
        assert (why + b". Ignoring argument --unpaired1") in err or not u1
    assert ("f.fq" in exist) == bool(f)
    digests = json.load(open(DIGESTS))
    assert [hashlib.md5(x).hexdigest() for x in files] == digests[f"{name}/{wset}"], "tests/golden/make_fastq_outs_digests.py is out of date"


def test_committed_digests_are_the_ports():
    """Runs without the reference binary too: the committed CLI digests equal what the port says the files hold."""
    digests = json.load(open(DIGESTS))
    assert set(digests) == {f"{n}/{w}" for n, w in RUNS}
    for name, ws in RUNS:
        assert [hashlib.md5(x).hexdigest() for x in O.expected_files(name, ws)] == digests[f"{name}/{ws}"], (name, ws)


def failed_records(text):
    lines = text.split(b"\n")
    return [lines[k:k + 4] for k in range(0, len(lines) - 1, 4)]


def test_cases_cover_what_they_claim():
    """Every tag, dropped reads written whole, failed reads with corrected bases, duplicates among one-sided pairs, strand lines."""
    tags = set()
    for name in O.fastq_outs_cases():
        got = O.port_text_path(name, O.port_writers(name, "f"))
        tags |= {t for t in O.TAGS if t in got["failed"]}
    assert tags == set(O.TAGS)
    for name in ("trim_null_pe", "trim_null_se"):                 # dropped reads: the whole row as read
        got = O.port_text_path(name, 0)
        d1 = got["dec"][0]
        r1 = got["res"]["out1"]
        dropped = np.nonzero((r1["flags"] & 0x01) != 0)[0]
        assert len(dropped) > 100
        body = {bytes(d1["seq"][i, :d1["len"][i]]) for i in dropped if d1["len"][i] > 0}
        written = {rec[1] for rec in failed_records(got["failed"])}
        assert len(body & written) > 50
    c = O.port_text_path("correction_pe", 0)["res"]
    one_sided = (c["out1"]["verdict"] == 0) != (c["out2"]["verdict"] == 0)
    corrected_fail = (((c["out1"]["flags"] & 0x08) != 0) & (c["out1"]["verdict"] != 0) | ((c["out2"]["flags"] & 0x08) != 0) & (c["out2"]["verdict"] != 0))
    assert (one_sided & corrected_fail).sum() > 20
    d = O.port_text_path("dedup_pe", 0)["res"]
    dup = (d["out1"]["flags"] & 0x40) != 0
    assert (dup & ((d["out1"]["verdict"] == 0) != (d["out2"]["verdict"] == 0))).sum() > 10
    e = O.port_text_path("edge256_pe", 3)
    assert b"\n+again\n" in e["failed"] and b"\n+again\n" in e["unpaired1"] and b"\n+again\n" in e["unpaired2"]
    m = O.port_text_path("merge_pe", 1)
    assert m["merged"].count(b" merged_") > 10 and len(m["unpaired1"]) > 0


def test_port_out_cap():
    """A record that does not fit under out_cap is left out whole; the total still counts it."""
    name = "filters_pe"
    full = O.port_text_path(name, 0)["failed"]
    _, _, paired, t1, t2, S = O.fastq_outs_cases()[name][:6]
    got = O.port_text_path(name, 0)
    d1, d2 = got["dec"]
    n, res, a = got["n"], got["res"], got["res"]["arrs"]
    part, total = O.oracle_fastq_encode_rejects(O.FAILED, 0, O.case_params(name), t1, d1["recs"][:n], res["out1"], a["seq1"], a["qual1"], d1["len"][:n],
                                                text2=t2, recs2=d2["recs"][:n], res2=res["out2"], seq2=a["seq2"], qual2=a["qual2"], len2=d2["len"][:n],
                                                stride=S, out_cap=len(full) - 1)
    assert total == len(full)
    last = full.rfind(b"\n@", 0, len(full) - 1) + 1
    assert part[:last] == full[:last] and set(part[last:]) <= {0}
