"""The C port of the index filter (oracle/fastp_oracle_index.c, tests/fp_index.py) against the unmodified reference CLI: every output
file and the -j counters of each case, the list loading rules and their error, and the committed digests.  No GPU."""
import hashlib
import json
import os

import pytest

import fp_index as X
from fp_testlib import REF_CLI

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fastq_index_cli_digests.json")
CASES = sorted(X.index_cases())
need_ref = pytest.mark.skipif(not os.path.exists(REF_CLI), reason="reference CLI not built (oracle/_ref/fastp_ref)")


def test_read_test_vector():
    """Read::test (src/read.cpp:173-180): lastIndex of its name is GGTCCCGA."""
    name = b"@NS500713:64:HFKJJBGXY:1:11101:20469:1097 1:N:0:TATAGCCT+GGTCCCGA"
    assert X.index_of(name, False) == b"GGTCCCGA"
    assert X.index_of(name, True) == b"TATAGCCT"


@pytest.mark.parametrize("name,first,last", [
    (b"@a", b"", b""), (b"@a:b", b"", b""), (b"@a:bc", b"bc", b"bc"), (b"@ab:cd", b"cd", b"cd"),
    (b"@SRR1.1 1 length=150", b"", b""), (b"@M:1 1:N:0:AC:+", b"AC:+", b"AC:+"), (b"@M1+A:", b"", b"A:"),
    (b"@M:1:ACGT+GG+TT", b"ACGT", b"TT"), (b"@M:1 1:N:0:+TTGG", b"", b"TTGG"), (b"@x:ACGT+", b"ACGT+", b"ACGT+"),
])
def test_index_shapes(name, first, last):
    assert X.index_of(name, True) == first
    assert X.index_of(name, False) == last


def test_match_rules():
    assert X.match([b"ACGT"], b"", 0) and X.match([b""], b"ACGT", 0)                 # empty index / barcode
    assert X.match([b"ACG"], b"ACGTT", 0) and X.match([b"ACGTTA"], b"ACG", 0)        # prefixes either way
    assert not X.match([b"ACGT"], b"ACGA", 0) and X.match([b"ACGT"], b"ACGA", 1)
    assert not X.match([b"ACGT"], b"", -1) and not X.match([], b"ACGT", 5)
    assert not X.match([b"ACGT"], b"acgt", 3) and X.match([b"ACGT"], b"acgt", 4)      # lower case never equals


@pytest.mark.parametrize("data,want", [
    (b"ACGT\nTTGG\n", [b"ACGT", b"TTGG"]), (b"ACGT\n\nTTGG", [b"ACGT", b"", b"TTGG"]), (b"ACGT\r\nTT\r\n", [b"ACGT", b"TT"]),
    (b"", []), (b"\n", [b""]), (b"A\r\n", [b"A"]), (b"\r\n", None), (b"ACGT\nACNT\n", None), (b"AC\0GG\n", [b"AC"]),
    (b"A" * 999 + b"\nCC\n", [b"A" * 999, b"CC"]), (b"A" * 1000 + b"\nCC\n", []),
])
def test_list_loading(data, want):
    assert X.load_list(data) == want


def _digest(streams, counts):
    return {"files": {k: hashlib.md5(v).hexdigest() for k, v in streams.items()}, "counts": counts}


@pytest.mark.parametrize("name", CASES)
def test_port_matches_digests(name):
    want = json.load(open(DIGESTS))[name]
    got = X.port_text_path(name)
    paired = X.index_cases()[name][2]
    assert _digest(X.expected_streams(name), X.summary_counts(got["res"]["counters"], paired)) == want


@need_ref
@pytest.mark.parametrize("name", CASES)
def test_port_matches_reference_cli(tmp_path, name):
    out, js, r = X.run_cli(REF_CLI, tmp_path, name)
    assert r.returncode == 0, r.stderr[-2000:]
    exp = X.expected_streams(name)
    for k in X.STREAMS:
        assert out[k] == exp[k], (name, k, len(out[k]), len(exp[k]))
    paired = X.index_cases()[name][2]
    assert X.json_counts(js) == X.summary_counts(X.port_text_path(name)["res"]["counters"], paired)


@need_ref
@pytest.mark.parametrize("name", ["l96_t0_pe", "dedup_pe"])
def test_port_matches_reference_cli_interleaved(tmp_path, name):
    out, js, r = X.run_cli(REF_CLI, tmp_path, name, interleaved=True)
    assert r.returncode == 0, r.stderr[-2000:]
    exp = X.expected_streams(name)
    for k in X.STREAMS:
        assert out[k] == exp[k], (name, k)


@need_ref
def test_reference_refuses_non_acgt(tmp_path):
    (tmp_path / "r1.fq").write_bytes(X.named_texts(10, 1, 0)[0])
    (tmp_path / "bad.txt").write_bytes(b"ACGT\nACNT\n")
    import subprocess
    r = subprocess.run([REF_CLI, "-i", str(tmp_path / "r1.fq"), "-o", str(tmp_path / "o.fq"), "--filter_by_index1", str(tmp_path / "bad.txt")],
                       capture_output=True, cwd=tmp_path)
    assert r.returncode == 255
    assert b"each line should be one barcode, which can only contain A/T/C/G" in r.stderr
