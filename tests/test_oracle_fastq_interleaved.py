"""The C port of interleaved pairs (oracle/fastp_oracle_interleaved.c) against the reference itself: the decode port against its own
FastqReaderPair(..., interleaved = true) through the harness, and the whole port path (interleaved decode, operator chain, the streams
--stdout writes) against the UNMODIFIED reference CLI's stdout and files.  The device (tests/test_gpu_fastq_interleaved.py) is compared
with this port, so the port is pinned here first."""
import hashlib
import json
import os

import numpy as np
import pytest

import fp_interleaved as IL
import fp_outs as O
import fp_testlib as T

DIGESTS = os.path.join(os.path.dirname(__file__), "golden", "fastq_interleaved_cli_digests.json")
needs_cli = pytest.mark.skipif(not os.path.exists(T.REF_CLI), reason="oracle/_ref/fastp_ref (the reference CLI) is not built")
needs_harness = pytest.mark.skipif(not IL.have_ref_interleaved(), reason="oracle/_ref/libfastp_ref.so without fp_ref_fastq_read_interleaved")


def rec(i, L=12, tag="1", strand=b"+", eol=b"\n", q=b"I"):
    s = bytes(np.random.default_rng(i).choice(np.frombuffer(b"ACGTN", np.uint8), L))
    return b"@r%d/%s" % (i, tag.encode()) + eol + s + eol + strand + eol + q * L + eol


def il_text(n, **kw):
    return b"".join(rec(i, L=5 + i % 20, tag="12"[i % 2], **kw) for i in range(n))


def decode_texts():
    """name -> (text, phred64): the reader rules the interleaved decode must follow."""
    t = {f"count{n}": (il_text(n), 0) for n in (0, 1, 2, 7, 8, 15, 16)}
    good = [rec(i, L=10) for i in range(10)]
    t["bad_mate1"] = (b"".join(good[:4]) + rec(4, strand=b"-") + b"".join(good[5:]), 0)             # record 4: mate 1 of pair 2
    t["bad_mate2"] = (b"".join(good[:5]) + rec(5, strand=b"x") + b"".join(good[6:]), 0)             # record 5: mate 2 of pair 2
    t["bad_length"] = (b"".join(good[:7]) + b"@r7\nACGT\n+\nIII\n" + b"".join(good[8:]), 0)
    t["junk_between_mates"] = (b"".join(g + (b"\n\njunk line\n" if k % 2 == 0 else b"") for k, g in enumerate(good)), 0)
    t["crlf"] = (il_text(9, eol=b"\r\n"), 0)
    t["phred64"] = (il_text(8, q=b"h"), 1)
    t["no_final_newline"] = (il_text(6)[:-1], 0)
    t["strand_text"] = (il_text(6, strand=b"+again"), 0)
    return t


@needs_harness
@pytest.mark.parametrize("name", list(decode_texts()))
def test_decode_port_equals_fastq_reader_pair(tmp_path, name):
    text, ph = decode_texts()[name]
    path = tmp_path / "il.fq"
    path.write_bytes(text)
    want = IL.ref_read_interleaved(path, ph)
    d = IL.oracle_decode_il(text, phred64=ph)
    assert IL.il_fields(text, d) == want
    assert d["info"]["n_records"] == len(want)
    if name.startswith("bad"):
        assert d["info"]["error"] != 0 and d["info"]["error_record"] in (4, 5, 7)
    else:
        assert d["info"]["error"] == 0 and d["info"]["consumed"] == len(text)


def test_decode_port_cuts_at_every_record_phase():
    """A chunk cut anywhere: non-final decodes followed by the rest give the pairs of one whole decode (a lone mate 1 is read again with
    its mate), and capacity cuts resume at record 2 * capacity."""
    text = il_text(15)
    whole = IL.il_fields(text, IL.oracle_decode_il(text))
    assert len(whole) == 7                                        # the 15th record has no mate: dropped
    for cut in range(0, len(text) + 1, 7):
        got, start = [], 0
        for final, end in ((0, cut), (1, len(text))):
            chunk = text[start:end]
            d = IL.oracle_decode_il(chunk, final=final)
            got += IL.il_fields(chunk, d)
            start += d["info"]["consumed"]
        assert got == whole and start == len(text), cut
    for cap in (1, 2, 3):
        got, start = [], 0
        while True:
            chunk = text[start:]
            d = IL.oracle_decode_il(chunk, capacity=cap)
            got += IL.il_fields(chunk, d)
            start += d["info"]["consumed"]
            if not d["info"]["more"]:
                break
        assert got == whole and start == len(text), cap


@needs_cli
@pytest.mark.parametrize("run", list(IL.RUNS))
def test_port_equals_reference_cli(tmp_path, run):
    outs, err = IL.run_ref_cli(tmp_path, run)
    assert outs == IL.expected_outputs(run), run
    digests = json.load(open(DIGESTS))
    assert [hashlib.md5(x).hexdigest() for x in outs] == digests[run], "tests/golden/make_fastq_interleaved_digests.py is out of date"
    if IL.RUNS[run][2] == "o1_merged":
        assert b"Using --out1 to store the merged reads to be compatible with fastp 0.19.8" in err


def test_committed_digests_are_the_ports():
    """Runs without the reference binary too: the committed CLI digests equal what the port says the CLI writes."""
    digests = json.load(open(DIGESTS))
    assert set(digests) == set(IL.RUNS)
    for run in IL.RUNS:
        assert [hashlib.md5(x).hexdigest() for x in IL.expected_outputs(run)] == digests[run], run


def test_interleaved_stream_is_out1_out2_interleaved():
    """The --stdout stream of a paired run is out1 and out2 interleaved record by record, and interleaved input decodes to the pairs of the
    two files."""
    for run in ("filters_pe/stdout", "filters_pe/il_stdout", "dedup_pe/il_stdout", "edge48_pe/il_stdout"):
        g = IL.port_streams(run)
        assert len(g["out1"]) > 0 and g["stdout_il"] == IL.interleave(g["out1"], g["out2"]), run
    two = IL.port_streams("filters_pe/stdout")
    one = IL.port_streams("filters_pe/il_stdout")
    assert one["n"] == two["n"] and one["stdout_il"] == two["stdout_il"] and one["failed"] == two["failed"]


def test_encode_port_out_cap():
    g = IL.port_streams("filters_pe/il_stdout")
    full = g["stdout_il"]
    text, _, _ = IL.run_inputs("filters_pe/il_stdout")
    S = O.fastq_outs_cases()["filters_pe"][5]
    d = IL.oracle_decode_il(text, stride=S)
    n = len(d["sides"][0]["recs"])
    sd1, sd2 = d["sides"]
    arrs = {"seq1": sd1["seq"].copy(), "qual1": sd1["qual"].copy(), "len1": sd1["len"].copy(),
            "seq2": sd2["seq"].copy(), "qual2": sd2["qual"].copy(), "len2": sd2["len"].copy()}
    res = T.run_cpu("oracle", O.case_params("filters_pe"), arrs, S)
    a = res["arrs"]
    part, total = IL.oracle_encode_il(text, sd1["recs"][:n], text, sd2["recs"][:n], res["out1"], res["out2"], a["seq1"], a["qual1"], a["seq2"],
                                      a["qual2"], S, out_cap=len(full) - 1)
    assert total == len(full)
    last = full.rfind(b"\n@", 0, len(full) - 1) + 1
    assert part[:last] == full[:last] and set(part[last:]) <= {0}
