"""The C port of the merging-mode output streams (fp_oracle_fastq_encode_merge: --merged_out, --out1, --out2 of
src/peprocessor.cpp:519-622, merged reads as OverlapAnalysis::merge builds them) against the UNMODIFIED reference CLI's files.
The device encoder (tests/test_gpu_fastq_merge.py) is compared with this port, so the port is pinned here first."""
import hashlib
import json
import os
import re

import numpy as np
import pytest

import fp_merge as M
import fp_testlib as T

CASES = M.fastq_merge_cases()
DIGESTS = os.path.join(os.path.dirname(__file__), "golden", "fastq_merge_cli_digests.json")
needs_cli = pytest.mark.skipif(not os.path.exists(T.REF_CLI), reason="oracle/_ref/fastp_ref (the reference CLI) is not built")


def port_streams(name):
    flags, kw, t1, t2, stride, dedup = CASES[name]
    p = M.merge_case_params(kw, 250 if stride == 256 else 150)
    return M.oracle_merge_text_path(p, t1, t2, stride, dup_level=3 if dedup else 0, dedup=dedup)     # -D: accuracy level 3 (main.cpp:203-209)


@needs_cli
@pytest.mark.parametrize("name", list(CASES))
def test_port_equals_reference_cli(tmp_path, name):
    flags, kw, t1, t2, stride, dedup = CASES[name]
    got = port_streams(name)
    m, o1, o2, js = M.run_ref_cli_merge(tmp_path, flags, t1, t2)
    assert len(m) > 10000 and m.count(b" merged_") > 300, "the case merges nothing"
    assert got["merged"] == m, name
    if "--include_unmerged" in flags:                     # the CLI drops --out1 / --out2 (options.cpp:127-135); nothing is left for them
        assert got["out1"] == b"" and got["out2"] == b""
    else:
        assert got["out1"] == o1 and got["out2"] == o2, name
    af, c = js["summary"]["after_filtering"], got["counters"]
    from fastp_b200 import capi
    assert c.summary(capi.STATS_POST1)["reads"] == af["total_reads"] and c.summary(capi.STATS_POST1)["bases"] == af["total_bases"]
    digests = json.load(open(DIGESTS))
    assert [hashlib.md5(x).hexdigest() for x in (m, o1, o2)] == digests[name], "tests/golden/make_fastq_merge_digests.py is out of date"


def test_committed_digests_are_the_ports():
    """Runs without the reference binary too: the committed CLI digests equal the port's streams."""
    digests = json.load(open(DIGESTS))
    assert set(digests) == set(CASES)
    for name in CASES:
        got = port_streams(name)
        assert [hashlib.md5(got[k]).hexdigest() for k in ("merged", "out1", "out2")] == digests[name], name


def suffixes(merged):
    return [(int(a), int(b)) for a, b in re.findall(rb" merged_(\d+)_(\d+)\n", merged)]


def test_cases_cover_what_they_claim():
    """Suffix widths of one to three digits on both lengths, len2 = 0 (offset <= 0), suffixed strand lines, duplicates of both kinds."""
    sx = suffixes(port_streams("digit_borders")["merged"])
    l1 = {a for a, _ in sx}; l2 = {b for _, b in sx}
    assert {9, 10, 99, 100} <= l1 | l2 and min(l2) == 0
    assert any(a >= 100 for a in l1) and any(b >= 100 for b in l2) and any(0 < b < 10 for b in l2) and any(10 <= b < 100 for b in l2)
    tail = suffixes(port_streams("short_tail")["merged"])
    assert {b for _, b in tail} >= set(range(0, 10))
    named = port_streams("named_strand")["merged"]
    assert re.search(rb"\n\+inst:7:FC:1:\d+:9 merged_\d+_\d+\n", named) and b"\n+\n" in named and re.search(rb"\n\+  merged_\d+_\d+\n", named)
    assert max(a + b for a, b in suffixes(port_streams("pe250")["merged"])) > 256
    for name in ("dedup", "dedup_include_unmerged"):
        s = port_streams(name)
        f1, fl = s["res"]["out1"]["flags"], s["res"]["out1"]["verdict"]
        dup_merged = int(((f1 & 0x40) != 0).astype(int) @ (((f1 & 0x80) != 0) & (fl == 0)).astype(int))
        dup_unmerged = int((((f1 & 0x40) != 0) & ((f1 & 0x80) == 0) & (s["res"]["out1"]["pair_verdict"] == 0)).sum())
        assert dup_merged > 20 and dup_unmerged > 20, (name, dup_merged, dup_unmerged)


ODD = [b for b in range(256) if b not in (10, 13)]            # every byte a FASTQ line can hold


def odd_byte_pairs():
    """Pairs whose read 2 starts with bytes outside A/C/G/T (lower case, IUPAC codes, controls, the upper half): that stretch is the part of
    read 2 beyond the overlap, so the merged read ends with its reverse complement and the overlap analysis never looks at it."""
    rng = np.random.default_rng(11)
    t1, t2, chunks = [], [], []
    for k in range(0, len(ODD), 64):
        odd = bytes(ODD[k:k + 64])
        r1 = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), 70))
        r2 = odd + M._revcomp_text(r1)[:50]
        t1.append(b"@o%d 1\n%s\n+\n%s\n" % (k, r1, b"I" * len(r1)))
        t2.append(b"@o%d 2\n%s\n+\n%s\n" % (k, r2, b"I" * len(r2)))
        chunks.append(odd)
    return b"".join(t1), b"".join(t2), chunks


def test_complement_map_is_the_scalar_rule():
    lib = M.merge_oracle()
    want = {ord("A"): "T", ord("a"): "T", ord("T"): "A", ord("t"): "A", ord("C"): "G", ord("c"): "G", ord("G"): "C", ord("g"): "C"}
    for b in range(256):                                      # src/simd.cpp:296-308
        assert lib.fp_oracle_merge_complement(b) == ord(want.get(b, "N")), b


@needs_cli
def test_complement_of_every_line_byte_equals_reference_cli(tmp_path):
    """254 byte values through the reference's own reverse complement: the CLI's merged reads end with what the port writes."""
    t1, t2, chunks = odd_byte_pairs()
    flags = ["-A", "-Q", "-G"]                                 # nothing trims the odd stretch or rejects it for its 'N's (filter.cpp:19-33)
    kw = dict(adapter_enabled=0, qual_filter_enabled=0)
    m, o1, o2, _ = M.run_ref_cli_merge(tmp_path, flags, t1, t2)
    got = M.oracle_merge_text_path(M.merge_case_params(kw, 150), t1, t2, 160)
    assert m.count(b" merged_70_") == len(chunks), m[:300]
    assert got["merged"] == m and got["out1"] == o1 and got["out2"] == o2
