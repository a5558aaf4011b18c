"""-m gpu: merging-mode output on the device text path.  fp_fastq_encode_merge (the three streams --merged_out / --out1 / --out2 of
src/peprocessor.cpp:519-622) against its C port on the records the device chain itself produced; fp_fastq_process_host_merge and
fastp_gpu_cli --device_fastq -m against the port's whole text path, the committed digests of the UNMODIFIED reference CLI's files
(tests/golden/fastq_merge_cli_digests.json) and, where oracle/_ref/fastp_ref travelled along, that CLI itself.  The port is pinned to
the CLI on the CPU by tests/test_oracle_fastq_merge.py."""
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import edge_inputs as E
import fp_merge as M
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "fastp_b200", "host", "fastp_gpu_cli")
DIGESTS = os.path.join(ROOT, "tests", "golden", "fastq_merge_cli_digests.json")
CASES = M.fastq_merge_cases()
STREAMS = (("merged", M.FQ_OUT_MERGED), ("out1", M.FQ_OUT_R1), ("out2", M.FQ_OUT_R2))


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def merge_params(include_unmerged, base="cfg4_full"):
    return T.config_params(("mergeu_" if include_unmerged else "merge_") + base, 1)


def device_streams(gpu, ctx, t1, t2, n):
    """decode -> chain -> the three encodes, all on the device; the port encodes the same device records for comparison."""
    d1 = gpu.gpu_fastq_decode(ctx, t1, capacity=n); d2 = gpu.gpu_fastq_decode(ctx, t2, capacity=n)
    assert d1["info"]["n_records"] == n == d2["info"]["n_records"]
    ch = M.gpu_chain_on_decoded(ctx, d1, d2, n)
    h = ch["host"]
    got, want = {}, {}
    for key, which in STREAMS:
        got[key] = M.gpu_fastq_encode_merge(ctx, which, d1, d2, ch, n)
        want[key] = M.oracle_fastq_encode_merge(which, ctx.params.merge_include_unmerged, t1, d1["recs"], t2, d2["recs"], h["res1"], h["res2"], h["ov"],
                                                h["seq1"], h["qual1"], h["seq2"], h["qual2"], ctx.stride)[0]
    return got, want, (d1, d2, ch)


def texts_of(arrs, strand="+"):
    return (T.fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0", strand=strand), T.fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0", strand=strand))


@pytest.mark.parametrize("include_unmerged", [0, 1])
def test_encode_large_enriched(gpu, include_unmerged):
    """60 K enriched pairs at stride 160: every stream equals the port, and the merged stream is not trivially small."""
    n = 60000
    _, arrs = T.synth_host(n, 160, 1, 0, 99, 1, 150)
    t1, t2 = texts_of(arrs)
    ctx = gpu.GpuCtx(merge_params(include_unmerged), n, 160, 320)
    got, want, _ = device_streams(gpu, ctx, t1, t2, n)
    ctx.close()
    for key, _ in STREAMS:
        assert got[key] == want[key], key
    assert got["merged"].count(b" merged_") > 5000
    assert (len(got["out1"]) == 0) == bool(include_unmerged)


@pytest.mark.parametrize("include_unmerged", [0, 1])
@pytest.mark.parametrize("stride", [48, 160, 256])
def test_encode_edge_lengths(gpu, stride, include_unmerged):
    """Lengths 0..stride, independent per side, quality extremes; strand lines that are not '+' so that the suffix lands on them."""
    n = 3 * stride + 500
    p = merge_params(include_unmerged, "default")
    arrs = E.edge_batch(n, stride, 1, 17 + stride, p)
    t1, t2 = texts_of(arrs, strand="+again")
    ctx = gpu.GpuCtx(p, n, stride, 2 * stride)
    got, want, _ = device_streams(gpu, ctx, t1, t2, n)
    ctx.close()
    for key, _ in STREAMS:
        assert got[key] == want[key], (key, stride)


@pytest.mark.parametrize("n", [1, 7, 2047, 2048, 2049])
def test_encode_batch_sizes_around_one_block(gpu, n):
    """The encode block walks 2 048 units: one short, exact, one over; and tiny batches."""
    flags, kw, t1, t2, stride, _ = CASES["digit_borders_include_unmerged"]
    reps = (n + 1199) // 1200
    cut = lambda t: b"\n".join((t * reps).split(b"\n")[:4 * n]) + b"\n"      # noqa: E731
    t1, t2 = cut(t1), cut(t2)
    for iu in (0, 1):
        ctx = gpu.GpuCtx(M.merge_case_params(dict(merge_include_unmerged=iu), 150), 4096, stride, 2 * stride)
        got, want, _ = device_streams(gpu, ctx, t1, t2, n)
        ctx.close()
        for key, _ in STREAMS:
            assert got[key] == want[key], (key, n, iu)
        assert n < 7 or len(got["merged"]) > 0


def test_encode_complement_of_all_256_byte_values(gpu):
    """Rows are the caller's: read 2's part beyond the overlap holds every byte value; the device writes what the port writes."""
    import torch
    n, S = 8, 160
    rng = np.random.default_rng(3)
    r1 = rng.choice(E.ACGT, (n, 70))
    recs1, recs2 = [], []
    for i in range(n):
        recs1.append(b"@c%d 1\n%s\n+\n%s\n" % (i, bytes(r1[i]), b"I" * 70))
        recs2.append(b"@c%d 2\n%s\n+\n%s\n" % (i, b"A" * 32 + M._revcomp_text(bytes(r1[i]))[:50], b"I" * 82))
    t1, t2 = b"".join(recs1), b"".join(recs2)
    p = M.merge_case_params(dict(adapter_enabled=0, qual_filter_enabled=0), 150)
    ctx = gpu.GpuCtx(p, n, S, 2 * S)
    d1 = gpu.gpu_fastq_decode(ctx, t1, capacity=n); d2 = gpu.gpu_fastq_decode(ctx, t2, capacity=n)
    ch = M.gpu_chain_on_decoded(ctx, d1, d2, n)
    h = ch["host"]
    assert ((h["res1"]["flags"] & 0x80) != 0).all() and (h["res1"]["verdict"] == 0).all() and (h["ov"]["offset"] == 20).all()
    # after the chain: the 32 bases of read 2 that the merged read takes reversed become all 256 byte values, 32 per pair
    rows = h["seq2"].copy()
    rows[:, :32] = np.arange(256, dtype=np.uint8).reshape(n, 32)
    d2["dev"][1][:n * S].copy_(torch.from_numpy(rows.reshape(-1)))
    got = M.gpu_fastq_encode_merge(ctx, M.FQ_OUT_MERGED, d1, d2, ch, n)
    want = M.oracle_fastq_encode_merge(M.FQ_OUT_MERGED, 0, t1, d1["recs"], t2, d2["recs"], h["res1"], h["res2"], h["ov"], h["seq1"], h["qual1"], rows, h["qual2"], S)[0]
    ctx.close()
    assert got == want and got.count(b" merged_70_32\n") == n
    tails = b"".join(rec.split(b"\n")[1][70:][::-1] for rec in got.split(b"@c")[1:])
    comp = {ord("A"): "T", ord("a"): "T", ord("T"): "A", ord("t"): "A", ord("C"): "G", ord("c"): "G", ord("G"): "C", ord("g"): "C"}
    assert tails == bytes(ord(comp.get(b, "N")) for b in range(256))          # src/simd.cpp:296-308


def test_encode_out_cap(gpu):
    """One byte short of the total: the last unit that writes is left out whole and nothing lands at or behind its offset; the size
    query (cap 0, NULL buffer) is what device_streams sizes its buffers with."""
    flags, kw, t1, t2, stride, _ = CASES["named_strand_include_unmerged"]
    n = 500
    for iu in (0, 1):
        ctx = gpu.GpuCtx(M.merge_case_params(dict(merge_include_unmerged=iu), 150), n, stride, 2 * stride)
        got, want, (d1, d2, ch) = device_streams(gpu, ctx, t1, t2, n)
        h = ch["host"]
        for key, which in STREAMS:
            total = len(want[key])
            if total == 0:
                continue

            def port(k):
                return M.oracle_fastq_encode_merge(which, iu, t1, d1["recs"][:k], t2, d2["recs"][:k], h["res1"][:k], h["res2"][:k], h["ov"][:k],
                                                   h["seq1"][:k], h["qual1"][:k], h["seq2"][:k], h["qual2"][:k], stride)[0]
            k = n
            while len(port(k - 1)) == total:                                    # unit k - 1 is the last one that writes to this stream
                k -= 1
            head = port(k - 1)
            rc, buf, tot, guard_ok = M.gpu_fastq_encode_merge(ctx, which, d1, d2, ch, n, out_cap=total - 1)
            assert rc == 0 and tot == total and guard_ok, key
            assert buf[:len(head)] == head and set(buf[len(head):]) <= {M.GUARD}, key
        ctx.close()


def test_refusals(gpu):
    flags, kw, t1, t2, stride, _ = CASES["default"]
    lib = capi.load()
    total = T.C.c_int64(7)
    for p in (T.config_params("default", 0), T.config_params("cfg3_overlap_correction", 1)):       # single-end ctx, paired ctx that does not merge
        ctx = gpu.GpuCtx(p, 1024, 160, 320)
        rc = lib.fp_fastq_encode_merge(ctx.h, M.FQ_OUT_MERGED, *([None] * 11), 0, None, 0, T.C.byref(total))
        assert rc == -1 and total.value == 0                                    # FP_E_INVAL
        if p.paired:
            r = M.gpu_fastq_process_host_merge(ctx, t1, t2)
            assert r["rc"] == -1 and r["untouched"]
        ctx.close()
    ctx = gpu.GpuCtx(M.merge_case_params({}, 150), 1024, 160, 320)
    assert lib.fp_fastq_encode_merge(ctx.h, 3, *([None] * 11), 0, None, 0, T.C.byref(total)) == -1
    r = M.gpu_fastq_process_host_merge(ctx, t1, t2, entry="fp_fastq_process_host")              # the two-stream entry point on a merging ctx
    assert r["rc"] == -1 and r["untouched"] and b"fp_fastq_process_host_merge" in lib.fp_last_error()
    full = M.gpu_fastq_process_host_merge(ctx, t1, t2)
    ctx.close()
    ctx = gpu.GpuCtx(M.merge_case_params({}, 150), 1024, 160, 320)
    short = M.gpu_fastq_process_host_merge(ctx, t1, t2, out_cap=(len(full["out1"]), len(full["out2"]), len(full["merged"]) - 1))
    ctx.close()
    assert short["rc"] == -4 and short["guard_ok"]                              # FP_E_TOOLARGE


@pytest.mark.parametrize("name", list(CASES))
def test_text_path_equals_port_digests_and_reference_cli(gpu, tmp_path, name):
    """fp_fastq_process_host_merge over several rounds (max_batch well below the unit count) == C-port decode -> chain -> C-port encode;
    counters too; and the committed digests of the reference CLI's files (the CLI itself where it is present)."""
    flags, kw, t1, t2, stride, dedup = CASES[name]
    p = M.merge_case_params(kw, 250 if stride == 256 else 150)
    want = M.oracle_merge_text_path(p, t1, t2, stride, dup_level=3 if dedup else 0, dedup=dedup)
    ctx = gpu.GpuCtx(p, 700, stride, 2 * stride)                                # 3 000 pairs: five rounds
    if dedup:
        capi.check(ctx.lib.fp_fastq_set_dedup(ctx.h, 3, 1), ctx.lib)           # duplicates sit 3 000 pairs behind their first copy: another round
    got = M.gpu_fastq_process_host_merge(ctx, t1, t2)
    cnt = ctx.counters()
    ctx.close()
    assert got["rc"] == 0 and got["guard_ok"] and got["n"] == want["n"] and got["consumed"] == (len(t1), len(t2))
    for key, _ in STREAMS:
        assert got[key] == want[key], (name, key)
    T.assert_counters_equal(cnt, want["counters"], name)
    digests = json.load(open(DIGESTS))
    assert [hashlib.md5(got[k]).hexdigest() for k in ("merged", "out1", "out2")] == digests[name], name
    if os.path.exists(T.REF_CLI):
        m, o1, o2, _ = M.run_ref_cli_merge(tmp_path, flags, t1, t2)
        assert got["merged"] == m and got["out1"] == o1 and got["out2"] == o2


def test_text_path_three_upload_pieces(gpu):
    """Texts longer than two upload pieces (4 MiB each at this batch size), so rounds start on text that is still arriving."""
    n = 30000
    _, arrs = T.synth_host(n, 160, 1, 0, 57, 1, 150)
    t1, t2 = texts_of(arrs)
    assert len(t1) > 2 * (4 << 20)
    p = merge_params(0)
    want = M.oracle_merge_text_path(p, t1, t2, 160)
    ctx = gpu.GpuCtx(p, 4096, 160, 320)
    got = M.gpu_fastq_process_host_merge(ctx, t1, t2)
    cnt = ctx.counters()
    ctx.close()
    for key, _ in STREAMS:
        assert got[key] == want[key], key
    T.assert_counters_equal(cnt, want["counters"], "three pieces")


@pytest.mark.parametrize("name,gz", [("full", False), ("include_unmerged_full", True), ("dedup", False), ("named_strand", True)])
def test_mirror_cli(gpu, tmp_path, name, gz):
    """fastp_gpu_cli --device_fastq -m at two chunk sizes (records straddle chunk ends): files equal the port's streams and the committed
    reference digests, JSON after-filtering totals equal the port's counters (and the reference CLI's JSON where it is present)."""
    assert os.path.exists(CLI), "build with __graft_entry__.build()"
    flags, kw, t1, t2, stride, dedup = CASES[name]
    p = M.merge_case_params(kw, 150)
    want = M.oracle_merge_text_path(p, t1, t2, stride, dup_level=3 if dedup else 0, dedup=dedup)
    digests = json.load(open(DIGESTS))[name]
    (tmp_path / "r1.fq").write_bytes(t1); (tmp_path / "r2.fq").write_bytes(t2)
    ref_js = None
    if os.path.exists(T.REF_CLI):
        (tmp_path / "ref").mkdir()
        ref_js = M.run_ref_cli_merge(tmp_path / "ref", flags, t1, t2)[3]
    iu = "--include_unmerged" in flags
    for chunk in (100003, 1 << 20):
        d = tmp_path / str(chunk); d.mkdir()
        mname = "m.fq.gz" if gz else "m.fq"
        cmd = [CLI, "-i", str(tmp_path / "r1.fq"), "-I", str(tmp_path / "r2.fq"), "--device_fastq", "-m", "--merged_out", str(d / mname), "-j", str(d / "s.json"),
               "--chunk_bytes", str(chunk), "--pack_size", "2048", "--max_read_len", "150"] + flags
        cmd += ["-o", str(d / "o1.fq"), "-O", str(d / "o2.fq")]                # with --include_unmerged they are dropped with a warning
        if not dedup:
            cmd.append("--dont_eval_duplication")
        r = subprocess.run(cmd, capture_output=True, timeout=600)
        assert r.returncode == 0, r.stderr[-500:]
        m = (d / mname).read_bytes()
        m = gzip.decompress(m) if gz else m
        rd = lambda f: (d / f).read_bytes() if (d / f).exists() else b""       # noqa: E731
        o1, o2 = rd("o1.fq"), rd("o2.fq")
        assert (m, o1, o2) == (want["merged"], want["out1"], want["out2"]), (name, chunk)
        assert [hashlib.md5(x).hexdigest() for x in (m, o1, o2)] == digests
        if iu:
            assert b"Ignoring argument --out1" in r.stderr and not (d / "o1.fq").exists()
        js = json.load(open(d / "s.json"))
        c = want["counters"]
        for key, field in (("reads", "total_reads"), ("bases", "total_bases"), ("q20", "q20_bases"), ("q30", "q30_bases")):
            assert js["after_filtering"][field] == c.summary(capi.STATS_POST1)[key], (field, chunk)
            if ref_js is not None:
                assert js["after_filtering"][field] == ref_js["summary"]["after_filtering"][field]


def test_mirror_cli_argument_rules(gpu, tmp_path):
    (tmp_path / "r.fq").write_bytes(b"@a\nACGT\n+\nIIII\n")
    base = [CLI, "-i", str(tmp_path / "r.fq")]
    for extra, msg in ((["-I", str(tmp_path / "r.fq"), "-m", "--merged_out", str(tmp_path / "m.fq")], b"--device_fastq"),
                       (["--device_fastq", "-m", "--merged_out", str(tmp_path / "m.fq")], b"--in2"),
                       (["--device_fastq", "-I", str(tmp_path / "r.fq"), "-m"], b"--merged_out")):
        r = subprocess.run(base + extra, capture_output=True, timeout=120)
        assert r.returncode == 2 and msg in r.stderr, (extra, r.stderr)
    assert not (tmp_path / "m.fq").exists()
