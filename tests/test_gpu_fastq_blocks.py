"""-m gpu: the device FASTQ codec past one warp of lines.  fq_fsm_kernel carries the 4-state record automaton across lanes, warps
(256 lines) and blocks (2 048 lines); clean four-line records start every one of them in state 0, so the texts here shift the
records by 1-3 lines, end lines with "\\r\\n" / "\\r" across thread and block borders, break several records in different blocks
and cut the chunk in late blocks.  Device == C port (tests/test_oracle_dedup.py pins the C port to FastqReader on the same texts).
Then fp_fastq_encode under an output cap, and fp_fastq_process_host over many rounds against
C-port decode -> C-port chain -> C-port encode."""
import ctypes as C

import numpy as np
import pytest

import fp_testlib as T
from fastp_b200 import capi
from test_duplicate_oracle import planted
from test_gpu_fastq import same_decode

pytestmark = pytest.mark.gpu
S = 160
FP_E_TOOLARGE = -4
FP_F_DUPLICATE = 0x40


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


@pytest.fixture(scope="module")
def ctx(gpu):
    c = gpu.GpuCtx(T.config_params("default", 0), 4096, S, S)
    yield c
    c.close()


def both(gpu, ctx, text, what, **kw):
    want = T.oracle_fastq_decode(text, stride=S, **kw)
    same_decode(gpu.gpu_fastq_decode(ctx, text, **kw), want, what)
    return want


# ---------------- decode ----------------
def test_block_warp_and_thread_starts_in_every_automaton_state(gpu, ctx):
    text = T.fastq_shifted_text()
    want = both(gpu, ctx, text, "shifted", capacity=12000)
    assert want["info"]["n_records"] == 12000 and want["info"]["n_lines"] > 20 * T.FQ_LINES_PER_BLOCK
    st = T.states_at_block_starts(text, want["recs"])
    assert set(st[1:]) == {0, 1, 2, 3}, st
    ls = T.line_starts(text)
    at = [b for b, s in enumerate(st) if s == 3 and text[ls[b * T.FQ_LINES_PER_BLOCK]] == ord("@")]
    assert at, "no quality line beginning with '@' on a block's first line"
    for cap in (5000, 11999):                                  # capacity reached in a later block: more, consumed
        w = both(gpu, ctx, text, f"capacity {cap}", capacity=cap)
        assert w["info"]["more"] == 1 and w["info"]["consumed"] == int(want["recs"]["name_off"][cap])
    for cut in (len(text) // 3, len(text) - 7):                # non-final cuts inside a record of a later block
        both(gpu, ctx, text[:cut], f"cut {cut}", final=0, capacity=12000)
        both(gpu, ctx, text[:cut], f"cut {cut} final", final=1, capacity=12000)


@pytest.mark.parametrize("seed", [11, 12])
def test_long_fuzz_text(gpu, ctx, seed):
    rng = np.random.default_rng(seed)
    text = T.fastq_fuzz_text(rng, nrec=5000)
    assert text.count(b"\n") + text.count(b"\r") > 10000
    both(gpu, ctx, text, "fuzz whole")
    for cut in rng.integers(len(text) // 2, len(text), 4):
        both(gpu, ctx, text[:int(cut)], f"fuzz prefix {cut}", final=0)
    # no broken records: every record is decoded, with junk lines and all three line ends between and inside them
    text = T.fastq_fuzz_text(np.random.default_rng(seed), nrec=5000, broken=0)
    w = both(gpu, ctx, text, "fuzz unbroken")
    assert w["info"]["n_records"] == 5000 and w["info"]["error"] == 0
    both(gpu, ctx, text, "fuzz unbroken, capacity", capacity=4321)
    for cut in rng.integers(len(text) // 2, len(text), 4):
        both(gpu, ctx, text[:int(cut)], f"fuzz unbroken prefix {cut}", final=0)


@pytest.mark.parametrize("eol", ["\r\n", "\r"])
def test_cr_line_ends_across_thread_and_block_borders(gpu, ctx, eol):
    text = T.fastq_eol_text(eol)
    assert len(text) > 3 * T.FQ_BYTES_PER_BLOCK
    both(gpu, ctx, text, "eol whole")
    cr = [o for o in (T.FQ_BYTES_PER_BLOCK - 1, 3 * T.FQ_BYTES_PER_BLOCK - 1, text.rindex(b"\r"))]
    for o in cr:                                               # the chunk ends on '\r', final and not
        assert text[o] == 13
        for final in (0, 1):
            both(gpu, ctx, text[:o + 1], f"ends on CR at {o} final {final}", final=final)


@pytest.mark.parametrize("misalign", [0, 1, 15])
def test_text_alignment(gpu, ctx, misalign):
    """The terminator pass reads 16 bytes at a time where the address allows it and byte by byte elsewhere."""
    text = T.fastq_eol_text("\r\n", nrec=1500, seed=5, straddle=(63, T.FQ_BYTES_PER_BLOCK - 1))
    want = T.oracle_fastq_decode(text, stride=S)
    same_decode(gpu.gpu_fastq_decode(ctx, text, misalign=misalign), want, f"misalign {misalign}")


@pytest.mark.parametrize("bad", [(("length", 9000), ("strand", 5200)), (("strand", 9000), ("length", 5200)),
                                 (("strand", 11000), ("length", 700), ("strand", 6000))])
def test_first_bad_record_of_several_blocks(gpu, ctx, bad):
    text = T.fastq_shifted_text(at_quality_on_block_start=False)
    recs = T.oracle_fastq_decode(text, stride=S, capacity=12000)["recs"]
    for how, idx in sorted(bad, key=lambda x: -x[1]):          # from the back: earlier offsets stay valid
        text = T.fastq_break_record(text, recs, idx, how)
    first = min(bad, key=lambda x: x[1])
    w = both(gpu, ctx, text, f"bad {bad}", capacity=12000)
    assert w["info"]["error"] == {"strand": 1, "length": 2}[first[0]] and w["info"]["error_record"] == first[1] == w["info"]["n_records"]


def test_read_longer_than_the_stride_in_a_late_block(gpu, ctx):
    text = T.fastq_shifted_text(nrec=6000)
    recs = T.oracle_fastq_decode(text, stride=S, capacity=6000)["recs"]
    o = int(recs["name_off"][5500])
    text = text[:o] + b"@long\n" + b"A" * (S + 1) + b"\n+\n" + b"I" * (S + 1) + b"\n" + text[o:]
    w = both(gpu, ctx, text, "stride", capacity=6001)
    assert w["info"]["error"] == 3 and w["info"]["error_record"] == 5500


# ---------------- encode under a cap ----------------
def test_encode_cap_and_dropped_records(gpu, ctx):
    import torch
    text = T.fastq_shifted_text(nrec=6000, seed=3)
    want = T.oracle_fastq_decode(text, stride=S, capacity=6000)
    got = gpu.gpu_fastq_decode(ctx, text, capacity=6000)
    n = 6000
    rng = np.random.default_rng(4)
    res = np.zeros(n, capi.READ_RESULT_DTYPE)
    ln = want["len"].astype(np.int64)
    res["front"] = rng.integers(0, ln // 2 + 1)
    res["len"] = rng.integers(0, ln - res["front"] + 1)
    res["pair_verdict"] = np.where(rng.random(n) < 0.3, 1, 0)
    res["flags"] = np.where(rng.random(n) < 0.3, FP_F_DUPLICATE, 0)
    res["pair_verdict"][256:512] = 1                           # a whole 256-record group and a whole 2 048-record block written nothing
    res["flags"][2048:4096] |= FP_F_DUPLICATE
    kept = (res["pair_verdict"] == 0) & (res["flags"] & FP_F_DUPLICATE == 0)
    assert kept[:256].any() and kept[4096:].any() and not kept[256:512].any() and not kept[2048:4096].any()
    assert ((res["pair_verdict"] == 0) & (res["flags"] & FP_F_DUPLICATE != 0)).sum() > 500
    olib = T.oracle(); T._bind_fastq(olib)
    tbuf = np.frombuffer(text, np.uint8).copy()
    keep = (np.ascontiguousarray(want["recs"]), np.ascontiguousarray(want["seq"]), np.ascontiguousarray(want["qual"]))
    oargs = (tbuf.ctypes.data, keep[0].ctypes.data, res.ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data, S, n)
    total = olib.fp_oracle_fastq_encode(*oargs, None, 0)
    assert total > 50000
    d_text, d_seq, d_qual, d_len, d_recs = got["dev"]
    d_res = torch.from_numpy(res.view(np.uint8).copy()).cuda()
    for cap in (0, total // 2, total - 1, total):
        ref = np.full(total + 64, 0xA5, np.uint8)
        assert olib.fp_oracle_fastq_encode(*oargs, ref.ctypes.data, cap) == total
        d_out = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device="cuda:0")
        nb = C.c_int64()
        capi.check(ctx.lib.fp_fastq_encode(ctx.h, d_text.data_ptr(), d_recs.data_ptr(), d_res.data_ptr(), d_seq.data_ptr(), d_qual.data_ptr(), n,
                                           d_out.data_ptr(), cap, C.byref(nb)), ctx.lib)
        out = d_out.cpu().numpy()
        assert nb.value == total, cap
        assert (out[cap:] == 0xA5).all(), f"bytes written behind out_cap {cap}"
        assert np.array_equal(out, ref), cap


# ---------------- fp_fastq_process_host over many rounds ----------------
def pipeline(p, texts, is_dup=None):
    """C-port decode -> chain -> encode of one or two whole texts: (outputs, units, counters, decodes)."""
    dec = [T.oracle_fastq_decode(t, stride=S, capacity=t.count(b"\n") // 4 + 2) for t in texts]
    n = min(int(d["info"]["n_records"]) for d in dec)
    arrs = {}
    for k, d in enumerate(dec):
        sd = str(k + 1)
        arrs["seq" + sd], arrs["qual" + sd], arrs["len" + sd] = d["seq"][:n].copy(), d["qual"][:n].copy(), d["len"][:n].copy()
    r = T.run_cpu("oracle", p, arrs, S, is_dup=is_dup(arrs) if is_dup else None)
    outs = [T.oracle_fastq_encode(t, d["recs"][:n], r["out" + str(k + 1)], r["arrs"]["seq" + str(k + 1)], r["arrs"]["qual" + str(k + 1)], S)
            for k, (t, d) in enumerate(zip(texts, dec))]
    return outs, n, r["counters"], dec


def stream_texts(paired, n, seed=41, name_pad=0):
    _, arrs = T.synth_host(n, S, paired, 0, seed, 1, 150)
    tag = lambda sd: sd + ":N:0" + "x" * name_pad               # noqa: E731
    return [T.fastq_text(arrs["seq" + sd], arrs["qual" + sd], arrs["len" + sd], tag(sd)) for sd in ("1", "2")[: 2 if paired else 1]]


def same_outputs(got, outs, what):
    for k, o in enumerate(outs):
        g = got["out%d" % (k + 1)]
        assert len(g) == len(o), (what, k, len(g), len(o))
        assert g == o, (what, k)


@pytest.mark.parametrize("paired", [1, 0])
def test_process_host_many_rounds_and_upload_pieces(gpu, paired):
    p = T.config_params("cfg4_full", paired)
    texts = stream_texts(paired, 27000)
    assert all(len(t) > 8 << 20 for t in texts)
    outs, n, cnt, dec = pipeline(p, texts)
    c = gpu.GpuCtx(p, 1000, S, S)
    got = gpu.gpu_fastq_process_host(c, *texts)
    assert got["n"] == n == 27000 and got["consumed"] == tuple(len(t) for t in texts) and got["guard_ok"]
    same_outputs(got, outs, "27 rounds")
    T.assert_counters_equal(c.counters(), cnt, "27 rounds")
    # the same stream in two calls: a non-final call cut inside a record, its remainder carried into the final call
    c.reset()
    cuts = [len(t) * 2 // 5 + 13 for t in texts]
    a = gpu.gpu_fastq_process_host(c, *[t[:k] for t, k in zip(texts, cuts)], final=0)
    assert 0 < a["n"] < n and all(x <= k for x, k in zip(a["consumed"], cuts))
    for t, x, d in zip(texts, a["consumed"], dec):
        assert x == int(d["recs"]["name_off"][a["n"]])
    b = gpu.gpu_fastq_process_host(c, *[t[x:] for t, x in zip(texts, a["consumed"])], final=1)
    assert a["n"] + b["n"] == n
    same_outputs({k: a[k] + b[k] for k in ("out1", "out2") if k in a}, outs, "two calls")
    T.assert_counters_equal(c.counters(), cnt, "two calls")
    c.close()


@pytest.mark.parametrize("short", [1, 0])
def test_process_host_sides_of_different_length(gpu, short):
    p = T.config_params("cfg4_full", 1)
    texts = stream_texts(1, 6000)
    full = T.oracle_fastq_decode(texts[short], stride=S, capacity=6000)
    texts[short] = texts[short][:int(full["recs"]["name_off"][6000 - 137])]
    outs, n, cnt, dec = pipeline(p, texts)
    assert n == 6000 - 137
    c = gpu.GpuCtx(p, 1000, S, S)
    got = gpu.gpu_fastq_process_host(c, *texts)
    want_consumed = [len(texts[short])] * 2
    want_consumed[1 - short] = int(dec[1 - short]["recs"]["name_off"][n])
    assert got["n"] == n and list(got["consumed"]) == want_consumed, (got["n"], got["consumed"], want_consumed)
    same_outputs(got, outs, f"side {short + 1} short")
    T.assert_counters_equal(c.counters(), cnt, "short side")
    assert [i["n_records"] for i in got["info"]] == [n, n] and all(i["error"] == 0 for i in got["info"])
    c.close()


@pytest.mark.parametrize("side,how", [(1, "strand"), (0, "length")])
def test_process_host_reader_error_in_round_seven(gpu, side, how):
    p = T.config_params("cfg4_full", 1)
    texts = stream_texts(1, 9000)
    recs = T.oracle_fastq_decode(texts[side], stride=S, capacity=9000)["recs"]
    texts[side] = T.fastq_break_record(texts[side], recs, 6500, how)
    outs, n, cnt, dec = pipeline(p, texts)
    assert n == 6500 and dec[side]["info"]["error_record"] == 6500
    c = gpu.GpuCtx(p, 1000, S, S)
    got = gpu.gpu_fastq_process_host(c, *texts)
    assert got["n"] == 6500
    same_outputs(got, outs, "reader error")
    T.assert_counters_equal(c.counters(), cnt, "reader error")
    assert got["info"][side]["error"] == dec[side]["info"]["error"] and got["info"][side]["error_record"] == 6500
    assert got["info"][1 - side]["error"] == 0 and got["info"][side]["n_records"] == 6500
    c.close()


def test_process_host_long_names_and_small_output_buffer(gpu):
    p = T.config_params("cfg4_full", 0)
    texts = stream_texts(0, 2500, name_pad=500)
    outs, n, cnt, _ = pipeline(p, texts)
    total = len(outs[0])
    assert total > n * (2 * S + 256)                            # more per record than the first encode attempt allows for
    c = gpu.GpuCtx(p, 1000, S, S)
    got = gpu.gpu_fastq_process_host(c, texts[0], out_cap=(total,))
    assert got["rc"] == 0 and got["guard_ok"]
    same_outputs(got, outs, "long names")
    c.reset()
    small = gpu.gpu_fastq_process_host(c, texts[0], out_cap=(total - 1,))
    assert small["rc"] == FP_E_TOOLARGE and small["guard_ok"]
    c.close()


@pytest.mark.parametrize("paired", [1, 0])
def test_process_host_dedup_across_rounds(gpu, paired):
    """fp_fastq_set_dedup(level 1, dedup): the filter's arrays live across rounds, so a copy whose original went through an earlier
    round is dropped and left out of the post-filter stats -- the sequential filter over the whole stream says which."""
    p = T.config_params("cfg4_full", paired)
    arrs = planted(paired)
    n = len(arrs["len1"])
    texts = [T.fastq_text(arrs["seq" + sd], arrs["qual" + sd], arrs["len" + sd], sd + ":N:0") for sd in ("1", "2")[: 2 if paired else 1]]
    flags, total, dups = T.oracle_dup_flags([arrs], paired, 1)
    key = [arrs["seq1"][i].tobytes() + (arrs["seq2"][i].tobytes() if paired else b"") for i in range(n)]
    first = {}
    for i, k in enumerate(key):
        first.setdefault(k, i)
    assert sum(1 for i, k in enumerate(key) if flags[0][i] and first[k] < i // 1000 * 1000) > 300
    outs, nn, cnt, _ = pipeline(p, texts, is_dup=lambda a: flags[0])
    assert nn == n
    c = gpu.GpuCtx(p, 1000, S, S)
    capi.check(c.lib.fp_fastq_set_dedup(c.h, 1, 1), c.lib)
    got = gpu.gpu_fastq_process_host(c, *texts)
    same_outputs(got, outs, "dedup")
    T.assert_counters_equal(c.counters(), cnt, "dedup")
    t, d = C.c_int64(), C.c_int64()
    capi.check(c.lib.fp_dup_totals(c.h, C.byref(t), C.byref(d)), c.lib)
    assert (t.value, d.value) == (total, dups)
    c.close()
