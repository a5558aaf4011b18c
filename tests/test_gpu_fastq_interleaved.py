"""-m gpu: interleaved pairs on the device text path (--interleaved_in, --stdin, --stdout).  fp_fastq_decode_interleaved and
fp_fastq_encode_interleaved against their C port; fp_fastq_process_host* with fp_fastq_set_interleaved against the port's whole text path,
the committed digests of the UNMODIFIED reference CLI's outputs (tests/golden/fastq_interleaved_cli_digests.json) and, where
oracle/_ref/fastp_ref travelled along, that CLI itself; fastp_gpu_cli --device_fastq through a pipe.  The port is pinned to the reference
on the CPU by tests/test_oracle_fastq_interleaved.py."""
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import fp_interleaved as IL
import fp_outs as O
import fp_testlib as T
from fastp_b200 import capi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "fastp_b200", "host", "fastp_gpu_cli")
DIGESTS = os.path.join(ROOT, "tests", "golden", "fastq_interleaved_cli_digests.json")
CASES = O.fastq_outs_cases()
GUARD = 0xA5
R1, R2 = capi.FP_FQ_OUT_R1, capi.FP_FQ_OUT_R2


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def gpu_decode_il(ctx, text, final=1, capacity=None):
    """fp_fastq_decode_interleaved on cuda:0 -> same shape as fp_interleaved.oracle_decode_il (+ device tensors per side)."""
    import torch
    lib, S = ctx.lib, ctx.stride
    cap = capacity if capacity is not None else text.count(b"@") // 2 + 2
    c1 = max(cap, 1)
    d_text = torch.from_numpy(np.concatenate([np.frombuffer(text, np.uint8), np.zeros(1, np.uint8)])).cuda()
    dev = [dict(seq=torch.full((c1 * S + 64,), 0xEE, dtype=torch.uint8, device="cuda:0"), qual=torch.full((c1 * S + 64,), 0xEE, dtype=torch.uint8, device="cuda:0"),
                len=torch.zeros(c1, dtype=torch.int16, device="cuda:0"), recs=torch.zeros(c1 * 16, dtype=torch.uint8, device="cuda:0")) for _ in range(2)]
    info = capi.FastqInfo()
    ptrs = [dev[s][k].data_ptr() for s in range(2) for k in ("seq", "qual", "len", "recs")]
    capi.check(lib.fp_fastq_decode_interleaved(ctx.h, d_text.data_ptr(), len(text), final, 0, *ptrs, cap, C.byref(info)), lib)
    n = int(info.n_records)
    sides = [{"seq": d["seq"].cpu().numpy()[:c1 * S].reshape(c1, S)[:n], "qual": d["qual"].cpu().numpy()[:c1 * S].reshape(c1, S)[:n],
              "len": d["len"].cpu().numpy().view(np.uint16)[:n], "recs": d["recs"].cpu().numpy().view(capi.FASTQ_REC_DTYPE)[:n].copy()} for d in dev]
    return {"sides": sides, "info": {k: int(getattr(info, k)) for k, _ in capi.FastqInfo._fields_}, "dev": dev, "text": d_text}


def same_decode(a, b, what):
    assert a["info"] == b["info"], (what, a["info"], b["info"])
    for s in range(2):
        for k in ("seq", "qual", "len", "recs"):
            assert np.array_equal(a["sides"][s][k], b["sides"][s][k]), (what, s, k)


def texts_around_blocks():
    """Interleaved texts of 2 x 150 reads whose record and line counts sit around the decode's 2 048-line and 16 KiB blocks, with odd counts."""
    _, arrs = T.synth_host(1200, 160, 1, 0, 31, 1, 150)
    t1 = T.fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0"); t2 = T.fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0")
    recs = [r for a, b in zip(IL.records(t1), IL.records(t2)) for r in (a, b)]
    return {k: b"".join(recs[:k]) for k in (1, 2, 3, 47, 48, 511, 512, 513, 1023, 2047, 2048, 2049)}


def test_decode_equals_port(gpu):
    """Whole, non-final (a lone mate 1 at the end is left for the next chunk) and capacity-cut decodes, at record counts around the blocks."""
    ctx = gpu.GpuCtx(capi.default_params(1, lib=T.oracle()), 4096, 160, 160)
    for k, text in texts_around_blocks().items():
        for final in (1, 0):
            same_decode(gpu_decode_il(ctx, text, final), IL.oracle_decode_il(text, final), (k, final))
            cut = text[:len(text) * 2 // 3]                        # mid-record
            same_decode(gpu_decode_il(ctx, cut, final), IL.oracle_decode_il(cut, final), (k, final, "cut"))
        for cap in (1, 5, k // 2, (k + 1) // 2):                   # capacity cuts at odd records
            if cap > 0:
                same_decode(gpu_decode_il(ctx, text, 1, cap), IL.oracle_decode_il(text, 1, capacity=cap), (k, "cap", cap))
    for name, (text, ph) in __import__("test_oracle_fastq_interleaved").decode_texts().items():
        if ph == 0:
            same_decode(gpu_decode_il(ctx, text), IL.oracle_decode_il(text), name)
    ctx.close()


def device_chain_il(gpu, ctx, text, n):
    """interleaved decode -> fp_process_pe on the device -> the decode, the device records and host copies of the rows and records."""
    import torch
    lib, S = ctx.lib, ctx.stride
    d = gpu_decode_il(ctx, text, capacity=n)
    assert d["info"]["n_records"] == n
    m = max(n, 1)
    res = [torch.zeros(m * 16, dtype=torch.uint8, device="cuda:0") for _ in range(2)]
    b = capi.Batch()
    b.n, b.stride = n, S
    b.seq1, b.qual1, b.len1 = (d["dev"][0][k].data_ptr() for k in ("seq", "qual", "len"))
    b.seq2, b.qual2, b.len2 = (d["dev"][1][k].data_ptr() for k in ("seq", "qual", "len"))
    ov = torch.zeros(m * 8, dtype=torch.uint8, device="cuda:0")
    capi.check(lib.fp_process_pe(ctx.h, C.byref(b), res[0].data_ptr(), res[1].data_ptr(), ov.data_ptr(), None, 0, None, None), lib)
    torch.cuda.synchronize()
    host = {}
    for s in range(2):
        host[f"res{s + 1}"] = res[s].cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy()
        host[f"seq{s + 1}"] = d["dev"][s]["seq"].cpu().numpy()[:m * S].reshape(m, S)[:n].copy()
        host[f"qual{s + 1}"] = d["dev"][s]["qual"].cpu().numpy()[:m * S].reshape(m, S)[:n].copy()
    return d, res, host


def gpu_encode_il(ctx, d, res, n, out_cap=None):
    import torch
    lib = ctx.lib
    dv = d["dev"]
    args = [d["text"].data_ptr(), dv[0]["recs"].data_ptr(), d["text"].data_ptr(), dv[1]["recs"].data_ptr(), res[0].data_ptr(), res[1].data_ptr(),
            dv[0]["seq"].data_ptr(), dv[0]["qual"].data_ptr(), dv[1]["seq"].data_ptr(), dv[1]["qual"].data_ptr(), n]
    total = C.c_int64()
    capi.check(lib.fp_fastq_encode_interleaved(ctx.h, *args, None, 0, C.byref(total)), lib)
    cap = total.value if out_cap is None else out_cap
    d_out = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda:0")
    t2 = C.c_int64()
    capi.check(lib.fp_fastq_encode_interleaved(ctx.h, *args, d_out.data_ptr(), cap, C.byref(t2)), lib)
    h = d_out.cpu().numpy()
    assert t2.value == total.value and bool((h[cap:] == GUARD).all())
    return h[:cap].tobytes(), total.value


@pytest.mark.parametrize("n", [1, 7, 2047, 2048, 2049])
def test_encode_equals_port_and_interleaved_sides(gpu, n):
    """The device's interleaved stream == the port on the device chain's own records == fp_fastq_encode's out1 and out2 interleaved
    (filters and -D flags; batch sizes around the 2 048-unit encode block)."""
    flags, kw, paired, t1, t2, S, _ = CASES["filters_pe"]
    text = IL.interleave(t1, t2)
    text = b"".join(IL.records(text)[:2 * n])
    ctx = gpu.GpuCtx(O.case_params("filters_pe"), 4096, S, S)
    d, res, h = device_chain_il(gpu, ctx, text, n)
    got, total = gpu_encode_il(ctx, d, res, n)
    sd1, sd2 = d["sides"]
    want = IL.oracle_encode_il(text, sd1["recs"], text, sd2["recs"], h["res1"], h["res2"], h["seq1"], h["qual1"], h["seq2"], h["qual2"], S)[0]
    assert got == want
    o1 = gpu.gpu_fastq_encode(ctx, (d["text"], d["dev"][0]["seq"], d["dev"][0]["qual"], d["dev"][0]["len"], d["dev"][0]["recs"]), h["res1"], n)
    o2 = gpu.gpu_fastq_encode(ctx, (d["text"], d["dev"][1]["seq"], d["dev"][1]["qual"], d["dev"][1]["len"], d["dev"][1]["recs"]), h["res2"], n)
    assert got == IL.interleave(o1, o2)
    if n > 100:
        part, tot = gpu_encode_il(ctx, d, res, n, out_cap=total - 1)   # one byte short: the last writing unit is left out whole
        head = part.rstrip(bytes([GUARD]))
        assert tot == total and want.startswith(head) and want[len(head):len(head) + 1] == b"@" and 1 <= len(IL.records(want[len(head):])) <= 2
    ctx.close()


def process_host_il(ctx, text1, text2, want, il_in, il_out, caps=None, final=1):
    """fp_fastq_set_interleaved + fp_fastq_process_host_outs -> dict(rc, streams, n, consumed, info, guard_ok, untouched)."""
    lib = ctx.lib
    rc = lib.fp_fastq_set_interleaved(ctx.h, il_in, il_out)
    if rc:
        return {"rc": rc, "set": False}
    if caps is None:
        caps = [2 * (len(text1) + len(text2)) + 256] * 6
    b1 = np.frombuffer(text1, np.uint8).copy() if text1 else np.zeros(1, np.uint8)
    b2 = np.frombuffer(text2, np.uint8).copy() if text2 else None
    outs = [np.full(caps[s] + 64, GUARD, np.uint8) if s in want else None for s in range(6)]
    optr = (C.c_void_p * 6)(*[o.ctypes.data if o is not None else None for o in outs])
    ocap = (C.c_int64 * 6)(*[caps[s] if s in want else 0 for s in range(6)])
    ob = (C.c_int64 * 6)(*([-7] * 6))
    nu, c1, c2 = C.c_int64(), C.c_int64(-3), C.c_int64(-3)
    i1, i2 = capi.FastqInfo(), capi.FastqInfo()
    i2.n_records = -5
    rc = lib.fp_fastq_process_host_outs(ctx.h, b1.ctypes.data, len(text1), b2.ctypes.data if b2 is not None else None, len(text2), final, 0,
                                        optr, ocap, ob, C.byref(nu), C.byref(c1), C.byref(c2), C.byref(i1), C.byref(i2))
    r = {"rc": rc, "set": True, "n": nu.value, "consumed": (c1.value, c2.value), "i1": {k: int(getattr(i1, k)) for k, _ in capi.FastqInfo._fields_},
         "i2": {k: int(getattr(i2, k)) for k, _ in capi.FastqInfo._fields_},
         "guard_ok": all(o is None or bool((o[caps[s]:] == GUARD).all()) for s, o in enumerate(outs)),
         "untouched": all(o is None or bool((o == GUARD).all()) for o in outs) and list(ob) == [-7] * 6}
    for s in range(6):
        r[s] = outs[s][:min(ob[s], caps[s])].tobytes() if (rc == 0 and outs[s] is not None) else b""
    return r


HOST_RUNS = ["filters_pe/il", "filters_pe/il_stdout", "filters_pe/stdout", "filters_pe/il_stdout_f", "filters_pe/stdout_u1u2f", "dedup_pe/il_stdout",
             "merge_pe/il", "merge_pe/il_stdout", "merge_iu_pe/il_stdout", "edge48_pe/il_stdout", "edge256_pe/il"]


@pytest.mark.parametrize("run", HOST_RUNS)
def test_text_path_equals_port_digests_and_reference_cli(gpu, tmp_path, run):
    """fp_fastq_process_host_outs with both switches over many rounds (max_batch 700) == the port; what the reference CLI writes from those
    streams matches the committed digests and, where present, the CLI itself."""
    name, inp, outm, wset = IL.RUNS[run]
    flags, kw, paired, _, _, S, dedup = CASES[name]
    p = O.case_params(name)
    merging = "-m" in flags
    iu = "--include_unmerged" in flags
    t1, t2, _ = IL.run_inputs(run)
    il_in = 1 if inp.endswith("il") else 0
    il_out = 1 if (outm == "stdout" and not merging) else 0
    u1, u2, f = O.WRITER_SETS[wset] if wset else (0, 0, 0)
    want = set()
    if outm == "stdout":
        want |= {0} if merging else {R1}
    else:
        want |= ({0} if merging else set()) | (set() if iu else {R1, R2})
    want |= ({O.U1} if u1 else set()) | ({O.U2} if u2 else set()) | ({O.FAILED} if f else set())
    ctx = gpu.GpuCtx(p, 700, S, 2 * S if merging else S)
    if dedup:
        capi.check(ctx.lib.fp_fastq_set_dedup(ctx.h, 3, 1), ctx.lib)
    r = process_host_il(ctx, t1, t2, want, il_in, il_out)
    ctx.close()
    g = IL.port_streams(run)
    assert r["rc"] == 0 and r["guard_ok"] and r["n"] == g["n"], run
    assert r["consumed"] == ((len(t1), 0) if il_in else (len(t1), len(t2)))
    if il_in:
        assert r["i2"] == {k: 0 for k in r["i2"]} and r["i1"]["n_records"] == g["n"]
    if il_out:
        assert r[R1] == g["stdout_il"] == IL.interleave(g["out1"], g["out2"]) and r[R2] == b""
    else:
        assert r[R1] == (g["out1"] if R1 in want else b"") and r[R2] == (g["out2"] if R2 in want else b"")
        assert r[0] == (g["merged"] if 0 in want else b"")
    exp = IL.expected_outputs(run)
    stdout = r[0] if (outm == "stdout" and merging) else (r[R1] if outm == "stdout" else b"")
    files = (stdout, b"" if outm == "stdout" else r[R1], b"" if outm == "stdout" else r[R2], b"" if outm == "stdout" else r[0],
             r[O.U1], r[O.U2] if u1 else b"", r[O.FAILED])
    assert files == exp, run
    assert [hashlib.md5(x).hexdigest() for x in files] == json.load(open(DIGESTS))[run], run
    if os.path.exists(T.REF_CLI):
        assert IL.run_ref_cli(tmp_path, run)[0] == files


def test_text_path_many_pieces(gpu):
    """60 K enriched pairs in one interleaved text (several upload pieces, max_batch 4 093 so that rounds end on odd records): the interleaved
    stream equals the two-file path's out1 and out2 interleaved, and the port; a chunk that is not final leaves its lone mate 1."""
    n = 60001
    _, arrs = T.synth_host(n, 160, 1, 0, 77, 1, 150)
    t1 = T.fastq_text(arrs["seq1"], arrs["qual1"], arrs["len1"], "1:N:0"); t2 = T.fastq_text(arrs["seq2"], arrs["qual2"], arrs["len2"], "2:N:0")
    text = IL.interleave(t1, t2)
    p = capi.default_params(1, lib=T.oracle(), seq_len1=150, seq_len2=150, qualified_qual=33 + 30, unqualified_percent_limit=10, length_required=120)
    ctx = gpu.GpuCtx(p, 4093, 160, 160)
    two = process_host_il(ctx, t1, t2, {R1, R2, O.FAILED}, 0, 0)
    ctx.close()
    ctx = gpu.GpuCtx(p, 4093, 160, 160)
    one = process_host_il(ctx, text, b"", {R1, O.FAILED}, 1, 1)
    ctx.close()
    assert two["rc"] == 0 and one["rc"] == 0 and one["n"] == two["n"] == n
    assert one[R1] == IL.interleave(two[R1], two[R2]) and one[O.FAILED] == two[O.FAILED] and len(one[R1]) > 0
    d = IL.oracle_decode_il(text, stride=160)
    sd1, sd2 = d["sides"]
    a = {"seq1": sd1["seq"].copy(), "qual1": sd1["qual"].copy(), "len1": sd1["len"].copy(), "seq2": sd2["seq"].copy(), "qual2": sd2["qual"].copy(),
         "len2": sd2["len"].copy()}
    res = T.run_cpu("oracle", p, a, 160)
    ra = res["arrs"]
    want = IL.oracle_encode_il(text, sd1["recs"], text, sd2["recs"], res["out1"], res["out2"], ra["seq1"], ra["qual1"], ra["seq2"], ra["qual2"], 160)[0]
    assert one[R1] == want
    lone = text + IL.records(t1)[0]                                   # a trailing mate 1: not final -> left; final -> dropped
    ctx = gpu.GpuCtx(p, 4093, 160, 160)
    nf = process_host_il(ctx, lone, b"", {R1}, 1, 1, final=0)
    fin = process_host_il(ctx, lone, b"", {R1}, 1, 1, final=1)
    ctx.close()
    assert nf["consumed"][0] == len(text) and nf["n"] == n and fin["consumed"][0] == len(lone) and fin["n"] == n


def test_refusals(gpu):
    flags, kw, paired, t1, t2, S, _ = CASES["filters_pe"]
    lib = capi.load()
    se = gpu.GpuCtx(O.case_params("filters_se"), 700, S, S)
    for i, o in ((1, 0), (0, 1), (1, 1)):
        assert lib.fp_fastq_set_interleaved(se.h, i, o) == -1, (i, o)        # single-end ctx
    assert lib.fp_fastq_set_interleaved(se.h, 0, 0) == 0
    total = C.c_int64(5)
    assert lib.fp_fastq_encode_interleaved(se.h, *([None] * 10), 0, None, 0, C.byref(total)) == -1 and total.value == 0
    se.close()
    mg = gpu.GpuCtx(O.case_params("merge_pe"), 700, S, 2 * S)
    assert lib.fp_fastq_set_interleaved(mg.h, 0, 1) == -1 and lib.fp_fastq_set_interleaved(mg.h, 1, 1) == -1
    assert lib.fp_fastq_encode_interleaved(mg.h, *([None] * 10), 0, None, 0, C.byref(total)) == -1
    assert lib.fp_fastq_set_interleaved(mg.h, 1, 0) == 0                      # merging mode reads interleaved input
    mg.close()
    pe = gpu.GpuCtx(O.case_params("filters_pe"), 700, S, S)
    text = IL.interleave(t1, t2)
    r = process_host_il(pe, text, t2, {R1, R2}, 1, 0)                         # text2 with interleaved input
    assert r["rc"] == -1 and r["untouched"]
    r = process_host_il(pe, t1, t2, {R1, R2}, 0, 1)                           # an out2 buffer with interleaved output
    assert r["rc"] == -1 and r["untouched"]
    capi.check(lib.fp_fastq_set_interleaved(pe.h, 0, 0), lib)                 # off again: the ordinary two-file path
    r = process_host_il(pe, t1, t2, {R1, R2}, 0, 0)
    g = IL.port_streams("filters_pe/stdout")
    assert r["rc"] == 0 and r[R1] == g["out1"] and r[R2] == g["out2"]
    pe.close()


MIRROR = ["filters_pe/stdin_il_stdout", "edge160_pe/stdin_il_stdout", "filters_se/stdin_stdout", "filters_pe/stdout", "filters_pe/il",
          "filters_pe/il_stdout_f", "dedup_pe/il_stdout", "merge_pe/il_stdout", "merge_pe/stdout_merged_out", "merge_pe/il_o1_merged",
          "merge_iu_pe/il_stdout"]


@pytest.mark.parametrize("run", MIRROR)
def test_mirror_cli(gpu, tmp_path, run):
    """fastp_gpu_cli --device_fastq at two chunk sizes, input through a pipe where the run says --stdin: stdout and files equal the committed
    digests of the reference CLI's; the stride comes from the piped bytes themselves (no --max_read_len)."""
    assert os.path.exists(CLI), "build with __graft_entry__.build()"
    digests = json.load(open(DIGESTS))[run]
    for chunk in (100003, 1 << 20):
        d = tmp_path / str(chunk); d.mkdir()
        outs, err = IL.run_cli(CLI, d, run, ["--device_fastq", "--chunk_bytes", str(chunk), "--pack_size", "2048"])
        assert [hashlib.md5(x).hexdigest() for x in outs] == digests, (run, chunk, err[-400:])


def test_mirror_cli_gz_interleaved_input(gpu, tmp_path):
    """.gz interleaved input via --interleaved_in, --stdout: the bytes of the reference's run on the plain text."""
    run = "filters_pe/il_stdout"
    text, _, _ = IL.run_inputs(run)
    (tmp_path / "r1.fq.gz").write_bytes(gzip.compress(text))
    flags = CASES["filters_pe"][0]
    for chunk in (100003, 1 << 20):
        r = subprocess.run([CLI, "-i", str(tmp_path / "r1.fq.gz"), "--interleaved_in", "--stdout", "--device_fastq", "--dont_eval_duplication",
                            "--chunk_bytes", str(chunk)] + flags, capture_output=True, timeout=600)
        assert r.returncode == 0, r.stderr[-400:]
        assert hashlib.md5(r.stdout).hexdigest() == json.load(open(DIGESTS))[run][0]


def test_mirror_cli_argument_rules(gpu, tmp_path):
    pair = b"@a\nACGTTGCAACGTTGCAACGT\n+\nIIIIIIIIIIIIIIIIIIII\n@b\nTTGCAACGTTGCAACGTTGC\n+\nIIIIIIIIIIIIIIIIIIII\n"
    (tmp_path / "r.fq").write_bytes(pair)
    r = str(tmp_path / "r.fq")
    for args, msg in (([r, "-I", r, "--interleaved_in", "--device_fastq", "--stdout"], b"<in2> is not allowed when <in1> is specified as interleaved mode"),
                      ([r, "-I", r, "-m", "--device_fastq"], b"In merging mode, you should either specify --merged_out or enable --stdout"),
                      ([r, "-m", "--device_fastq", "--stdout"], b"read2 input should be specified by --in2 for merging mode"),
                      ([r, "--interleaved_in", "--stdout"], b"--device_fastq")):
        p = subprocess.run([CLI, "-i"] + args, capture_output=True, timeout=120)
        assert p.returncode == 2 and msg in p.stderr, (args, p.stderr)
    p = subprocess.run([CLI, "-i", r, "--interleaved_in", "--device_fastq", "--stdout", "-o", str(tmp_path / "o.fq")], capture_output=True, timeout=120)
    assert p.returncode == 0 and b"In STDOUT mode, ignore the out1 filename" in p.stderr and not (tmp_path / "o.fq").exists()
    assert p.stdout == pair
