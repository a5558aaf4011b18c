"""-m gpu: the CUDA adapter trimmers against the CPU port on the adapter shapes and lists of tests/adapter_edges.py, bit-exact (records,
rows, the whole counter block): device mode at SE strides 160 / 512 and PE 160 / 256, with the adapter events replayed into the
reference's adapter-string maps; the host entry point at the tight pitch and with FP_B_PACK2BIT; a 40-entry list whose reads trim
up to 40 times each, over several host chunks of a 1 024-unit ctx.  The C-ABI's adapter limits, and the bound CLI against the
unmodified CLI on --adapter_fasta files, including those past the limits that the bound CLI hands to the stock body.
tests/test_oracle_adapter_edges.py pins the port to the reference's objects on the same inputs."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import adapter_edges as A
import fp_testlib as T
from fastp_b200 import capi
from test_oracle_adapter_edges import PE_CASES, PE_STRIDES, SE_CASES, SE_STRIDES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GPU_CLI = os.path.join(ROOT, "oracle", "_ref", "fastp_gpu")
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    import fp_gpu
    return fp_gpu


def adapters_of(p):
    return [(p.adapter_seq_r1 or b"").decode(), (p.adapter_seq_r2 or b"").decode()] + [p.fasta_adapters[i].decode() for i in range(p.n_fasta_adapters)]


def device_events(gpu, ctx, p, arrs, S, splits=1):
    import torch
    n = len(arrs["len1"])
    cap = (2 + 2 * p.n_fasta_adapters) * max(n, 1)
    d_ev = torch.zeros(cap * 16, dtype=torch.uint8, device="cuda:0"); d_n = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    capi.check(ctx.lib.fp_set_event_sink(ctx.h, d_ev.data_ptr(), cap, d_n.data_ptr()), ctx.lib)
    try:
        got = gpu.run_gpu(p, arrs, S, mode="device", ctx=ctx, splits=splits)
    finally:
        capi.check(ctx.lib.fp_set_event_sink(ctx.h, None, 0, None), ctx.lib)
    ne = int(d_n.item())
    assert ne <= cap
    return got, np.sort(d_ev.cpu().numpy().view(capi.EVENT_DTYPE)[:ne].copy(), order=["unit", "key"])


def host_events(gpu, ctx, p, arrs, S, mode):
    cap = (2 + 2 * p.n_fasta_adapters) * max(len(arrs["len1"]), 1)
    h_ev = np.zeros(cap, capi.EVENT_DTYPE); h_n = C.c_uint64()
    capi.check(ctx.lib.fp_set_host_event_sink(ctx.h, h_ev.ctypes.data, cap, C.byref(h_n)), ctx.lib)
    try:
        got = gpu.run_gpu(p, arrs, S, mode=mode, ctx=ctx)
    finally:
        capi.check(ctx.lib.fp_set_host_event_sink(ctx.h, None, 0, None), ctx.lib)
    assert h_n.value <= cap
    return got, np.sort(h_ev[:h_n.value].copy(), order=["unit", "key"])


def check(gpu, name, paired, S, host_modes=()):
    p = A.case_params(name, paired)
    arrs, _ = A.case_batch(name, paired, S, 3 + S)
    want = T.run_cpu("oracle", p, arrs, S)
    ctx = gpu.GpuCtx(p, len(arrs["len1"]), S, S)
    try:
        got, ev = device_events(gpu, ctx, p, arrs, S)
        T.assert_results_equal(got, want, paired, what=f"{name}/S{S}/device")
        if T.have_ref():
            maps, _ = T.ref_adapter_maps(p, arrs, S)
            got_maps = T.rebuild_adapter_maps(ev, got["arrs"], adapters_of(p))
            assert got_maps[0] == maps[0] and got_maps[1] == maps[1], f"{name}/S{S}: adapter-string maps differ"
        for mode in host_modes:
            hgot, hev = host_events(gpu, ctx, p, arrs, S, mode)
            T.assert_results_equal(hgot, want, paired, what=f"{name}/S{S}/{mode}")
            assert (hev == ev).all(), f"{name}/S{S}/{mode}: event list differs from device mode"
    finally:
        ctx.close()


@pytest.mark.parametrize("S", SE_STRIDES)
@pytest.mark.parametrize("name", SE_CASES)
def test_adapter_edges_se(gpu, name, S):
    check(gpu, name, 0, S, ("host_tight", "host_tight_pack2bit") if S == 160 else ())


@pytest.mark.parametrize("S", PE_STRIDES)
@pytest.mark.parametrize("name", PE_CASES)
def test_adapter_edges_pe(gpu, name, S):
    check(gpu, name, 1, S, ("host_tight", "host_tight_pack2bit") if S == 160 else ())


def test_64_base_one_gap_reads_are_trimmed(gpu):
    """A 64-base adapter whose last base is not A, reads of 65 bases and more with one inserted base and exactly 64/8 - 1 mismatches:
    the reference trims them to length 0 in scan 2.  The one-gap quick reject read bit 63 of its shifted field, which compares
    read[64] with adapter[63], as an A, and so rejected them (DESIGN §3)."""
    for paired, S in ((0, 160), (1, 256)):
        arrs, labels = A.case_batch("seq.rand64", paired, S, 3 + S)
        p = A.case_params("seq.rand64", paired)
        want = T.run_cpu("oracle", p, arrs, S)
        got = gpu.run_gpu(p, arrs, S)
        for tag in ("1", "2")[: 1 + paired]:
            sel = (labels[tag]["kind"] == A.K["gap2"]) & (labels[tag]["at"] == 0) & (arrs["len" + tag] >= 65)
            w, g = want["out" + tag]["len"][sel], got["out" + tag]["len"][sel]
            assert np.count_nonzero(w == 0) >= 8
            assert (g == w).all(), f"S{S} side {tag}: {int(np.count_nonzero(g != w))} of {int(sel.sum())} insertion reads differ"
        T.assert_results_equal(got, want, paired, what=f"rand64 one-gap S{S}")


def test_many_events_per_unit_over_host_chunks(gpu):
    """40 fasta adapters, reads trimmed up to 40 times each: more than 62 events for some pairs, through the host entry point of a
    1 024-unit ctx (several chunks) and in device mode on the first 1 000 pairs (one launch: the device sink numbers units per
    launch); the sorted event lists agree, and with the reference present the maps replayed from the host list equal the reference's."""
    n, S, m = 3000, 256, 1000
    p, arrs = A.many_trims_input(n)
    want = T.run_cpu("oracle", p, arrs, S)
    ctx = gpu.GpuCtx(p, 1024, S, S)
    try:
        host, host_ev = host_events(gpu, ctx, p, arrs, S, "host")
        T.assert_results_equal(host, want, 1, what="many events/host")
        per_unit = np.bincount(host_ev["unit"].astype(np.int64), minlength=n)
        assert per_unit.max() > 62
        head = {k: v[:m] for k, v in arrs.items()}
        dev, dev_ev = device_events(gpu, ctx, p, head, S)
        T.assert_results_equal(dev, T.run_cpu("oracle", p, head, S), 1, what="many events/device")
        host_head = host_ev[host_ev["unit"] < m]
        assert len(host_head) == len(dev_ev) and (host_head == dev_ev).all()
        if T.have_ref():
            maps, _ = T.ref_adapter_maps(p, arrs, S)
            got = T.rebuild_adapter_maps(host_ev, host["arrs"], adapters_of(p))
            assert got[0] == maps[0] and got[1] == maps[1]
    finally:
        ctx.close()


@pytest.mark.parametrize("what,adapters,ok", [
    ("255 bases", [A.SHAPES["rand255"]], True),
    ("256 bases", [A.SHAPES["rand255"] + "A"], False),
    ("512 entries", A.LISTS["list512"], True),
    ("513 entries", A.LISTS["list512"] + ["ACGTACGT"], False),
])
def test_ctx_adapter_limits(gpu, what, adapters, ok):
    """FP_MAX_ADAPTER_LEN (255) and FP_MAX_ADAPTERS (512 fasta entries) are accepted; one base or one entry more is FP_E_INVAL."""
    lib = capi.load()
    p = capi.default_params(1, fasta_adapters=adapters)
    h = C.c_void_p()
    rc = lib.fp_ctx_create(C.byref(p), 0, 1024, 160, 160, C.byref(h))
    if ok:
        assert rc == 0, lib.fp_last_error()
        lib.fp_ctx_destroy(h)
    else:
        assert rc == -1 and not h.value, (rc, lib.fp_last_error())             # FP_E_INVAL
        assert b"adapter" in lib.fp_last_error()


# ---------------- the bound CLI on --adapter_fasta files ----------------
def _fasta(items):
    return "".join(f">a{i}\n{s}\n" for i, s in enumerate(items))


FASTA_FILES = {
    # the 64-base adapter, N at both ends, a lower-case base
    "shapes": [A.SHAPES["rand64"], A.SHAPES["n_start_end64"], A.SHAPES["lower_a33"]],
    "contigs300": A.LISTS["list512"][:300],
    # past fp_ctx_create's limits: the bound CLI runs these on the stock body
    "adapter300": [A.SHAPES["rand200"] + A.SHAPES["rand97"] + "GGG", A.SHAPES["rand33"]],
    "contigs513": [],
}
_distinct = list(dict.fromkeys(A.LISTS["list512"]))                    # the reference's loader drops repeated entries
FASTA_FILES["contigs513"] = _distinct + [A.SHAPES["rand12"] + "T" * k for k in range(1, 514 - len(_distinct))]
ON_DEVICE = {"shapes": True, "contigs300": True, "adapter300": False, "contigs513": False}


def _cli_reads(name, paired):
    """FASTQ texts: synthetic reads, then (for the file that starts with it) the reads planted for the 64-base adapter."""
    import bench
    _, syn = T.synth_host(1500, 160, paired, 0, 31, 1, 150)
    parts = [syn]
    if FASTA_FILES[name][0] == A.SHAPES["rand64"]:
        parts.append(A.case_batch("seq.rand64", paired, 160, 5)[0])
    texts = []
    for sd in ("1", "2")[: 1 + paired]:
        t = b"".join(bench.fastq_text_np(np, a["seq" + sd], a["qual" + sd], a["len" + sd], f"{sd}:N:0").tobytes() for a in parts)
        texts.append(t)
    return texts


def _binding_has_stock_trace():
    """fastp_gpu comes from a binding that reports the option sets it hands to the stock body -- the binding that also hands over
    adapters past fp_ctx_create's limits.  The Makefile relinks it whenever the binding's content changes, but only where the reference
    sources are; a prebuilt _ref/ from an older binding exits in fp_ctx_create on those files."""
    with open(GPU_CLI, "rb") as f:
        return b"units on the stock body" in f.read()


@pytest.mark.skipif(not (os.path.exists(GPU_CLI) and os.path.exists(T.REF_CLI)), reason="oracle/_ref/fastp_gpu not built (needs the reference sources at build time)")
@pytest.mark.parametrize("paired", [1, 0])
@pytest.mark.parametrize("name", list(FASTA_FILES))
def test_bound_cli_adapter_fasta(tmp_path, name, paired):
    """Output files byte-identical and JSON reports equal; the files within fp_ctx_create's limits run on the device, the ones past
    them on the stock body (before, the bound CLI exited in fp_ctx_create)."""
    if not ON_DEVICE[name] and not _binding_has_stock_trace():
        pytest.skip("oracle/_ref/fastp_gpu was linked from an older reference_binding.cpp (a prebuilt _ref/ that travelled without the "
                    "reference sources): rebuild it with `make -C oracle` where they are")
    (tmp_path / "ad.fa").write_text(_fasta(FASTA_FILES[name]))
    for k, t in enumerate(_cli_reads(name, paired)):
        (tmp_path / f"r{k + 1}.fq").write_bytes(t)
    outs = {}
    for tag, cli in (("ref", T.REF_CLI), ("gpu", GPU_CLI)):
        d = tmp_path / tag
        os.makedirs(d)
        cmd = [cli, "-i", str(tmp_path / "r1.fq"), "-o", "o1.fq", "-w", "1", "-j", "t.json", "-h", "t.html", "--adapter_fasta", str(tmp_path / "ad.fa")]
        if paired:
            cmd += ["-I", str(tmp_path / "r2.fq"), "-O", "o2.fq"]
        r = subprocess.run(cmd, capture_output=True, text=True, cwd=d, env=dict(os.environ, FASTP_B200_TRACE="1"), timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        if tag == "gpu":
            where = "units on the device" if ON_DEVICE[name] else "units on the stock body"
            assert where in r.stderr and ("units on the device" in r.stderr) == ON_DEVICE[name], r.stderr[-2000:]
        js = json.load(open(d / "t.json"))
        js.pop("command", None)
        outs[tag] = (js, {f: open(d / f, "rb").read() for f in sorted(os.listdir(d)) if f.endswith(".fq")})
    assert outs["gpu"][1].keys() == outs["ref"][1].keys()
    for f in outs["ref"][1]:
        assert outs["gpu"][1][f] == outs["ref"][1][f], f"{f} differs"
    jr, jg = outs["ref"][0], outs["gpu"][0]
    assert jg.keys() == jr.keys()
    for k in jr:
        assert jg[k] == jr[k], f"JSON section {k} differs"
    if name == "shapes" and paired:                                        # (the SE report has no adapter_cutting section)
        assert jr["adapter_cutting"]["adapter_trimmed_reads"] > 0
