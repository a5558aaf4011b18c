"""GPU-side test helper: runs the C-ABI of libfastp_b200.so on cuda:0.
torch is used for device memory only (plumbing); every compute call goes through the C-ABI."""
import ctypes as C

import numpy as np

from fastp_b200 import capi


def _torch():
    import torch
    return torch


class GpuCtx:
    def __init__(self, params, max_batch, stride, cycles, device=0):
        self.lib = capi.load()
        self.params = params
        self.h = C.c_void_p()
        capi.check(self.lib.fp_ctx_create(C.byref(params), device, max_batch, stride, cycles, C.byref(self.h)), self.lib)
        self.L = capi.CounterLayout()
        capi.check(self.lib.fp_ctx_layout(self.h, C.byref(self.L)), self.lib)
        self.stride = stride
        self.device = device

    def close(self):
        if self.h:
            self.lib.fp_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def counters(self):
        out = np.zeros(self.L.total, np.int64)
        capi.check(self.lib.fp_counters_fetch(self.h, out.ctypes.data), self.lib)
        return capi.CounterView(self.L, out)

    def reset(self):
        capi.check(self.lib.fp_counters_reset(self.h), self.lib)

    def kernel_time_ms(self, reset=True):
        ms = C.c_double()
        n = C.c_int64()
        capi.check(self.lib.fp_kernel_time_ms(self.h, C.byref(ms), C.byref(n), 1 if reset else 0), self.lib)
        return ms.value, n.value


def device_batch(arrs, device=0):
    """Copy numpy host arrays to torch cuda tensors; returns (Batch with device pointers, tensors)."""
    torch = _torch()
    t = {k: torch.from_numpy(v).to(f"cuda:{device}") for k, v in arrs.items()}
    b = capi.Batch()
    b.n = arrs["seq1"].shape[0]
    b.stride = arrs["seq1"].shape[1]
    for k, v in t.items():
        setattr(b, k, v.data_ptr())
    b._keepalive = t
    return b, t


def pack_rows(lib, b, arrs, paired, threads=4):
    """fp_host_pack_rows into fresh numpy buffers; returns (PackedBatch, keepalive dict)."""
    n, S = arrs["seq1"].shape
    L = int(max(arrs["len1"].max(initial=0), arrs["len2"].max(initial=0) if paired else 0))
    pitch_b, pitch_q = (L + 3) // 4 + 1, L + 2
    keep = {"npos": np.zeros(max(2 * n, 1024) * 8 + 64, np.uint8)}
    pb = capi.PackedBatch()
    pb.pitch_b, pb.pitch_q = pitch_b, pitch_q
    for sd in ("1", "2")[: 2 if paired else 1]:
        keep["bases" + sd] = np.zeros(max(n, 1) * pitch_b + 64, np.uint8); keep["qual" + sd] = np.zeros(max(n, 1) * pitch_q + 64, np.uint8)
        keep["len" + sd] = np.zeros(max(n, 1), np.uint16)
        setattr(pb, "bases" + sd, keep["bases" + sd].ctypes.data); setattr(pb, "qual" + sd, keep["qual" + sd].ctypes.data); setattr(pb, "len" + sd, keep["len" + sd].ctypes.data)
    pb.npos = keep["npos"].ctypes.data; pb.npos_cap = keep["npos"].size // 8
    capi.check(lib.fp_host_pack_rows(C.byref(b), 1 if paired else 0, C.byref(pb), threads), lib)
    keep["bytes"] = (2 if paired else 1) * n * (pitch_b + pitch_q + 2) + pb.n_npos * 8
    pb._keep = keep
    return pb, keep


def run_gpu(params, arrs, cycles, mode="device", ctx=None, splits=1, is_dup=None, bounds=None, first_index=None, indexed=None):
    """Run the CUDA hot path over a COPY of arrs; same return shape as fp_testlib.run_cpu.
    is_dup (mode "device" only): --dedup flags of the units, uploaded and given to every launch through fp_set_dup_flags at that
    launch's first unit, and cleared afterwards.
    bounds (mode "device"): the launches' unit boundaries [0, ..., n] instead of `splits` even ones.  first_index: launches carry
    FP_B_INDEXED with first_read_index = first_index + their first unit -- all of them, or those whose number is in `indexed`."""
    torch = _torch()
    paired = bool(params.paired)
    n, stride = arrs["seq1"].shape
    own = ctx is None
    if own:
        ctx = GpuCtx(params, max(n, 1), stride, cycles)
    lib = ctx.lib
    ctx.reset()
    a = {k: v.copy() for k, v in arrs.items()}
    out1 = np.zeros(n, capi.READ_RESULT_DTYPE)
    out2 = np.zeros(n, capi.READ_RESULT_DTYPE)
    ov = np.zeros(n, capi.OV_RESULT_DTYPE)
    if mode == "device":
        b, t = device_batch(a)
        d_out1 = torch.zeros(max(n, 1) * 16, dtype=torch.uint8, device="cuda:0")
        d_out2 = torch.zeros(max(n, 1) * 16, dtype=torch.uint8, device="cuda:0")
        d_ov = torch.zeros(max(n, 1) * 8, dtype=torch.uint8, device="cuda:0")
        if paired:
            cap = 4 * n + 16
            d_patch = torch.zeros(cap * 12, dtype=torch.uint8, device="cuda:0")
            d_np = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        d_dup = None
        if is_dup is not None:
            flags = np.ascontiguousarray(is_dup, np.uint8)
            assert flags.shape == (n,)
            d_dup = torch.from_numpy(np.concatenate([flags, np.zeros(1, np.uint8)])).cuda()
        bounds = bounds if bounds is not None else [n * i // splits for i in range(splits + 1)]
        for launch, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):     # consecutive sub-batches of one stream (counters accumulate)
            if d_dup is not None:
                capi.check(lib.fp_set_dup_flags(ctx.h, d_dup.data_ptr() + lo), lib)
            sb = capi.Batch()
            sb.n, sb.stride = hi - lo, stride
            if first_index is not None and (indexed is None or launch in indexed):
                sb.flags, sb.first_read_index = capi.FP_B_INDEXED, first_index + lo
            for k, v in t.items():
                setattr(sb, k, v.data_ptr() + lo * (2 if k.startswith("len") else stride))
            if paired:
                assert len(bounds) == 2 or not params.correction_enabled, "patch indices are batch-local"
                capi.check(lib.fp_process_pe(ctx.h, C.byref(sb), d_out1.data_ptr() + lo * 16, d_out2.data_ptr() + lo * 16, d_ov.data_ptr() + lo * 8,
                                             d_patch.data_ptr(), cap, d_np.data_ptr(), None), lib)
            else:
                capi.check(lib.fp_process_se(ctx.h, C.byref(sb), d_out1.data_ptr() + lo * 16, None), lib)
        torch.cuda.synchronize()
        if d_dup is not None:
            capi.check(lib.fp_set_dup_flags(ctx.h, None), lib)
        out1 = d_out1.cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy()
        if paired:
            out2 = d_out2.cpu().numpy().view(capi.READ_RESULT_DTYPE)[:n].copy()
            ov = d_ov.cpu().numpy().view(capi.OV_RESULT_DTYPE)[:n].copy()
            npatch = int(d_np.cpu().item())
            patches = d_patch.cpu().numpy().view(capi.PATCH_DTYPE)[:min(npatch, cap)].copy()
        for k in a:
            a[k] = t[k].cpu().numpy()
        extra = {"patches": patches, "n_patches": npatch} if paired else {}
    elif is_dup is not None:
        raise ValueError("is_dup goes with mode='device': the host entry points refuse a set flag pointer")
    elif mode in ("host_tight", "host_tight_pack2bit"):
        # host rows at pitch = longest read (no padding bytes over PCIe); corrected rows come back at that pitch.
        # _pack2bit: FP_B_PACK2BIT, the library's host threads pack the bases chunk by chunk under the copies
        Lmax = int(max(a["len1"].max(initial=1), a["len2"].max(initial=1) if paired else 1))
        tight = {k: (np.ascontiguousarray(v[:, :Lmax]) if v.ndim == 2 else v) for k, v in a.items()}
        b = capi.batch_from_arrays(tight)
        assert b.stride == Lmax
        if mode.endswith("pack2bit"):
            b.flags |= capi.FP_B_PACK2BIT
        if paired:
            capi.check(lib.fp_process_pe_host(ctx.h, C.byref(b), out1.ctypes.data, out2.ctypes.data, ov.ctypes.data), lib)
        else:
            capi.check(lib.fp_process_se_host(ctx.h, C.byref(b), out1.ctypes.data), lib)
        for k, v in tight.items():
            if v.ndim == 2:
                a[k][:, :Lmax] = v
        extra = {}
    elif mode == "packed":
        # fp_host_pack_rows -> fp_process_*_host_packed; the corrected rows are rebuilt from the returned patch list
        b = capi.batch_from_arrays(a)
        pb, keep = pack_rows(lib, b, a, paired)
        cap = 4 * n + 16
        hp = np.zeros(cap, capi.PATCH_DTYPE); hn = C.c_uint64()
        if paired:
            capi.check(lib.fp_process_pe_host_packed(ctx.h, C.byref(pb), out1.ctypes.data, out2.ctypes.data, ov.ctypes.data, hp.ctypes.data, cap, C.byref(hn)), lib)
            for pt in hp[:hn.value]:
                side = "2" if pt["which"] else "1"
                a["seq" + side][pt["pair"], pt["pos"]] = pt["base"]; a["qual" + side][pt["pair"], pt["pos"]] = pt["qual"]
        else:
            capi.check(lib.fp_process_se_host_packed(ctx.h, C.byref(pb), out1.ctypes.data), lib)
        extra = {"packed_bytes": keep["bytes"]}
    else:
        b = capi.batch_from_arrays(a)
        if mode == "host_pack2bit":
            b.flags |= capi.FP_B_PACK2BIT
        if paired:
            capi.check(lib.fp_process_pe_host(ctx.h, C.byref(b), out1.ctypes.data, out2.ctypes.data, ov.ctypes.data), lib)
        else:
            capi.check(lib.fp_process_se_host(ctx.h, C.byref(b), out1.ctypes.data), lib)
        extra = {}
    cnt = ctx.counters()
    res = {"out1": out1, "out2": out2, "ov": ov, "counters": cnt, "arrs": a, "layout": ctx.L}
    res.update(extra)
    if own:
        ctx.close()
    return res


# ---------------- FASTQ text <-> rows ----------------
def gpu_fastq_decode(ctx, text, final=1, phred64=0, capacity=None, misalign=0):
    """fp_fastq_decode on cuda:0; same return shape as fp_testlib.oracle_fastq_decode (+ the device tensors).
    misalign: the text starts that many bytes behind a 256-byte aligned device address."""
    torch = _torch()
    lib = ctx.lib
    cap = capacity if capacity is not None else text.count(b"@") + 2
    cap1 = max(cap, 1)
    d_text = torch.from_numpy(np.concatenate([np.zeros(misalign, np.uint8), np.frombuffer(text, np.uint8), np.zeros(1, np.uint8)])).cuda()[misalign:]
    assert d_text.data_ptr() % 16 == misalign % 16
    d_seq = torch.full((cap1 * ctx.stride + 64,), 0xEE, dtype=torch.uint8, device="cuda:0")
    d_qual = torch.full((cap1 * ctx.stride + 64,), 0xEE, dtype=torch.uint8, device="cuda:0")
    d_len = torch.zeros(cap1, dtype=torch.int16, device="cuda:0")
    d_recs = torch.zeros(cap1 * 16, dtype=torch.uint8, device="cuda:0")
    info = capi.FastqInfo()
    capi.check(lib.fp_fastq_decode(ctx.h, d_text.data_ptr(), len(text), final, phred64, d_seq.data_ptr(), d_qual.data_ptr(), d_len.data_ptr(), cap,
                                   d_recs.data_ptr(), C.byref(info)), lib)
    n = int(info.n_records)
    S = ctx.stride
    out = {"seq": d_seq.cpu().numpy()[:cap1 * S].reshape(cap1, S)[:n], "qual": d_qual.cpu().numpy()[:cap1 * S].reshape(cap1, S)[:n],
           "len": d_len.cpu().numpy().view(np.uint16)[:n], "recs": d_recs.cpu().numpy().view(capi.FASTQ_REC_DTYPE)[:n].copy(),
           "info": {k: int(getattr(info, k)) for k, _ in capi.FastqInfo._fields_},
           "dev": (d_text, d_seq, d_qual, d_len, d_recs)}
    return out


def gpu_fastq_encode(ctx, dev, res, n):
    torch = _torch()
    lib = ctx.lib
    d_text, d_seq, d_qual, d_len, d_recs = dev
    d_res = torch.from_numpy(np.ascontiguousarray(res).view(np.uint8).copy() if n else np.zeros(16, np.uint8)).cuda()
    total = C.c_int64()
    capi.check(lib.fp_fastq_encode(ctx.h, d_text.data_ptr(), d_recs.data_ptr(), d_res.data_ptr(), d_seq.data_ptr(), d_qual.data_ptr(), n, None, 0, C.byref(total)), lib)
    d_out = torch.zeros(max(total.value, 1), dtype=torch.uint8, device="cuda:0")
    t2 = C.c_int64()
    capi.check(lib.fp_fastq_encode(ctx.h, d_text.data_ptr(), d_recs.data_ptr(), d_res.data_ptr(), d_seq.data_ptr(), d_qual.data_ptr(), n, d_out.data_ptr(), total.value,
                                   C.byref(t2)), lib)
    assert t2.value == total.value
    return d_out.cpu().numpy()[:total.value].tobytes()


GUARD = 0xA5


def gpu_fastq_process_host(ctx, text1, text2=None, final=1, phred64=0, out_cap=None):
    """fp_fastq_process_host: text in, filtered text out (host buffers).  out_cap = (cap1, cap2) gives the output buffers exactly
    that size, with 64 guard bytes behind them that must come back untouched ("guard_ok")."""
    lib = ctx.lib
    texts = [text1] + ([text2] if text2 is not None else [])
    caps = list(out_cap) if out_cap is not None else [len(t) + 64 for t in texts]
    bufs = [np.frombuffer(t, np.uint8).copy() if len(t) else np.zeros(1, np.uint8) for t in texts]
    outs = [np.full(c + 64, GUARD, np.uint8) for c in caps]
    nout = [C.c_int64(), C.c_int64()]; cons = [C.c_int64(), C.c_int64()]; nu = C.c_int64()
    infos = [capi.FastqInfo(), capi.FastqInfo()]
    if text2 is not None:
        rc = lib.fp_fastq_process_host(ctx.h, bufs[0].ctypes.data, len(text1), bufs[1].ctypes.data, len(text2), final, phred64,
                                       outs[0].ctypes.data, caps[0], C.byref(nout[0]), outs[1].ctypes.data, caps[1], C.byref(nout[1]),
                                       C.byref(nu), C.byref(cons[0]), C.byref(cons[1]), C.byref(infos[0]), C.byref(infos[1]))
    else:
        rc = lib.fp_fastq_process_host(ctx.h, bufs[0].ctypes.data, len(text1), None, 0, final, phred64,
                                       outs[0].ctypes.data, caps[0], C.byref(nout[0]), None, 0, None,
                                       C.byref(nu), C.byref(cons[0]), None, C.byref(infos[0]), None)
    guard_ok = all(bool((o[c:] == GUARD).all()) for o, c in zip(outs, caps))
    if out_cap is None:
        capi.check(rc, lib)
    res = {"rc": rc, "guard_ok": guard_ok, "n": nu.value, "consumed": tuple(c.value for c in cons[:len(texts)]),
           "info": [{k: int(getattr(i, k)) for k, _ in capi.FastqInfo._fields_} for i in infos[:len(texts)]]}
    for k, (o, c, nb) in enumerate(zip(outs, caps, nout)):
        res["out%d" % (k + 1)] = o[:min(nb.value, c)].tobytes() if rc == 0 else b""
    return res
