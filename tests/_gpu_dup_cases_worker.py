"""Child process of tests/test_gpu_dedup.py: fp_dup_check at ONE accuracy level (argv[1]) against the sequential C port, over the row
strides a ctx takes (PE 48 / 160 / 256, SE 160 / 512), one ctx -- one set of bit arrays -- at a time.  Per ctx:
  sizes     batches of 0 / 1 / 7 / 33 / 20 000 units, then fp_dup_reset and the same units in batches of 20 000 / 33 / 7 / 1 / 0 (scratch
            buffers grow, the table mask changes); one batch without a flag array (totals only), one on a caller's stream
  same unit one unit 4 096 times: every thread meets the same table slots
  copies    six batches, each later one holding copies of batch 0
  refusals  another accuracy level, another stride: FP_E_INVAL
Exit code 0 and one "ok:" line per ctx = equal everywhere."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, HERE)
import edge_inputs as E  # noqa: E402
import fp_testlib as T  # noqa: E402
from fastp_b200 import capi  # noqa: E402

FP_E_INVAL = -1
SHAPES = [(1, 48), (1, 160), (1, 256), (0, 160), (0, 512)]


def units(paired, S, seed, n0=14500):
    """n0 edge-length units (0, 1, ..., the full stride; bytes outside A/C/G/T in some), 40 % of them again as exact copies, 200
    one-base variants, shuffled."""
    rng = np.random.default_rng(seed)
    a = E.edge_batch(n0, S, paired, seed, T.config_params("default", paired), read_len=min(150, S) if S <= 256 else S - 12)
    odd = np.frombuffer(b"Nacgtn.", np.uint8)
    for sd in ("1", "2")[: 2 if paired else 1]:
        rows = rng.integers(0, n0, n0 // 10)
        a["seq" + sd][rows, rng.integers(0, S, len(rows))] = rng.choice(odd, len(rows))      # may land in the padding: put back below
        a["len" + sd][:4] = (0, 1, S, S)
        if paired and sd == "1":
            a["len1"][4:6] = 0                                                               # read 1 empty, read 2 not
        a["seq" + sd][:6] = rng.choice(E.ACGT, (6, S))
    E._zero_padding(a)
    pick = rng.integers(0, n0, int(n0 * 0.4))
    out = {k: np.concatenate([v, v[pick]]) for k, v in a.items()}
    for i in rng.integers(n0, len(out["len1"]), 200):
        if out["len1"][i] > 3:
            out["seq1"][i, 2] = ord("A") if out["seq1"][i, 2] != ord("A") else ord("C")
    perm = rng.permutation(len(out["len1"]))
    return {k: np.ascontiguousarray(v[perm]) for k, v in out.items()}


def cut(arrs, sizes):
    out, lo = [], 0
    for s in sizes:
        out.append({k: np.ascontiguousarray(v[lo:lo + s]) for k, v in arrs.items()}); lo += s
    return out


def device_run(fp_gpu, torch, ctx, level, batches, no_flags=(), on_stream=()):
    """fp_dup_check over `batches`; the flags of each (None where no array was given) and the totals."""
    got = []
    side = torch.cuda.Stream()
    for i, sub in enumerate(batches):
        n = len(sub["len1"])
        if n:
            db, _t = fp_gpu.device_batch(sub)
        else:
            db = capi.Batch(); db.n, db.stride = 0, ctx.stride
        d_flags = None if i in no_flags else torch.full((max(n, 1),), 7, dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        st = C.c_void_p(side.cuda_stream) if i in on_stream else None
        capi.check(ctx.lib.fp_dup_check(ctx.h, C.byref(db), level, d_flags.data_ptr() if d_flags is not None else None, st), ctx.lib)
        torch.cuda.synchronize()
        got.append(None if d_flags is None else d_flags.cpu().numpy()[:n])
    t, d = C.c_int64(), C.c_int64()
    capi.check(ctx.lib.fp_dup_totals(ctx.h, C.byref(t), C.byref(d)), ctx.lib)
    return got, t.value, d.value


def compare(what, got, want):
    gf, gt, gd = got
    wf, wt, wd = want
    for i, (g, w) in enumerate(zip(gf, wf)):
        if g is not None and not np.array_equal(g, w):
            bad = np.flatnonzero(g != w)
            raise SystemExit(f"{what}: flags of batch {i} differ at {len(bad)} of {len(w)} units, first {bad[:5]}: {g[bad[:5]]} vs {w[bad[:5]]}")
    if (gt, gd) != (wt, wd):
        raise SystemExit(f"{what}: totals {gt, gd} vs {wt, wd}")


def main(level):
    import torch
    import fp_gpu
    buf_num = 4 if level == 3 else 2
    for paired, S in SHAPES:
        what = f"level {level} {'PE' if paired else 'SE'} S{S}"
        arrs = units(paired, S, seed=100 * level + S + paired)
        total_len = arrs["len1"].astype(int) + (arrs["len2"].astype(int) if paired else 0)
        assert total_len.max() == (2 if paired else 1) * S and total_len.min() == 0
        # the prime index (q * buf_num + i) & mask never wraps inside a ctx's strides (PE <= 256, SE <= 512): the C port is
        # pinned on wrapping pairs at stride 512 by tests/test_oracle_dedup.py
        assert (total_len.max() - 1) * buf_num + buf_num - 1 <= 512 * buf_num - 1
        ctx = fp_gpu.GpuCtx(T.config_params("default", paired), 20000, S, S)
        sizes = [0, 1, 7, 33, 20000]
        assert sum(sizes) <= len(arrs["len1"])
        fwd = cut(arrs, sizes)
        compare(what + " sizes", device_run(fp_gpu, torch, ctx, level, fwd), T.oracle_dup_flags(fwd, paired, level))
        capi.check(ctx.lib.fp_dup_reset(ctx.h), ctx.lib)
        rev = cut(arrs, sizes[::-1])
        want = T.oracle_dup_flags(rev, paired, level)
        assert want[2] > 3000
        compare(what + " sizes reversed", device_run(fp_gpu, torch, ctx, level, rev, no_flags=(1,), on_stream=(0, 2)), want)
        capi.check(ctx.lib.fp_dup_reset(ctx.h), ctx.lib)
        one = [{k: np.ascontiguousarray(np.repeat(v[40:41], 4096, axis=0)) for k, v in arrs.items()}]
        want = T.oracle_dup_flags(one, paired, level)
        assert want[0][0][0] == 0 and want[0][0][1:].all()
        compare(what + " same unit", device_run(fp_gpu, torch, ctx, level, one), want)
        capi.check(ctx.lib.fp_dup_reset(ctx.h), ctx.lib)
        parts = cut(arrs, [500] * 6)
        rng = np.random.default_rng(S)
        six = [parts[0]]
        for k in range(1, 6):
            perm = rng.permutation(700)
            six.append({key: np.ascontiguousarray(np.concatenate([parts[k][key], parts[0][key][:200]])[perm]) for key in parts[0]})
        compare(what + " copies of batch 0", device_run(fp_gpu, torch, ctx, level, six), T.oracle_dup_flags(six, paired, level))
        db, _t = fp_gpu.device_batch(parts[1])
        if ctx.lib.fp_dup_check(ctx.h, C.byref(db), level % 3 + 1, None, None) != FP_E_INVAL:
            raise SystemExit(what + ": another accuracy level was accepted")
        db.stride = S + 16
        if ctx.lib.fp_dup_check(ctx.h, C.byref(db), level, None, None) != FP_E_INVAL:
            raise SystemExit(what + ": another stride was accepted")
        ctx.close()
        torch.cuda.synchronize()
        print("ok:", what, flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main(int(sys.argv[1])))
