#!/usr/bin/env python
"""Throughput of interleaved pairs on the text path: profile-1 synthetic 2x150 pairs as FASTQ text in pinned host memory through
fp_fastq_process_host_outs, interleaved in -> interleaved out (fp_fastq_set_interleaved(1, 1), what `--stdin --interleaved_in --stdout`
runs) against two texts in -> out1 / out2, the two calls alternated step by step in one process, on one ctx each.  Filters -q 30 -u 10 -l 120
as in bench_fastq_outs.py.  Checks that the interleaved stream is out1 and out2 interleaved.  Host clock around the synchronous call.  Prints
one JSON line with the card's name and power limit read in the same run.  Needs a GPU: there is nothing to measure without one."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
STRIDE, READ_LEN, SEED = 160, 150, 20240607
FILTERS = dict(qualified_qual=33 + 30, unqualified_percent_limit=10, length_required=120)


def records(text):
    lines = text.split(b"\n")
    return [b"\n".join(lines[k:k + 4]) + b"\n" for k in range(0, len(lines) - 1, 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4_000_000, help="pairs per timed call")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-batch", type=int, default=1 << 20, help="pairs per round of the text path")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_fastq_interleaved: no CUDA device")
    from bench import fastq_text_np
    from fastp_b200 import capi
    lib = capi.load()
    dev = torch.cuda.current_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(dev)], capture_output=True, text=True).stdout.strip()
    gen = min(args.pairs, 250_000)
    reps = max(1, args.pairs // gen)
    n = gen * reps
    result = {"card": card, "pairs_per_call": n, "steps": args.steps, "read_len": READ_LEN, "profile": 1, "filters": "-q 30 -u 10 -l 120"}

    p = capi.default_params(1, lib=lib, seq_len1=READ_LEN, seq_len2=READ_LEN, **FILTERS)
    h = C.c_void_p()
    capi.check(lib.fp_ctx_create(C.byref(p), dev, args.max_batch, STRIDE, STRIDE, C.byref(h)), lib)
    t = {k: torch.empty(gen * (2 if k.startswith("len") else STRIDE), dtype=torch.uint8, device="cuda") for k in ("seq1", "qual1", "len1", "seq2", "qual2", "len2")}
    b = capi.Batch(); b.n, b.stride = gen, STRIDE
    for k, v in t.items():
        setattr(b, k, v.data_ptr())
    capi.check(lib.fp_synth_fill(h, C.byref(b), 0, SEED, 1, READ_LEN, None), lib)
    torch.cuda.synchronize()
    lib.fp_ctx_destroy(h)
    sides = [fastq_text_np(np, t["seq" + s].cpu().numpy().reshape(gen, STRIDE), t["qual" + s].cpu().numpy().reshape(gen, STRIDE),
                           t["len" + s].cpu().numpy().view(np.uint16), s + ":N:0") for s in ("1", "2")]
    del t
    il = np.frombuffer(b"".join(a + c for a, c in zip(records(sides[0].tobytes()), records(sides[1].tobytes()))), np.uint8)
    pin = [torch.from_numpy(np.tile(x, reps)).pin_memory() for x in (sides[0], sides[1], il)]
    caps = [pin[0].numel() + 64, pin[1].numel() + 64, pin[2].numel() + 64]
    outs = [torch.empty(c, dtype=torch.uint8).pin_memory() for c in caps]

    ctxs = {}
    for mode in ("two_files", "interleaved"):
        h = C.c_void_p()
        capi.check(lib.fp_ctx_create(C.byref(p), dev, args.max_batch, STRIDE, STRIDE, C.byref(h)), lib)
        if mode == "interleaved":
            capi.check(lib.fp_fastq_set_interleaved(h, 1, 1), lib)
        ctxs[mode] = h
    ob = {m: (C.c_int64 * 6)() for m in ctxs}
    nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64()

    def call(mode):
        h = ctxs[mode]
        if mode == "two_files":
            optr = (C.c_void_p * 6)(None, outs[0].data_ptr(), outs[1].data_ptr(), None, None, None)
            ocap = (C.c_int64 * 6)(0, caps[0], caps[1], 0, 0, 0)
            text = (pin[0].data_ptr(), pin[0].numel(), pin[1].data_ptr(), pin[1].numel())
        else:
            optr = (C.c_void_p * 6)(None, outs[2].data_ptr(), None, None, None, None)
            ocap = (C.c_int64 * 6)(0, caps[2], 0, 0, 0, 0)
            text = (pin[2].data_ptr(), pin[2].numel(), None, 0)
        capi.check(lib.fp_fastq_process_host_outs(h, *text, 1, 0, optr, ocap, ob[mode], C.byref(nu), C.byref(c1), C.byref(c2), None, None), lib)
        assert nu.value == n, (mode, nu.value, n)

    for _ in range(args.warmup):
        for m in ctxs:
            call(m)
    times = {m: [] for m in ctxs}
    for _ in range(args.steps):                          # alternated: both modes see the same card state
        for m in ctxs:
            t0 = time.perf_counter()
            call(m)
            times[m].append(time.perf_counter() - t0)
    o1 = outs[0][:ob["two_files"][1]].numpy().tobytes(); o2 = outs[1][:ob["two_files"][2]].numpy().tobytes()
    oi = outs[2][:ob["interleaved"][1]].numpy().tobytes()
    assert oi == b"".join(a + c for a, c in zip(records(o1), records(o2))), "interleaved stream != out1 / out2 interleaved"
    for m, h in ctxs.items():
        lib.fp_ctx_destroy(h)
        dt = sum(times[m]) / len(times[m])
        result[m] = {"pairs_per_s": n / dt, "seconds_per_call": [round(x, 4) for x in times[m]]}
    result["interleaved_out_bytes"] = len(oi)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
