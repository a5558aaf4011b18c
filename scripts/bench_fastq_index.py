#!/usr/bin/env python
"""Throughput of the paired text path with the index filter off and on: profile-1 synthetic 2x150 pairs with Illumina-style names
(`1:N:0:ACGTACGT+TTGGCCAA`) as FASTQ text in pinned host memory through fp_fastq_process_host, out1 / out2.  The filter runs with random
barcode lists of 1 / 96 / 10 000 barcodes (8 bases) at threshold 0 and 2 that do not hold the reads' index, so every unit is compared with
the whole list and the outputs stay the same as with the filter off -- the matcher's cost, not fewer pairs to write.  The modes alternate
in one process, call by call, on one ctx.  Host clock around the synchronous call.  Prints one JSON line with the card's name and power
limit read in the same run.  Needs a GPU: there is nothing to measure without one."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4_000_000, help="pairs per timed call")
    ap.add_argument("--steps", type=int, default=5, help="timed calls per mode")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-batch", type=int, default=1 << 20, help="pairs per round of the text path")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_fastq_index: no CUDA device")
    from bench import fastq_text_np
    from fastp_b200 import capi
    lib = capi.load()
    dev = torch.cuda.current_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(dev)], capture_output=True, text=True).stdout.strip()
    gen = min(args.pairs, 250_000)
    reps = max(1, args.pairs // gen)
    n = gen * reps
    result = {"card": card, "units_per_call": n, "steps": args.steps, "read_len": READ_LEN, "profile": 1, "options": "defaults"}
    p = capi.default_params(1, lib=lib, seq_len1=READ_LEN, seq_len2=READ_LEN)
    h = C.c_void_p()
    capi.check(lib.fp_ctx_create(C.byref(p), dev, args.max_batch, STRIDE, STRIDE, C.byref(h)), lib)
    t = {k: torch.empty(gen * (2 if k.startswith("len") else STRIDE), dtype=torch.uint8, device="cuda") for k in ("seq1", "qual1", "len1", "seq2", "qual2", "len2")}
    b = capi.Batch(); b.n, b.stride = gen, STRIDE
    for k, v in t.items():
        setattr(b, k, v.data_ptr())
    capi.check(lib.fp_synth_fill(h, C.byref(b), 0, SEED, 1, READ_LEN, None), lib)
    torch.cuda.synchronize()
    pin = []
    for side in ("1", "2"):
        one = fastq_text_np(np, t["seq" + side].cpu().numpy().reshape(gen, STRIDE), t["qual" + side].cpu().numpy().reshape(gen, STRIDE),
                            t["len" + side].cpu().numpy().view(np.uint16), side + ":N:0:ACGTACGT+TTGGCCAA")
        pin.append(torch.from_numpy(np.tile(one, reps)).pin_memory())
    del t
    outs = [torch.empty(x.numel() + 64, dtype=torch.uint8).pin_memory() for x in (pin[0], pin[1])]
    o1, o2, nu, c1, c2 = (C.c_int64() for _ in range(5))
    rng = np.random.default_rng(SEED)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    far = lambda bc: all(sum(x != y for x, y in zip(bc, ix)) > 2 for ix in (b"ACGTACGT", b"TTGGCCAA"))     # noqa: E731
    lists = {k: [bc for bc in (bytes(rng.choice(acgt, 8)) for _ in range(2 * k)) if far(bc)][:k] for k in (1, 96, 10000)}
    modes = [("off", None, 0)] + [(f"list{k}_t{thr}", k, thr) for k in (1, 96, 10000) for thr in (0, 2)]

    def call(mode):
        _, k, thr = mode
        if k:
            arr = (C.c_char_p * k)(*lists[k])
            capi.check(lib.fp_fastq_set_index_filter(h, arr, k, arr, k, thr), lib)
        t0 = time.perf_counter()
        capi.check(lib.fp_fastq_process_host(h, pin[0].data_ptr(), pin[0].numel(), pin[1].data_ptr(), pin[1].numel(), 1, 0,
                                             outs[0].data_ptr(), outs[0].numel() - 64, C.byref(o1), outs[1].data_ptr(), outs[1].numel() - 64, C.byref(o2),
                                             C.byref(nu), C.byref(c1), C.byref(c2), None, None), lib)
        dt = time.perf_counter() - t0
        if k:
            capi.check(lib.fp_fastq_set_index_filter(h, None, 0, None, 0, 0), lib)
        assert nu.value == n, (nu.value, n)
        return dt, (o1.value, o2.value)

    for _ in range(args.warmup):
        for m in modes:
            call(m)
    times = {m[0]: [] for m in modes}
    sizes = set()
    for _ in range(args.steps):
        for m in modes:
            dt, sz = call(m)
            times[m[0]].append(dt)
            sizes.add(sz)
    lib.fp_ctx_destroy(h)
    assert len(sizes) == 1, sizes                     # no list holds the reads' index: every mode writes the same bytes
    for key, ts in times.items():
        s = sorted(ts)
        result[key] = {"units_per_s_median": n / s[len(s) // 2], "seconds_per_call": [round(x, 4) for x in ts]}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
