#!/usr/bin/env python
"""Throughput of the merging-mode text path: profile-1 synthetic 2x150 pairs as FASTQ text in pinned host memory through
fp_fastq_process_host_merge (H2D of the text, device decode, duplicate-free operator chain with its merging branch, the three device
encodes, D2H of the three streams), with and without --include_unmerged.  Host clock around the synchronous call.  Prints one JSON line
with pairs/s, output bytes per stream, the share of pairs that merged, and the card's name and power limit read in the same run.
Needs a GPU: there is nothing to measure without one."""
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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-batch", type=int, default=1 << 20, help="pairs per round of the text path")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_fastq_merge: no CUDA device")
    from bench import fastq_text_np
    from fastp_b200 import capi
    lib = capi.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                          capture_output=True, text=True).stdout.strip()
    gen = min(args.pairs, 250_000)
    reps = max(1, args.pairs // gen)
    n = gen * reps
    result = {"card": card, "pairs_per_call": n, "steps": args.steps, "read_len": READ_LEN, "profile": 1}
    pin = None
    for mode, iu in (("merge", 0), ("merge_include_unmerged", 1)):
        p = capi.default_params(1, lib=lib, seq_len1=READ_LEN, seq_len2=READ_LEN, merge_enabled=1, correction_enabled=1, merge_include_unmerged=iu)
        h = C.c_void_p()
        capi.check(lib.fp_ctx_create(C.byref(p), torch.cuda.current_device(), args.max_batch, STRIDE, 2 * STRIDE, C.byref(h)), lib)
        if pin is None:
            t = {k: torch.empty(gen * (2 if k.startswith("len") else STRIDE), dtype=torch.uint8, device="cuda") for k in ("seq1", "qual1", "len1", "seq2", "qual2", "len2")}
            b = capi.Batch(); b.n, b.stride = gen, STRIDE
            for k, v in t.items():
                setattr(b, k, v.data_ptr())
            capi.check(lib.fp_synth_fill(h, C.byref(b), 0, SEED, 1, READ_LEN, None), lib)
            torch.cuda.synchronize()
            pin = []
            for side in ("1", "2"):
                one = fastq_text_np(np, t["seq" + side].cpu().numpy().reshape(gen, STRIDE), t["qual" + side].cpu().numpy().reshape(gen, STRIDE),
                                    t["len" + side].cpu().numpy().view(np.uint16), side + ":N:0")
                pin.append(torch.from_numpy(np.tile(one, reps)).pin_memory())
            del t
            outs = [torch.empty(x.numel() + 64, dtype=torch.uint8).pin_memory() for x in pin]
            outs.append(torch.empty(pin[0].numel() + pin[1].numel() + 40 * n + 64, dtype=torch.uint8).pin_memory())
        ob = [C.c_int64(), C.c_int64(), C.c_int64()]; nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64()
        i1, i2 = capi.FastqInfo(), capi.FastqInfo()

        def call():
            capi.check(lib.fp_fastq_process_host_merge(h, pin[0].data_ptr(), pin[0].numel(), pin[1].data_ptr(), pin[1].numel(), 1, 0,
                                                       outs[0].data_ptr(), outs[0].numel(), C.byref(ob[0]), outs[1].data_ptr(), outs[1].numel(), C.byref(ob[1]),
                                                       outs[2].data_ptr(), outs[2].numel(), C.byref(ob[2]),
                                                       C.byref(nu), C.byref(c1), C.byref(c2), C.byref(i1), C.byref(i2)), lib)
        for _ in range(args.warmup):
            call()
        assert nu.value == n, (nu.value, n)
        capi.check(lib.fp_counters_reset(h), lib)
        ms, kn = C.c_double(), C.c_int64()
        capi.check(lib.fp_kernel_time_ms(h, C.byref(ms), C.byref(kn), 1), lib)        # drop the warm-up's chain kernel time
        times = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            call()
            times.append(time.perf_counter() - t0)
        L = capi.CounterLayout()
        capi.check(lib.fp_ctx_layout(h, C.byref(L)), lib)
        cnt = np.zeros(L.total, np.int64)
        capi.check(lib.fp_counters_fetch(h, cnt.ctypes.data), lib)
        merged_pairs = int(capi.CounterView(L, cnt).filter[107]) / args.steps      # FP_FR_MERGED_PAIRS: merged reads that passed
        capi.check(lib.fp_kernel_time_ms(h, C.byref(ms), C.byref(kn), 1), lib)
        lib.fp_ctx_destroy(h)
        dt = sum(times) / len(times)
        result[mode] = {"pairs_per_s": n / dt, "seconds_per_call": [round(x, 4) for x in times], "input_bytes": int(pin[0].numel() + pin[1].numel()),
                        "out1_bytes": ob[0].value, "out2_bytes": ob[1].value, "merged_bytes": ob[2].value,
                        "merged_and_passed_share": merged_pairs / n, "chain_kernel_ms_per_call": ms.value / args.steps}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
