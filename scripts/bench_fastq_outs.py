#!/usr/bin/env python
"""Throughput of the text path with --unpaired1 / --unpaired2 / --failed_out: profile-1 synthetic 2x150 reads as FASTQ text in pinned host
memory through fp_fastq_process_host_outs, under a filter set that fails a real share of reads (-q 30 -u 10 -l 120: the share is printed).
Modes: PE with out1 / out2 only, PE with the three extra streams as well, SE with --failed_out.  --plain times only the plain path
(fp_fastq_process_host, out1 / out2) and prints the md5 of its output; with --lib it loads another build of libfastp_b200.so (for example
the parent commit's), so that a shell loop can alternate the two libraries, one process each, in one session.
Host clock around the synchronous call.  Prints one JSON line with the card's name and power limit read in the same run.
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
FILTERS = dict(qualified_qual=33 + 30, unqualified_percent_limit=10, length_required=120)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4_000_000, help="pairs (or reads) per timed call")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-batch", type=int, default=1 << 20, help="units per round of the text path")
    ap.add_argument("--plain", action="store_true", help="time only the plain path (fp_fastq_process_host)")
    ap.add_argument("--lib", default=None, help="load this build of libfastp_b200.so instead of the tree's")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_fastq_outs: no CUDA device")
    from bench import fastq_text_np
    from fastp_b200 import capi
    if args.lib:                                         # an older build may lack the newer entry points: bind what it has
        raw = C.CDLL(os.path.abspath(args.lib), mode=C.RTLD_GLOBAL)
        lib = capi.bind(raw, [k for k in capi.SYMBOLS if hasattr(raw, k)])
    else:
        lib = capi.load()
    dev = torch.cuda.current_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(dev)], capture_output=True, text=True).stdout.strip()
    gen = min(args.pairs, 250_000)
    reps = max(1, args.pairs // gen)
    n = gen * reps
    result = {"card": card, "units_per_call": n, "steps": args.steps, "read_len": READ_LEN, "profile": 1, "filters": "-q 30 -u 10 -l 120"}

    p0 = capi.default_params(1, lib=lib, seq_len1=READ_LEN, seq_len2=READ_LEN, **FILTERS)
    h = C.c_void_p()
    capi.check(lib.fp_ctx_create(C.byref(p0), dev, args.max_batch, STRIDE, STRIDE, C.byref(h)), lib)
    t = {k: torch.empty(gen * (2 if k.startswith("len") else STRIDE), dtype=torch.uint8, device="cuda") for k in ("seq1", "qual1", "len1", "seq2", "qual2", "len2")}
    b = capi.Batch(); b.n, b.stride = gen, STRIDE
    for k, v in t.items():
        setattr(b, k, v.data_ptr())
    capi.check(lib.fp_synth_fill(h, C.byref(b), 0, SEED, 1, READ_LEN, None), lib)
    torch.cuda.synchronize()
    lib.fp_ctx_destroy(h)
    pin = []
    for side in ("1", "2"):
        one = fastq_text_np(np, t["seq" + side].cpu().numpy().reshape(gen, STRIDE), t["qual" + side].cpu().numpy().reshape(gen, STRIDE),
                            t["len" + side].cpu().numpy().view(np.uint16), side + ":N:0")
        pin.append(torch.from_numpy(np.tile(one, reps)).pin_memory())
    del t
    both = pin[0].numel() + pin[1].numel()
    caps = [0, pin[0].numel() + 64, pin[1].numel() + 64, both + 64, pin[1].numel() + 64, both + 24 * 2 * n + 64]
    outs = [torch.empty(max(c, 1), dtype=torch.uint8).pin_memory() for c in caps]

    def timed(call):
        for _ in range(args.warmup):
            call()
        times = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            call()
            times.append(time.perf_counter() - t0)
        return times

    for mode, paired, want in () if args.plain else (("pe_out1_out2", 1, (1, 2)), ("pe_all_streams", 1, (1, 2, 3, 4, 5)), ("se_failed_out", 0, (1, 5))):
        p = capi.default_params(paired, lib=lib, seq_len1=READ_LEN, seq_len2=READ_LEN, **FILTERS)
        h = C.c_void_p()
        capi.check(lib.fp_ctx_create(C.byref(p), dev, args.max_batch, STRIDE, STRIDE, C.byref(h)), lib)
        optr = (C.c_void_p * 6)(*[outs[s].data_ptr() if s in want else None for s in range(6)])
        ocap = (C.c_int64 * 6)(*[caps[s] if s in want else 0 for s in range(6)])
        ob = (C.c_int64 * 6)()
        nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64()
        i1, i2 = capi.FastqInfo(), capi.FastqInfo()

        def call():
            capi.check(lib.fp_fastq_process_host_outs(h, pin[0].data_ptr(), pin[0].numel(), pin[1].data_ptr() if paired else None, pin[1].numel() if paired else 0,
                                                      1, 0, optr, ocap, ob, C.byref(nu), C.byref(c1), C.byref(c2) if paired else None, C.byref(i1),
                                                      C.byref(i2) if paired else None), lib)
        times = timed(call)
        assert nu.value == n, (nu.value, n)
        passed = ob[1] / pin[0].numel()
        lib.fp_ctx_destroy(h)
        dt = sum(times) / len(times)
        result[mode] = {"units_per_s": n / dt, "seconds_per_call": [round(x, 4) for x in times],
                        "out_bytes": {k: ob[s] for s, k in enumerate(("merged", "out1", "out2", "unpaired1", "unpaired2", "failed")) if s in want},
                        "out1_bytes_over_input1_bytes": round(passed, 4)}

    if args.plain:
        import hashlib
        p = capi.default_params(1, lib=lib, seq_len1=READ_LEN, seq_len2=READ_LEN, **FILTERS)
        h = C.c_void_p()
        capi.check(lib.fp_ctx_create(C.byref(p), dev, args.max_batch, STRIDE, STRIDE, C.byref(h)), lib)
        o1, o2, nu, c1, c2 = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()

        def call():
            capi.check(lib.fp_fastq_process_host(h, pin[0].data_ptr(), pin[0].numel(), pin[1].data_ptr(), pin[1].numel(), 1, 0,
                                                 outs[1].data_ptr(), caps[1], C.byref(o1), outs[2].data_ptr(), caps[2], C.byref(o2),
                                                 C.byref(nu), C.byref(c1), C.byref(c2), None, None), lib)
        times = timed(call)
        lib.fp_ctx_destroy(h)
        result["plain"] = {"lib": args.lib or "tree", "units_per_s": n / (sum(times) / len(times)), "seconds_per_call": [round(x, 4) for x in times],
                           "md5": hashlib.md5(outs[1][:o1.value].numpy().tobytes() + outs[2][:o2.value].numpy().tobytes()).hexdigest()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
