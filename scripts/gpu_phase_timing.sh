#!/bin/bash
# phase timing on an H100: swaps in the -DFP_PHASE_TIMING build (scripts/timing/libfastp_b200.so), prints what the 16 warps of CTA 0
# spent per phase, then their means in M cycles.  Phases A and C are split into the dense column pass ("col": mean over the warps that
# hold columns, measured up to the end of dense_tile / dense_remove), the items that follow it ("items": mean over all warps) and the
# wait at the CTA barrier ("wait").  The bench logs go to $OUT (default: a new temporary directory).
OUT="${OUT:-$(mktemp -d)}"; mkdir -p "$OUT"
[ -f scripts/timing/libfastp_b200.so ] || { echo "build it first: nvcc ... -DFP_PHASE_TIMING ... -o scripts/timing/libfastp_b200.so (same line as __graft_entry__.build)"; exit 1; }
cp fastp_b200/libfastp_b200.so /tmp/lib_orig.so; cp scripts/timing/libfastp_b200.so fastp_b200/libfastp_b200.so
for wl in ${WLS:-pe150_overlap_correction}; do
  python bench.py --workload $wl --units ${U:-8000000} --steps 1 --warmup 1 --no-cpu-baseline --no-e2e --fastq-units 0 --no-workloads > "$OUT/timing_$wl.log" 2>&1
  grep PHASE "$OUT/timing_$wl.log" | tail -16
  grep PHASE "$OUT/timing_$wl.log" | tail -16 | python3 -c '
import sys
rows = []
for ln in sys.stdin:
    t = ln.split()[1:]
    rows.append({t[i]: int(t[i + 1]) for i in range(0, len(t) - 1, 2)})
if not rows: sys.exit("no PHASE lines")
M = lambda v: v / len(rows) / 1e6
cw = [r for r in rows if r["col"]] or rows
col = lambda k: sum(r[k] for r in cw) / len(cw) / 1e6
s = lambda *ks: M(sum(r[k] for r in rows for k in ks))
print("%s: %d column warps | tma %.2f | A %.2f (col %.2f, items %.2f, wait %.2f) | B to decision %.2f | correction list %.2f | B after %.2f"
      " | C %.2f (col %.2f, items %.2f, wait %.2f) | total %.2f M cycles" % (sys.argv[1], sum(r["col"] for r in rows),
      s("tma"), s("colA", "itemsA", "totA"), col("colA"), s("itemsA"), s("totA"), s("busyB1", "totB1"), s("corr"), s("busyB2", "totB2"),
      s("colC", "itemsC", "totC"), col("colC"), s("itemsC"), s("totC"),
      s("tma", "colA", "itemsA", "totA", "busyB1", "totB1", "corr", "busyB2", "totB2", "colC", "itemsC", "totC")))
' "$wl"
done
cp /tmp/lib_orig.so fastp_b200/libfastp_b200.so
