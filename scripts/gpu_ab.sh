#!/bin/bash
# A/B on an H100: quick parity subset, then short bench lines for a list of env settings (VARIANTS="A=1 B=2|A=0"), 8 M units each.
# The logs go to $OUT (default: a new temporary directory).
OUT="${OUT:-$(mktemp -d)}"; mkdir -p "$OUT"
if [ -n "$TESTS" ]; then
  timeout ${TEST_TIMEOUT:-600} python -m pytest $TESTS -m gpu -q -x --timeout 600 ${TESTK:+-k "$TESTK"} 2>&1 | tail -8 > "$OUT/ab_pytest.log"; cat "$OUT/ab_pytest.log"
fi
U=${U:-8000000}
IFS='|' read -ra VS <<< "${VARIANTS:-FP_NONE=0}"
for v in "${VS[@]}"; do
  for wl in ${WLS:-pe150_overlap_correction}; do
    env $v FP_TRACE=1 python bench.py --workload $wl --units $U --steps 3 --warmup 3 --no-cpu-baseline --no-e2e --fastq-units 0 --no-workloads ${BENCH_ARGS} > "$OUT/ab.json" 2> "$OUT/ab.err"
    python - "$v" "$wl" "$OUT" <<'PY'
import json,sys
try:
    d=json.load(open(sys.argv[3] + '/ab.json'))
    print('AB %-40s %-28s %8.1f M/s kernel_ms %.2f' % (sys.argv[1], sys.argv[2], d['value']/1e6, d['roofline']['kernel_ms']), {k:v for k,v in d['checks'].items() if not v} or 'checks ok')
except Exception as e:
    print('AB', sys.argv[1], sys.argv[2], 'FAILED', e); print(open(sys.argv[3] + '/ab.err').read()[-1500:])
PY
    grep -m1 "chain kernel:" "$OUT/ab.err"
  done
done
