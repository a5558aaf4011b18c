#!/usr/bin/env python
"""md5 of the UNMODIFIED reference CLI's --overlapped_out file (oracle/_ref/fastp_ref -w 1 ... --overlapped_out) for the cases of
fp_overlapped.overlapped_cases() -> tests/golden/fastq_overlapped_cli_digests.json (for boxes without the reference binary)."""
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import fp_overlapped as O  # noqa: E402

out = {}
for name, (flags, p, t1, t2, stride, dedup) in O.overlapped_cases().items():
    with tempfile.TemporaryDirectory() as d:
        out[name] = hashlib.md5(O.run_ref_cli(Path(d), flags, t1, t2)).hexdigest()
json.dump(out, open(os.path.join(HERE, "fastq_overlapped_cli_digests.json"), "w"), indent=1)
print(out)
