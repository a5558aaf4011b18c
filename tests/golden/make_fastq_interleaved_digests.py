#!/usr/bin/env python
"""md5 of what the UNMODIFIED reference CLI (oracle/_ref/fastp_ref -w 1) writes to stdout and to its six files for the runs of
fp_interleaved.RUNS (--interleaved_in, --stdin, --stdout, -m with --stdout / --merged_out, the 0.19.8 rule; b"" for an output it does not
write) -> tests/golden/fastq_interleaved_cli_digests.json (for boxes without the reference binary)."""
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import fp_interleaved as IL  # noqa: E402

out = {}
for run in IL.RUNS:
    with tempfile.TemporaryDirectory() as d:
        outs, _ = IL.run_ref_cli(Path(d), run)
    out[run] = [hashlib.md5(x).hexdigest() for x in outs]
json.dump(out, open(os.path.join(HERE, "fastq_interleaved_cli_digests.json"), "w"), indent=1)
print(len(out), "digests")
