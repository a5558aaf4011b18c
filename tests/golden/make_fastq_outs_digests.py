#!/usr/bin/env python
"""md5 of the UNMODIFIED reference CLI's six files (oracle/_ref/fastp_ref -w 1 ... -o -O --merged_out --unpaired1 --unpaired2 --failed_out,
as far as a case and writer set name them; b"" for a file it does not write) for the cases of fp_outs.fastq_outs_cases()
-> tests/golden/fastq_outs_cli_digests.json (for boxes without the reference binary)."""
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import fp_outs as O  # noqa: E402

out = {}
for name in O.fastq_outs_cases():
    for ws in O.case_writer_sets(name):
        with tempfile.TemporaryDirectory() as d:
            files, _, _ = O.run_ref_cli_outs(Path(d), name, ws)
        out[f"{name}/{ws}"] = [hashlib.md5(x).hexdigest() for x in files]
json.dump(out, open(os.path.join(HERE, "fastq_outs_cli_digests.json"), "w"), indent=1)
print(len(out), "digests")
