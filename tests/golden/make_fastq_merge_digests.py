#!/usr/bin/env python
"""md5 of the UNMODIFIED reference CLI's three merging-mode files (oracle/_ref/fastp_ref -w 1 -m --merged_out ... -o -O, or
--include_unmerged) for the cases of fp_merge.fastq_merge_cases() -> tests/golden/fastq_merge_cli_digests.json
(for boxes without the reference binary)."""
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import fp_merge as M  # noqa: E402

out = {}
for name, (flags, kw, t1, t2, stride, dedup) in M.fastq_merge_cases().items():
    with tempfile.TemporaryDirectory() as d:
        m, o1, o2, _ = M.run_ref_cli_merge(Path(d), flags, t1, t2)
    out[name] = [hashlib.md5(x).hexdigest() for x in (m, o1, o2)]
json.dump(out, open(os.path.join(HERE, "fastq_merge_cli_digests.json"), "w"), indent=1)
print(out)
