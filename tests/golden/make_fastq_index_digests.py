#!/usr/bin/env python
"""md5 of every output file of the UNMODIFIED reference CLI (oracle/_ref/fastp_ref -w 1 ... --filter_by_index1/2), and its -j counts that the
index filter decides, for the cases of fp_index.index_cases() -> tests/golden/fastq_index_cli_digests.json (for boxes without the
reference binary)."""
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import fp_index as X  # noqa: E402
from fp_testlib import REF_CLI  # noqa: E402

out = {}
for name in sorted(X.index_cases()):
    with tempfile.TemporaryDirectory() as d:
        files, js, r = X.run_cli(REF_CLI, Path(d), name)
        assert r.returncode == 0, r.stderr
        out[name] = {"files": {k: hashlib.md5(files[k]).hexdigest() for k in X.STREAMS}, "counts": X.json_counts(js)}
json.dump(out, open(os.path.join(HERE, "fastq_index_cli_digests.json"), "w"), indent=1)
print(len(out), "cases")
