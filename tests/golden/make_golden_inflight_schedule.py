#!/usr/bin/env python
"""Record the in-flight schedule oracles' decisions on the seeded scripts of tests/test_oracle_schedule_trace.py:
python tests/golden/make_golden_inflight_schedule.py [OUT.npz]  (default: the committed tests/golden/inflight_schedule_trace.npz).
The trace pins the rules as they were when it was recorded; it is not rewritten to make a changed rule pass."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.test_oracle_schedule_trace import SCRIPTS, trace  # noqa: E402

OUT = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "inflight_schedule_trace.npz")
res = {}
for name, run in SCRIPTS.items():
    for k, v in trace(run).items():
        res[f"{name}:{k}"] = v
np.savez_compressed(OUT, **res)
print("wrote", len(SCRIPTS), "scripts,", sum(len(v) for k, v in res.items() if k.endswith(":plan")), "schedule calls")
