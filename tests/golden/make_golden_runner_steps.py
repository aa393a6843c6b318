#!/usr/bin/env python
"""Golden output bits of every decode-runner step kind (tests/test_gpu_runner_steps.runner_step_outputs) at w4a8kv4, w4a8kv4-g128 and
w8a8kv8.  The runs are rebuilt from fixed seeds by the test, so only the outputs are stored.  Needs the built library and an H100; run from
the repository root:
    python tests/golden/make_golden_runner_steps.py /tmp/runner_steps.npz [/tmp/runner_kernels.json]
and copy the .npz to tests/golden/.  tests/test_gpu_runner_steps.py::test_runner_steps_reproduce_the_pinned_bits compares against it.

With a second argument it also records, under torch.profiler, the names of the CUDA kernels (and memcpy / memset) one eager step of each
kind launches, in launch order, and writes them as JSON: two versions of the runner that should launch the same sequence give equal files."""
import contextlib
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.test_gpu_runner_steps import PRECISIONS, _as_numpy, runner_step_outputs  # noqa: E402

dev = torch.device("cuda:0")
kernels = {}


def recorder(precision):
    @contextlib.contextmanager
    def around(name):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            yield
            torch.cuda.synchronize()
        events = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
        kernels[f"{precision}.{name}"] = [e.name for e in events]
    return around


record = len(sys.argv) > 2
arrays = {}
for precision in PRECISIONS:
    around = recorder(precision) if record else (lambda name: contextlib.nullcontext())
    for key, t in runner_step_outputs(dev, precision, around).items():
        arrays[f"{precision}.{key}"] = _as_numpy(t)
np.savez_compressed(sys.argv[1], **arrays)
if record:
    with open(sys.argv[2], "w") as f:
        json.dump(kernels, f, indent=1)
print("wrote", sys.argv[1:], len(arrays), "arrays", torch.cuda.get_device_name(dev))
