#!/usr/bin/env python
"""Golden output bits of the paged-attention kernels (multi-token chain and tree verify, shared-prefix decode, single-query decode with
idle rows and non-power-of-two groups), the pages after every appending call, and the planned workspace sizes, at the cases of
tests/test_gpu_paged_attention_bits.py, KV4 and KV8.  The inputs are rebuilt from fixed seeds by the test, so only the outputs are stored.
Needs the built library and an H100 (the context-split count depends on the SM count); run from the repository root:
    python tests/golden/make_golden_paged_attn.py /tmp/paged_attn_bits.npz
and copy the result to tests/golden/.  tests/test_gpu_paged_attention_bits.py compares against it."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.test_gpu_paged_attention_bits import all_outputs  # noqa: E402

dev = torch.device("cuda:0")
np.savez_compressed(sys.argv[1], **{key: t.numpy() for key, t in all_outputs(dev).items()})
print("wrote", sys.argv[1], torch.cuda.get_device_name(dev), torch.cuda.get_device_properties(dev).multi_processor_count, "SMs")
