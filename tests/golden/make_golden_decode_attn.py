#!/usr/bin/env python
"""Golden output bits of the decode-attention kernel: single_query_attention (fp16 out) and single_query_attention_quant (int8 codes,
fp16 scale and sum) at tests/test_gpu_attention.GOLDEN_CASES, KV4 and KV8.  The inputs are rebuilt from fixed seeds by the test, so only
the outputs are stored.  Needs the built library and an H100 (the context-split count depends on the SM count); run from the repository root:
    python tests/golden/make_golden_decode_attn.py /tmp/decode_attn_bits.npz
and copy the result to tests/golden/.  tests/test_gpu_attention.py::test_decode_attention_output_bits_are_pinned compares against it."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.test_gpu_attention import GOLDEN_CASES, decode_attn_outputs  # noqa: E402

dev = torch.device("cuda:0")
arrays = {}
for bits in (4, 8):
    for case in range(len(GOLDEN_CASES)):
        for key, t in decode_attn_outputs(dev, case, bits).items():
            arrays[f"kv{bits}_{case}_{key}"] = t.numpy()
np.savez_compressed(sys.argv[1], **arrays)
print("wrote", sys.argv[1], torch.cuda.get_device_name(dev), torch.cuda.get_device_properties(dev).multi_processor_count, "SMs")
