"""CPU tests: the C-ABI library loads and exports every symbol include/qserve_b200.h declares, with the ctypes types of its prototype; the
drop-in package exposes the reference's module and function names; ops fail loudly without a GPU (no fallback)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CTYPES = {"int": ctypes.c_int, "int32_t": ctypes.c_int, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "unsigned": ctypes.c_uint,
           "size_t": ctypes.c_size_t, "float": ctypes.c_float}


def _ctype(c_type: str, ret: bool = False):
    """The ctypes type a C type of the header is bound with: every pointer is c_void_p, except a `const char*` result (c_char_p)."""
    c_type = " ".join(c_type.replace("*", " * ").split())
    if "*" in c_type:
        return ctypes.c_char_p if ret and c_type == "const char *" else ctypes.c_void_p
    return _CTYPES[c_type]


def _declared():
    """name -> (restype, argtypes) of every qs_* prototype in include/qserve_b200.h, in ctypes terms."""
    text = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "qserve_b200.h")).read(), flags=re.S)
    protos = {}
    for ret, name, params in re.findall(r"QS_API\s+([^;(]*?)\s*\b(qs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        params = [] if params.strip() == "void" else [re.fullmatch(r"(.*?)\s*\w+", p.strip()).group(1) for p in params.split(",")]
        protos[name] = (_ctype(ret, ret=True), [_ctype(p) for p in params])
    return protos


def test_library_exports_every_declared_symbol():
    from qserve_b200 import _lib

    protos = _declared()
    names = sorted(protos)
    assert len(names) >= 25
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in include/qserve_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == names, "python binding and header disagree"
    wrong = {n: (_lib.SIGNATURES[n], protos[n]) for n in names if _lib.SIGNATURES[n] != protos[n]}
    assert not wrong, f"ctypes (restype, argtypes) differ from include/qserve_b200.h (binding, header): {wrong}"
    assert raw.qs_abi_version() == _lib.ABI_VERSION


def test_dropin_module_surface():
    """SURVEY.md 8b: module and function names of the seven reference extensions."""
    import qserve_backend as qb

    want = {
        "qgemm_w4a8_per_chn": ["gemm_forward_cuda"],
        "qgemm_w4a8_per_group": ["gemm_forward_cuda"],
        "qgemm_w8a8": ["w8a8_gemm_forward_cuda"],
        "fused_attention": ["single_query_attention", "apply_bias_rope_update_kv_cache", "compute_padding_offsets"],
        "layernorm_ops": ["rms_norm", "rms_norm_general", "rms_norm_general_fuse_sum", "invoke_dequant_add_residual_rms_norm_quant"],
        "fused_kernels": ["invoke_quant", "invoke_quant_fuse_sum", "invoke_dequant_add_residual", "invoke_dequant"],
        "activation_ops": ["silu_and_mul", "gelu_new", "gelu_fast", "invoke_dequant_silu_and_mul_quant"],
    }
    for mod, fns in want.items():
        m = getattr(qb, mod)
        for f in fns:
            assert callable(getattr(m, f)), f"{mod}.{f}"
    # keyword names that the reference binds with py::arg (layernorm.cpp:48-58)
    sig = inspect.signature(qb.layernorm_ops.rms_norm_general_fuse_sum)
    assert list(sig.parameters) == ["out", "input", "weight", "input_sum", "scaling", "epsilon", "use_per_token_quant"]
    sig = inspect.signature(qb.layernorm_ops.rms_norm)
    assert list(sig.parameters) == ["out", "input", "weight", "epsilon", "use_quant"]
    assert len(inspect.signature(qb.fused_attention.single_query_attention).parameters) == 15
    assert len(inspect.signature(qb.fused_attention.apply_bias_rope_update_kv_cache).parameters) == 15


def test_prompt_attention_has_the_call_site_signature():
    """`backend.flash_attn_varlen_func` stands in for flash_attn.flash_attn_varlen_func at llama_w4a8_unpad.py:232-242, which passes q, k, v
    positionally and cu_seqlens_q / cu_seqlens_k / max_seqlen_q / max_seqlen_k / dropout_p / causal by keyword: same names, same positional order
    as flash-attn 2.x for the leading parameters; CPU tensors are rejected like everywhere else."""
    from qserve_b200 import backend

    params = list(inspect.signature(backend.flash_attn_varlen_func).parameters)
    assert params[:10] == ["q", "k", "v", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k", "dropout_p", "softmax_scale", "causal"]
    q = torch.zeros(4, 2, 128, dtype=torch.half)
    cu = torch.tensor([0, 4], dtype=torch.int32)
    with pytest.raises(RuntimeError):
        backend.flash_attn_varlen_func(q, q, q, cu_seqlens_q=cu, cu_seqlens_k=cu, max_seqlen_q=4, max_seqlen_k=4, dropout_p=0.0, causal=True)


def test_no_cpu_fallback():
    """CPU tensors are rejected (the reference's CHECK_DEVICE); nothing silently computes on the host."""
    import qserve_backend as qb

    x = torch.zeros(4, 128, dtype=torch.int8)
    with pytest.raises(RuntimeError):
        qb.qgemm_w8a8.w8a8_gemm_forward_cuda(x, torch.zeros(128, 128, dtype=torch.int8), torch.ones(128, dtype=torch.half),
                                            torch.ones(4, dtype=torch.half), torch.zeros(4, 128, dtype=torch.half))
    with pytest.raises(RuntimeError):
        qb.fused_kernels.invoke_quant(torch.zeros(4, 128, dtype=torch.int8), torch.zeros(4, 128, dtype=torch.half), torch.zeros(4, dtype=torch.half))


def test_product_never_imports_oracle():
    for pkg in ("qserve_b200", "qserve_backend"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, pkg)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h")):
                    src = open(os.path.join(dirpath, f)).read()
                    assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f"{pkg}/{f} imports the oracle"
