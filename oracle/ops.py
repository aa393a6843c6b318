"""Oracle: fused norm / activation / per-token quant kernels (TEST INFRASTRUCTURE, not product).

Restates kernels/csrc/{fused_kernels.cu, layernorm_kernels.cu, activation_kernels.cu}.
Source-level IEEE semantics are used (the reference is *built* with --use_fast_math,
kernels/setup.py:33, which only perturbs results at the fp32-ulp level; the tests state
where a tolerance is needed because of that or because of reduction order).

fp16 helpers: every fp16 operation is evaluated in float64 and rounded once to float16.
"""
from __future__ import annotations

import numpy as np


def f16(x):
    return np.asarray(x, dtype=np.float64).astype(np.float16)


def f32(x):
    return np.asarray(x).astype(np.float32)


def cvt_rni_sat_s8(x):
    """cvt.rni.sat.s8.f32 (utils.cuh:79-84): round-half-even, saturate, NaN -> 0."""
    x = np.asarray(x, dtype=np.float32)
    r = np.rint(np.nan_to_num(x, nan=0.0, posinf=127.0, neginf=-128.0))
    return np.clip(r, -128, 127).astype(np.int8)


def cvt_rni_sat_u8(x):
    x = np.asarray(x, dtype=np.float32)
    r = np.rint(np.nan_to_num(x, nan=0.0, posinf=255.0, neginf=0.0))
    return np.clip(r, 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------------
# Q1: invoke_quant / invoke_quant_fuse_sum (tensor-scale overloads)   fused_kernels.cu:52-137
# ------------------------------------------------------------------------------------------------


def quant_per_token(x, fuse_sum: bool = True):
    """x fp16 [M,H] -> (q int8 [M,H], scale fp16 [M], sum fp16 [M] or None).

    amax = max|x| (fp32, init 0) ; scale = half(amax/127) ; tmp = 127/amax ;
    q = cvt.rni.sat.s8(float(x)*tmp) ; sum = half(sum_fp32(x))        fused_kernels.cu:104-131
    The fp32 row sum is order dependent on the GPU; the oracle uses a float64 sum rounded to fp32.
    Non-finite rows: the amax is taken with `if (val > amax)`, which never picks a NaN, so NaN elements are ignored
    (and quantise to 0); the sum follows IEEE: an inf makes it inf, +inf with -inf or any NaN makes it NaN.
    """
    xf = f32(x)
    return quant_given_amax(x, _absmax(xf), fuse_sum)


def _absmax(xf):
    """max |x| per row, initialised to 0 and ignoring NaN (the reference's `if (val > amax) amax = val`)."""
    return np.fmax.reduce(np.abs(f32(xf)), axis=1, initial=np.float32(0.0)).astype(np.float32)


def quant_given_amax(x, amax_f32, fuse_sum: bool = True):
    """The per-token quantiser with an amax supplied from outside (fp32 [M], e.g. the max over all tensor-parallel shards):
    scale = half(amax/127) ; q = cvt.rni.sat.s8(float(x)*(127/amax)) ; sum = half(sum of this row), as in quant_per_token."""
    xf = f32(x)
    amax = f32(amax_f32).reshape(-1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        scale = (amax / np.float32(127.0)).astype(np.float32).astype(np.float16)
        tmp = (np.float32(127.0) / amax).astype(np.float32)
        q = cvt_rni_sat_s8((xf * tmp[:, None]).astype(np.float32))
        s = None
        if fuse_sum:
            s = xf.astype(np.float64).sum(axis=1).astype(np.float32).astype(np.float16)
    return q, scale, s


def quant_scalar_scale(x, scale):
    """invoke_quant(out, input, at::Half scale): q = rni_sat(float(x) / float(scale))  fused_kernels.cu:84-88."""
    return cvt_rni_sat_s8((f32(x) / np.float32(np.float16(scale))).astype(np.float32))


# ------------------------------------------------------------------------------------------------
# N1: rms_norm_general[_fuse_sum]  == generalLayerNorm[_fuse_sum]    layernorm_kernels.cu:53-326
# ------------------------------------------------------------------------------------------------


def _ref_block(hidden: int) -> int:
    """blockDim the reference launches with: min(H,1024) rounded up to 32 (layernorm_kernels.cu:433-436)."""
    b = min(hidden, 1024)
    return 32 * ((b + 31) // 32)


def layernorm_general_quant(x, gamma, eps: float, fuse_sum: bool = True):
    """Despite the op name this is a mean-subtracting LayerNorm without beta (layernorm_kernels.cu:21-29,241-268).

    mean = sum(x)/H ; var = sum((x-mean)^2)/H ; y = (x-mean)*rsqrt(var+eps)*gamma    (fp32)
    y_h = half(y) ; amax = max(|y_h|, 1e-6) in fp16 ; sum: each of the `blockDim` threads adds its own
    y_h values IN FP16 (thread t owns elements t, t+B, t+2B, ...), then an fp32 block reduce  (:274-306)
    q = cvt.rni.sat.s8(y_fp32 * (127/amax)) using the UN-rounded fp32 y                     (:307-318)
    scale = half(amax/127) ; input_sum = half(sum)                                           (:320-324)
    Returns (q int8, scale fp16 [M], sum fp16 [M] or None, y fp32) -- y for diagnostics.
    """
    xf = f32(x)
    M, H = xf.shape
    g = f32(gamma)
    mean = (xf.astype(np.float64).sum(axis=1) / H).astype(np.float32)
    diff = (xf - mean[:, None]).astype(np.float32)
    var = ((diff.astype(np.float64) ** 2).sum(axis=1)).astype(np.float32)
    rstd = (1.0 / np.sqrt((var / np.float32(H) + np.float32(eps)).astype(np.float64))).astype(np.float32)
    y = ((diff * rstd[:, None]).astype(np.float32) * g[None, :]).astype(np.float32)
    yh = y.astype(np.float16)
    amax_h = np.maximum(np.abs(yh).max(axis=1), np.float16(1e-6))
    amax = amax_h.astype(np.float32)
    tmp = (np.float32(127.0) / amax).astype(np.float32)
    q = cvt_rni_sat_s8((y * tmp[:, None]).astype(np.float32))
    scale = (amax / np.float32(127.0)).astype(np.float32).astype(np.float16)
    s = None
    if fuse_sum:
        B = _ref_block(H)
        n_iter = (H + B - 1) // B
        pad = n_iter * B - H
        yp = np.concatenate([yh, np.zeros((M, pad), np.float16)], axis=1).reshape(M, n_iter, B)
        acc = np.zeros((M, B), np.float16)
        for j in range(n_iter):  # sequential fp16 accumulation per thread
            acc = f16(acc.astype(np.float64) + yp[:, j].astype(np.float64))
        s = acc.astype(np.float64).sum(axis=1).astype(np.float32).astype(np.float16)
    return q, scale, s, y


def layernorm_general_quant_per_tensor(x, gamma, eps: float, scale):
    """rms_norm_general with use_per_token_quant=False: a static per-tensor scale (fp16, read) instead of the row amax.

    mean, variance and y as in layernorm_general_quant ; q = cvt.rni.sat.s8(float(half(y)) * float(scale))
    (layernorm_kernels.cu:153-157: the fp16-rounded y, not the fp32 y the per-token form quantises).
    Returns (q int8 [M, H], y fp32) -- y for diagnostics.
    """
    xf = f32(x)
    H = xf.shape[1]
    g = f32(gamma)
    mean = (xf.astype(np.float64).sum(axis=1) / H).astype(np.float32)
    diff = (xf - mean[:, None]).astype(np.float32)
    var = ((diff.astype(np.float64) ** 2).sum(axis=1)).astype(np.float32)
    rstd = (1.0 / np.sqrt((var / np.float32(H) + np.float32(eps)).astype(np.float64))).astype(np.float32)
    y = ((diff * rstd[:, None]).astype(np.float32) * g[None, :]).astype(np.float32)
    sc = np.float32(np.float16(scale))
    q = cvt_rni_sat_s8((y.astype(np.float16).astype(np.float32) * sc).astype(np.float32))
    return q, y


# ------------------------------------------------------------------------------------------------
# N2: rms_norm (final norm)   layernorm_kernels.cu:330-360
# ------------------------------------------------------------------------------------------------


def rms_norm(x, weight, eps: float, use_quant: bool = False):
    """out = half(x * rsqrt(mean(x^2)+eps)) * weight   (fp16 multiply)   or   rni_sat_s8(float(x*s)*w)."""
    xf = f32(x)
    H = xf.shape[1]
    var = (xf.astype(np.float64) ** 2).sum(axis=1).astype(np.float32)
    s = (1.0 / np.sqrt((var / np.float32(H) + np.float32(eps)).astype(np.float64))).astype(np.float32)
    xs = (xf * s[:, None]).astype(np.float32)
    if use_quant:
        return cvt_rni_sat_s8((xs * f32(weight)[None, :]).astype(np.float32))
    return f16(xs.astype(np.float16).astype(np.float64) * np.asarray(weight, np.float16).astype(np.float64)[None, :])


# ------------------------------------------------------------------------------------------------
# A0: silu_and_mul   activation_kernels.cu:10-30
# ------------------------------------------------------------------------------------------------


def silu_and_mul(x):
    """x fp16 [M, 2d] -> fp16 [M, d]:  half( x/(1+expf(-x)) ) * y   with the product in fp16."""
    x = np.asarray(x, dtype=np.float16)
    d = x.shape[1] // 2
    g = x[:, :d].astype(np.float32)
    silu = (g / (np.float32(1.0) + np.exp(-g).astype(np.float32))).astype(np.float32).astype(np.float16)
    return f16(silu.astype(np.float64) * x[:, d:].astype(np.float64))


# ------------------------------------------------------------------------------------------------
# Legacy exports (not reached by llama_w4a8/w8a8, kept for API completeness)
# ------------------------------------------------------------------------------------------------


def dequant_add_residual(inp_i32, residual, scale):
    """out = T(float(in)*scale + float(residual)); scale scalar or [M]   fused_kernels.cu:19-38."""
    sc = f32(scale)
    sc = sc[:, None] if sc.ndim == 1 else sc
    return ((np.asarray(inp_i32).astype(np.float32) * sc).astype(np.float32) + f32(residual)).astype(np.float32).astype(np.float16)


def dequant(inp_i32, scale):
    return (np.asarray(inp_i32).astype(np.float32) * np.float32(np.float16(scale))).astype(np.float32).astype(np.float16)


def _hmul(a, b):
    return f16(np.asarray(a, np.float16).astype(np.float64) * np.asarray(b, np.float16).astype(np.float64))


def _hadd(a, b):
    return f16(np.asarray(a, np.float16).astype(np.float64) + np.asarray(b, np.float16).astype(np.float64))


def gelu_new(x):
    """activation_kernels.cu:166-170 with scalar_t = half: every `T` expression is rounded to fp16."""
    x = np.asarray(x, np.float16)
    x3 = _hmul(_hmul(x, x), x).astype(np.float32)
    inner = (np.float32(0.044715) * x3).astype(np.float32).astype(np.float16)
    arg = (np.float32(0.79788456) * _hadd(x, inner).astype(np.float32)).astype(np.float32).astype(np.float16)
    t = np.tanh(arg.astype(np.float32)).astype(np.float32).astype(np.float16)
    return _hmul(_hmul(np.float16(0.5), x), _hadd(np.float16(1.0), t))


def gelu_fast(x):
    """activation_kernels.cu:172-178 with scalar_t = half."""
    x = np.asarray(x, np.float16)
    f = x.astype(np.float32)
    a = (f * np.float32(0.79788456)).astype(np.float32).astype(np.float16)
    b = _hadd(np.float16(1.0), _hmul((np.float32(0.044715) * f).astype(np.float32).astype(np.float16), x))
    t = np.tanh(_hmul(a, b).astype(np.float32)).astype(np.float32).astype(np.float16)
    return _hmul(_hmul(np.float16(0.5), x), _hadd(np.float16(1.0), t))


def dequant_add_residual_rms_norm_quant(inp_i32, residual, gamma, scale, eps):
    """layernorm_kernels.cu:365-401; returns (q int8, new_residual fp16)."""
    sc = f32(scale)
    sc = sc[:, None] if sc.ndim == 1 else sc
    d = ((np.asarray(inp_i32).astype(np.float32) * sc).astype(np.float32) + f32(residual)).astype(np.float32)
    res = d.astype(np.float16)
    H = d.shape[1]
    var = (d.astype(np.float64) ** 2).sum(axis=1).astype(np.float32)
    s = (1.0 / np.sqrt((var / np.float32(H) + np.float32(eps)).astype(np.float64))).astype(np.float32)
    q = cvt_rni_sat_s8(((res.astype(np.float32) * s[:, None]).astype(np.float32) * f32(gamma)[None, :]).astype(np.float32))
    return q, res


def dequant_silu_and_mul_quant(inp_i32, scale_gate, scale_up, scale_out):
    """activation_kernels.cu:33-80 (scalar scale_out variant): q = rni_sat(silu(x)*y/scale_out)."""
    a = np.asarray(inp_i32)
    d = a.shape[1] // 2
    x = (a[:, :d].astype(np.float32) * np.float32(scale_gate)).astype(np.float32)
    y = (a[:, d:].astype(np.float32) * np.float32(scale_up)).astype(np.float32)
    silu = (x / (np.float32(1.0) + np.exp(-x).astype(np.float32))).astype(np.float32)
    return cvt_rni_sat_s8(((silu * y).astype(np.float32) / np.float32(scale_out)).astype(np.float32))


def dequant_silu_and_mul_quant_per_token(inp_i32, scale_gate, scale_up):
    """activation_kernels.cu:33-70 (per-token variant): t = silu(x)*y in fp32 ; amax = max|t| (init 0, NaN ignored) ;
    scale_out = amax/127 (fp32) ; q = rni_sat((127/amax) * t).   Returns (q int8 [M, d], scale_out fp32 [M], tmp fp32 [M, d])."""
    a = np.asarray(inp_i32)
    d = a.shape[1] // 2
    x = (a[:, :d].astype(np.float32) * np.float32(scale_gate)).astype(np.float32)
    y = (a[:, d:].astype(np.float32) * np.float32(scale_up)).astype(np.float32)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        silu = (x / (np.float32(1.0) + np.exp(-x).astype(np.float32))).astype(np.float32)
        t = (silu * y).astype(np.float32)
        amax = _absmax(t)
        scale_out = (amax / np.float32(127.0)).astype(np.float32)
        q = cvt_rni_sat_s8(((np.float32(127.0) / amax).astype(np.float32)[:, None] * t).astype(np.float32))
    return q, scale_out, t
