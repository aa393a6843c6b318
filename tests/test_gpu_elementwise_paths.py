"""GPU: every kernel the elementwise host launchers (csrc/elementwise.cu) can pick, compared with the oracle, on smooth rows mixed with
edge rows in the same call.

The launchers choose a kernel from the row width, the token count and the SM count.  `_norm_plan`, `_quant_plan` and `_silu_plan` below mirror those rules
(launch_norm_fast, quant_per_token, silu_and_mul_quant with its cluster-size loop); every case names the kernel it is meant to reach,
the mirror must agree, and `test_launched_kernel_names` checks under torch.profiler that the library really launches it.  Cluster sizes
depend on the SM count, so silu_and_mul_quant cases choose their token count from the mirror at run time.

Edge rows (mixed into ordinary rows): zero, constant non-zero (the norm subtracts the mean: y = 0, amax clamps to half(1e-6)),
one-hot +-2000 and +-65504 over N(0, 1) (the outlier's code must be exactly +-127), +-65504 throughout, subnormal only; and for the
quantisers and silu_and_mul_quant one +inf, two +inf, +inf with -inf, one NaN.  silu_and_mul_quant gets its infinities by fp16
overflow (g = u = 300) and its NaN from a NaN input.  Norm rows with non-finite input are not tested: every output is NaN there, in
this library and in the reference alike.

Non-finite contract (the reference's fused_kernels.cu:104-131): amax ignores NaN (`if (val > amax)`); the row sum is an IEEE sum,
so inf for infinities of one sign and NaN for +inf with -inf or any NaN; with amax = inf every code is 0.

Stated tolerances (none looser than tests/test_gpu_elementwise.py):
  * invoke_quant[_fuse_sum], row_absmax + invoke_quant_given_amax: codes, fp16 scales, fp32 amax and row sums bit-exact (NaN == NaN).
  * Norms (per-token): scale <= 1 fp16 ulp; codes differ by <= 1 and only where y*127/amax is within 2e-3 of a rounding boundary,
    on < 0.2 % of the elements -- or anywhere in a row whose scale moved by its ulp; row sum within 2e-3*sqrt(H) (the mean /
    variance are fp32 reductions in another order).
    add_rms_norm_general: hidden_out bit-exact to half(float(x) + float(delta)) and every output bit-exact to rms_norm_general on it.
  * Norm (per-tensor): codes differ by <= 1, only where the code of half(y*(1 +- 2e-6)) * scale differs, on < 0.2 % of the elements.
  * rms_norm: fp16 output between the oracle's outputs for rstd * (1 -+ 1e-5), and different from the oracle on < 1 % of the
    elements; INT8 output <= 1.
  * silu_and_mul_quant: bit-exact to silu_and_mul -> invoke_quant[_fuse_sum], and bit-exact to the quantiser oracle applied to the
    GPU activation.  Against the oracle end to end, ops.quant_per_token(ops.silu_and_mul(x)): the activations differ by <= 2 fp16 ulp
    on < 0.1 % of the elements (expf differs in the last fp32 bit); codes by <= 1 LSB, and only where half(silu)*u itself differs or
    x*127/amax is within 2e-3 of a rounding boundary -- or anywhere in a row whose largest element differs; the scale is bit-exact
    unless the row's largest element differs, and then by no more fp16 ulps than that element.
  * invoke_dequant_silu_and_mul_quant (per-token): tmp and scale_out within 8 fp32 ulps (expf), codes within 1 LSB.
  * Live reference (oracle/_ref present): invoke_quant_fuse_sum codes <= 1 LSB, scale bit-exact, sum <= 1 fp16 ulp; silu_and_mul
    <= 2 ulp on < 0.2 %; rms_norm_general_fuse_sum codes <= 1 on < 0.2 %, scale <= 1 ulp, sum within 2e-3*sqrt(H); and the non-finite
    sums and scales are inf / NaN exactly where the reference's are.
"""
import re
import zlib

import numpy as np
import pytest
import torch

from oracle import ops
from tests.util import bits16, np_of, to_dev, ulp16_diff

pytestmark = pytest.mark.gpu

THREADS, SILU_THREADS, SMEM_NO_ATTR = 512, 256, 40 * 1024
EPS = 1e-5


# ------------------------------------------------------------------------------------------------------------------------------------
# mirror of the host dispatch in csrc/elementwise.cu
# ------------------------------------------------------------------------------------------------------------------------------------
def _norm_plan(H, add, per_token, with_sum):
    nvec = H // 8
    if per_token and nvec <= 2 * THREADS:  # launch_norm_fast
        return [f"norm_quant_fast_kernel<{'true' if add else 'false'}, false, {1 if nvec <= THREADS else 2}>"], False
    smem = 2 * H * (2 if with_sum else 1)
    return ["add_layernorm_quant_kernel<false>" if add else "layernorm_quant_kernel"], smem > SMEM_NO_ATTR


def _quant_plan(H):
    nvec = H // 8
    for ch in (1, 2, 4):
        if nvec <= ch * THREADS:
            return [f"quant_per_token_fast_kernel<{ch}>"], False
    return ["quant_per_token_kernel"], 2 * H > SMEM_NO_ATTR


def _silu_plan(M, d, sms):
    csize = 1
    while csize < 8 and M * csize < 2 * sms and d % (csize * 2 * 8) == 0 and d // (csize * 2) >= 512:
        csize *= 2
    nvec = d // csize // 8
    if nvec <= 2 * SILU_THREADS:
        return csize, f"silu_mul_quant_fast_kernel<{1 if nvec <= SILU_THREADS else 2}>", False
    return csize, "silu_mul_quant_kernel", (d // csize) * 2 > SMEM_NO_ATTR


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _silu_tokens(target, d, prefer):
    """A token count that reaches `target` = (cluster size, kernel, dynamic-smem attribute) on this GPU: `prefer` if it does
    (the numbers are chosen for a 132-SM H100), else the smallest that does."""
    sms = _sms()
    for M in [prefer] + list(range(24, 8 * sms)):
        if _silu_plan(M, d, sms) == target:
            return M
    pytest.fail(f"silu_and_mul_quant branch {target} at d={d} is unreachable with {sms} SMs")


# ------------------------------------------------------------------------------------------------------------------------------------
# cases: (op, params, the branch it targets)
# ------------------------------------------------------------------------------------------------------------------------------------
WIDTHS = [4096, 8192, 12288, 16384, 24576]
CASES = []
for H in WIDTHS:
    for s in (True, False):
        CASES.append(("norm", dict(H=H, with_sum=s, per_token=True)))
        CASES.append(("add_norm", dict(H=H, with_sum=s)))
    CASES.append(("norm", dict(H=H, with_sum=False, per_token=False)))
for H in (4096, 24576):
    for q in (False, True):
        CASES.append(("rms_norm", dict(H=H, use_quant=q)))
for H in (4096, 8192, 16384, 24576, 28672):
    for s in (True, False):
        CASES.append(("quant", dict(H=H, with_sum=s)))
for H in (4096, 24576):
    for s in (True, False):
        CASES.append(("given_amax", dict(H=H, with_sum=s)))
# (cluster size, kernel, smem attribute), d, preferred token count on 132 SMs
SILU_TARGETS = [
    ((8, "silu_mul_quant_fast_kernel<1>", False), 14336, 64),
    ((8, "silu_mul_quant_fast_kernel<2>", False), 24576, 40),
    ((4, "silu_mul_quant_fast_kernel<2>", False), 14336, 96),
    ((4, "silu_mul_quant_kernel", False), 24576, 96),
    ((2, "silu_mul_quant_kernel", False), 14336, 256),   # verify step, B = 64, n = 4
    ((1, "silu_mul_quant_kernel", False), 14336, 512),   # verify step, B = 64, n = 8
    ((1, "silu_mul_quant_kernel", True), 24576, 300),    # Qwen1.5-72B at TP = 1: 48 KiB of dynamic smem
    ((1, "silu_mul_quant_fast_kernel<2>", False), 3584, 300),
    ((1, "silu_mul_quant_fast_kernel<1>", False), 1000, 40),  # d % 16 != 0: no cluster
]
for target, d, prefer in SILU_TARGETS:
    for s in (True, False):
        CASES.append(("silu", dict(target=target, d=d, prefer=prefer, with_sum=s)))
for d in (4096, 1000):
    CASES.append(("dequant_silu", dict(d=d)))


def _case_id(c):
    op, p = c
    if op == "silu":
        return f"silu-c{p['target'][0]}-{p['target'][1].replace('silu_mul_quant_', '')}-d{p['d']}-{'sum' if p['with_sum'] else 'nosum'}"
    return op + "-" + "-".join(f"{k}{int(v) if isinstance(v, bool) else v}" for k, v in p.items())


def _expected(op, p, M):
    """kernel names the launch must consist of (in order), and whether the dynamic-smem attribute path is taken"""
    if op in ("norm", "add_norm"):
        return _norm_plan(p["H"], op == "add_norm", p.get("per_token", True), p["with_sum"])
    if op == "rms_norm":
        return ["rms_norm_kernel"], 2 * p["H"] > SMEM_NO_ATTR
    if op == "quant":
        return _quant_plan(p["H"])
    if op == "given_amax":
        return ["row_absmax_kernel", "quant_given_amax_kernel"], False
    if op == "silu":
        csize, kern, attr = _silu_plan(M, p["d"], _sms())
        assert (csize, kern, attr) == p["target"], "the mirror does not reach the branch this case targets"
        return [kern], attr
    return ["dequant_silu_and_mul_quant_kernel"], False


# ------------------------------------------------------------------------------------------------------------------------------------
# inputs: ordinary rows with edge rows mixed in (odd row indices)
# ------------------------------------------------------------------------------------------------------------------------------------
def _edge_rows(rng, H, nonfinite):
    """name -> (fp64 row, outlier index or None)"""
    e = {"zero": (np.zeros(H), None), "constant": (np.full(H, 0.75), None)}
    for v in (2000.0, -2000.0, 65504.0, -65504.0):
        r, i = rng.standard_normal(H), int(rng.integers(H))
        r[i] = v
        e[f"onehot{v:+.0f}"] = (r, i)
    e["pm65504"] = (rng.choice([-65504.0, 65504.0], H), None)
    e["subnormal"] = (rng.integers(-1023, 1024, H) * 2.0 ** -24, None)
    if nonfinite:
        for name, vals in (("inf", [np.inf]), ("two_inf", [np.inf, np.inf]), ("inf_ninf", [np.inf, -np.inf]), ("nan", [np.nan])):
            r = rng.standard_normal(H)
            r[rng.choice(H, len(vals), replace=False)] = vals
            e[name] = (r, None)
    return e


def _mix(rng, base, edges):
    """put the edge rows into `base` (fp16 [M, H]) at rows 1, 3, 5, ...; returns name -> (row, outlier index)"""
    where = {}
    for k, (name, (r, i)) in enumerate(edges.items()):
        row = 2 * k + 1
        assert row < base.shape[0]
        with np.errstate(over="ignore"):
            base[row] = r.astype(np.float16)
        where[name] = (row, i)
    return where


def _silu_edges(rng, d):
    """name -> (g row, u row, outlier index): half(silu(g)) * u produces the edge activation"""
    n = lambda: rng.standard_normal(d)
    e = {"zero": (n(), np.zeros(d), None), "constant": (np.full(d, 8.0), np.full(d, 0.5), None)}
    for name, (gv, uv) in (("onehot+2000", (50.0, 40.0)), ("onehot-2000", (50.0, -40.0)),
                           ("onehot+65504", (256.0, 255.875)), ("onehot-65504", (256.0, -255.875))):
        g, u, i = n(), n(), int(rng.integers(d))
        g[i], u[i] = gv, uv
        e[name] = (g, u, i)
    e["pm65504"] = (np.full(d, 256.0), rng.choice([-255.875, 255.875], d), None)
    e["subnormal"] = (np.ones(d), rng.integers(-1023, 1024, d) * 2.0 ** -24, None)
    for name, us in (("inf", [300.0]), ("two_inf", [300.0, 300.0]), ("inf_ninf", [300.0, -300.0])):
        g, u = n(), n()
        idx = rng.choice(d, len(us), replace=False)
        g[idx], u[idx] = 300.0, us  # half(silu(300)) * 300 = 90000 overflows fp16
        e[name] = (g, u, None)
    g, u = n(), n()
    u[int(rng.integers(d))] = np.nan
    e["nan"] = (g, u, None)
    return e


def _same16(a, b):
    """bit-exact fp16 equality where NaN matches NaN (the NaN payload is not part of the contract)"""
    a, b = np.asarray(a, np.float16), np.asarray(b, np.float16)
    return bool(np.all((bits16(a) == bits16(b)) | (np.isnan(a) & np.isnan(b))))


def _codes_close(q_gpu, q_ref, exact_product, name, allow_rows=None):
    d = np.abs(q_gpu.astype(np.int32) - q_ref.astype(np.int32))
    assert d.max() <= 1, f"{name}: int8 differs by more than 1 LSB"
    frac = exact_product - np.floor(exact_product)
    ok = np.abs(frac - 0.5) < 2e-3
    if allow_rows is not None:
        ok = ok | allow_rows
    bad = (d > 0) & ~ok
    assert not np.any(bad), f"{name}: mismatch away from a rounding boundary at {np.argwhere(bad)[:5].tolist()}"
    assert (d > 0).mean() < 2e-3, f"{name}: too many boundary flips ({(d > 0).mean():.2e})"


def _outliers_exact(q, where, name):
    for label, (row, i) in where.items():
        if i is not None:
            want = 127 if "+" in label else -127
            assert int(q[row, i]) == want, f"{name}: outlier of row '{label}' quantised to {int(q[row, i])}, want {want}"


def _ref(name):
    from tests import refmods

    return refmods.load(name)


# ------------------------------------------------------------------------------------------------------------------------------------
# one case: build the inputs, and a `launch` that runs only the op under test (for the kernel-name check)
# ------------------------------------------------------------------------------------------------------------------------------------
class _Case:
    def __init__(self, op, p, dev):
        self.op, self.p, self.dev = op, p, dev
        rng = np.random.default_rng(zlib.crc32(_case_id((op, p)).encode()))
        self.rng = rng
        if op == "silu":
            self.M = _silu_tokens(p["target"], p["d"], p["prefer"])
            d = p["d"]
            g = rng.standard_normal((self.M, d)) * 2
            u = rng.standard_normal((self.M, d)) * 2
            self.where = {}
            for k, (name, (ge, ue, i)) in enumerate(_silu_edges(rng, d).items()):
                g[2 * k + 1], u[2 * k + 1] = ge, ue
                self.where[name] = (2 * k + 1, i)
            self.x = np.concatenate([g, u], axis=1).astype(np.float16)
        elif op == "dequant_silu":
            self.M, d = 24, p["d"]
            self.acc = rng.integers(-3000, 3000, size=(self.M, 2 * d)).astype(np.int32)
            self.acc[1] = 0
            for row, v in ((3, 20000), (5, -20000)):  # one-hot: silu(20) * (+-40)
                i = int(rng.integers(d))
                self.acc[row, i], self.acc[row, d + i] = 20000, v
        else:
            H = p["H"]
            self.M = 32
            nonfinite = op in ("quant", "given_amax")
            if op == "quant" or op == "given_amax":
                base = rng.standard_normal((self.M, H)) * rng.uniform(0.1, 4, size=(self.M, 1))
            else:
                base = rng.standard_normal((self.M, H)) * 2 + rng.uniform(-1, 1, size=(self.M, 1))
            self.x = base.astype(np.float16)
            self.where = _mix(rng, self.x, _edge_rows(rng, H, nonfinite))
            self.gamma = (1 + 0.1 * rng.standard_normal(H)).astype(np.float16)
            if op == "add_norm":
                self.delta = rng.standard_normal((self.M, H)).astype(np.float16)
                for row, _ in self.where.values():
                    self.delta[row] = 0  # edge rows reach the norm unchanged
        self._alloc()

    def _alloc(self):
        dev, M = self.dev, self.M
        width = self.p["d"] if self.op in ("silu", "dequant_silu") else self.p["H"]
        self.q = torch.full((M, width), 99, dtype=torch.int8, device=dev)  # sentinel: a skipped store shows
        self.s = torch.full((M,), 7.0, dtype=torch.half, device=dev)
        self.m = torch.full((M,), 7.0, dtype=torch.half, device=dev) if self.p.get("with_sum", True) else None
        if self.op == "dequant_silu":
            self.acc_d = to_dev(self.acc, dev)
            self.so = torch.full((M,), 7.0, dtype=torch.float32, device=dev)
            self.tmp = torch.full((M, width), 7.0, dtype=torch.float32, device=dev)
            return
        self.x_d = to_dev(self.x, dev)
        if self.op in ("norm", "add_norm", "rms_norm"):
            self.g_d = to_dev(self.gamma, dev)
        if self.op == "add_norm":
            self.delta_d = to_dev(self.delta, dev)
            self.h = torch.full_like(self.x_d, 7.0)
        if self.op == "norm" and not self.p["per_token"]:
            self.s.fill_(31.75)  # static per-tensor scale (read)
        if self.op == "rms_norm":
            self.out = torch.full((M, self.p["H"]), 99, dtype=torch.int8, device=dev) if self.p["use_quant"] else torch.full_like(self.x_d, 7.0)
        if self.op == "given_amax":
            self.amax = torch.full((M,), 7.0, dtype=torch.float32, device=dev)

    def launch(self):
        from qserve_b200 import backend as ext

        op, p = self.op, self.p
        if op == "norm":
            if self.m is not None:
                ext.rms_norm_general_fuse_sum(self.q, self.x_d, self.g_d, self.m, self.s, EPS, True)
            else:
                ext.rms_norm_general(self.q, self.x_d, self.g_d, self.s, EPS, p["per_token"])
        elif op == "add_norm":
            ext.add_rms_norm_general(self.q, self.h, self.x_d, self.delta_d, self.g_d, self.m, self.s, EPS)
        elif op == "rms_norm":
            ext.rms_norm(self.out, self.x_d, self.g_d, EPS, p["use_quant"])
        elif op == "quant":
            if self.m is not None:
                ext.invoke_quant_fuse_sum(self.q, self.x_d, self.m, self.s)
            else:
                ext.invoke_quant(self.q, self.x_d, self.s)
        elif op == "given_amax":
            ext.row_absmax(self.amax, self.x_d)
            ext.invoke_quant_given_amax(self.q, self.x_d, self.amax, self.m, self.s)
        elif op == "silu":
            ext.silu_and_mul_quant(self.q, self.x_d, self.m, self.s)
        else:
            ext.invoke_dequant_silu_and_mul_quant(self.q, self.acc_d, 1e-3, 2e-3, self.so, self.tmp)


# ------------------------------------------------------------------------------------------------------------------------------------
# checks per op
# ------------------------------------------------------------------------------------------------------------------------------------
def _check_norm(c):
    from qserve_b200 import backend as ext

    H, M = c.p["H"], c.M
    q = np_of(c.q)
    if not c.p.get("per_token", True):
        q_o, y = ops.layernorm_general_quant_per_tensor(c.x, c.gamma, EPS, np.float16(31.75))
        d = np.abs(q.astype(np.int32) - q_o.astype(np.int32))
        assert d.max() <= 1
        sc = np.float32(31.75)
        near = np.zeros_like(d, dtype=bool)
        for f in (1 - 2e-6, 1 + 2e-6):
            near |= ops.cvt_rni_sat_s8((y * np.float32(f)).astype(np.float32).astype(np.float16).astype(np.float32) * sc) != q_o
        assert not np.any((d > 0) & ~near), "per-tensor codes differ where half(y) * scale is not at a rounding boundary"
        assert (d > 0).mean() < 2e-3
        assert np.all(np_of(c.s) == np.float16(31.75)), "the per-tensor scale is an input and must not be written"
        return
    hid = (c.x.astype(np.float32) + c.delta.astype(np.float32)).astype(np.float16) if c.op == "add_norm" else c.x
    q_o, s_o, sum_o, y = ops.layernorm_general_quant(hid, c.gamma, EPS, c.m is not None)
    ds = ulp16_diff(np_of(c.s), s_o)
    assert ds.max() <= 1
    amax = np.maximum(np.abs(y.astype(np.float16)).max(axis=1), np.float16(1e-6)).astype(np.float32)  # what 127/amax divides by
    # a row whose amax of half(y) moved by an ulp quantises with another 127/amax: there any code may move by one
    _codes_close(q, q_o, y.astype(np.float64) * (127.0 / amax.astype(np.float64))[:, None], f"{c.op} H={H}", (ds > 0)[:, None])
    _outliers_exact(q, c.where, c.op)
    for label in ("zero", "constant"):
        assert not np.any(q[c.where[label][0]]), f"{label} row: y = 0 must quantise to 0"
    if c.m is not None:
        got, want = np_of(c.m).astype(np.float32), sum_o.astype(np.float32)
        assert np.abs(got - want).max() <= 2e-3 * np.sqrt(H)
    if c.op == "add_norm":
        assert np.array_equal(bits16(np_of(c.h)), bits16(hid)), "hidden_out must be half(float(x) + float(delta))"
        q2, s2 = torch.full_like(c.q, 99), torch.full_like(c.s, 7.0)
        m2 = torch.full_like(c.m, 7.0) if c.m is not None else None
        if m2 is not None:
            ext.rms_norm_general_fuse_sum(q2, c.h, c.g_d, m2, s2, EPS, True)
        else:
            ext.rms_norm_general(q2, c.h, c.g_d, s2, EPS, True)
        torch.cuda.synchronize()
        assert torch.equal(q2, c.q) and torch.equal(s2, c.s) and (m2 is None or torch.equal(m2, c.m)), "fused add + norm != norm(x + delta)"


def _check_norm_live(c):
    ln = _ref("layernorm_ops")
    if ln is None or c.op != "norm" or c.m is None:
        return
    q0, s0, m0 = torch.empty_like(c.q), torch.empty_like(c.s), torch.empty_like(c.m)
    ln.rms_norm_general_fuse_sum(q0, c.x_d, c.g_d, m0, s0, EPS, True)
    torch.cuda.synchronize()
    rows = np.ones(c.M, bool)
    if c.p["H"] & (c.p["H"] - 1):
        # the reference divides by H with the fast-math reciprocal: its mean of a constant row can be off by an ulp, which leaves
        # y ~ 1e-5 instead of 0 and amax far above the clamp -- a reference artefact, not a contract
        rows[c.where["constant"][0]] = False
    dq = np.abs(np_of(q0).astype(np.int32) - np_of(c.q).astype(np.int32))[rows]
    assert dq.max() <= 1 and (dq > 0).mean() < 2e-3, "rms_norm_general_fuse_sum vs the live reference"
    assert ulp16_diff(np_of(c.s), np_of(s0))[rows].max() <= 1
    dm = np.abs(np_of(c.m).astype(np.float32) - np_of(m0).astype(np.float32))
    assert dm[rows].max() <= 2e-3 * np.sqrt(c.p["H"]), "row sum vs the live reference"


def _check_rms(c):
    if c.p["use_quant"]:
        want = ops.rms_norm(c.x, c.gamma, EPS, True)
        assert np.abs(np_of(c.out).astype(np.int32) - want.astype(np.int32)).max() <= 1
    else:
        want = ops.rms_norm(c.x, c.gamma, EPS)
        got = np_of(c.out)
        d = ulp16_diff(got, want)
        # half(x * rstd) * w rounds twice: an rstd that moved in its last bits (the fp32 sum of squares of a row with a +-65504
        # outlier drops the small squares: 5e-6 relative) can move the result by 2 ulps.  Bar: the output lies between the oracle's
        # outputs for rstd * (1 -+ 1e-5), and < 1 % of the elements differ from the oracle at all.
        key = lambda a: np.where(bits16(a).astype(np.int32) & 0x8000, -(bits16(a).astype(np.int32) & 0x7FFF), bits16(a).astype(np.int32) & 0x7FFF)
        lo, hi = (key(_rms_scaled(c.x, c.gamma, f)) for f in (1 - 1e-5, 1 + 1e-5))
        assert np.all((key(got) >= np.minimum(lo, hi)) & (key(got) <= np.maximum(lo, hi))), f"max {d.max()} ulp"
        assert (d > 0).mean() < 1e-2


def _rms_scaled(x, w, f):
    """ops.rms_norm with rstd scaled by f"""
    xf = x.astype(np.float32)
    var = (xf.astype(np.float64) ** 2).sum(axis=1).astype(np.float32)
    r = (1.0 / np.sqrt((var / np.float32(x.shape[1]) + np.float32(EPS)).astype(np.float64)) * f).astype(np.float32)
    xs = (xf * r[:, None]).astype(np.float32)
    return ops.f16(xs.astype(np.float16).astype(np.float64) * w.astype(np.float64)[None, :])


def _check_quant_nonfinite(q, s, m, where, name):
    """the reference's verdicts, spelled out: these rows are also covered by the bit-exact oracle comparison"""
    if m is not None:
        for label, want in (("inf", np.inf), ("two_inf", np.inf), ("inf_ninf", np.nan), ("nan", np.nan)):
            got = m[where[label][0]]
            assert (np.isnan(got) if np.isnan(want) else got == want), f"{name}: row sum of '{label}' row is {got}, want {want}"
    for label in ("inf", "two_inf", "inf_ninf"):
        row = where[label][0]
        assert s[row] == np.inf and not np.any(q[row]), f"{name}: '{label}' row: amax = inf gives scale inf and all codes 0"
    assert np.isfinite(s[where["nan"][0]]), f"{name}: amax must ignore NaN"


def _check_quant(c):
    q, s = np_of(c.q), np_of(c.s)
    m = np_of(c.m) if c.m is not None else None
    q_o, s_o, m_o = ops.quant_per_token(c.x, c.m is not None)
    assert np.array_equal(q, q_o), "codes must be bit-exact"
    assert _same16(s, s_o), "scales must be bit-exact"
    if m is not None:
        assert _same16(m, m_o), "row sums must be bit-exact (exact fixed-point sum; IEEE verdict for non-finite rows)"
    _outliers_exact(q, c.where, "invoke_quant")
    _check_quant_nonfinite(q, s, m, c.where, "invoke_quant")
    fk = _ref("fused_kernels")
    if fk is not None:  # live reference on the same rows
        q0, s0, m0 = torch.empty_like(c.q), torch.empty_like(c.s), torch.empty_like(c.s)
        fk.invoke_quant_fuse_sum(q0, c.x_d, m0, s0)
        torch.cuda.synchronize()
        assert np.abs(np_of(q0).astype(np.int32) - q.astype(np.int32)).max() <= 1
        assert _same16(np_of(s0), s), "scale vs the live reference"
        if m is not None:
            m0 = np_of(m0)
            assert np.array_equal(np.isnan(m0), np.isnan(m)), "NaN row sums where the reference has them"
            assert np.array_equal(np.where(np.isinf(m0), np.sign(m0), 0), np.where(np.isinf(m), np.sign(m), 0)), "inf row sums"
            fin = np.isfinite(m0)
            assert ulp16_diff(m[fin], m0[fin]).max() <= 1


def _check_given_amax(c):
    from qserve_b200 import backend as ext

    amax = np_of(c.amax)
    assert np.array_equal(amax.view(np.uint32), ops._absmax(c.x).view(np.uint32)), "row_absmax must be bit-exact (NaN ignored)"
    # with the row's own amax: bit-identical to invoke_quant[_fuse_sum]
    q1, s1 = torch.full_like(c.q, 99), torch.full_like(c.s, 7.0)
    m1 = torch.full_like(c.m, 7.0) if c.m is not None else None
    if m1 is not None:
        ext.invoke_quant_fuse_sum(q1, c.x_d, m1, s1)
    else:
        ext.invoke_quant(q1, c.x_d, s1)
    torch.cuda.synchronize()
    assert torch.equal(q1, c.q) and _same16(np_of(s1), np_of(c.s)) and (m1 is None or _same16(np_of(m1), np_of(c.m)))
    # with a larger amax, as another shard would supply: codes and scale follow it, the sum stays this row's own
    big = (np.maximum(np.nan_to_num(amax, posinf=0), 1.0) * c.rng.uniform(1.1, 3.0, c.M)).astype(np.float32)
    big[np.isinf(amax)] = np.inf
    c.amax.copy_(torch.from_numpy(big))
    ext.invoke_quant_given_amax(c.q, c.x_d, c.amax, c.m, c.s)
    torch.cuda.synchronize()
    q_o, s_o, m_o = ops.quant_given_amax(c.x, big, c.m is not None)
    assert np.array_equal(np_of(c.q), q_o) and _same16(np_of(c.s), s_o)
    if c.m is not None:
        assert _same16(np_of(c.m), m_o)
    _check_quant_nonfinite(np_of(c.q), np_of(c.s), np_of(c.m) if c.m is not None else None, c.where, "invoke_quant_given_amax")


def _check_silu(c):
    from qserve_b200 import backend as ext

    M, d = c.M, c.p["d"]
    a = torch.full((M, d), 7.0, dtype=torch.half, device=c.dev)
    ext.silu_and_mul(a, c.x_d)
    q1, s1 = torch.full_like(c.q, 99), torch.full_like(c.s, 7.0)
    m1 = torch.full_like(c.m, 7.0) if c.m is not None else None
    if m1 is not None:
        ext.invoke_quant_fuse_sum(q1, a, m1, s1)
    else:
        ext.invoke_quant(q1, a, s1)
    torch.cuda.synchronize()
    q, s = np_of(c.q), np_of(c.s)
    m = np_of(c.m) if c.m is not None else None
    # 1. the fused kernel is the unfused pair, bit for bit
    assert torch.equal(q1, c.q) and _same16(np_of(s1), s) and (m1 is None or _same16(np_of(m1), m)), "fused != silu_and_mul -> invoke_quant"
    # 2. ... and the quantiser oracle applied to the GPU activation, bit for bit
    a_g = np_of(a)
    q_g, s_g, m_g = ops.quant_per_token(a_g, m is not None)
    assert np.array_equal(q, q_g) and _same16(s, s_g) and (m is None or _same16(m, m_g))
    _check_quant_nonfinite(q, s, m, c.where, "silu_and_mul_quant")
    # 3. end to end against ops.quant_per_token(ops.silu_and_mul(x))
    with np.errstate(over="ignore", invalid="ignore"):
        a_o = ops.silu_and_mul(c.x)
    both_nan = np.isnan(a_g) & np.isnan(a_o)
    da = np.where(both_nan, 0, ulp16_diff(a_g, a_o))
    assert da.max() <= 2 and (da > 0).mean() < 1e-3, "silu_and_mul activation vs the oracle"
    q_o, s_o, _ = ops.quant_per_token(a_o, False)
    amax_g, amax_o = ops._absmax(a_g), ops._absmax(a_o)
    row_moved = amax_g != amax_o
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        prod = np.nan_to_num(a_o.astype(np.float64) * (127.0 / amax_o.astype(np.float64))[:, None])
    allow = (da > 0) | row_moved[:, None]
    dq = np.abs(q.astype(np.int32) - q_o.astype(np.int32))
    assert dq.max() <= 1
    frac = prod - np.floor(prod)
    assert not np.any((dq > 0) & ~(allow | (np.abs(frac - 0.5) < 2e-3))), "codes differ away from a rounding boundary"
    ds = ulp16_diff(s, s_o)
    assert not np.any(ds[~row_moved]), "scale must be bit-exact where the row's largest activation agrees"
    if row_moved.any():
        dmax = ulp16_diff(amax_g.astype(np.float16), amax_o.astype(np.float16))
        assert np.all(ds[row_moved] <= dmax[row_moved])
    _outliers_exact(q, c.where, "silu_and_mul_quant")
    # 4. the live reference: its silu_and_mul -> invoke_quant_fuse_sum on the same rows
    act, fk = _ref("activation_ops"), _ref("fused_kernels")
    if act is not None and fk is not None:
        a0 = torch.empty_like(a)
        act.silu_and_mul(a0, c.x_d)
        q0, s0, m0 = torch.empty_like(c.q), torch.empty_like(c.s), torch.empty_like(c.s)
        fk.invoke_quant_fuse_sum(q0, a0, m0, s0)
        torch.cuda.synchronize()
        a0 = np_of(a0)
        dr = np.where(np.isnan(a0) & np.isnan(a_g), 0, ulp16_diff(a_g, a0))
        assert dr.max() <= 2 and (dr > 0).mean() < 2e-3, "silu_and_mul vs the live reference"
        s0, m0 = np_of(s0), np_of(m0)
        assert np.array_equal(np.isinf(s0), np.isinf(s)), "inf scales where the reference has them"
        if m is not None:
            assert np.array_equal(np.isnan(m0), np.isnan(m)), "NaN row sums where the reference has them"
            assert np.array_equal(np.where(np.isinf(m0), np.sign(m0), 0), np.where(np.isinf(m), np.sign(m), 0)), "inf row sums"


def _check_dequant_silu(c):
    q_o, so_o, t_o = ops.dequant_silu_and_mul_quant_per_token(c.acc, 1e-3, 2e-3)
    t = np_of(c.tmp)
    tol = 8 * 2.0 ** -23
    assert np.all(np.abs(t - t_o) <= tol * np.abs(t_o) + 1e-30), "tmp vs the oracle (expf)"
    assert np.all(np.abs(np_of(c.so) - so_o) <= tol * so_o), "scale_out vs the oracle"
    assert np.abs(np_of(c.q).astype(np.int32) - q_o.astype(np.int32)).max() <= 1
    assert np_of(c.so)[1] == 0 and not np.any(np_of(c.q)[1]), "zero row"
    for row in (3, 5):
        assert np.abs(np_of(c.q)[row]).max() == 127, "one-hot row: the outlier's code is +-127"


CHECKS = {"norm": _check_norm, "add_norm": _check_norm, "rms_norm": _check_rms, "quant": _check_quant, "given_amax": _check_given_amax,
          "silu": _check_silu, "dequant_silu": _check_dequant_silu}


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_against_oracle(dev, case):
    op, p = case
    c = _Case(op, p, dev)
    _expected(op, p, c.M)  # the case reaches the branch it names
    with np.errstate(over="ignore", invalid="ignore"):
        c.launch()
        torch.cuda.synchronize()
        CHECKS[op](c)
        if op == "norm":
            _check_norm_live(c)


def _kernel_names(prof):
    names = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and not re.match(r"(?i)mem(cpy|set)", e.name):
            names.append(e.name)
    return names


def test_launched_kernel_names(dev):
    """every case launches exactly the kernel(s) the mirror of the host rules predicts -- so a change of a dispatch rule fails here
    instead of quietly moving what the oracle tests cover"""
    from torch.profiler import ProfilerActivity, profile

    rows, seen_any, wrong = [], False, []
    for op, p in CASES:
        c = _Case(op, p, dev)
        want, attr = _expected(op, p, c.M)
        c.launch()  # first launch outside the trace: module loading, smem attributes
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            c.launch()
            torch.cuda.synchronize()
        got = _kernel_names(prof)
        seen_any |= bool(got)
        ok = len(got) == len(want) and all(re.search(r"(?<![\w])" + re.escape(w) + r"(?![\w<])", g) for w, g in zip(want, got))
        rows.append(f"{_case_id((op, p)):55s} M={c.M:<4d} -> {', '.join(want)}{' (smem attribute)' if attr else ''}")
        if got and not ok:
            wrong.append(f"{_case_id((op, p))}: want {want}, launched {got}")
    if not seen_any:
        pytest.skip("torch.profiler recorded no CUDA kernel events")
    print("\n" + "\n".join(rows))
    assert not wrong, "\n".join(wrong)
