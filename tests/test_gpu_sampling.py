"""GPU: temperature / top-p / top-k sampling (qs_sample_rows) and sampled acceptance of draft trees (qs_tree_accept_sampling) against the
float64 oracle (oracle/sampling.py), with the oracle's own Philox draws.

Bar for a drawn token: the oracle's token, or one whose float64 CDF interval lies within delta = 4e-6 * S_kept of u * S_kept.  The kernels
compute the weights with fp32 expf (a few ulp: ~3e-7 relative) and sum them exactly in 64-bit fixed point after rounding each weight to
2^-41, so a CDF value is off by at most ~3e-7 S plus V * 2^-41 <= 1e-7 S; delta leaves an order of magnitude.  A top-p threshold whose
crossing lies within delta of a tie group's boundary, and an acceptance decision within delta of flipping, may go either way: such rows /
sequences are counted and must stay below 1 %.
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import sampling as osm

pytestmark = pytest.mark.gpu
DELTA = 4e-6
SEED = 0x9E3779B97F4A7C15


def _backend():
    from qserve_b200 import backend
    return backend


def _rows(rng, R, V):
    """fp16 rows of several kinds, cycled: normal at two scales, a few levels (heavy ties), -inf entries, one finite value, NaN."""
    x = np.empty((R, V), np.float16)
    for r in range(R):
        kind = r % 6
        if kind == 0:
            x[r] = rng.standard_normal(V) * 1.0
        elif kind == 1:
            x[r] = rng.standard_normal(V) * 4.0
        elif kind == 2:
            x[r] = rng.integers(-3, 4, V) * 1.25
        elif kind == 3:
            x[r] = rng.standard_normal(V) * 2.0
            x[r, rng.random(V) < 0.3] = -np.inf
        elif kind == 4:
            x[r] = -np.inf
            x[r, rng.integers(V)] = rng.standard_normal()
        else:
            x[r] = rng.standard_normal(V) * 2.0
            x[r, rng.integers(V, size=3)] = np.nan
    return x


def _grid(V):
    return list(itertools.product([0.0, 0.3, 0.7, 1.0, 1.5], [-1, 1, 2, 50, V, V + 5], [1.0, 0.95, 0.5, 1e-9]))


def _call(x, T, K, P, offsets, dev):
    be = _backend()
    t = lambda a, dt: torch.tensor(np.asarray(a), dtype=dt, device=dev)
    off = t(offsets, torch.int64)
    out = be.sample_rows(torch.from_numpy(x).to(dev), t(T, torch.float32), t(np.minimum(K, 2**31 - 1), torch.int32), t(P, torch.float32), SEED, off)
    torch.cuda.synchronize()
    return out.cpu().numpy(), off.cpu().numpy()


def _check_rows(x, T, K, P, offsets, got):
    want, ws, margins, u = osm.sample_rows(x, T, K, P, SEED, offsets)
    bad, ambiguous = [], 0
    for r in range(x.shape[0]):
        if got[r] == want[r]:
            continue
        greedy = osm.is_greedy(T[r], P[r]) or not (~np.isnan(x[r].astype(np.float32)) & (x[r] != -np.inf)).any()
        if not greedy and osm.cdf_ok(int(got[r]), ws[r], u[r], DELTA):
            continue
        if not greedy and margins[r] < DELTA:
            ambiguous += 1
            continue
        bad.append((r, int(got[r]), int(want[r]), T[r], K[r], P[r]))
    return bad, ambiguous


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. sample_rows against the oracle
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [64, 1024, 32000, 128256, 152064])
def test_sample_rows_matches_oracle(dev, V):
    rng = np.random.default_rng(V)
    grid = _grid(V)
    total, amb = 0, 0
    for rows in ([64] if V > 1024 else [1, 7, 64]):
        for start in range(0, len(grid), rows):
            params = [grid[(start + i) % len(grid)] for i in range(rows)]
            T, K, P = (np.array(a) for a in zip(*params))
            x = _rows(rng, rows, V)
            offsets = rng.integers(0, 1 << 40, rows)
            got, off_after = _call(x, T, K, P, offsets, dev)
            assert np.array_equal(off_after, offsets + 1)
            bad, a = _check_rows(x, T, K, P, offsets, got)
            assert not bad, bad[:5]
            total += rows
            amb += a
            if rows < 64:
                break
    assert amb < 0.01 * total, (amb, total)


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. greedy rows: bitwise argmax_rows; (1, 1, 1) samples a maximal logit
# ---------------------------------------------------------------------------------------------------------------------------------
def test_greedy_rows_are_argmax_rows(dev):
    be = _backend()
    rng = np.random.default_rng(2)
    R, V = 48, 4096
    x = (rng.integers(-2, 3, (R, V)) * 0.5).astype(np.float16)  # many tied maxima
    x[5, [7, 900]] = np.nan
    x[6] = np.nan
    x[7] = -np.inf
    xd = torch.from_numpy(x).to(dev)
    ref = be.argmax_rows(xd)
    off = torch.zeros(R, dtype=torch.int64, device=dev)
    for T, P in ((0.0, 1.0), (1.0, 1e-9), (0.0, 1e-9)):
        assert torch.equal(be.sample_rows(xd, T, 50, P, SEED, off), ref)
    tok = be.sample_rows(xd, 1.0, 1, 1.0, SEED, off)
    rowmax = torch.where(xd.isnan(), float("-inf"), xd.float()).amax(-1)
    ok = torch.gather(xd.float(), 1, tok[:, None])[:, 0] == rowmax
    assert ok[torch.arange(R, device=dev) != 6].all()  # row 6 is all NaN: the argmax_rows answer
    assert len(set(tok[8:].tolist())) > 1  # ties are sampled, not resolved to the first index
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. offsets: determinism, advance, CUDA-graph replays
# ---------------------------------------------------------------------------------------------------------------------------------
def test_offsets_determinism_and_graph_replay(dev):
    be = _backend()
    rng = np.random.default_rng(3)
    R, V = 64, 32000
    x = torch.from_numpy(_rows(rng, R, V)).to(dev)
    T = torch.full((R,), 0.8, device=dev)
    K = torch.full((R,), -1, dtype=torch.int32, device=dev)
    P = torch.full((R,), 0.95, device=dev)
    start = torch.arange(R, dtype=torch.int64, device=dev) * 1000
    off = start.clone()
    a = be.sample_rows(x, T, K, P, SEED, off).clone()
    off.copy_(start)
    b = be.sample_rows(x, T, K, P, SEED, off).clone()
    assert torch.equal(a, b)
    off.copy_(start)
    eager = [be.sample_rows(x, T, K, P, SEED, off).clone() for _ in range(3)]
    assert torch.equal(off, start + 3)
    assert not all(torch.equal(eager[0], e) for e in eager[1:])
    out = torch.empty(R, dtype=torch.int64, device=dev)
    off.copy_(start)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.sample_rows(x, T, K, P, SEED, off, out=out)  # warm-up
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.sample_rows(x, T, K, P, SEED, off, out=out)
    off.copy_(start)
    for e in eager:
        g.replay()
        assert torch.equal(out, e)
    assert torch.equal(off, start + 3)


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. distribution: G-test against the oracle's warped probabilities
# ---------------------------------------------------------------------------------------------------------------------------------
def _g_test(counts, probs):
    from scipy import stats

    counts, probs = np.asarray(counts, np.float64).ravel(), np.asarray(probs, np.float64).ravel()
    assert counts[probs == 0].sum() == 0, "a token of probability 0 was emitted"
    e = probs * counts.sum()
    big = e >= 5
    o = np.append(counts[big], counts[~big & (probs > 0)].sum())
    e = np.append(e[big], e[~big & (probs > 0)].sum())
    keep = e > 0
    o, e = o[keep], e[keep]
    g = 2 * np.sum(np.where(o > 0, o * np.log(np.where(o > 0, o, 1) / e), 0))
    return stats.chi2.sf(g, max(1, o.size - 1))


@pytest.mark.parametrize("setting", [(1.0, -1, 1.0), (0.7, 50, 0.9), (1.3, -1, 0.8)])
def test_sample_rows_distribution(dev, setting):
    be = _backend()
    rng = np.random.default_rng(4)
    V, R, calls = 1024, 1 << 16, 64
    row = (rng.standard_normal(V) * 2.5).astype(np.float16)
    w = osm.warp(row, *setting)[0]
    x = torch.from_numpy(row).to(dev)[None].expand(R, V).contiguous()
    off = torch.arange(R, dtype=torch.int64, device=dev) * 977
    counts = torch.zeros(V, dtype=torch.int64, device=dev)
    for _ in range(calls):
        counts += torch.bincount(be.sample_rows(x, *setting, SEED, off), minlength=V)
    assert _g_test(counts.cpu().numpy(), w / w.sum()) > 1e-6


# ---------------------------------------------------------------------------------------------------------------------------------
# 5-7. tree_accept_sampling
# ---------------------------------------------------------------------------------------------------------------------------------
def _parents(shape, n, rng):
    if shape == "chain":
        return [i - 1 for i in range(n)]
    if shape == "star":
        return [-1] + [0] * (n - 1)
    if shape == "binary":
        return [-1] + [(i - 1) // 2 for i in range(1, n)]
    if shape == "medusa":  # 3 candidates at depth 1, 3 below each of the first two, the rest below the first grandchild
        par = [-1, 0, 0, 0, 1, 1, 1, 2, 2, 2] + [4] * 6
        return par[:n]
    return [-1] + [int(rng.integers(0, i)) for i in range(1, n)]


def _mask(parents):
    m = [0] * len(parents)
    for i, p in enumerate(parents):
        if p >= 0:
            m[i] = m[p] | (1 << p)
    return np.array(m, np.int32)


def _tree_case(rng, B, n, V, shape, qmode, setting, logit_scale=2.0):
    """Drafts drawn on the host from q (Dirichlet, q = the warped target of the parent) or the parent's best tokens (one-hot q)."""
    logits = (rng.standard_normal((B, n, V)) * logit_scale).astype(np.float16)
    draft = np.zeros((B, n), np.int64)
    mask = np.zeros((B, n), np.int32)
    q = None if qmode == "none" else np.zeros((B, n, V), np.float32)
    for b in range(B):
        par = _parents(shape, n, rng)
        mask[b] = _mask(par)
        draft[b, 0] = rng.integers(V)
        for c in range(1, n):
            lp = logits[b, par[c]]
            if qmode == "none":
                rank = sum(1 for j in range(1, c) if par[j] == par[c])
                draft[b, c] = np.argsort(-lp.astype(np.float32), kind="stable")[rank]
                continue
            if qmode == "p":
                w = osm.warp(lp, *setting)[0]
                qc = w / w.sum()
            else:
                qc = rng.dirichlet(np.ones(V) * 0.3)
            q[b, c] = qc.astype(np.float32)
            qq = q[b, c].astype(np.float64)
            draft[b, c] = rng.choice(V, p=qq / qq.sum())
    if B and n > 3:
        draft[0, 3] = -1  # a padding node
    return draft, mask, logits, q


def _run_tree(dev, draft, mask, logits, q, setting, offsets):
    be = _backend()
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
    off = t(offsets, torch.int64)
    acc, path, bonus = be.tree_accept_sampling(t(draft, torch.int64), t(mask, torch.int32), t(logits, torch.float16), *setting, SEED, off,
                                               draft_probs=None if q is None else t(q, torch.float32))
    torch.cuda.synchronize()
    return acc.cpu().numpy(), path.cpu().numpy(), bonus.cpu().numpy(), off.cpu().numpy()


TREE_SETTINGS = [(1.0, -1, 1.0), (0.7, 50, 0.9), (1.0, 1, 1.0), (0.0, -1, 1.0)]


@pytest.mark.parametrize("shape", ["chain", "star", "binary", "medusa", "random"])
@pytest.mark.parametrize("qmode", ["none", "dirichlet", "p"])
def test_tree_accept_sampling_matches_oracle(dev, shape, qmode):
    rng = np.random.default_rng(hash((shape, qmode)) & 0xFFFF)
    B, n, V = 24, 16 if shape != "star" else 6, 512
    marked = total = 0
    for setting in TREE_SETTINGS:
        draft, mask, logits, q = _tree_case(rng, B, n, V, shape, qmode, setting)
        offsets = rng.integers(0, 1 << 33, B)
        acc, path, bonus, off = _run_tree(dev, draft, mask, logits, q, setting, offsets)
        assert np.array_equal(off, offsets + 1)
        w_acc, w_path, w_bonus, info = osm.tree_accept_sampling(draft, mask, logits, *setting, SEED, offsets, q)
        for b in range(B):
            total += 1
            same_path = acc[b] == w_acc[b] and np.array_equal(path[b], w_path[b])
            if same_path and (bonus[b] == w_bonus[b] or osm.cdf_ok(int(bonus[b]), info[b]["bonus_p"], info[b]["u0"], DELTA)):
                continue
            assert info[b]["margin"] < DELTA or info[b]["top_p_margin"] < DELTA, (setting, b, acc[b], w_acc[b], path[b], w_path[b], bonus[b], w_bonus[b])
            marked += 1
    assert marked < 0.01 * total, (marked, total)


def test_tree_first_child_accepted_when_q_is_the_target(dev):
    """q_c = the warped target of c's parent and p(d) > 0 for every draft: u q(d) < p(d) always holds, so the walk takes the first child."""
    rng = np.random.default_rng(6)
    B, n, V = 32, 16, 1024
    for shape in ("chain", "binary", "medusa", "random"):
        draft, mask, logits, q = _tree_case(rng, B, n, V, shape, "p", (1.0, -1, 1.0), logit_scale=0.5)
        acc, path, _, _ = _run_tree(dev, draft, mask, logits, q, (1.0, -1, 1.0), rng.integers(0, 1 << 20, B))
        for b in range(B):
            par = osm.parents_of(mask[b], n)
            cur, want = 0, [0]
            while True:
                kids = [c for c in range(1, n) if par[c] == cur and draft[b, c] >= 0]
                if not kids:
                    break
                cur = kids[0]
                want.append(cur)
            assert acc[b] == len(want) and list(path[b, : len(want)]) == want, (shape, b)


def test_tree_greedy_limit_is_tree_accept_greedy(dev):
    be = _backend()
    rng = np.random.default_rng(7)
    B, n, V = 64, 16, 4096
    for shape in ("chain", "star", "binary", "medusa", "random"):
        draft, mask, logits, q = _tree_case(rng, B, n, V, shape, "dirichlet", (1.0, -1, 1.0))
        logits[:, :, :8] = np.float16(3.0)  # tied maxima: first index wins, as in argmax_rows
        logits[1, 2, 5] = np.nan
        target = logits.astype(np.float32).argmax(-1)
        for b in range(B):  # make some drafts the target's choice so that paths get long
            for c in range(1, n):
                if rng.random() < 0.7:
                    draft[b, c] = target[b, osm.parents_of(mask[b], n)[c]]
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
        lg = t(logits, torch.float16)
        tgt = be.argmax_rows(lg.view(B * n, V)).view(B, n)
        want = [x.clone() for x in be.tree_accept_greedy(t(draft, torch.int64), t(mask, torch.int32), tgt)]
        for T, P in ((0.0, 1.0), (0.9, 1e-9)):
            got = be.tree_accept_sampling(t(draft, torch.int64), t(mask, torch.int32), lg, T, -1, P, SEED, torch.zeros(B, dtype=torch.int64, device=dev),
                                          draft_probs=t(q, torch.float32))
            assert all(torch.equal(a, b) for a, b in zip(got, want)), shape


def _first_tokens(acc, path, bonus, draft):
    B = acc.size
    b = np.arange(B)
    t1 = np.where(acc >= 2, draft[b, np.maximum(path[:, 1], 0)], bonus)
    return t1


@pytest.mark.parametrize("case", ["chain3", "iid_star4", "wor_star4", "onehot4"])
def test_tree_lossless_on_gpu(dev, case):
    rng = np.random.default_rng(8)
    B, V = 1 << 16, 64
    setting = (0.9, -1, 0.95)
    row0 = (rng.standard_normal(V) * 1.5).astype(np.float16)
    w0 = osm.warp(row0, *setting)[0]
    p1 = w0 / w0.sum()
    q1 = rng.dirichlet(np.ones(V) * 0.5)
    if case == "chain3":
        n = 4
        cond = (rng.standard_normal((V, V)) * 1.5).astype(np.float16)  # target logits after token t
        p2 = np.array([osm.warp(r, *setting)[0] for r in cond])
        p2 /= p2.sum(1, keepdims=True)
        q2 = rng.dirichlet(np.ones(V) * 0.5, size=V)
        d1 = rng.choice(V, size=B, p=q1)
        u = rng.random(B)
        cdf2 = np.cumsum(q2, 1)
        d2 = np.minimum((cdf2[d1] < u[:, None]).sum(1), V - 1)
        d3 = rng.integers(V, size=B)
        draft = np.stack([np.zeros(B, np.int64), d1, d2, d3], 1)
        mask = np.tile(_mask([-1, 0, 1, 2]), (B, 1))
        logits = np.empty((B, n, V), np.float16)
        logits[:, 0] = row0
        logits[:, 1] = cond[d1]
        logits[:, 2:] = (rng.standard_normal((B, 2, V)) * 1.5).astype(np.float16)
        q = np.zeros((B, n, V), np.float32)
        q[:, 1] = q1
        q[:, 2] = q2[d1]
        q[:, 3] = 1.0 / V
    else:
        k, n = 4, 5
        mask = np.tile(_mask([-1, 0, 0, 0, 0]), (B, 1))
        logits = np.broadcast_to(row0, (B, n, V)).copy()
        q = np.zeros((B, n, V), np.float32) if case != "onehot4" else None
        draft = np.zeros((B, n), np.int64)
        if case == "iid_star4":
            draft[:, 1:] = rng.choice(V, size=(B, k), p=q1)
            q[:, 1:] = q1
        elif case == "wor_star4":
            g = rng.gumbel(size=(B, V)) + np.log(q1)
            order = np.argsort(-g, 1)[:, :k]  # Gumbel top-k: k draws without replacement from q1
            draft[:, 1:] = order
            rem = np.broadcast_to(q1, (B, V)).copy()
            for j in range(k):
                q[:, 1 + j] = rem / rem.sum(1, keepdims=True)
                rem[np.arange(B), order[:, j]] = 0
        else:
            draft[:, 1:] = np.argsort(-p1)[:k]
    acc, path, bonus, _ = _run_tree(dev, draft, mask, logits, q, setting, np.arange(B) * 3 + 1)
    t1 = _first_tokens(acc, path, bonus, draft)
    assert _g_test(np.bincount(t1, minlength=V), p1) > 1e-6
    if case == "chain3":
        t2 = np.where(acc >= 3, draft[np.arange(B), 2], bonus)
        nxt = acc == 1  # node 1 rejected: the second token comes from the next step, drawn from p2(. | t1)
        cdf = np.cumsum(p2[t1[nxt]], 1)
        t2[nxt] = np.minimum((cdf < rng.random(nxt.sum())[:, None]).sum(1), V - 1)
        joint = np.bincount(t1 * V + t2, minlength=V * V)
        assert _g_test(joint, (p1[:, None] * p2).ravel()) > 1e-6


# ---------------------------------------------------------------------------------------------------------------------------------
# 8. the decode runner
# ---------------------------------------------------------------------------------------------------------------------------------
def test_runner_sampled_step_and_sampled_tree_graph(dev):
    from qserve_b200.decode import DecodeRunner
    B, ctx, n = 6, 130, 5
    a = DecodeRunner("tiny", "w4a8kv4", batch=B, ctx=ctx, device=dev, seed=5)
    b = DecodeRunner("tiny", "w4a8kv4", batch=B, ctx=ctx, device=dev, seed=5)
    V = a.cfg.vocab
    a.tokens_in.copy_(torch.arange(B, device=dev) * 7 % V)
    b.tokens_in.copy_(a.tokens_in)
    b.s_temperature.fill_(0.0)
    a.capture()
    b.capture(sample=True)
    a.step(); b.step()
    torch.cuda.synchronize()
    assert torch.equal(a.tokens_out, b.tokens_out)
    b.s_temperature.fill_(1.0); b.s_top_k.fill_(-1)
    o0 = b.s_offsets.clone()
    for _ in range(3):
        b.step()
    torch.cuda.synchronize()
    assert torch.equal(b.s_offsets, o0 + 3)
    # the sampled tree graph at T = 0 is the greedy tree graph: outputs and pages
    g = DecodeRunner("tiny", "w4a8kv4", batch=B, ctx=ctx, device=dev, seed=9, verify_len=n)
    s = DecodeRunner("tiny", "w4a8kv4", batch=B, ctx=ctx, device=dev, seed=9, verify_len=n)
    s.s_temperature.fill_(0.0)
    parents = [-1, 0, 0, 1, 3]
    mask = torch.tensor(_mask(parents), dtype=torch.int32, device=dev).repeat(B, 1)
    with torch.no_grad():
        root = torch.arange(B, device=dev) * 13 % V
        tgt = g.verify_forward(torch.stack([root] * n, 1), tree_mask=mask)
    toks = torch.stack([root, tgt[:, 0], (tgt[:, 0] + 1) % V, torch.zeros_like(root), torch.zeros_like(root)], 1)
    for r in (g, s):
        r.v_tokens_in[:, :n].copy_(toks)
        r.v_tree_mask[:, :n].copy_(mask)
    g.capture_verify(n, tree=True)
    s.capture_verify(n, tree=True, sampled=True, draft_probs=True)
    for r, kw in ((g, {}), (s, {"sampled": True, "draft_probs": True})):
        r.v_accept_len.zero_(); r.v_path.zero_(); r.v_bonus.zero_()
        r.verify_step(n, tree=True, **kw)
    torch.cuda.synchronize()
    assert torch.equal(g.v_accept_len, s.v_accept_len) and torch.equal(g.v_path, s.v_path) and torch.equal(g.v_bonus, s.v_bonus)
    assert (g.v_accept_len >= 2).all()
    assert all(torch.equal(x, y) for x, y in zip(g.kpools + g.vpools, s.kpools + s.vpools))
    s.s_temperature.fill_(1.0)
    o0 = s.s_offsets.clone()
    s.verify_step(n, tree=True, sampled=True, draft_probs=True)
    s.verify_step(n, tree=True, sampled=True, draft_probs=True)
    torch.cuda.synchronize()
    assert torch.equal(s.s_offsets, o0 + 2)


# ---------------------------------------------------------------------------------------------------------------------------------
# 9. full size, determinism, argument errors
# ---------------------------------------------------------------------------------------------------------------------------------
def test_full_size_determinism(dev):
    be = _backend()
    B, n, V = 64, 16, 128256
    gen = torch.Generator(device=dev).manual_seed(11)
    logits = (torch.randn((B, n, V), device=dev, generator=gen) * 3).half()
    draft = torch.randint(0, V, (B, n), device=dev, generator=gen)
    draft[:, 1] = logits[:, 0].float().argmax(-1)
    mask = torch.tensor(_mask(_parents("medusa", n, None)), dtype=torch.int32, device=dev).repeat(B, 1)
    q = torch.softmax(torch.randn((B, n, V), device=dev, generator=gen), -1)
    # a small vocabulary first: the full-size calls below need more dynamic shared memory (6 B per logit of a CTA's slice, 94 KB here) than
    # the kernel's limit set for this one, so the library must raise the limit again
    small = torch.zeros((B, n, 512), dtype=torch.float16, device=dev)
    be.tree_accept_sampling(draft % 512, mask, small, 1.0, -1, 1.0, SEED, torch.zeros(B, dtype=torch.int64, device=dev))
    for setting in ((0.7, 50, 0.9), (0.8, -1, 0.95), (1.0, -1, 1.0)):
        rows, res = [], []
        for _ in range(3):
            off = torch.arange(B, dtype=torch.int64, device=dev)
            rows.append(be.sample_rows(logits[:, 0].contiguous(), *setting, SEED, off).clone())
            off = torch.arange(B, dtype=torch.int64, device=dev)
            res.append([x.clone() for x in be.tree_accept_sampling(draft, mask, logits, *setting, SEED, off, draft_probs=q)])
        assert all(torch.equal(rows[0], r) for r in rows[1:])
        assert all(all(torch.equal(x, y) for x, y in zip(res[0], r)) for r in res[1:])
    torch.cuda.synchronize()


def test_argument_errors(dev):
    be = _backend()
    x = torch.zeros((4, 64), dtype=torch.float16, device=dev)
    off = torch.zeros(4, dtype=torch.int64, device=dev)

    def bad(fn, *a, **k):
        with pytest.raises(RuntimeError):
            fn(*a, **k)

    be.sample_rows(x, 1.0, -1, 1.0, 0, off)  # valid
    bad(be.sample_rows, x.float(), 1.0, -1, 1.0, 0, off)
    bad(be.sample_rows, torch.zeros((4, 60), dtype=torch.float16, device=dev), 1.0, -1, 1.0, 0, off)
    bad(be.sample_rows, torch.zeros((1, 196616), dtype=torch.float16, device=dev), 1.0, -1, 1.0, 0, off[:1])
    bad(be.sample_rows, x, 1.0, 0, 1.0, 0, off)
    bad(be.sample_rows, x, 1.0, -2, 1.0, 0, off)
    bad(be.sample_rows, x, 1.0, -1, 0.0, 0, off)
    bad(be.sample_rows, x, 1.0, -1, 1.5, 0, off)
    bad(be.sample_rows, x, -0.5, -1, 1.0, 0, off)
    bad(be.sample_rows, x, 1.0, -1, 1.0, 0, off.int())
    bad(be.sample_rows, x, 1.0, -1, 1.0, 0, off[:3])
    bad(be.sample_rows, x, torch.ones(4, dtype=torch.float64, device=dev), -1, 1.0, 0, off)
    bad(be.sample_rows, x, 1.0, -1, 1.0, -1, off)
    d = torch.zeros((4, 5), dtype=torch.int64, device=dev)
    m = torch.zeros((4, 5), dtype=torch.int32, device=dev)
    lg = torch.zeros((4, 5, 64), dtype=torch.float16, device=dev)
    be.tree_accept_sampling(d, m, lg, 1.0, -1, 1.0, 0, off)  # valid
    bad(be.tree_accept_sampling, d.int(), m, lg, 1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m.long(), lg, 1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg.float(), 1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg[:, :4].contiguous(), 1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, torch.zeros((4, 5, 60), dtype=torch.float16, device=dev), 1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg, 1.0, 0, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg, 1.0, -1, 0.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg, -1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg, 1.0, -1, 1.0, 0, off, draft_probs=torch.zeros((4, 5, 64), dtype=torch.float16, device=dev))
    bad(be.tree_accept_sampling, d, m, lg, 1.0, -1, 1.0, 0, off, draft_probs=torch.zeros((4, 5, 32), device=dev))
    z17 = dict(dtype=torch.int64, device=dev)
    bad(be.tree_accept_sampling, torch.zeros((4, 17), **z17), torch.zeros((4, 17), dtype=torch.int32, device=dev),
        torch.zeros((4, 17, 64), dtype=torch.float16, device=dev), 1.0, -1, 1.0, 0, off)
    bad(be.tree_accept_sampling, d, m, lg, 1.0, -1, 1.0, 0, off, accept_len=torch.zeros(3, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
