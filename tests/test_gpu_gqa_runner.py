"""GPU: the decode runner at a GQA group of 7 (Qwen2.5-7B at TP = 2 has 14 query / 2 KV heads).

The attention kernels at non-power-of-two groups are pinned by test_gpu_attention_gqa.py; these tests run them through the runner's own
plumbing (buffer and plan sizing for Hq = 14, captured graphs, the verify, fork-group and chunked-prompt routes) on `tiny-g7`, a 2-layer
model registered here only: 14 heads / 2 KV heads of 128, hidden 1792, intermediate 2048, vocab 1024.  The step equivalences are the ones
the suite holds the tiny model (G = 2) to, with the same bars:
  * the fused step gives `_forward_reference`'s greedy tokens, and its graph replay gives the eager bits (test_gpu_refmodel.py);
  * chain and tree verify rows equal sequential decode steps (test_gpu_multi_token_attention.py, test_gpu_tree_verify.py);
  * shared_prefix=True equals the plain route (test_gpu_shared_prefix_runner.py);
  * a chunked prompt equals a whole prompt (test_gpu_prefill_runner.py).
"""
import pytest
import torch

from tests.test_gpu_prefill_runner import _prompts, _slots

pytestmark = pytest.mark.gpu
MODEL = "tiny-g7"


@pytest.fixture(autouse=True)
def tiny_g7(monkeypatch):
    from qserve_b200 import decode, modelcfg
    monkeypatch.setitem(modelcfg.MODELS, MODEL, modelcfg.ModelConfig("tiny-g7", 1792, 2048, 14, 2, 2, 1024, 10000.0))
    monkeypatch.setattr(decode, "SHARED_PREFIX_MIN_PAGES", 1)  # route the short prompts below through shared_prefix_decode_attention


def _runner(dev, **kw):
    from qserve_b200.decode import DecodeRunner
    run = DecodeRunner(MODEL, **kw, device=dev)
    assert (run.Hq, run.Hkv) == (14, 2)
    return run


def _snap(run):
    return [(k.clone(), v.clone()) for k, v in zip(run.kpools, run.vpools)]


def _restore(run, snap):
    for (k, v), (k0, v0) in zip(zip(run.kpools, run.vpools), snap):
        k.copy_(k0)
        v.copy_(v0)


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. the fused step: the reference op sequence's greedy tokens; graph replay = eager
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
@pytest.mark.parametrize("ctx", [150, 700])  # 700: the decode attention plans context splits
def test_fused_step_gives_the_reference_greedy_tokens(dev, precision, ctx):
    run = _runner(dev, precision=precision, batch=6, ctx=ctx, seed=5, fused=False)
    tokens = torch.randint(0, run.cfg.vocab, (run.batch,), generator=torch.Generator().manual_seed(5)).to(dev)
    snap = _snap(run)
    with torch.no_grad():
        logits_ref = run._forward_reference(tokens, return_logits=True).clone()
        _restore(run, snap)
        run.fused = True
        tok = run.forward(tokens).clone()
        logits = run.last_logits.clone()
        pages = _snap(run)
    torch.cuda.synchronize()
    assert torch.isfinite(logits_ref.float()).all()
    assert torch.equal(tok, torch.argmax(logits_ref, dim=-1))
    _restore(run, snap)
    run.capture()
    _restore(run, snap)
    run.tokens_in.copy_(tokens)
    run.step()
    torch.cuda.synchronize()
    assert torch.equal(run.tokens_out, tok) and torch.equal(run.last_logits, logits)
    assert all(torch.equal(k, k0) and torch.equal(v, v0) for (k, v), (k0, v0) in zip(zip(run.kpools, run.vpools), pages))


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. chain and tree verify against sequential decode steps
# ---------------------------------------------------------------------------------------------------------------------------------
def _sequential(run, tokens, ctx):
    """Decode steps of tokens [B, k] at positions ctx .. ctx + k - 1 -> logits [B, k, vocab] (float)."""
    out = []
    for i in range(tokens.size(1)):
        run.context_lens.fill_(ctx + 1 + i)
        run.max_seq_len = ctx + 1 + i
        out.append(run._forward_fused(tokens[:, i].contiguous(), return_logits=True).float())
    return torch.stack(out, dim=1)


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
@pytest.mark.parametrize("n", [1, 3, 5])  # 7, 21 and 35 columns per KV head: one n8 tile, two and three column parts
def test_chain_verify_equals_sequential_decode(dev, precision, n):
    B, ctx = 5, 130
    seq = _runner(dev, precision=precision, batch=B, ctx=ctx, seed=3, verify_len=n)
    ver = _runner(dev, precision=precision, batch=B, ctx=ctx, seed=3, verify_len=n)
    tokens = (torch.arange(B * n, device=dev).view(B, n) * 37) % seq.cfg.vocab
    with torch.no_grad():
        want = _sequential(seq, tokens, ctx)
        got = ver.verify_forward(tokens, return_logits=True).float()
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert float((got - want).abs().max()) <= 1e-2 * float(want.abs().max())
    assert torch.equal(seq.kpools[0], ver.kpools[0]) and torch.equal(seq.vpools[0], ver.vpools[0])  # layer 0: the same bytes appended
    with torch.no_grad():
        eager = ver.verify_forward(tokens).clone()
    ver.v_tokens_in.copy_(tokens)
    ver.capture_verify(n)
    ver.verify_step(n)
    torch.cuda.synchronize()
    assert torch.equal(ver.v_tokens_out, eager)
    assert torch.equal(ver.last_verify_logits.float(), got)


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
def test_tree_verify_equals_sequential_decode(dev, precision):
    """Six nodes (42 columns per KV head, three column parts) on two branches, 0 -> 2 -> 3 -> 5 and 0 -> 1 -> 4: every node's logits equal
    the decode step of its token after its root path's tokens."""
    from tests.test_gpu_tree_verify import mask_of
    B, ctx, n = 5, 130, 6
    parents = [-1, 0, 0, 2, 1, 3]
    tre = _runner(dev, precision=precision, batch=B, ctx=ctx, seed=3, verify_len=n)
    tokens = (torch.arange(B * n, device=dev).view(B, n) * 53 + 7) % tre.cfg.vocab
    mask = torch.tensor(mask_of(parents), dtype=torch.int32, device=dev).repeat(B, 1)
    with torch.no_grad():
        got = tre.verify_forward(tokens, return_logits=True, tree_mask=mask).float()
        want = torch.empty_like(got)
        for path in ([0, 2, 3, 5], [0, 1, 4]):
            seq = _runner(dev, precision=precision, batch=B, ctx=ctx, seed=3, verify_len=n)
            want[:, path] = _sequential(seq, tokens[:, path], ctx)
            del seq
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert float((got - want).abs().max()) <= 1e-2 * float(want.abs().max())


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. shared_prefix=True against the plain route
# ---------------------------------------------------------------------------------------------------------------------------------
def test_shared_prefix_equals_the_plain_route(dev):
    """Groups of 4 and 3 rows (28 and 21 columns of (member, head) per KV head).  Children follow their parent bit for bit; against the
    runner without the flag, the first step's logits agree to the bar of test_gpu_shared_prefix_runner.py (the attention differs only in
    its fp32 summation order) and layer-0 pages are byte-identical."""
    B, CTX = 8, 200
    lens = [193, 150, 1, 1, 1, 130, 1, 1]
    with torch.no_grad():
        runs = [_runner(dev, precision="w4a8kv4", batch=B, ctx=CTX, seed=3, prompt_tokens=B * CTX, max_new_tokens=8, generate=True,
                        shared_prefix=f) for f in (False, True)]
        logits, pages = [], []
        for run in runs:
            prompts, lens_d = _prompts(dev, lens, CTX, seed=13)
            run.prefill(prompts, lens_d)
            run.fork(0, [2, 3, 4])
            run.fork(5, [6, 7])
            run.generate_forward(1)
            logits.append(run.last_logits.float().clone())
            pages.append((run.kpools[0].clone(), run.vpools[0].clone()))
        assert runs[1].sp_groups == [((0, 2, 3, 4), 3), ((5, 6, 7), 2)]
    a, b = logits
    assert torch.isfinite(b).all()
    for c in (2, 3, 4):
        assert torch.equal(b[c], b[0]), f"child {c}: logits differ from the parent's"
    for c in (6, 7):
        assert torch.equal(b[c], b[5]), f"child {c}: logits differ from the parent's"
    assert torch.equal(a[1], b[1]), "a row outside every group changed"
    tol = 5e-2 * max(1.0, a.abs().max().item())
    assert (a - b).abs().max().item() <= tol, (a - b).abs().max().item()
    assert torch.equal(pages[0][0], pages[1][0]) and torch.equal(pages[0][1], pages[1][1]), "layer-0 pages differ"


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. a chunked prompt against a whole prompt
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [16, 64, 100])
def test_chunked_prompt_equals_whole_prompt(dev, chunk):
    """Layer 0 sees the same K / V whole or in pieces, and the chunked append promises the whole append's bytes; deeper layers read the
    earlier pieces back quantised, so the logits agree exactly for rows whose prompt fits one piece and to a cosine of 0.99 for the
    others (the bar of test_gpu_prefill_runner.py::test_chunked_prefill_matches_chunked_sequence)."""
    B, CTX = 5, 130
    LENS = [1, 63, 64, 65, 130]
    with torch.no_grad():
        run, whole = (_runner(dev, precision="w4a8kv4", batch=B, ctx=CTX, seed=3, prompt_tokens=512) for _ in range(2))
        prompts, lens = _prompts(dev, LENS, CTX)
        run.prefill(prompts, lens, chunk=chunk)
        whole.prefill(prompts, lens)
    torch.cuda.synchronize()
    for b, n in enumerate(LENS):
        assert torch.equal(_slots(run, b, n, [0]), _slots(whole, b, n, [0])), f"row {b}: layer-0 pages differ from the whole prompt's"
    a, w = run.last_logits.float(), whole.last_logits.float()
    assert torch.isfinite(a).all()
    cos = torch.nn.functional.cosine_similarity(a, w, dim=-1)
    for b, n in enumerate(LENS):
        assert torch.equal(a[b], w[b]) if n <= chunk else cos[b].item() >= 0.99, (b, cos)
