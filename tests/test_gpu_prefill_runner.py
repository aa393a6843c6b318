"""GPU: the decode runner's prompt step (DecodeRunner.prefill) and copy-on-write fork (DecodeRunner.fork, qs_kv_cache_fork).

The yardstick of the prompt step is a composition in this file of the unfused drop-in calls in the reference's prompt order
(llama_w4a8_unpad.py:186-242, 330-361) over a second runner built from the same seed, so with the same weights and pages.  The prompt step
must reproduce it bit for bit: the last positions' hidden rows, the logits, and every byte of every row's pages below its prompt length."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

B, CTX = 5, 130
LENS = [1, 63, 64, 65, 130]


def _runner(dev, precision="w4a8kv4", **kw):
    from qserve_b200.decode import DecodeRunner

    kw.setdefault("batch", B)
    kw.setdefault("ctx", CTX)
    return DecodeRunner("tiny", precision, device=dev, seed=3, **kw)


def _prompts(dev, lens, width, seed=5, vocab=1024):
    g = torch.Generator(device=dev).manual_seed(seed)
    p = torch.randint(0, vocab, (len(lens), width), device=dev, generator=g)
    return p, torch.tensor(lens, dtype=torch.int32, device=dev)


def _slots(run, b, n, layers=None):
    """The bytes of slots 0 .. n - 1 of row b's own pages (codes, scales, zeros; K and V), layer by layer."""
    kRow, cb = 128 * run.kv_bits // 8, 64 * run.size_per_token
    out = []
    for li in range(run.L) if layers is None else layers:
        for pool in (run.kpools[li], run.vpools[li]):
            for j in range((n + 63) // 64):
                s = min(64, n - 64 * j)
                page = pool[b * run.blocks_per_seq + j]
                out += [page[:cb].view(run.Hkv, 64, kRow)[:, :s].flatten(), page[cb:].view(2, run.Hkv, 128)[:, :, : 2 * s].flatten()]
    return torch.cat(out)


def _compose(run, prompts, lens_h, chunk=None):
    """The reference's prompt op sequence with the unfused drop-in calls, over run's weights and pages; piece by piece for chunk=C
    (apply_bias_rope_update_kv_cache_at at the cached length, prefix_prefill_attention).  Returns the final hidden state of every prompt
    position [sum(lens), H], in prompt order."""
    import qserve_backend as qb
    from qserve_b200 import backend
    from qserve_b200.decode import prompt_pieces

    cfg, dev = run.cfg, run.dev
    D, int4, maxpos = cfg.head_dim, run.kv_bits == 4, min(8192, cfg.max_pos)
    per_row = [[] for _ in lens_h]
    for start, c in prompt_pieces(lens_h, run.ctx, 1 << 30, chunk):
        T, maxc = sum(c), max(c)
        cu_h = np.concatenate([[0], np.cumsum(c)]).astype(np.int32)
        cu, clens = torch.from_numpy(cu_h).to(dev), torch.tensor(c, dtype=torch.int32, device=dev)
        pad = backend.compute_padding_offsets(cu, maxc, T)
        tokens = torch.cat([prompts[b, start:start + c[b]] for b in range(len(c))])
        prefix = torch.tensor([min(n, start) for n in lens_h], dtype=torch.int32, device=dev)
        hidden = run.embed[tokens]
        W = run.q_size + 2 * run.kv_size
        qkv = torch.empty((T, W), dtype=torch.half, device=dev)
        out = torch.empty((T, cfg.hidden), dtype=torch.half, device=dev)
        gate_up = torch.empty((T, 2 * run.Iloc), dtype=torch.half, device=dev)
        act = torch.empty((T, run.Iloc), dtype=torch.half, device=dev)
        qh = torch.empty((T, cfg.hidden), dtype=torch.int8, device=dev)
        qa = torch.empty((T, run.q_size), dtype=torch.int8, device=dev)
        qm = torch.empty((T, run.Iloc), dtype=torch.int8, device=dev)
        sc, sm = torch.empty(T, dtype=torch.half, device=dev), torch.empty(T, dtype=torch.half, device=dev)

        def norm_quant(x, g):
            if run.act_sum:
                qb.layernorm_ops.rms_norm_general_fuse_sum(qh, x, g, sm, sc, cfg.eps, True)
            else:
                qb.layernorm_ops.rms_norm_general(qh, x, g, sc, cfg.eps, True)

        def quant(o, x):
            if run.act_sum:
                qb.fused_kernels.invoke_quant_fuse_sum(o, x, sm, sc)
            else:
                qb.fused_kernels.invoke_quant(o, x, sc)

        for li, ly in enumerate(run.layers):
            table = run.block_tables[li]
            residual = hidden
            norm_quant(hidden, ly["ln1"])
            ly["qkv"](qh, sc, sm, qkv)
            q, k, v = run._heads(qkv)
            if chunk is None:
                qb.fused_attention.apply_bias_rope_update_kv_cache(qkv, clens, pad, table, run.Hq, run.Hkv, maxc, 64, run.size_per_token, D,
                                                                   cfg.rope_theta, maxpos, True, int4, True)
                attn = backend.flash_attn_varlen_func(q, k, v, cu_seqlens_q=cu, cu_seqlens_k=cu, max_seqlen_q=maxc, max_seqlen_k=maxc,
                                                      dropout_p=0.0, causal=True)
            else:
                backend.apply_bias_rope_update_kv_cache_at(qkv, clens, pad, prefix, table, run.Hq, run.Hkv, maxc, 64, run.size_per_token, D,
                                                           cfg.rope_theta, maxpos, True, int4, True)
                attn = backend.prefix_prefill_attention(q, k, v, cu, maxc, prefix, start, table, 64, run.size_per_token, int4)
            quant(qa, attn.reshape(T, -1))
            ly["o"](qa, sc, sm, out)
            hidden = residual + out
            residual = hidden
            norm_quant(hidden, ly["ln2"])
            ly["gate_up"](qh, sc, sm, gate_up)
            qb.activation_ops.silu_and_mul(act, gate_up)
            quant(qm, act)
            ly["down"](qm, sc, sm, out)
            hidden = residual + out
        for b in range(len(c)):
            per_row[b].append(hidden[cu_h[b]:cu_h[b + 1]])
    return torch.cat([torch.cat(r) for r in per_row])


def _last(hidden, lens_h):
    return hidden[torch.tensor(np.cumsum(lens_h) - 1, device=hidden.device)]


def _norm(run, x):
    import qserve_backend as qb

    out = torch.empty_like(x)
    qb.layernorm_ops.rms_norm(out, x, run.norm_w, run.cfg.eps, False)
    return out


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv4-g128", "w8a8kv8", "w4a8kv8"])
def test_prefill_matches_reference_sequence(dev, precision):
    with torch.no_grad():
        run, ref = _runner(dev, precision, prompt_tokens=512), _runner(dev, precision)
        prompts, lens = _prompts(dev, LENS, CTX + 3)
        tok = run.prefill(prompts, lens)
        hidden = _compose(ref, prompts, LENS)
        last = _last(hidden, LENS)
        assert torch.equal(_norm(run, run.last_prompt_hidden), _norm(ref, last))
        assert torch.equal(run.last_logits, ref._logits(last))
        assert torch.equal(tok, run.last_logits.float().argmax(-1))
        for b, n in enumerate(LENS):
            assert torch.equal(_slots(run, b, n), _slots(ref, b, n)), f"row {b}: pages differ"


@pytest.mark.parametrize("chunk", [1, 16, 64, 100])
def test_chunked_prefill_matches_chunked_sequence(dev, chunk):
    with torch.no_grad():
        run, ref, whole = _runner(dev, prompt_tokens=512), _runner(dev), _runner(dev, prompt_tokens=512)
        prompts, lens = _prompts(dev, LENS, CTX)
        run.prefill(prompts, lens, chunk=chunk)
        whole.prefill(prompts, lens)
        last = _last(_compose(ref, prompts, LENS, chunk), LENS)
        assert torch.equal(run.last_prompt_hidden, last)
        assert torch.equal(run.last_logits, ref._logits(last))
        for b, n in enumerate(LENS):
            assert torch.equal(_slots(run, b, n), _slots(ref, b, n)), f"row {b}: pages differ from the chunked sequence"
            # layer 0 sees the same K / V whole or in pieces, and the chunked append promises the whole append's bytes
            assert torch.equal(_slots(run, b, n, [0]), _slots(whole, b, n, [0])), f"row {b}: layer-0 pages differ from the whole prompt's"
        # Deeper layers attend to the earlier pieces' keys and values dequantised from the INT4 pages instead of in fp16, so the logits
        # move by the KV quantisation noise: rows whose prompt fits in one piece must agree exactly, the others to a cosine of 0.99 (the
        # tiny model's random weights amplify the noise; the lowest seen on an H100 was 0.994 at chunk 1, where every earlier key is read
        # back quantised as in decoding, and 0.998 at chunk >= 16).  A key at a wrong position
        # is not noise, and it could not hide here: the pages and hidden rows above equal the chunked composition bit for bit, and the
        # needle tests of prefix_prefill_attention pin every position of the prefix.
        a, w = run.last_logits.float(), whole.last_logits.float()
        cos = torch.nn.functional.cosine_similarity(a, w, dim=-1)
        for b, n in enumerate(LENS):
            assert torch.equal(a[b], w[b]) if n <= chunk else cos[b].item() >= 0.99, (b, cos)


def test_prefill_pages_match_token_by_token_decode(dev):
    with torch.no_grad():
        run, dec = _runner(dev, layers=1, prompt_tokens=512), _runner(dev, layers=1)
        prompts, lens = _prompts(dev, LENS, CTX)
        run.prefill(prompts, lens)
        for i in range(max(LENS)):
            dec.context_lens.fill_(i + 1)
            dec.forward(prompts[:, i].contiguous())
        for b, n in enumerate(LENS):
            assert torch.equal(_slots(run, b, n), _slots(dec, b, n)), f"row {b}: the prompt append and the decode append differ"


@pytest.mark.parametrize("chunk", [None, 64])
def test_prompt_logprobs(dev, chunk):
    from qserve_b200 import backend

    with torch.no_grad():
        run, ref = _runner(dev, prompt_tokens=512), _runner(dev)
        prompts, lens = _prompts(dev, LENS, CTX)
        tok = run.prefill(prompts, lens, chunk=chunk, prompt_logprobs=5)
        hidden = _compose(ref, prompts, LENS, chunk)
        cu = np.concatenate([[0], np.cumsum(LENS)])
        src = [cu[b] + j for b, n in enumerate(LENS) for j in range(n - 1)]
        dst = [cu[b] + j + 1 for b, n in enumerate(LENS) for j in range(n - 1)]
        nxt = torch.cat([prompts[b, 1:n] for b, n in enumerate(LENS)])
        if chunk is None:  # the same rows in one lm_head call, as the runner's single block
            lp, ids, tlp = backend.logprobs_rows(ref._logits(hidden[torch.tensor(src, device=dev)]), nxt, 5)
            assert torch.equal(run.p_logprob[dst], lp) and torch.equal(run.p_top_ids[dst], ids) and torch.equal(run.p_top_logprobs[dst], tlp)
        else:  # one lm_head call per piece in the runner: the logits agree to the last fp16 bit up to cuBLAS's choice of kernel per M
            lp, ids, tlp = backend.logprobs_rows(ref._logits(hidden[torch.tensor(src, device=dev)]), nxt, 5)
            assert torch.allclose(run.p_logprob[dst], lp, atol=2e-3, rtol=0)
        first = torch.tensor(cu[:-1], device=dev)
        assert torch.isnan(run.p_logprob[first]).all() and (run.p_top_ids[first] == -1).all()
        assert torch.equal(tok, ref._logits(_last(hidden, LENS)).float().argmax(-1))


def _gen_runner(dev, **kw):
    return _runner(dev, prompt_tokens=B * CTX, max_new_tokens=24, generate=True, verify_len=4, **kw)


@pytest.mark.parametrize("n", [1, 4])
def test_handoff_matches_reset_generation(dev, n):
    steps = 8
    with torch.no_grad():
        run = _gen_runner(dev)
        prompts, lens = _prompts(dev, [CTX] * B, CTX, seed=9, vocab=64)  # a small alphabet gives the n-gram drafter matches
        run.prefill(prompts, lens)
        assert torch.equal(run.s_history[:, :CTX], prompts) and (run.s_seq_lens == CTX + 1).all() and (run.context_lens == CTX + 1).all()
        root = run.s_history[:, :CTX + 1].clone()
        for _ in range(steps):
            run.generate_forward(n)
        want = run.s_history.clone()
        run.prefill(prompts, lens)
        run.reset_generation(root)
        run.g_budget.add_(1)
        for _ in range(steps):
            run.generate_forward(n)
        assert torch.equal(run.s_history, want)


@pytest.mark.parametrize("n", [1, 4])
def test_handoff_captured_generate_matches_eager(dev, n):
    steps = 6
    with torch.no_grad():
        run = _gen_runner(dev)
        run.capture_generate(n)
        prompts, lens = _prompts(dev, LENS, CTX, seed=11, vocab=64)
        run.prefill(prompts, lens)
        for _ in range(steps):
            run.generate_forward(n)
        want = (run.s_history.clone(), run.s_seq_lens.clone(), run.context_lens.clone())
        run.prefill(prompts, lens)
        for _ in range(steps):
            run.generate_step(n)
        assert torch.equal(run.s_history, want[0]) and torch.equal(run.s_seq_lens, want[1]) and torch.equal(run.context_lens, want[2])
        # a first token equal to the row's eos finishes it
        first = run.prefill(prompts, lens)
        run.g_eos[1::2] = first[1::2]
        run.prefill(prompts, lens)
        assert run.g_finished.tolist() == [0, 1, 0, 1, 0]


@pytest.mark.parametrize("lens", [[128, 100, 128, 100, 128], [100, 128, 100, 128, 100]])
def test_fork(dev, lens):
    with torch.no_grad():
        run = _runner(dev, prompt_tokens=B * CTX, max_new_tokens=80, generate=True)
        prompts, lens_d = _prompts(dev, lens, CTX, seed=13)
        run.prefill(prompts, lens_d)
        p, kids = 0, [2, 3, 4]
        snap = _slots(run, p, lens[p])
        run.fork(p, kids)
        assert torch.equal(run.context_lens[kids], run.context_lens[[p] * 3]) and torch.equal(run.s_history[kids], run.s_history[[p] * 3])
        run.generate_forward(1)
        for c in kids:
            assert torch.equal(run.last_logits[c], run.last_logits[p]), f"child {c}: logits differ from the parent's"
        for _ in range(69):  # crosses a page boundary in every row
            run.generate_forward(1)
        for c in kids:
            assert torch.equal(run.s_history[c], run.s_history[p]), f"greedy child {c} left its parent"
        assert torch.equal(_slots(run, p, lens[p]), snap), "a child wrote into the parent's pages"
        # sampled children with their own Philox streams diverge; a prefill gives every row its own pages back
        run.prefill(prompts, lens_d)
        assert torch.equal(run.block_tables, run.own_tables)
        run.fork(p, kids)
        run.s_temperature.fill_(1.0); run.s_top_k.fill_(-1)
        run.s_offsets.copy_(torch.arange(B, device=dev) * 1000)
        for _ in range(8):
            run.generate_forward(1, sampled=True)
        h = run.s_history
        assert not torch.equal(h[2], h[3]) and not torch.equal(h[3], h[4]) and not torch.equal(h[2], h[4])


def test_prompt_tokens_changes_nothing_else(dev):
    with torch.no_grad():
        runs = [_runner(dev, max_new_tokens=8, generate=True, verify_len=4, prompt_tokens=pt) for pt in (0, 4096)]
        g = torch.Generator(device=dev).manual_seed(21)
        toks = torch.randint(0, 1024, (B,), device=dev, generator=g)
        drafts = torch.randint(0, 1024, (B, 4), device=dev, generator=g)
        assert all(torch.equal(a, b) for a, b in zip(runs[0].kpools + runs[0].vpools, runs[1].kpools + runs[1].vpools))
        assert all(torch.equal(a, b) for a, b in zip(runs[0].embed, runs[1].embed))
        out = []
        for run in runs:
            t = run.forward(toks)
            lg = run.last_logits.clone()
            v = run.verify_forward(drafts, return_logits=True).clone()
            run.capture_generate(1)
            run.reset_generation(torch.cat([torch.zeros((B, CTX), dtype=torch.int64, device=dev), toks[:, None]], 1))
            for _ in range(4):
                run.generate_step(1)
            out.append((t, lg, v, run.s_history.clone()))
        for a, b in zip(*out):
            assert torch.equal(a, b)


def test_llama3_8b_prefill(dev):
    with torch.no_grad():
        from qserve_b200.decode import DecodeRunner

        run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=2, ctx=1000, device=dev, layers=2, prompt_tokens=2000)
        prompts, lens = _prompts(dev, [1000, 1000], 1000, vocab=128256)
        run.prefill(prompts, lens)
        whole = run.last_logits.float()
        run.prefill(prompts, lens, chunk=256)
        chunked = run.last_logits.float()
        assert torch.isfinite(whole).all() and torch.isfinite(chunked).all()
        assert torch.nn.functional.cosine_similarity(whole, chunked, dim=-1).min().item() >= 0.99
