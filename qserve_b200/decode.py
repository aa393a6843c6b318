"""Decode-step runner: the reference's per-layer op sequence over the drop-in `qserve_backend` API, with persistent
activation buffers and whole-step CUDA-graph capture.

This is the measurement harness for BASELINE.json's metric (tokens/s, Llama-3-8B W4A8KV4 decode) and the
"step-level CUDA-graph runner under the unchanged model code" of SURVEY.md section 8f-2.  It issues exactly the calls
`LlamaDecoderLayer.forward` issues (qserve/modeling/models/llama_w4a8_unpad.py:330-361, 69-93, 186-291; W8A8:
llama_w8a8_unpad.py) with the same argument marshalling, on synthetic weights of the named architecture
(random INT4/INT8 codes, scales chosen so that activations stay O(1); there is no network for checkpoints).

Tensor parallelism (SURVEY.md section 8e) is Megatron style: qkv / gate_up column parallel, o_proj / down_proj row parallel
(split along K in multiples of 128), KV heads sharded, one NCCL sum-allreduce of [M, hidden] fp16 after each row-parallel
GEMM.  Two quantisation modes for the inputs of the row-parallel GEMMs:
  * `tp_exact=True` -- SURVEY.md 8e parity rule: the per-token amax is max-all-reduced ([M] fp32) so every rank uses the SAME
    scale, the activation sum stays the local K shard's: the INT32 partial sums of the ranks add up to the single-GPU
    accumulators bit for bit (tests/test_gpu_tp.py); costs one extra tiny collective per row-parallel GEMM;
  * `tp_exact=False` (throughput mode) -- every rank quantises its shard with its own per-token scale inside the fused
    attention / silu kernels; each partial product is a correctly de-quantised partial sum (agrees with the single-GPU run to
    quantisation noise, not bit for bit).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import NamedTuple, Optional

import torch

import qserve_backend.activation_ops as activation_ops
import qserve_backend.fused_attention as fused_attention
import qserve_backend.fused_kernels as fused_kernels
import qserve_backend.layernorm_ops as layernorm_ops
import qserve_backend.qgemm_w4a8_per_chn as qgemm_chn
import qserve_backend.qgemm_w4a8_per_group as qgemm_grp
import qserve_backend.qgemm_w8a8 as qgemm_w8
from qserve_b200 import backend as _ext


@dataclass(frozen=True)
class OpSet:
    """The seven `qserve_backend` modules a step is made of.  Default: this repo's sm_90a library.  `bench.py --impl reference-gpu`
    and the live parity tests pass the reference's own extensions (oracle/_ref, compiled unmodified for sm_90a) instead, so the
    SAME op sequence runs on the legacy mma.sync kernels -- same buffers, same shapes, same harness."""
    layernorm_ops: object = layernorm_ops
    fused_kernels: object = fused_kernels
    activation_ops: object = activation_ops
    fused_attention: object = fused_attention
    qgemm_chn: object = qgemm_chn
    qgemm_grp: object = qgemm_grp
    qgemm_w8: object = qgemm_w8


DEFAULT_OPS = OpSet()


from qserve_b200.modelcfg import MODELS, PRECISIONS, ModelConfig  # noqa: E402,F401  (pure-Python table; re-exported)


class _Linear:
    """Weights of one quantised linear layer in the reference's buffer layout (w4a8_linear.py:38-103, w8a8_linear.py:45-54)."""

    def __init__(self, N: int, K: int, mode: str, dev, gen, ops: OpSet = DEFAULT_OPS):
        self.N, self.K, self.mode, self.ops = N, K, mode, ops
        r = lambda lo, hi, shape, dt: torch.randint(lo, hi, shape, dtype=dt, device=dev, generator=gen)
        u = lambda lo, hi, shape: (torch.rand(shape, device=dev, generator=gen) * (hi - lo) + lo)
        target = 1.0 / (K ** 0.5)  # output std ~ O(1) for unit-variance inputs
        if mode == "w8":
            self.weight = r(-127, 128, (N, K), torch.int8)
            self.wscale = (u(0.8, 1.2, (N,)) * target / 73.0).half()
        else:
            self.qweight = r(-128, 128, (N, K // 2), torch.int8)  # uniform random nibbles
            if mode == "chn":
                self.s1 = (u(0.8, 1.2, (N,)) * target / 4.6).half()
                z = r(7, 9, (N,), torch.int8).float()
                self.s1z = (z * self.s1.float()).half()
            else:
                g = K // 128
                s2 = r(1, 9, (g, N), torch.int8)
                z = r(7, 9, (g, N), torch.int8)
                self.s2_scales = s2.contiguous()
                self.s2_zeros = (-(z.int()) * s2.int()).to(torch.int8).contiguous()
                self.s1 = (u(0.8, 1.2, (N,)) * target / (4.6 * 4.5)).half()

    def __call__(self, x_q, scale, asum, out):
        if self.mode == "chn":    # w4a8_linear.py:106-115
            self.ops.qgemm_chn.gemm_forward_cuda(x_q, self.qweight, self.s1, scale, self.s1z, asum, out)
        elif self.mode == "grp":  # w4a8_linear.py:121-131
            self.ops.qgemm_grp.gemm_forward_cuda(x_q, self.qweight, self.s2_zeros, self.s2_scales, self.s1, scale, out)
        else:                     # w8a8_linear.py:98-101
            self.ops.qgemm_w8.w8a8_gemm_forward_cuda(x_q, self.weight, self.wscale, scale, out)

    def weight_bytes(self) -> int:
        return self.N * self.K if self.mode == "w8" else self.N * self.K // 2


class _Rows(NamedTuple):
    """Views of the first M rows of the ActivationBuffer: what one step's layers read and write."""
    qkv: torch.Tensor       # fp16 [M, q + 2 kv]
    out: torch.Tensor       # fp16 [M, hidden], aliases qkv
    gate_up: torch.Tensor   # fp16 [M, 2 I], aliases qkv
    q_hidden: torch.Tensor  # int8 [M, hidden]
    q_attn: torch.Tensor    # int8 [M, q], aliases q_hidden
    q_mlp: torch.Tensor     # int8 [M, I], aliases q_hidden
    q_scale: torch.Tensor   # fp16 [M]
    q_sum: torch.Tensor     # fp16 [M]


def fork_groups(groups: list, parents, children, cached) -> list:
    """The shared-prefix groups after a fork (DecodeRunner(shared_prefix=True)): groups is a list of (rows, S) with the group's first row
    first; each parent of the fork and its children form one group with S = cached[parent] // 64 (the parent's full pages, which fork points
    the children's tables at).  A fork dissolves every earlier group that holds a row it touches."""
    touched = set(parents) | set(children)
    kept = [(tuple(rows), int(s)) for rows, s in groups if not touched & set(rows)]
    new: dict = {}
    for p, c in zip(parents, children):
        new.setdefault(int(p), [int(p)]).append(int(c))
    return kept + [(tuple(rows), int(cached[p]) // 64) for p, rows in new.items()]


# Layouts the plain decode step sends to qs_shared_prefix_decode_attention; every other layout keeps single_query_attention_quant.  From the
# sweep of tools/shared_prefix_bench.py in DESIGN.md 5 (Llama-3-8B heads, B = 64, H100 80GB HBM3, 700 W): with 1024 shared tokens the op took
# 1.08-2.10x the decode launch at every group size; with 4096 shared tokens and groups of >= 2 rows it took 0.69-0.99x, and groups of one row
# 1.09-1.36x.  End to end (8 prompts x 8 forks, captured step) ctx 1024 went 3.85 -> 4.45 ms and ctx 4096 5.50 -> 5.31 ms.  Shared prefixes
# between 1024 and 4096 tokens were not measured and keep the decode kernel.
SHARED_PREFIX_MIN_ROWS = 2
SHARED_PREFIX_MIN_PAGES = 64


def shared_prefix_route(groups: list) -> bool:
    """True when the layout has a group of at least SHARED_PREFIX_MIN_ROWS rows sharing at least SHARED_PREFIX_MIN_PAGES pages."""
    return any(len(rows) >= SHARED_PREFIX_MIN_ROWS and s >= SHARED_PREFIX_MIN_PAGES for rows, s in groups)


def prompt_pieces(lens, ctx: int, prompt_tokens: int, chunk: Optional[int] = None) -> list:
    """The pieces of a prompt step (DecodeRunner.prefill), planned on the host: lens (ints, one prompt length per row) -> [(start, [tokens
    of each row in this piece])].  chunk=None: one piece (0, lens).  chunk=C: piece k starts at k C and row b takes min(C, lens[b] - k C)
    tokens (0 once its prompt is done).  Raises RuntimeError if a length lies outside [1, ctx], chunk < 1 or a piece holds more than
    prompt_tokens tokens."""
    lens = [int(x) for x in lens]
    if not lens or min(lens) < 1 or max(lens) > ctx:
        raise RuntimeError(f"prompt lengths must lie in [1, ctx={ctx}], got {lens}")
    if chunk is not None and int(chunk) < 1:
        raise RuntimeError(f"chunk={chunk}: a piece takes at least one token per row")
    C = max(lens) if chunk is None else int(chunk)
    pieces = []
    for start in range(0, max(lens), C):
        c = [min(C, max(n - start, 0)) for n in lens]
        if sum(c) > prompt_tokens:
            raise RuntimeError(f"a prompt piece of {sum(c)} tokens exceeds prompt_tokens={prompt_tokens}: construct a larger runner or pass a smaller chunk")
        pieces.append((start, c))
    return pieces


class InflightPoll(NamedTuple):
    """DecodeRunner.poll: the requests retired since the last poll and the prompt tokens still to prefill."""
    finished: list
    pending_tokens: int


_PROMPT_LOGITS_BYTES = 64 << 20  # prompt_logprobs: fp16 logits of at most this many bytes exist at once


class DecodeRunner:
    def __init__(self, model: str = "llama-3-8b", precision: str = "w4a8kv4", batch: int = 64, ctx: int = 1024,
                 device: Optional[torch.device] = None, tp_rank: int = 0, tp_size: int = 1, seed: int = 0, layers: Optional[int] = None,
                 process_group=None, fused: bool = True, ops: Optional[OpSet] = None, tp_exact: bool = False, tp_peer: bool = False, no_comm: bool = False,
                 verify_len: int = 0, max_new_tokens: int = 0, generate: bool = False, prompt_tokens: int = 0, shared_prefix: bool = False,
                 beam_width: int = 0, inflight: int = 0):
        """verify_len > 0 (single GPU, fused path) adds the speculative-decoding verify step (`verify_forward`): the page tables cover
        ctx + verify_len tokens and the activation buffers hold batch * verify_len rows.  verify_len = 0 leaves the decode step, its buffers
        and its random draws exactly as they are without it.

        max_new_tokens > 0 adds penalties and log-probabilities to the decode step (forward(..., penalties=True, logprobs=n)): the token
        history s_history int64 [batch, ctx + max_new_tokens] (the caller writes the prompts into [:, :ctx]; the step appends its token),
        s_prompt_lens / s_seq_lens (= ctx), the per-row s_repetition / s_presence / s_frequency (neutral: 1, 0, 0) and the log-probability
        outputs s_logprob [batch], s_top_ids / s_top_logprobs [batch, n].  All made with torch.full / torch.zeros: max_new_tokens = 0 and
        max_new_tokens > 0 give the same weights, pages and greedy / sampled steps.

        generate=True (single GPU, fused path, max_new_tokens = T >= 1) adds the generation loop (reset_generation, generate_forward,
        capture_generate / generate_step): plain decode steps (n = 1) and prompt-lookup speculative steps (2 <= n <= verify_len) that advance
        every row by what it accepted.  The history is [batch, ctx + 1 + T] (the prompt is ctx cached tokens and the root), the page tables
        cover ctx + T + max(1, verify_len) tokens (the pages past blocks_per_seq come from zero-filled pools made after every random draw, so
        the weights and the first blocks_per_seq pages of each row are those of generate=False), and the per-row state is g_budget (tokens a
        row may generate, default T), g_eos (-1: none), g_stop (up to 8 stop tokens, -1 pads) and g_finished.  generate_forward(...,
        penalties=True, logprobs=n) adds the penalties and log-probabilities of forward to plain and speculative steps; the log-probabilities
        go to history-aligned buffers (g_logprob, g_top_view).

        prompt_tokens > 0 (single GPU, fused path) adds the prompt step (`prefill`): at most prompt_tokens prompt tokens per piece, so the
        activation buffers hold max(batch * max(1, verify_len), prompt_tokens) rows.  It makes no generator draws: the weights, pages and
        decode / verify / generate steps are those of prompt_tokens = 0.

        shared_prefix=True (single GPU, fused path): fork records groups (a parent and its children share the parent's full pages) and prefill
        dissolves them.  While shared_prefix_route(sp_groups) holds, the plain decode step (forward, capture / step, generate_forward(1),
        capture_generate(1)) runs its attention through shared_prefix_decode_attention, which reads each group's shared pages once; otherwise
        through single_query_attention_quant.  The layout lives in buffers made with torch.zeros, so the weights, pages and every step
        without a group are those of shared_prefix=False.  The plain-step graph keys end in the layout's launch plan: after a fork or prefill
        that changes it, replaying the old key raises instead of running under a stale plan.

        beam_width = W >= 1 (single GPU, fused path, max_new_tokens = T >= 1, prompt_tokens > 0; not with generate or verify_len) adds beam
        search (beam_start, beam_forward, capture_beam / beam_step, beam_results): batch / W requests of W beams, request r in rows
        r W .. r W + W - 1.  The page tables cover ctx + T + 1 tokens as with generate=True, and the beam state (b_live, b_cum, b_parent, the
        per-request b_length_penalty (1), b_early_stopping (0), b_eos (-1), b_stop (-1 pads), b_budget (T), b_done and the hypothesis pool
        b_pool) is made with torch.full / torch.zeros, so the weights, pages and every other step are those of beam_width = 0.

        inflight = Q >= 1 (single GPU, fused path, generate=True, max_new_tokens = T >= 1, prompt_tokens = C >= 1; not with verify_len,
        beam_width or shared_prefix) adds in-flight batching (submit, inflight_forward, capture_inflight / inflight_step, poll): a queue of Q
        requests, rows that take queued prompts as they free up, and a step that carries up to C prompt tokens of the prefilling rows in the
        same forward pass as the decode tokens of the others (DESIGN.md 3.12).  The activation buffers hold batch + C rows and the page tables
        cover max(ctx + T + 1, ctx - 1 + C) tokens; every row keeps its own pages.  All its state is made with torch.full / torch.zeros after
        every random draw, so inflight = 0 leaves the weights, pages and every other step as they are."""
        beam_width = int(beam_width)
        if beam_width:
            if not 1 <= beam_width <= _ext.MAX_BEAM_WIDTH:
                raise RuntimeError(f"beam_width={beam_width}: 1 .. {_ext.MAX_BEAM_WIDTH}")
            if batch % beam_width:
                raise RuntimeError(f"batch={batch} is not a multiple of beam_width={beam_width}")
            if tp_size != 1 or not fused or generate or verify_len:
                raise RuntimeError("beam search is single-GPU, uses the fused path and is not combined with generate=True or verify_len")
            if max_new_tokens < 1 or prompt_tokens < 1:
                raise RuntimeError("beam search needs max_new_tokens >= 1 and prompt_tokens >= 1")
            if ctx + max_new_tokens + 1 > min(8192, MODELS[model].max_pos):
                raise RuntimeError("beam search runs past the positions the attention supports")
        self.beam_width = beam_width
        inflight = int(inflight)
        if inflight:
            if tp_size != 1 or not fused or not generate or verify_len or beam_width or shared_prefix:
                raise RuntimeError("in-flight batching is single-GPU, uses the fused path, needs generate=True and is not combined with verify_len, "
                                   "beam_width or shared_prefix")
            if max_new_tokens < 1 or prompt_tokens < 1 or inflight < 1:
                raise RuntimeError("in-flight batching needs max_new_tokens >= 1, prompt_tokens >= 1 and a queue of at least one request")
            if not 1 <= batch <= _ext.MAX_INFLIGHT_ROWS:
                raise RuntimeError(f"in-flight batching runs 1 .. {_ext.MAX_INFLIGHT_ROWS} rows")
        self.inflight = inflight
        assert precision in PRECISIONS, precision
        assert not shared_prefix or (tp_size == 1 and fused), "shared_prefix is single-GPU and uses the fused path"
        self.shared_prefix = shared_prefix
        assert prompt_tokens >= 0 and (prompt_tokens == 0 or (tp_size == 1 and fused)), "the prompt step is single-GPU and uses the fused path"
        self.prompt_tokens = prompt_tokens
        assert 0 <= verify_len <= 16, "verify_len: at most 16 draft tokens per sequence"
        assert verify_len == 0 or (tp_size == 1 and fused), "the verify step is single-GPU and uses the fused path"
        assert max_new_tokens == 0 or 0 < ctx + max_new_tokens <= _ext.MAX_PENALTY_HISTORY, "the token history holds at most 32768 tokens per row"
        self.generate = generate
        if generate:
            assert tp_size == 1 and fused, "generation is single-GPU and uses the fused path"
            assert max_new_tokens >= 1, "generate=True needs max_new_tokens >= 1"
            assert ctx + 1 + max_new_tokens <= _ext.MAX_PENALTY_HISTORY, "the token history holds at most 32768 tokens per row"
            assert ctx + max_new_tokens + max(1, verify_len) <= min(8192, MODELS[model].max_pos), "generation runs past the positions the attention supports"
        self.verify_len = verify_len
        self.ops = ops = ops or DEFAULT_OPS
        self.tp_exact = tp_exact
        self.no_comm = no_comm  # debugging: run one rank's shard of a tensor-parallel model without the collectives (sanitizer / profiler runs)
        # tensor parallel, fused path: the all-reduce of the row-parallel GEMM outputs is folded into the following add+norm+quant kernel
        # (peer loads over NVLink symmetric memory) instead of an NCCL call
        self.tp_peer = tp_peer and tp_size > 1
        assert not (self.tp_peer and not fused), "tp_peer needs the fused path"
        assert ops is DEFAULT_OPS or not fused, "the fused extensions exist only in this repo's library"
        self.cfg = cfg = MODELS[model]
        self.precision, self.batch, self.ctx = precision, batch, ctx
        self.dev = dev = device or torch.device("cuda", torch.cuda.current_device())
        self.tp_rank, self.tp_size, self.pg = tp_rank, tp_size, process_group
        self.fused = fused  # fused residual+norm+quant and silu*mul+quant extensions (bit-identical to the reference op sequence)
        self.L = layers if layers is not None else cfg.layers
        gen = torch.Generator(device=dev)
        gen.manual_seed(seed + 1000 * tp_rank)
        self.wmode = "w8" if precision.startswith("w8a8") else ("grp" if precision.endswith("g128") else "chn")
        self.act_sum = self.wmode == "chn"  # per-channel W4 needs the activation sum (llama_w4a8_unpad.py:69, 165-168)
        self.kv_bits = 4 if "kv4" in precision else 8
        D, H, I = cfg.head_dim, cfg.hidden, cfg.intermediate
        assert cfg.heads % tp_size == 0 and I % (128 * tp_size) == 0
        self.Hq = cfg.heads // tp_size
        self.Hkv = max(1, cfg.kv_heads // tp_size)  # llama_w4a8_unpad.py:120-129
        self.Iloc = I // tp_size
        self.q_size, self.kv_size = self.Hq * D, self.Hkv * D
        M = batch

        # ---- weights --------------------------------------------------------------------------------------
        self.layers = []
        for _ in range(self.L):
            self.layers.append({
                "qkv": _Linear(self.q_size + 2 * self.kv_size, H, self.wmode, dev, gen, ops),
                "o": _Linear(H, self.q_size, self.wmode, dev, gen, ops),
                "gate_up": _Linear(2 * self.Iloc, H, self.wmode, dev, gen, ops),
                "down": _Linear(H, self.Iloc, self.wmode, dev, gen, ops),
                # W4A8 checkpoints skip the norm weights (gamma = 1, llama_w4a8_unpad.py:541-542); W8A8 loads them
                "ln1": torch.ones(H, dtype=torch.half, device=dev),
                "ln2": torch.ones(H, dtype=torch.half, device=dev),
            })
        self.norm_w = torch.ones(H, dtype=torch.half, device=dev)
        self.embed = (torch.randn((cfg.vocab, H), device=dev, generator=gen) * 1.0).half()
        self.lm_head = (torch.randn((cfg.vocab, H), device=dev, generator=gen) * (1.0 / H ** 0.5)).half()  # fp16, cuBLAS (:432)

        # ---- paged KV cache: ctx tokens present, the step decodes token ctx (length ctx+1) ---------------------
        self.blocks_per_seq = (ctx + max(1, verify_len) + 63) // 64
        self.size_per_token = self.Hkv * D * self.kv_bits // 8
        code_bytes = 64 * self.size_per_token
        self.page_bytes = code_bytes + self.Hkv * 64 * 4  # cache_engine.py:62-66
        n_pages = batch * self.blocks_per_seq
        self.kpools, self.vpools, tables = [], [], []
        blk = torch.arange(n_pages, device=dev, dtype=torch.int64).view(batch, self.blocks_per_seq)
        for _ in range(self.L):
            pools = []
            for _kv in range(2):
                pool = torch.randint(0, 256, (n_pages, self.page_bytes), dtype=torch.uint8, device=dev, generator=gen)
                meta = pool[:, code_bytes:].view(torch.float16).view(n_pages, 2, self.Hkv, 64)
                meta[:, 0] = (torch.rand((n_pages, self.Hkv, 64), device=dev, generator=gen) * 0.09 + 0.01).half()
                zmax = 15.0 if self.kv_bits == 4 else 255.0
                meta[:, 1] = (torch.rand((n_pages, self.Hkv, 64), device=dev, generator=gen) * zmax).half()
                pools.append(pool)
            self.kpools.append(pools[0]); self.vpools.append(pools[1])
            # [B, 2, blocks] absolute addresses (model_runner.py:506-530)
            tables.append(torch.stack([pools[0].data_ptr() + blk * self.page_bytes, pools[1].data_ptr() + blk * self.page_bytes], dim=1))
        self.table_blocks = self.blocks_per_seq
        self.kpools_gen, self.vpools_gen = [], []
        if generate or beam_width:  # pages for the generated tokens: zero-filled (no generator draws), after the pages above in every row's table
            # (in-flight batching: also the host bound ctx - 1 + C of the chunk segment's prompt attention)
            self.table_blocks = (max(ctx + max_new_tokens + max(1, verify_len), ctx - 1 + prompt_tokens if inflight else 0) + 63) // 64
            extra = self.table_blocks - self.blocks_per_seq
            if extra:
                blk = torch.arange(batch * extra, device=dev, dtype=torch.int64).view(batch, extra)
                for li in range(self.L):
                    kp = torch.zeros((batch * extra, self.page_bytes), dtype=torch.uint8, device=dev)
                    vp = torch.zeros_like(kp)
                    self.kpools_gen.append(kp); self.vpools_gen.append(vp)
                    more = torch.stack([kp.data_ptr() + blk * self.page_bytes, vp.data_ptr() + blk * self.page_bytes], dim=1)
                    tables[li] = torch.cat([tables[li], more], dim=2)
        self.block_tables = torch.stack(tables, dim=0).contiguous()  # [L, B, 2, blocks]
        self.own_tables = self.block_tables.clone()  # every row's own pages: fork() shares a parent's pages, prefill() restores these
        self.context_lens = torch.full((batch,), ctx + 1, dtype=torch.int32, device=dev)
        # host bounds of the attention launches: in generation the contexts grow up to ctx + 1 + max_new_tokens
        self.max_seq_len = ctx + 1 + (max_new_tokens if generate or beam_width else 0)
        self.max_prefix_len = ctx + (max_new_tokens if generate or beam_width else 0)

        # ---- persistent ActivationBuffer (input_metadata.py:71-109; aliasing kept) for the rows of the widest step --------------------
        # (H is in the max for tensor parallelism: at TP = 8 a 72B model's sharded qkv / gate_up rows are narrower than the full hidden row of out_buf)
        R = max(M * max(1, verify_len), prompt_tokens, M + prompt_tokens if inflight else 0)
        self.act_buffer = torch.empty(R * max(self.q_size + 2 * self.kv_size, 2 * self.Iloc, H), dtype=torch.half, device=dev)
        self.q_act = torch.empty(R * max(H, self.Iloc), dtype=torch.int8, device=dev)
        self.scale_buffer = torch.empty(R, dtype=torch.half, device=dev)
        self.sum_buffer = torch.empty(R, dtype=torch.half, device=dev)
        self.rows = self._row_views(M)  # the decode step's
        self.qkv_buf, self.out_buf, self.gate_up_buf, self.q_hidden, self.q_attn, self.q_mlp, self.q_scale, self.q_sum = self.rows
        self.q_amax = torch.empty(M, dtype=torch.float32, device=dev)  # TP parity mode: per-token amax, max-all-reduced
        self.mlp_act = torch.empty((M, self.Iloc), dtype=torch.half, device=dev)  # reference: fresh torch.empty per call (activation.py:26)
        self.peer = None
        if self.tp_peer:
            self.peer = _ext.PeerContext(M, H, dev, process_group if process_group is not None else torch.distributed.group.WORLD)
        self.tokens_in = torch.zeros(M, dtype=torch.int64, device=dev)
        self.tokens_out = torch.zeros(M, dtype=torch.int64, device=dev)
        self.graph: Optional[torch.cuda.CUDAGraph] = None  # the latest capture()
        self.graphs = {}  # ("decode" | "verify" | "generate", *arguments) -> CUDA graph
        self.launches_per_step = 0
        if verify_len:
            self._alloc_verify_buffers()
        # sampling (forward(sample=True), the sampled tree verify): per-row parameters the caller edits between replays, made with torch.full
        # (no generator draws).  Defaults: the reference ModelRunner's SamplingParams(temperature=1.0, top_p=1.0, top_k=1).
        self.s_seed = seed
        self.s_temperature = torch.full((batch,), 1.0, dtype=torch.float32, device=dev)
        self.s_top_k = torch.full((batch,), 1, dtype=torch.int32, device=dev)
        self.s_top_p = torch.full((batch,), 1.0, dtype=torch.float32, device=dev)
        self.s_offsets = torch.full((batch,), 0, dtype=torch.int64, device=dev)
        self._p_logprob = None  # prompt_logprobs outputs, allocated by the first prefill that asks for them
        self.max_new_tokens = max_new_tokens
        if max_new_tokens:
            self._alloc_penalty_buffers()
        if generate:
            self._alloc_generate_buffers()
        if beam_width:
            self._alloc_beam_buffers()
        if inflight:
            self._alloc_inflight_buffers()
        self.sp_groups = []  # shared-prefix groups: (rows, S), the group's first row first
        self._sp_layout = None  # the layout the plain step passes to shared_prefix_decode_attention (None: single_query_attention_quant)
        if shared_prefix:
            z = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)
            self._sp_buf = (z(batch + 1), z(batch), z(batch), z(batch))  # offsets, rows, pages, row_pages: updated in place (graphs hold them)

    # ---------------------------------------------------------------------------------------------------------
    def _set_groups(self, groups: list) -> None:
        """Record the shared-prefix groups and write their layout into the persistent buffers."""
        self.sp_groups = groups
        self._sp_layout = None
        if not shared_prefix_route(groups):
            return
        lay = _ext.shared_prefix_layout([rows for rows, _ in groups], [s for _, s in groups], self.batch)
        G, n = lay.num_groups, lay.group_rows.numel()
        off, rows, pages, row_pages = self._sp_buf
        off[: G + 1].copy_(lay.group_offsets)
        rows[:n].copy_(lay.group_rows)
        pages[:G].copy_(lay.group_pages)
        row_pages.copy_(lay.row_pages)
        self._sp_layout = lay._replace(group_offsets=off[: G + 1], group_rows=rows[:n], group_pages=pages[:G], row_pages=row_pages)

    def _sp_key(self) -> tuple:
        """Suffix of the plain-step graph keys: () without shared_prefix, else the launch plan of the current layout."""
        if not self.shared_prefix:
            return ()
        lay = self._sp_layout
        return ("shared_prefix",) + ((lay.num_groups, lay.max_group, lay.max_pages) if lay is not None else (None,))

    def _row_views(self, M: int) -> _Rows:
        H, W = self.cfg.hidden, self.q_size + 2 * self.kv_size
        a, q = self.act_buffer, self.q_act
        return _Rows(a[: M * W].view(M, W), a[: M * H].view(M, H), a[: M * 2 * self.Iloc].view(M, -1), q[: M * H].view(M, H),
                     q[: M * self.q_size].view(M, self.q_size), q[: M * self.Iloc].view(M, self.Iloc), self.scale_buffer[:M], self.sum_buffer[:M])

    def _norm_quant(self, r: _Rows, x, gamma):
        """Per-token quantised RMS norm of x into r.q_hidden, r.q_scale and r.q_sum."""
        if self.act_sum:  # layernorm.py:88
            self.ops.layernorm_ops.rms_norm_general_fuse_sum(r.q_hidden, x, gamma, r.q_sum, r.q_scale, self.cfg.eps, True)
        else:             # layernorm.py:72
            self.ops.layernorm_ops.rms_norm_general(r.q_hidden, x, gamma, r.q_scale, self.cfg.eps, True)

    def _quant(self, r: _Rows, out_q, x):
        """Per-token quantisation of the input of a ROW-parallel GEMM (o_proj, down_proj) into out_q, r.q_scale and r.q_sum."""
        if self.tp_size > 1 and self.tp_exact:
            # SURVEY.md 8e: same per-token scale on all ranks (global amax), local-K-shard activation sum
            _ext.row_absmax(self.q_amax, x)
            if not self.no_comm:
                torch.distributed.all_reduce(self.q_amax, op=torch.distributed.ReduceOp.MAX, group=self.pg)
            _ext.invoke_quant_given_amax(out_q, x, self.q_amax, r.q_sum if self.act_sum else None, r.q_scale)
        elif self.act_sum:  # llama_w4a8_unpad.py:177-183
            self.ops.fused_kernels.invoke_quant_fuse_sum(out_q, x, r.q_sum, r.q_scale)
        else:
            self.ops.fused_kernels.invoke_quant(out_q, x, r.q_scale)

    def _allreduce(self, t):
        if self.tp_size > 1 and not self.no_comm:
            torch.distributed.all_reduce(t, group=self.pg)

    def forward(self, tokens: torch.Tensor, sample: bool = False, penalties: bool = False, logprobs: int = 0) -> torch.Tensor:
        """One decode step for `batch` sequences; returns the greedy next tokens [batch] (device).  sample=True ends the step in sample_rows
        with the per-row s_temperature / s_top_k / s_top_p, seed s_seed and counters s_offsets (advanced by one) instead of argmax_rows.

        penalties / logprobs (need max_new_tokens > 0): logits -> apply_penalties (s_history, s_prompt_lens, s_seq_lens, s_repetition,
        s_presence, s_frequency) if penalties -> sample_rows / argmax_rows -> logprobs_rows of the penalised logits with n = logprobs
        (s_logprob, s_top_ids, s_top_logprobs: the distribution before the temperature / top-k / top-p warpers) if logprobs > 0 -> the token
        is appended to s_history at s_seq_lens (index clamped to the last column) and s_seq_lens advances by one.  A caller must not run
        more than max_new_tokens such steps (eager or replayed) without resetting s_seq_lens and s_history."""
        assert self.max_new_tokens or not (penalties or logprobs), "construct the runner with max_new_tokens > 0 for penalties / logprobs"
        logits = self._forward_fused(tokens, True) if self.fused else self._forward_reference(tokens, True)
        return self._next_tokens(logits, sample, penalties, logprobs)

    def _pick(self, logits, sample: bool, penalties: bool = False, logprobs: int = 0, out: Optional[torch.Tensor] = None):
        """logits -> apply_penalties (if penalties) -> sample_rows / argmax_rows: the step's tokens, written into out if given."""
        if penalties:
            _ext.apply_penalties(logits, self.s_history, self.s_prompt_lens, self.s_seq_lens, self.s_repetition, self.s_presence, self.s_frequency)
        if sample:
            return _ext.sample_rows(logits, self.s_temperature, self.s_top_k, self.s_top_p, self.s_seed, self.s_offsets, out=out)
        if self.fused or penalties or logprobs:
            return _ext.argmax_rows(logits, out=out)  # one launch instead of torch's two-pass reduction
        return torch.argmax(logits, dim=-1)  # the reference's greedy step

    def _next_tokens(self, logits, sample: bool, penalties: bool = False, logprobs: int = 0, out: Optional[torch.Tensor] = None):
        """logits -> the step's tokens as forward describes them, written into out if given."""
        tok = self._pick(logits, sample, penalties, logprobs, out)
        if logprobs:
            _ext.logprobs_rows(logits, tok, int(logprobs), self.s_logprob, *self.top_logprobs_view(int(logprobs)))
        if penalties or logprobs:
            col = self.s_seq_lens.clamp(max=self.s_history.size(1) - 1).long().unsqueeze(1)
            self.s_history.scatter_(1, col, tok.unsqueeze(1))
            self.s_seq_lens.add_(1)
        return tok

    def _alloc_penalty_buffers(self) -> None:
        B, dev = self.batch, self.dev
        self.s_history = torch.full((B, self.ctx + int(self.generate) + self.max_new_tokens), -1, dtype=torch.int64, device=dev)
        self.s_prompt_lens = torch.full((B,), self.ctx, dtype=torch.int32, device=dev)
        self.s_seq_lens = torch.full((B,), self.ctx, dtype=torch.int32, device=dev)
        self.s_repetition = torch.full((B,), 1.0, dtype=torch.float32, device=dev)
        self.s_presence = torch.zeros(B, dtype=torch.float32, device=dev)
        self.s_frequency = torch.zeros(B, dtype=torch.float32, device=dev)
        self.s_logprob = torch.zeros(B, dtype=torch.float32, device=dev)
        # flat, so that [:B n] viewed as [B, n] is contiguous for any n <= 20
        self.s_top_ids = torch.zeros(B * _ext.MAX_TOP_LOGPROBS, dtype=torch.int64, device=dev)
        self.s_top_logprobs = torch.zeros(B * _ext.MAX_TOP_LOGPROBS, dtype=torch.float32, device=dev)

    def top_logprobs_view(self, n: int):
        """(s_top_ids, s_top_logprobs) as the [batch, n] tensors a step with logprobs = n writes."""
        B = self.batch
        return self.s_top_ids[: B * n].view(B, n), self.s_top_logprobs[: B * n].view(B, n)

    def _heads(self, qkv):
        """q [M, Hq, D], k and v [M, Hkv, D]: views of the qkv GEMM output (:245-252)."""
        D = self.cfg.head_dim
        q, k, v = qkv.split([self.q_size, self.kv_size, self.kv_size], dim=-1)
        return q.reshape(q.size(0), self.Hq, D), k.reshape(k.size(0), self.Hkv, D), v.reshape(v.size(0), self.Hkv, D)

    def _attention(self, li):
        cfg = self.cfg
        q, k, v = self._heads(self.qkv_buf)
        attn = self.ops.fused_attention.single_query_attention(
            q, k, v, self.block_tables[li], self.context_lens, None, min(8192, cfg.max_pos), 64, self.size_per_token,
            self.max_seq_len, cfg.head_dim, cfg.rope_theta, True, self.kv_bits == 4, True)  # :265-281
        return attn.reshape(q.size(0), -1)

    def _attention_quant(self, li, r: _Rows) -> None:
        """The decode step's attention, quantised into r.q_attn: one launch, or with tp_exact on TP > 1 the attention and then _quant."""
        if self.tp_size > 1 and self.tp_exact:
            self._quant(r, r.q_attn, self._attention(li))
            return
        cfg = self.cfg
        q, k, v = self._heads(r.qkv)
        if self._sp_layout is not None:
            _ext.shared_prefix_decode_attention(q, k, v, self.block_tables[li], self.context_lens, self._sp_layout, 64, self.size_per_token,
                                                self.max_seq_len, cfg.head_dim, cfg.rope_theta, self.kv_bits == 4, True, out_q=r.q_attn,
                                                out_scale=r.q_scale, out_sum=r.q_sum if self.act_sum else None)
            return
        _ext.single_query_attention_quant(q, k, v, self.block_tables[li], self.context_lens, min(8192, cfg.max_pos), 64, self.size_per_token,
                                          self.max_seq_len, cfg.head_dim, cfg.rope_theta, self.kv_bits == 4, True, r.q_attn, r.q_scale,
                                          r.q_sum if self.act_sum else None)

    def _logits(self, hidden):
        """Final norm (:408) and the fp16 lm_head (cuBLAS, :474-476)."""
        out = torch.empty_like(hidden)
        self.ops.layernorm_ops.rms_norm(out, hidden, self.norm_w, self.cfg.eps, False)
        return torch.nn.functional.linear(out, self.lm_head)

    def _forward_reference(self, tokens: torch.Tensor, return_logits: bool = False) -> torch.Tensor:
        """Exactly the reference's op sequence (LlamaDecoderLayer.forward, llama_w4a8_unpad.py:330-361)."""
        r = self.rows
        n = 0
        hidden = self.embed[tokens]  # LlamaModel.forward (:401-404)
        for li, ly in enumerate(self.layers):
            residual = hidden
            self._norm_quant(r, hidden, ly["ln1"])
            ly["qkv"](self.q_hidden, self.q_scale, self.q_sum, self.qkv_buf)
            attn = self._attention(li)
            self._quant(r, self.q_attn, attn)
            ly["o"](self.q_attn, self.q_scale, self.q_sum, self.out_buf)
            self._allreduce(self.out_buf)
            hidden = residual + self.out_buf  # :348
            residual = hidden
            self._norm_quant(r, hidden, ly["ln2"])
            ly["gate_up"](self.q_hidden, self.q_scale, self.q_sum, self.gate_up_buf)
            self.ops.activation_ops.silu_and_mul(self.mlp_act, self.gate_up_buf)  # activation.py:24-29
            self._quant(r, self.q_mlp, self.mlp_act)
            ly["down"](self.q_mlp, self.q_scale, self.q_sum, self.out_buf)
            self._allreduce(self.out_buf)
            hidden = residual + self.out_buf  # :360
            n += 10
        logits = self._logits(hidden)
        self.launches_per_step = n + 1
        self.last_logits = logits  # what the step computed before sampling (bench.py --dump-outputs)
        return logits if return_logits else torch.argmax(logits, dim=-1)

    def _fused_layers(self, hidden: torch.Tensor, r: _Rows, attention):
        """The decoder layers over the M rows of r, from the embedded tokens hidden [M, H]: the reference's arithmetic, three launches fewer
        per layer (the two torch residual adds are folded into the following norm, `add_rms_norm_general`, and silu_and_mul into the
        following per-token quant, `silu_and_mul_quant`).  attention(li, r) reads r.qkv and writes r.q_attn, r.q_scale and r.q_sum.
        Returns the final hidden state [M, H] and the number of launches."""
        cfg = self.cfg
        exact = self.tp_size > 1 and self.tp_exact
        qsum = r.q_sum if self.act_sum else None
        nxt = torch.empty_like(hidden)
        self._norm_quant(r, hidden, self.layers[0]["ln1"])
        n = 1
        for li, ly in enumerate(self.layers):
            ly["qkv"](r.q_hidden, r.q_scale, r.q_sum, r.qkv)
            attention(li, r)
            if self.tp_peer:
                ly["o"](r.q_attn, r.q_scale, r.q_sum, self.peer.partial[0])
                _ext.add_rms_norm_general_peer(r.q_hidden, nxt, hidden, self.peer, 0, ly["ln2"], qsum, r.q_scale, cfg.eps)
            else:
                ly["o"](r.q_attn, r.q_scale, r.q_sum, r.out)
                self._allreduce(r.out)
                _ext.add_rms_norm_general(r.q_hidden, nxt, hidden, r.out, ly["ln2"], qsum, r.q_scale, cfg.eps)
            hidden, nxt = nxt, hidden
            ly["gate_up"](r.q_hidden, r.q_scale, r.q_sum, r.gate_up)
            if exact:
                activation_ops.silu_and_mul(self.mlp_act, r.gate_up)
                self._quant(r, r.q_mlp, self.mlp_act)
            else:
                _ext.silu_and_mul_quant(r.q_mlp, r.gate_up, qsum, r.q_scale)
            if self.tp_peer:
                ly["down"](r.q_mlp, r.q_scale, r.q_sum, self.peer.partial[1])
            else:
                ly["down"](r.q_mlp, r.q_scale, r.q_sum, r.out)
                self._allreduce(r.out)
            n += 11 if exact else 7
            if self.tp_peer:
                # the last layer has no following norm: the same kernel delivers hidden + sum(partials) (its quantised output is not used)
                gam = self.layers[li + 1]["ln1"] if li + 1 < len(self.layers) else ly["ln1"]
                _ext.add_rms_norm_general_peer(r.q_hidden, nxt, hidden, self.peer, 1, gam, qsum, r.q_scale, cfg.eps)
                hidden, nxt = nxt, hidden
                n += 1
            elif li + 1 < len(self.layers):
                _ext.add_rms_norm_general(r.q_hidden, nxt, hidden, r.out, self.layers[li + 1]["ln1"], qsum, r.q_scale, cfg.eps)
                hidden, nxt = nxt, hidden
                n += 1
            else:
                hidden = hidden + r.out
        return hidden, n

    def _forward_fused(self, tokens: torch.Tensor, return_logits: bool = False) -> torch.Tensor:
        """The decode step on the fused layers: the arithmetic of _forward_reference, three launches fewer per layer."""
        hidden, n = self._fused_layers(self.embed[tokens], self.rows, self._attention_quant)
        logits = self._logits(hidden)
        self.launches_per_step = n + 2
        self.last_logits = logits
        return logits if return_logits else _ext.argmax_rows(logits)  # one launch instead of torch's two-pass reduction

    # ---------------------------------------------------------------------------------------------------------
    # speculative-decoding verify: n draft tokens per sequence at positions ctx .. ctx + n - 1 in one step
    # ---------------------------------------------------------------------------------------------------------
    def _alloc_verify_buffers(self) -> None:
        """State of the verify step (torch.full / torch.zeros: no random draws)."""
        dev = self.dev
        self.v_start = torch.full((self.batch,), self.ctx, dtype=torch.int32, device=dev)  # tokens cached before the drafts
        self.v_meta = {}  # n -> (draft lengths [B], cu_seqlens [B + 1], padding offsets [B n]), built on first use (before any capture)
        self.v_tokens_in = torch.zeros((self.batch, self.verify_len), dtype=torch.int64, device=dev)
        self.v_tokens_out = torch.zeros((self.batch, self.verify_len), dtype=torch.int64, device=dev)
        # draft-tree verify (capture_verify(n, tree=True)): ancestor words in, acceptance out
        self.v_tree_mask = torch.zeros((self.batch, self.verify_len), dtype=torch.int32, device=dev)
        self.v_accept_len = torch.zeros(self.batch, dtype=torch.int32, device=dev)
        self.v_path = torch.zeros(self.batch * self.verify_len, dtype=torch.int32, device=dev)  # [:B n] viewed as [B, n] for n nodes
        self.v_bonus = torch.zeros(self.batch, dtype=torch.int64, device=dev)
        self.v_draft_probs = None  # fp32 [B * verify_len * vocab], allocated by capture_verify(..., draft_probs=True)

    def _verify_meta(self, n: int):
        if n not in self.v_meta:
            B, dev = self.batch, self.dev
            cu = torch.arange(0, B * n + 1, n, dtype=torch.int32, device=dev)
            self.v_meta[n] = (torch.full((B,), n, dtype=torch.int32, device=dev), cu, _ext.compute_padding_offsets(cu, n, B * n))
        return self.v_meta[n]

    def verify_forward(self, tokens: torch.Tensor, return_logits: bool = False, tree_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Score n = tokens.size(1) <= verify_len draft tokens per sequence at positions ctx .. ctx + n - 1 in one step: tokens [B, n] ->
        greedy tokens [B, n] (or fp16 logits [B, n, vocab]).  Per layer: qkv GEMM at M = B n, apply_bias_rope_update_kv_cache_at at ctx,
        multi_token_decode_attention (each draft token gets the numbers of its own decode step), invoke_quant[_fuse_sum], then o, gate_up,
        silu+quant and down as the fused decode step.  The drafts' K / V stay in the pages; a later step at the same positions overwrites
        them, so rejected drafts need no cleanup.

        tree_mask (int32 [B, n], ancestor words, see backend.multi_token_decode_attention): the tokens are the nodes of a draft tree, node i
        is rotated at ctx + depth(i), stored in slot ctx + i and attends to the prefix and its ancestors; follow with accept_and_compact."""
        assert self.verify_len, "construct the runner with verify_len > 0"
        B, n = tokens.shape
        assert B == self.batch and 1 <= n <= self.verify_len
        cfg, M = self.cfg, B * n
        lens, cu, pad = self._verify_meta(n)
        tm = None
        if tree_mask is not None:
            assert tuple(tree_mask.shape) == (B, n) and tree_mask.dtype == torch.int32
            tm = tree_mask.contiguous().view(-1)

        def attention(li, r):
            table = self.block_tables[li]
            _ext.apply_bias_rope_update_kv_cache_at(r.qkv, lens, pad, self.v_start, table, self.Hq, self.Hkv, n, 64, self.size_per_token,
                                                   cfg.head_dim, cfg.rope_theta, min(8192, cfg.max_pos), True, self.kv_bits == 4, True, tree_mask=tm)
            attn = _ext.multi_token_decode_attention(*self._heads(r.qkv), cu, n, self.v_start, self.max_prefix_len, table, 64, self.size_per_token,
                                                     self.kv_bits == 4, tree_mask=tm)
            self._quant(r, r.q_attn, attn.view(M, -1))

        hidden, _ = self._fused_layers(self.embed[tokens.reshape(-1)], self._row_views(M), attention)
        logits = self._logits(hidden)
        self.last_verify_logits = logits.view(B, n, -1)
        return self.last_verify_logits if return_logits else _ext.argmax_rows(logits).view(B, n)

    def accept_and_compact(self, tokens: torch.Tensor, tree_mask: torch.Tensor, target: torch.Tensor):
        """After verify_forward(tokens, tree_mask=tree_mask) returned the greedy targets [B, n]: greedy acceptance of the tree and compaction
        of the accepted path's K / V into slots ctx .. ctx + accept_len - 1 of every layer (one launch each).  Returns (accept_len int32 [B],
        path int32 [B, n], bonus int64 [B]), written into v_accept_len, v_path and v_bonus.  The runner's positions stay at ctx: the engine
        advances each context by accept_len and feeds bonus as the next root."""
        n = tokens.size(1)
        path = self.v_path[: self.batch * n].view(self.batch, n)
        acc, path, bonus = _ext.tree_accept_greedy(tokens.contiguous(), tree_mask.contiguous(), target.contiguous(), self.v_accept_len, path,
                                                   self.v_bonus)
        _ext.kv_cache_compact(self.block_tables, self.v_start, path, acc, self.Hkv, 64, self.size_per_token, self.kv_bits == 4)
        return acc, path, bonus

    def accept_sampled_and_compact(self, tokens: torch.Tensor, tree_mask: torch.Tensor, logits: torch.Tensor, draft_probs: Optional[torch.Tensor] = None):
        """accept_and_compact with sampled acceptance: after verify_forward(tokens, return_logits=True, tree_mask=tree_mask) returned the logits
        [B, n, vocab], tree_accept_sampling with the runner's per-row sampling parameters (s_temperature, s_top_k, s_top_p, s_seed,
        s_offsets advanced by one) and draft_probs (fp32 [B, n, vocab] or None: one-hot drafts), then kv_cache_compact of the accepted path.
        Returns (accept_len, path, bonus) in v_accept_len, v_path and v_bonus."""
        n = tokens.size(1)
        path = self.v_path[: self.batch * n].view(self.batch, n)
        acc, path, bonus = _ext.tree_accept_sampling(tokens.contiguous(), tree_mask.contiguous(), logits, self.s_temperature, self.s_top_k, self.s_top_p,
                                                     self.s_seed, self.s_offsets, draft_probs, self.v_accept_len, path, self.v_bonus)
        _ext.kv_cache_compact(self.block_tables, self.v_start, path, acc, self.Hkv, 64, self.size_per_token, self.kv_bits == 4)
        return acc, path, bonus

    def draft_probs_view(self, n: int) -> torch.Tensor:
        """The [B, n, vocab] fp32 draft distributions the sampled tree graph for n nodes reads (capture_verify(..., draft_probs=True))."""
        return self.v_draft_probs[: self.batch * n * self.cfg.vocab].view(self.batch, n, self.cfg.vocab)

    def _verify_graph_body(self, n: int, tree: bool, sampled: bool = False, draft_probs: bool = False) -> None:
        tin, tout = self.v_tokens_in[:, :n].contiguous(), self.v_tokens_out[:, :n]
        if sampled:
            mask = self.v_tree_mask[:, :n].contiguous()
            logits = self.verify_forward(tin, return_logits=True, tree_mask=mask)
            self.accept_sampled_and_compact(tin, mask, logits, self.draft_probs_view(n) if draft_probs else None)
            return
        if not tree:
            tout.copy_(self.verify_forward(tin))
            return
        mask = self.v_tree_mask[:, :n].contiguous()
        tout.copy_(self.verify_forward(tin, tree_mask=mask))
        self.accept_and_compact(tin, mask, tout)

    def _verify_key(self, n: int, tree: bool, sampled: bool, draft_probs: bool):
        return ("verify", int(n), bool(tree or sampled), bool(sampled), bool(sampled and draft_probs))

    def capture_verify(self, n: int, warmup: int = 2, tree: bool = False, sampled: bool = False, draft_probs: bool = False) -> None:
        """Capture the verify step for n draft tokens in a CUDA graph: v_tokens_in[:, :n] -> v_tokens_out[:, :n].  tree=True: the graph
        also reads v_tree_mask[:, :n] and runs accept_and_compact (v_accept_len, v_path, v_bonus).  sampled=True (needs tree=True): verify
        -> accept_sampled_and_compact -> the same outputs, with the per-row sampling parameters; draft_probs=True allocates v_draft_probs
        (fp32 [B, verify_len, vocab], filled through draft_probs_view(n)) and reads it as q, otherwise the drafts are one-hot.  The warm-up
        runs the step eagerly, so it writes the draft slots (and, with tree=True, compacts them) like a replay does."""
        assert not sampled or tree, "sampled acceptance runs on the tree step (a chain is a tree with mask (1 << i) - 1)"
        if sampled and draft_probs and self.v_draft_probs is None:
            self.v_draft_probs = torch.zeros(self.batch * self.verify_len * self.cfg.vocab, dtype=torch.float32, device=self.dev)
        self._capture(self._verify_key(n, tree, sampled, draft_probs), lambda: self._verify_graph_body(n, tree, sampled, draft_probs), warmup)

    def verify_step(self, n: int, tree: bool = False, sampled: bool = False, draft_probs: bool = False) -> None:
        """Replay the captured verify step for n draft tokens."""
        self.graphs[self._verify_key(n, tree, sampled, draft_probs)].replay()

    # ---------------------------------------------------------------------------------------------------------
    # generation: plain decode steps and prompt-lookup speculative steps that advance every row by what it accepted
    # ---------------------------------------------------------------------------------------------------------
    def _alloc_generate_buffers(self) -> None:
        """Row state and step buffers of the generation loop (torch.full / torch.zeros: no random draws)."""
        B, dev, n = self.batch, self.dev, max(1, self.verify_len)
        self.g_budget = torch.full((B,), self.max_new_tokens, dtype=torch.int32, device=dev)
        self.g_eos = torch.full((B,), -1, dtype=torch.int64, device=dev)
        self.g_stop = torch.full((B, _ext.MAX_STOP_TOKENS), -1, dtype=torch.int64, device=dev)  # SamplingParams.stop_token_ids, -1 pads
        self.g_logprob = None  # fp32 [B, W] and the top-n buffers: allocated by the first step with logprobs > 0 (before any capture)
        self.g_top_n = 0
        self.g_finished = torch.zeros(B, dtype=torch.int32, device=dev)
        # the verify step's cached length P = L - 1 (the verify step's v_start when there is one)
        self.g_start = self.v_start if self.verify_len else torch.full((B,), self.ctx, dtype=torch.int32, device=dev)
        self.g_path1 = torch.zeros((B, 1), dtype=torch.int32, device=dev)  # a plain step commits the path [0] ...
        self.g_accept1 = torch.ones(B, dtype=torch.int32, device=dev)      # ... of length 1, so only its token is appended
        # drafts of the speculative step, flat so that [:B n] viewed as [B, n] is contiguous for any n
        self.g_tokens = torch.zeros(B * n, dtype=torch.int64, device=dev)
        self.g_mask = torch.zeros(B * n, dtype=torch.int32, device=dev)

    def _alloc_generate_logprobs(self, n: int) -> None:
        """g_logprob fp32 [B, W] (W = s_history.size(1)) and the flat top-n buffers behind g_top_view, on first use (torch.full: no random
        draws).  Column c holds the entry of history token c."""
        B, W = self.s_history.shape
        if self.g_logprob is None:
            self.g_logprob = torch.full((B, W), float("nan"), dtype=torch.float32, device=self.dev)
            self._g_top_ids = torch.full((B * W * _ext.MAX_TOP_LOGPROBS,), -1, dtype=torch.int64, device=self.dev)
            self._g_top_logprobs = torch.full((B * W * _ext.MAX_TOP_LOGPROBS,), float("nan"), dtype=torch.float32, device=self.dev)
        self.g_top_n = n

    def g_top_view(self, n: int):
        """(top ids int64 [B, W, n], top log-probabilities fp32 [B, W, n]): the history-aligned top-n entries a step with logprobs = n writes."""
        B, W = self.s_history.shape
        return self._g_top_ids[: B * W * n].view(B, W, n), self._g_top_logprobs[: B * W * n].view(B, W, n)

    def reset_generation(self, prompt: torch.Tensor) -> None:
        """Start generating after prompt int64 [batch, ctx + 1]: the ctx tokens the pages hold, then the root (the latest token, not yet
        cached).  Sets the history and its lengths, the positions of both step kinds and tokens_in, and clears g_finished; g_budget, g_eos
        and g_stop stay as the caller set them."""
        assert self.generate, "construct the runner with generate=True"
        B, C = self.batch, self.ctx + 1
        assert tuple(prompt.shape) == (B, C) and prompt.dtype == torch.int64, f"prompt must be int64 [{B}, {C}]"
        self.s_history.fill_(-1)
        self.s_history[:, :C].copy_(prompt)
        self.s_prompt_lens.fill_(C)
        self.s_seq_lens.fill_(C)
        self.g_start.fill_(self.ctx)
        self.context_lens.fill_(C)
        self.tokens_in.copy_(prompt[:, self.ctx])
        self.g_finished.zero_()

    def generate_forward(self, n: int = 1, branches: int = 1, ngram: tuple = (1, 4), sampled: bool = False, penalties: bool = False,
                         logprobs: int = 0) -> None:
        """One generation step for every row; the tokens go to s_history (lengths s_seq_lens).  n = 1: the decode step at the rows' own
        lengths, argmax_rows (or sample_rows with the s_* parameters if sampled), spec_commit of that token.  2 <= n <= verify_len:
        ngram_propose (n nodes, `branches` continuations, match lengths ngram = (n_min, n_max)) -> verify_forward of the draft tree ->
        accept_and_compact (or accept_sampled_and_compact with one-hot drafts, which keeps sampling lossless) -> spec_commit.  The commit
        ends a row at g_eos, at any token of g_stop and at g_budget.  Finished rows (g_finished) are computed but not advanced.  No host
        synchronisation.

        penalties=True: the logits first go through apply_penalties (n = 1; the history up to and including the root) or apply_penalties_tree
        (every draft node's row penalised as the sequential step at its position would be, so acceptance stays exact) with s_repetition,
        s_presence and s_frequency.  logprobs = k (1 .. 20): logprobs_accepted of the (penalised) logits before the commit: the entry of history
        token c goes to g_logprob[b, c] and g_top_view(k)[.][b, c], valid for s_prompt_lens[b] <= c < s_seq_lens[b]."""
        assert self.generate, "construct the runner with generate=True"
        logprobs = int(logprobs)
        assert 0 <= logprobs <= _ext.MAX_TOP_LOGPROBS, f"logprobs={logprobs}: 0 .. {_ext.MAX_TOP_LOGPROBS}"
        if logprobs:
            self._alloc_generate_logprobs(logprobs)
        B = self.batch
        common = (self.s_history, self.s_seq_lens, self.s_prompt_lens, self.g_budget, self.g_eos, self.g_finished, self.g_start, self.context_lens,
                  self.tokens_in)
        if n == 1:
            logits = self._forward_fused(self.tokens_in, True)
            tok = self._pick(logits, sampled, penalties, logprobs, out=self.tokens_out)
            if logprobs:
                _ext.logprobs_accepted(logits.view(B, 1, -1), tok.view(B, 1), self.g_path1, self.g_accept1, tok, self.s_seq_lens, self.g_finished,
                                       logprobs, self.g_logprob, *self.g_top_view(logprobs))
            # the path [0] of length 1 never reads the drafts: any [B, 1] tensor that is not an output will do
            _ext.spec_commit(tok.view(B, 1), self.g_path1, self.g_accept1, tok, *common, stop_ids=self.g_stop)
            return
        assert 2 <= n <= self.verify_len, f"n={n}: 1, or 2 .. verify_len={self.verify_len}"
        n_min, n_max = ngram
        toks = self.g_tokens[: B * n].view(B, n)
        mask = self.g_mask[: B * n].view(B, n)
        _ext.ngram_propose(self.s_history, self.s_seq_lens, n, n_min, n_max, branches, tokens=toks, tree_mask=mask)
        emb = toks.clamp(min=0)  # padding nodes (-1) are embedded as token 0; they are never accepted
        if sampled or penalties or logprobs:
            logits = self.verify_forward(emb, return_logits=True, tree_mask=mask)
            if penalties:
                _ext.apply_penalties_tree(logits, toks, mask, self.s_history, self.s_prompt_lens, self.s_seq_lens, self.s_repetition, self.s_presence,
                                          self.s_frequency)
            if sampled:
                acc, path, bonus = self.accept_sampled_and_compact(toks, mask, logits, None)
            else:
                acc, path, bonus = self.accept_and_compact(toks, mask, _ext.argmax_rows(logits.view(B * n, -1)).view(B, n))
            if logprobs:
                _ext.logprobs_accepted(logits, toks, path, acc, bonus, self.s_seq_lens, self.g_finished, logprobs, self.g_logprob,
                                       *self.g_top_view(logprobs))
        else:
            target = self.verify_forward(emb, tree_mask=mask)
            acc, path, bonus = self.accept_and_compact(toks, mask, target)
        _ext.spec_commit(toks, path, acc, bonus, *common, stop_ids=self.g_stop)

    def _generate_key(self, n: int, branches: int, ngram: tuple, sampled: bool, penalties: bool = False, logprobs: int = 0):
        extra = (bool(penalties), int(logprobs)) if penalties or logprobs else ()  # the keys without the sampler flags are those of before
        return ("generate", int(n), int(branches), tuple(int(x) for x in ngram), bool(sampled)) + extra + (self._sp_key() if n == 1 else ())

    def capture_generate(self, n: int = 1, branches: int = 1, ngram: tuple = (1, 4), sampled: bool = False, warmup: int = 2, penalties: bool = False,
                         logprobs: int = 0) -> None:
        """Capture generate_forward(n, branches, ngram, sampled, penalties, logprobs) in a CUDA graph.  The warm-up runs the step eagerly, so
        it advances the rows like a replay does (and allocates the log-probability buffers): call reset_generation afterwards."""
        self._capture(self._generate_key(n, branches, ngram, sampled, penalties, logprobs),
                      lambda: self.generate_forward(n, branches, ngram, sampled, penalties, logprobs), warmup)

    def generate_step(self, n: int = 1, branches: int = 1, ngram: tuple = (1, 4), sampled: bool = False, penalties: bool = False,
                      logprobs: int = 0) -> None:
        """Replay the captured generation step."""
        self.graphs[self._generate_key(n, branches, ngram, sampled, penalties, logprobs)].replay()

    # ---------------------------------------------------------------------------------------------------------
    # prompt step: prefill every row's prompt into its pages, whole or in chunks, then the first token and the hand-off to generation
    # ---------------------------------------------------------------------------------------------------------
    def prefill(self, prompts: torch.Tensor, lens: torch.Tensor, chunk: Optional[int] = None, sample: bool = False, penalties: bool = False,
                logprobs: int = 0, prompt_logprobs: int = 0) -> torch.Tensor:
        """Prefill prompts int64 [batch, >= max(lens)] with lens int32 [batch] (1 <= lens[b] <= ctx) into positions 0 .. lens[b] - 1 of every
        row's pages in every layer; returns the first tokens int64 [batch].  Eager, one host synchronisation (the lengths plan the pieces).

        Per layer: the qkv GEMM at M = the piece's tokens, then chunk=None: apply_bias_rope_update_kv_cache and flash_attn_varlen_func over
        the whole prompts (llama_w4a8_unpad.py:199-242); chunk=C: pieces of at most C tokens per row, each appended with
        apply_bias_rope_update_kv_cache_at at the row's cached length and attended with prefix_prefill_attention over the dequantised prefix
        (rows whose prompt is done take 0 tokens); then invoke_quant[_fuse_sum], o, gate_up, silu+quant and down as the fused decode step.
        A piece holds at most prompt_tokens tokens.  Only each row's last position goes through the final norm and lm_head (:471-475); the
        first token then comes out of the composition of forward (sample, penalties, logprobs as there; penalties see the prompt only).

        prompt_logprobs = n (1 .. 20): p_logprob fp32, p_top_ids int64 [., n] and p_top_logprobs fp32 [., n], flat over the prompts by
        cu_seqlens = [0, lens[0], lens[0] + lens[1], ...]: entry cu[b] + i (i >= 1) is the log-probability of prompt token i given tokens
        0 .. i - 1 and the top n there (logprobs_rows of the unpenalised logits); entry cu[b] (the first token) is NaN with top ids -1.  The
        lm_head runs over blocks of prompt rows, never over all of them at once.

        Hand-off: the block tables get every row's own pages back (undoing fork), context_lens = lens + 1, tokens_in = the first token, and
        v_start / g_start = lens where they exist.  With max_new_tokens > 0: s_history[b] = the prompt, the first token at lens[b], then -1;
        s_prompt_lens = lens and s_seq_lens = lens + 1 (the first token counts as generated).  With generate=True, g_finished[b] = 1 when the
        first token is g_eos[b], one of g_stop[b] or g_budget[b] <= 1, and with logprobs = n the first token's entry goes to column lens[b] of
        g_logprob / g_top_view(n); generate_forward continues from there."""
        assert self.prompt_tokens, "construct the runner with prompt_tokens > 0"
        assert self.max_new_tokens or not (penalties or logprobs), "construct the runner with max_new_tokens > 0 for penalties / logprobs"
        B, cfg, dev = self.batch, self.cfg, self.dev
        if not (lens.dtype == torch.int32 and tuple(lens.shape) == (B,)):
            raise RuntimeError(f"lens must be int32 [{B}], got {lens.dtype} {tuple(lens.shape)}")
        lens_h = [int(x) for x in lens.tolist()]
        pieces = prompt_pieces(lens_h, self.ctx, self.prompt_tokens, chunk)
        if not (prompts.dtype == torch.int64 and prompts.dim() == 2 and prompts.size(0) == B and prompts.size(1) >= max(lens_h)):
            raise RuntimeError(f"prompts must be int64 [{B}, >= {max(lens_h)}], got {prompts.dtype} {tuple(prompts.shape)}")
        if not 0 <= int(prompt_logprobs) <= _ext.MAX_TOP_LOGPROBS:
            raise RuntimeError(f"prompt_logprobs={prompt_logprobs}: 0 .. {_ext.MAX_TOP_LOGPROBS}")
        prompts, lens = prompts.to(dev), lens.to(dev)
        cu_all = [0]
        for n in lens_h:
            cu_all.append(cu_all[-1] + n)
        if prompt_logprobs:
            self._alloc_prompt_logprobs(cu_all, int(prompt_logprobs))
        self.block_tables.copy_(self.own_tables)
        if self.shared_prefix:
            self._set_groups([])
        D, int4, max_pos = cfg.head_dim, self.kv_bits == 4, min(8192, cfg.max_pos)
        last = torch.empty((B, cfg.hidden), dtype=torch.half, device=dev)
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)
        for start, c in pieces:
            T, maxc = sum(c), max(c)
            cu_h = [0]
            for n in c:
                cu_h.append(cu_h[-1] + n)
            rows = [b for b in range(B) for _ in range(c[b])]
            cols = [start + j for b in range(B) for j in range(c[b])]
            tokens = prompts[torch.tensor(rows, device=dev), torch.tensor(cols, device=dev)]
            cu, clens = i32(cu_h), i32(c)
            pad = _ext.compute_padding_offsets(cu, maxc, T)
            if chunk is None:
                def attention(li, r):  # llama_w4a8_unpad.py:199-243
                    _ext.apply_bias_rope_update_kv_cache(r.qkv, clens, pad, self.block_tables[li], self.Hq, self.Hkv, maxc, 64, self.size_per_token, D,
                                                         cfg.rope_theta, max_pos, True, int4, True)
                    attn = _ext.flash_attn_varlen_func(*self._heads(r.qkv), cu_seqlens_q=cu, cu_seqlens_k=cu, max_seqlen_q=maxc, max_seqlen_k=maxc,
                                                       dropout_p=0.0, causal=True)
                    self._quant(r, r.q_attn, attn.view(T, -1))
            else:
                prefix = i32([min(n, start) for n in lens_h])

                def attention(li, r):
                    table = self.block_tables[li]
                    _ext.apply_bias_rope_update_kv_cache_at(r.qkv, clens, pad, prefix, table, self.Hq, self.Hkv, maxc, 64, self.size_per_token, D,
                                                            cfg.rope_theta, max_pos, True, int4, True)
                    attn = _ext.prefix_prefill_attention(*self._heads(r.qkv), cu, maxc, prefix, start, table, 64, self.size_per_token, int4)
                    self._quant(r, r.q_attn, attn.view(T, -1))

            hidden, _ = self._fused_layers(self.embed[tokens], self._row_views(T), attention)
            done = [b for b in range(B) if c[b] and start + c[b] == lens_h[b]]
            if done:
                last[torch.tensor(done, device=dev)] = hidden[torch.tensor([cu_h[b + 1] - 1 for b in done], device=dev)]
            if prompt_logprobs:
                self._prompt_logprobs(hidden, prompts, start, c, cu_h, cu_all, int(prompt_logprobs))
        self.last_prompt_hidden = last
        logits = self._logits(last)
        self.last_logits = logits
        if self.max_new_tokens:
            W = self.s_history.size(1)
            w = min(W, prompts.size(1))
            hist = torch.full((B, W), -1, dtype=torch.int64, device=dev)
            hist[:, :w] = prompts[:, :w]
            self.s_history.copy_(torch.where(torch.arange(W, device=dev) < lens.unsqueeze(1), hist, -1))
            self.s_prompt_lens.copy_(lens)
            self.s_seq_lens.copy_(lens)
        tok = self._next_tokens(logits, sample, penalties, logprobs, out=self.tokens_out)
        if self.max_new_tokens and not (penalties or logprobs):  # _next_tokens appends only when it penalises or scores
            self.s_history.scatter_(1, self.s_seq_lens.long().unsqueeze(1), tok.unsqueeze(1))
            self.s_seq_lens.add_(1)
        self.context_lens.copy_(lens + 1)
        if self.verify_len:
            self.v_start.copy_(lens)
        if self.generate:
            self.g_start.copy_(lens)
            stop = (tok.unsqueeze(1) == self.g_stop).any(dim=1)  # tokens are >= 0: the -1 pads never match
            self.g_finished.copy_(((tok == self.g_eos) | stop | (self.g_budget <= 1)).to(torch.int32))
            if logprobs:  # the first token's entry at its history column lens[b]
                self._alloc_generate_logprobs(int(logprobs))
                rows, col = torch.arange(B, device=dev), lens.long()
                self.g_logprob[rows, col] = self.s_logprob
                for dst, src in zip(self.g_top_view(int(logprobs)), self.top_logprobs_view(int(logprobs))):
                    dst[rows, col] = src
        self.tokens_in.copy_(tok)
        return tok.clone()

    def _alloc_prompt_logprobs(self, cu_all: list, n: int) -> None:
        """p_logprob / p_top_ids / p_top_logprobs as views of buffers grown to the prompts of cu_all, the first entry of every prompt NaN / -1."""
        total = cu_all[-1]
        if self._p_logprob is None or self._p_logprob.numel() < total:
            self._p_logprob = torch.zeros(total, dtype=torch.float32, device=self.dev)
            self._p_top_ids = torch.zeros(total * _ext.MAX_TOP_LOGPROBS, dtype=torch.int64, device=self.dev)
            self._p_top_logprobs = torch.zeros(total * _ext.MAX_TOP_LOGPROBS, dtype=torch.float32, device=self.dev)
        self.p_logprob = self._p_logprob[:total]
        self.p_top_ids = self._p_top_ids[: total * n].view(total, n)
        self.p_top_logprobs = self._p_top_logprobs[: total * n].view(total, n)
        first = torch.tensor(cu_all[:-1], device=self.dev)
        self.p_logprob[first] = float("nan")
        self.p_top_ids[first] = -1
        self.p_top_logprobs[first] = float("nan")

    def _prompt_logprobs(self, hidden, prompts, start: int, c: list, cu_h: list, cu_all: list, n: int) -> None:
        """The prompt log-probabilities the rows of one piece give: position start + j of row b (hidden row cu_h[b] + j) scores prompt
        token start + j + 1, written at cu_all[b] + start + j + 1; the lm_head runs over blocks of rows."""
        # (hidden row, output entry, row, position of the scored token) of every position but each prompt's last
        m = [(cu_h[b] + j, cu_all[b] + start + j + 1, b, start + j + 1) for b in range(self.batch) for j in range(c[b])
             if start + j + 1 < cu_all[b + 1] - cu_all[b]]
        if not m:
            return
        src, dst, row, pos = torch.tensor(m, device=self.dev).unbind(1)
        targets = prompts[row, pos]
        rows = max(1, _PROMPT_LOGITS_BYTES // (2 * self.cfg.vocab))
        for i in range(0, src.numel(), rows):
            logits = self._logits(hidden[src[i:i + rows]])
            lp, ids, tlp = _ext.logprobs_rows(logits, targets[i:i + rows].contiguous(), n)
            d = dst[i:i + rows]
            self.p_logprob[d] = lp
            self.p_top_ids[d] = ids
            self.p_top_logprobs[d] = tlp

    def fork(self, parent_rows, child_rows) -> None:
        """Copy-on-write fork between steps (SamplingParams.n / best_of: prefill a prompt once, decode n rows from it).  parent_rows: one row or
        one per child; child_rows: rows that are not parents.  With P = the parent's cached tokens (context_lens - 1): in every layer the child's
        block-table entries 0 .. P // 64 - 1 point at the parent's pages (shared and read-only from then on: a child writes only at positions
        >= P), the rest at the child's own pages; kv_cache_fork copies the parent's partial tail page into the child's own page; the child
        gets the parent's history, s_prompt_lens, s_seq_lens, context_lens, g_start / v_start, tokens_in, g_budget, g_eos, g_stop, g_finished,
        penalty parameters and history-aligned log-probabilities.  s_offsets and the sampling parameters stay the child's own, so sampled children diverge.  Eager; the table
        entries are written with torch ops (the attention kernels read the tables before their dependency wait)."""
        children = list(child_rows) if not isinstance(child_rows, int) else [child_rows]
        parents = [parent_rows] * len(children) if isinstance(parent_rows, int) else list(parent_rows)
        parents, children = _ext.fork_pairs(parents, children, self.batch)
        if not children:
            return
        dev = self.dev
        par, chi = torch.tensor(parents, device=dev), torch.tensor(children, device=dev)
        cached = (self.context_lens - 1).contiguous()
        shared = torch.arange(self.table_blocks, device=dev).unsqueeze(0) < (cached[par] // 64).unsqueeze(1)  # [pairs, blocks]
        self.block_tables[:, chi] = torch.where(shared[None, :, None, :], self.block_tables[:, par], self.own_tables[:, chi])
        _ext.kv_cache_fork(self.block_tables, parents, children, cached, self.Hkv, 64, self.size_per_token, self.kv_bits == 4)
        names = ["context_lens", "tokens_in", "s_history", "s_prompt_lens", "s_seq_lens", "s_repetition", "s_presence", "s_frequency", "v_start",
                 "g_start", "g_budget", "g_eos", "g_stop", "g_finished", "g_logprob"]
        state = [getattr(self, a) for a in names if getattr(self, a, None) is not None]
        if getattr(self, "g_logprob", None) is not None:
            state += list(self.g_top_view(self.g_top_n))
        for t in {id(t): t for t in state}.values():  # g_start may alias v_start
            t[chi] = t[par]
        if self.shared_prefix:
            self._set_groups(fork_groups(self.sp_groups, parents, children, cached.tolist()))

    # ---------------------------------------------------------------------------------------------------------
    # beam search: W beams per request; selection and re-parenting of every beam's pages on the GPU, inside the captured step
    # ---------------------------------------------------------------------------------------------------------
    def _alloc_beam_buffers(self) -> None:
        """Beam state (torch.full / torch.zeros: no random draws)."""
        B, W, T, dev = self.batch, self.beam_width, self.max_new_tokens, self.dev
        R = B // W
        self.b_live = torch.zeros(B, dtype=torch.int32, device=dev)
        self.b_cum = torch.zeros(B, dtype=torch.float32, device=dev)
        self.b_parent = torch.full((B,), -1, dtype=torch.int32, device=dev)
        self.b_length_penalty = torch.full((R,), 1.0, dtype=torch.float32, device=dev)
        self.b_early_stopping = torch.zeros(R, dtype=torch.int32, device=dev)  # 0 False, 1 True, 2 "never"
        self.b_eos = torch.full((R,), -1, dtype=torch.int64, device=dev)
        self.b_stop = torch.full((R, _ext.MAX_STOP_TOKENS), -1, dtype=torch.int64, device=dev)
        self.b_budget = torch.full((R,), T, dtype=torch.int32, device=dev)
        self.b_done = torch.zeros(R, dtype=torch.int32, device=dev)
        self.b_pool = _ext.beam_pool(R, W, T, dev)
        # the step's candidates: logprobs_rows with n = 2 W (b_logprob is its unused per-row output)
        self.b_top_ids = torch.zeros((B, 2 * W), dtype=torch.int64, device=dev)
        self.b_top_logprobs = torch.zeros((B, 2 * W), dtype=torch.float32, device=dev)
        self.b_logprob = torch.zeros(B, dtype=torch.float32, device=dev)
        self.max_model_len = self.ctx + T

    def _beam_tail(self, logits: torch.Tensor) -> None:
        """logits -> the 2 W candidates of every beam -> beam_select -> beam_reorder."""
        W = self.beam_width
        _ext.logprobs_rows(logits, self.tokens_in, 2 * W, self.b_logprob, self.b_top_ids, self.b_top_logprobs)
        _ext.beam_select(self.b_top_ids, self.b_top_logprobs, self.b_live, self.b_cum, self.s_seq_lens, self.context_lens, self.tokens_in, self.b_parent,
                         self.s_prompt_lens, self.s_history, self.b_length_penalty, self.b_early_stopping, self.b_eos, self.b_stop, self.b_budget,
                         self.b_done, self.b_pool, self.max_model_len)
        # the next step begins with the embedding gather, a launch without PDL: the attention kernels, which read the tables and context_lens
        # before their dependency wait, see the reorder's writes
        _ext.beam_reorder(self.block_tables, self.b_parent, self.context_lens, self.s_prompt_lens, self.tokens_in, self.s_history, W, self.Hkv, 64,
                          self.size_per_token, self.kv_bits == 4)

    def beam_start(self, prompts: torch.Tensor, lens: torch.Tensor, chunk: Optional[int] = None, penalties: bool = False) -> None:
        """Start a beam search for R = batch / W prompts: prompts int64 [R, >= max(lens)], lens int32 [R] (1 <= lens[r] <= ctx).  Prompt r is
        prefilled into row r W (the other rows of the request get a 1-token prompt, so the prompt is computed once); then every row of
        request r takes its prompt as history (s_history, s_prompt_lens = s_seq_lens = lens[r]), slot r W is the only live beam with cum 0,
        the pool is emptied, and the first beam step runs on the prefill logits (apply_penalties first if penalties): logprobs_rows with
        n = 2 W, beam_select and beam_reorder with every running child's parent r W.  b_length_penalty, b_early_stopping, b_eos, b_stop and
        b_budget stay as the caller set them.  With shared_prefix=True each request's rows become one group sharing lens[r] // 64 pages: the
        reorder never changes table entries below that, so the layout holds for the whole search.  Eager, with prefill's host synchronisation."""
        assert self.beam_width, "construct the runner with beam_width > 0"
        B, W, dev = self.batch, self.beam_width, self.dev
        R = B // W
        if not (lens.dtype == torch.int32 and tuple(lens.shape) == (R,)):
            raise RuntimeError(f"lens must be int32 [{R}], got {lens.dtype} {tuple(lens.shape)}")
        if not (prompts.dtype == torch.int64 and prompts.dim() == 2 and prompts.size(0) == R):
            raise RuntimeError(f"prompts must be int64 [{R}, >= max(lens)], got {prompts.dtype} {tuple(prompts.shape)}")
        lens_h = [int(x) for x in lens.tolist()]
        prompts, lens = prompts.to(dev), lens.to(dev)
        first = torch.arange(R, device=dev) * W
        full = torch.zeros((B, prompts.size(1)), dtype=torch.int64, device=dev)
        full[first] = prompts
        full_lens = torch.ones(B, dtype=torch.int32, device=dev)
        full_lens[first] = lens
        self.prefill(full, full_lens, chunk, penalties=penalties)
        logits = self.last_logits  # penalised in place by prefill when penalties
        rows = torch.arange(B, device=dev) // W * W
        self.s_prompt_lens.copy_(self.s_prompt_lens[rows])
        self.s_seq_lens.copy_(self.s_prompt_lens)  # prefill appended its first token: drop it
        cols = torch.arange(self.s_history.size(1), device=dev)
        self.s_history.copy_(torch.where(cols < self.s_prompt_lens.unsqueeze(1), self.s_history[rows], -1))
        self.b_live.zero_()
        self.b_live[first] = 1
        self.b_cum.zero_()
        self.b_parent.fill_(-1)
        self.b_done.zero_()
        self.b_pool.tokens.fill_(-1)
        for t in self.b_pool[1:]:
            t.zero_()
        self._beam_tail(logits)
        if self.shared_prefix:
            self._set_groups([(tuple(range(r * W, r * W + W)), lens_h[r] // 64) for r in range(R)])

    def beam_forward(self, penalties: bool = False) -> None:
        """One beam step for every request: the decode step at the beams' own lengths (tokens_in, context_lens), apply_penalties (s_history,
        s_prompt_lens, s_seq_lens, s_repetition / s_presence / s_frequency) if penalties, logprobs_rows with n = 2 W, beam_select and
        beam_reorder.  Done requests and dead slots are computed but not advanced.  No host synchronisation."""
        assert self.beam_width, "construct the runner with beam_width > 0"
        logits = self._forward_fused(self.tokens_in, True)
        if penalties:
            _ext.apply_penalties(logits, self.s_history, self.s_prompt_lens, self.s_seq_lens, self.s_repetition, self.s_presence, self.s_frequency)
        self._beam_tail(logits)

    def _beam_key(self, penalties: bool) -> tuple:
        return ("beam", bool(penalties)) + self._sp_key()

    def capture_beam(self, penalties: bool = False, warmup: int = 2) -> None:
        """Capture beam_forward(penalties) in a CUDA graph.  The warm-up runs the step eagerly and advances the beams like a replay does: call
        beam_start afterwards.  With shared_prefix=True the key ends in the layout beam_start sets, so when that layout takes the shared route
        capture after beam_start (the warm-up then advances the search by `warmup` steps)."""
        self._capture(self._beam_key(penalties), lambda: self.beam_forward(penalties), warmup)

    def beam_step(self, penalties: bool = False) -> None:
        """Replay the captured beam step."""
        self.graphs[self._beam_key(penalties)].replay()

    def beam_results(self, n: Optional[int] = None) -> list:
        """Per request, its best n (default W) finished hypotheses, best first: (generated tokens, cumulative log-probability, score).  Reads
        the pool back to the host."""
        assert self.beam_width, "construct the runner with beam_width > 0"
        n = self.beam_width if n is None else int(n)
        pool = _ext.BeamPool(*(t.cpu() for t in self.b_pool))
        out = []
        for r in range(pool.count.numel()):
            c = min(int(pool.count[r]), n)
            out.append([(pool.tokens[r, q, : int(pool.length[r, q])].tolist(), float(pool.cum[r, q]), float(pool.score[r, q])) for q in range(c)])
        return out

    # ---------------------------------------------------------------------------------------------------------
    # in-flight batching: queued prompts enter rows as they free up; one step carries their prompt chunks and the decode tokens of the others
    # ---------------------------------------------------------------------------------------------------------
    def _alloc_inflight_buffers(self) -> None:
        """Queue, row state, step plan and per-request outputs (torch.full / torch.zeros: no random draws)."""
        B, C, T = self.batch, self.prompt_tokens, self.max_new_tokens
        self._alloc_generate_logprobs(0)  # g_logprob: the schedule hands the chosen tokens' log-probabilities to the outputs
        self.i_queue, self.i_rows, self.i_plan, self.i_out = _ext.inflight_buffers(B, self.inflight, C, self.ctx, T, self.dev)
        self._i_submitted = 0       # requests submitted (the host's tail)
        self._i_lens: dict = {}     # prompt length of every request not yet polled
        self._i_unpolled: set = set()
        self._i_staged: list = []   # pinned host tensors of copies still in flight (released by poll)
        self._i_polled = 0          # entries of the retired ring handed out by poll

    def submit(self, prompts, lens, max_tokens=None, eos=-1, stop=None, temperature=1.0, top_k=1, top_p=1.0, repetition=1.0, presence=0.0,
               frequency=0.0) -> list:
        """Queue requests: prompts int64 [n, >= max(lens)] (host or device), lens (host ints, 1 .. ctx); per request (a host scalar for all,
        or a host sequence of n) max_tokens (1 .. max_new_tokens, default max_new_tokens), eos (-1: none), stop (up to 8 ids per request), temperature,
        top_k, top_p, repetition, presence and frequency as the runner's per-row s_* parameters.  Returns the request ids (consecutive).
        Stream-ordered copies into the queue slots, then the tail advances; no host synchronisation.  Request r uses slot r % Q, so it may only
        be submitted once request r - Q has been returned by poll; raises RuntimeError otherwise (at most Q requests are outstanding)."""
        assert self.inflight, "construct the runner with inflight > 0"
        lens = [int(x) for x in (lens.tolist() if isinstance(lens, torch.Tensor) else lens)]
        n, Q, T, dev = len(lens), self.inflight, self.max_new_tokens, self.dev
        if n == 0:
            return []
        if min(lens) < 1 or max(lens) > self.ctx:
            raise RuntimeError(f"prompt lengths must lie in [1, ctx={self.ctx}], got {lens}")
        if not (isinstance(prompts, torch.Tensor) and prompts.dtype == torch.int64 and prompts.dim() == 2 and prompts.size(0) == n
                and prompts.size(1) >= max(lens)):
            raise RuntimeError(f"prompts must be int64 [{n}, >= {max(lens)}]")
        ids = list(range(self._i_submitted, self._i_submitted + n))
        busy = [r for r in ids if r - Q >= 0 and (r - Q) in self._i_unpolled]
        if busy or n > Q:
            raise RuntimeError(f"more than {Q} requests would be outstanding: poll the finished ones first")

        def per(v, name, conv):
            v = list(v) if isinstance(v, (list, tuple)) or (isinstance(v, torch.Tensor) and v.dim() > 0) else [v] * n
            if len(v) != n:
                raise RuntimeError(f"{name}: one value per request ({n}), got {len(v)}")
            return [conv(x) for x in v]
        mt = per(T if max_tokens is None else max_tokens, "max_tokens", int)
        if min(mt) < 1 or max(mt) > T:
            raise RuntimeError(f"max_tokens must lie in [1, max_new_tokens={T}], got {mt}")
        stops = [list(x) for x in (stop if stop is not None and len(stop) and isinstance(stop[0], (list, tuple)) else [stop or []] * n)]
        if len(stops) != n or any(len(x) > _ext.MAX_STOP_TOKENS for x in stops):
            raise RuntimeError(f"stop: up to {_ext.MAX_STOP_TOKENS} ids per request")
        f32 = lambda name, v: torch.tensor(per(v, name, float), dtype=torch.float32)
        i32 = lambda name, v: torch.tensor(per(v, name, int), dtype=torch.int32)
        host = {"lens": torch.tensor(lens, dtype=torch.int32), "max_tokens": torch.tensor(mt, dtype=torch.int32),
                "eos": torch.tensor(per(eos, "eos", int), dtype=torch.int64),
                "stop": torch.tensor([x + [-1] * (_ext.MAX_STOP_TOKENS - len(x)) for x in stops], dtype=torch.int64),
                "temperature": f32("temperature", temperature), "top_k": i32("top_k", top_k), "top_p": f32("top_p", top_p),
                "repetition": f32("repetition", repetition), "presence": f32("presence", presence), "frequency": f32("frequency", frequency)}
        # every host tensor goes through a pinned staging buffer and a non-blocking copy: a plain host-to-device copy from pageable memory
        # (torch.tensor(..., device=cuda) included) would wait for every step already queued on the stream
        slots = torch.tensor([r % Q for r in ids], dtype=torch.int64).pin_memory()
        self._i_staged.append(slots)
        slots = slots.to(dev, non_blocking=True)
        P = self.ctx
        rows = torch.full((n, P), -1, dtype=torch.int64, device=prompts.device)
        w = min(P, prompts.size(1))
        rows[:, :w] = prompts[:, :w]
        for name, t in [("prompts", rows)] + list(host.items()):
            if t.device.type == "cpu":
                t = t.pin_memory()
                self._i_staged.append(t)
            getattr(self.i_queue, name).index_copy_(0, slots, t.to(dev, non_blocking=True))
        self._i_submitted += n
        self.i_queue.counters[1].fill_(self._i_submitted)
        for r, ln in zip(ids, lens):
            self._i_lens[r] = ln
            self._i_unpolled.add(r)
        return ids

    def _inflight_schedule(self, chunk_budget: int) -> None:
        _ext.inflight_schedule(self.i_queue, self.i_rows, self.s_history, self.s_prompt_lens, self.s_seq_lens, self.s_temperature, self.s_top_k,
                               self.s_top_p, self.s_repetition, self.s_presence, self.s_frequency, self.g_eos, self.g_stop, self.g_budget,
                               self.s_offsets, self.g_finished, self.g_start, self.tokens_in, self.g_logprob, self.i_plan, self.i_out, chunk_budget)

    def inflight_forward(self, mixed: bool = True, sampled: bool = False, penalties: bool = False, logprobs: int = 0) -> None:
        """One in-flight step; no host synchronisation.  inflight_schedule (chunk budget C, or 0 when mixed=False: nothing is admitted and no
        prompt token is carried), then the layers over M = B + C rows (B without mixed): the B decode rows, idle ones at context length 0,
        and the chunk segment, whose padding slots are neither appended nor attended.  Per layer: single_query_attention_quant over the decode
        rows; apply_bias_rope_update_kv_cache_at + prefix_prefill_attention + invoke_quant[_fuse_sum] over the chunk segment (host bounds
        max_seqlen = C, max_prefix_len = ctx - 1).  The B logit rows (the decode rows, and for a row whose prompt completes the logit of its
        last prompt token) go through lm_head at M = B, then the sampler of generate_forward(1): apply_penalties if penalties, argmax_rows or
        sample_rows if sampled, logprobs_accepted if logprobs, spec_commit with the stop ids.  A completing row's first token is committed in
        the same step.

        sample_rows keys its Philox stream on the row index and s_offsets, which admission resets to 0 and every step advances (idle steps
        too): a sampled request's tokens are deterministic for a given submission script but depend on its row and on its neighbours."""
        assert self.inflight, "construct the runner with inflight > 0"
        logprobs = int(logprobs)
        assert 0 <= logprobs <= _ext.MAX_TOP_LOGPROBS, f"logprobs={logprobs}: 0 .. {_ext.MAX_TOP_LOGPROBS}"
        if logprobs:
            self._alloc_generate_logprobs(logprobs)
        B, C, cfg = self.batch, self.prompt_tokens, self.cfg
        M = B + C if mixed else B
        self._inflight_schedule(C if mixed else 0)
        plan = self.i_plan
        D, int4, max_pos = cfg.head_dim, self.kv_bits == 4, min(8192, cfg.max_pos)

        def attention(li, r):
            table = self.block_tables[li]
            q, k, v = self._heads(r.qkv)
            _ext.single_query_attention_quant(q[:B], k[:B], v[:B], table, plan.context_lens, max_pos, 64, self.size_per_token, self.max_seq_len, D,
                                              cfg.rope_theta, int4, True, r.q_attn[:B], r.q_scale[:B], r.q_sum[:B] if self.act_sum else None)
            if not mixed:
                return
            seg = r.qkv[B:]
            _ext.apply_bias_rope_update_kv_cache_at(seg, plan.chunk_lens, plan.padding_offset, plan.prefix_lens, table, self.Hq, self.Hkv, C, 64,
                                                    self.size_per_token, D, cfg.rope_theta, max_pos, True, int4, True)
            attn = _ext.prefix_prefill_attention(*self._heads(seg), plan.cu_seqlens, C, plan.prefix_lens, self.ctx - 1, table, 64, self.size_per_token,
                                                 int4)
            self._quant(r._replace(q_scale=r.q_scale[B:], q_sum=r.q_sum[B:]), r.q_attn[B:], attn.view(C, -1))

        hidden, n = self._fused_layers(self.embed[plan.tokens[:M]], self._row_views(M), attention)
        logits = self._logits(hidden.index_select(0, plan.logit_rows))
        self.launches_per_step = n + 3
        self.last_logits = logits
        tok = self._pick(logits, sampled, penalties, logprobs, out=self.tokens_out)
        if logprobs:
            _ext.logprobs_accepted(logits.view(B, 1, -1), tok.view(B, 1), self.g_path1, self.g_accept1, tok, self.s_seq_lens, self.g_finished,
                                   logprobs, self.g_logprob, *self.g_top_view(logprobs))
        _ext.spec_commit(tok.view(B, 1), self.g_path1, self.g_accept1, tok, self.s_history, self.s_seq_lens, self.s_prompt_lens, self.g_budget,
                         self.g_eos, self.g_finished, self.g_start, self.context_lens, self.tokens_in, stop_ids=self.g_stop)

    def _inflight_key(self, mixed: bool, sampled: bool, penalties: bool, logprobs: int) -> tuple:
        return ("inflight", bool(mixed), bool(sampled), bool(penalties), int(logprobs))

    def capture_inflight(self, mixed: bool = True, sampled: bool = False, penalties: bool = False, logprobs: int = 0, warmup: int = 2) -> None:
        """Capture inflight_forward(mixed, sampled, penalties, logprobs) in a CUDA graph.  The warm-up runs the step eagerly on the current
        state (it schedules, admits and advances rows like a replay does): capture before submitting."""
        self._capture(self._inflight_key(mixed, sampled, penalties, logprobs), lambda: self.inflight_forward(mixed, sampled, penalties, logprobs),
                      warmup)

    def inflight_step(self, mixed: bool = True, sampled: bool = False, penalties: bool = False, logprobs: int = 0) -> None:
        """Replay the captured in-flight step."""
        self.graphs[self._inflight_key(mixed, sampled, penalties, logprobs)].replay()

    def poll(self, flush: bool = False, logprobs: bool = False) -> "InflightPoll":
        """The requests retired since the last poll, in retire order, as (request id, tokens, reason) with reason "eos", "stop" or "budget"
        (with logprobs=True a fourth entry: the chosen tokens' log-probabilities, NaN for tokens of steps without logprobs), and the prompt
        tokens still to prefill (queued requests and prefilling rows): with none, the decode-only step (mixed=False) does the same work.
        flush=True first runs the schedule with chunk budget 0, which retires the rows the last step finished and admits nothing.  One host
        synchronisation."""
        assert self.inflight, "construct the runner with inflight > 0"
        if flush:
            self._inflight_schedule(0)
        q, rows, out = self.i_queue, self.i_rows, self.i_out
        snap = [t.to("cpu", non_blocking=True) for t in (q.counters, rows.phase, rows.done, self.s_prompt_lens, out.ids, out.length, out.reason,
                                                         out.tokens, out.logprob)]
        torch.cuda.current_stream(self.dev).synchronize()
        ctr, phase, done, plen, ids, length, reason, toks, lps = snap
        self._i_staged.clear()
        Q = self.inflight
        finished = []
        for i in range(self._i_polled, int(ctr[2])):
            r = int(ids[i % Q])
            s, k = r % Q, int(length[r % Q])
            entry = (r, toks[s, :k].tolist(), _ext.INFLIGHT_REASONS.get(int(reason[s]), "?"))
            finished.append(entry + (lps[s, :k].tolist(),) if logprobs else entry)
            self._i_unpolled.discard(r)
            self._i_lens.pop(r, None)
        self._i_polled = int(ctr[2])
        queued = sum(self._i_lens[r] for r in range(int(ctr[0]), self._i_submitted))
        prefilling = int(((plen - done) * (phase == _ext.INFLIGHT_PREFILL)).sum())
        return InflightPoll(finished, queued + prefilling)

    # ---------------------------------------------------------------------------------------------------------
    def load_shard_of(self, full: "DecodeRunner") -> None:
        """Make this tensor-parallel runner (rank tp_rank of tp_size) the shard of `full` (a tp_size = 1 runner of the same model /
        precision / batch / ctx living on the same or another device): weights by qserve_b200.tp (column parallel: the q | k | v and
        gate | up parts are sliced separately; row parallel: K slices of every band), KV pages by kv head, everything else replicated."""
        from qserve_b200 import tp

        r, n, dev = self.tp_rank, self.tp_size, self.dev
        assert full.tp_size == 1 and full.cfg == self.cfg and full.precision == self.precision and full.batch == self.batch and full.ctx == self.ctx
        assert self.cfg.kv_heads % n == 0, "KV-head replication (tp_size > kv_heads) is not needed by the benchmark models"
        D = self.cfg.head_dim

        def col_parts(lin, sizes):  # column-parallel shard of a fused layer: slice every part, then concatenate
            out, o = {}, 0
            attrs = ("weight", "wscale") if lin.mode == "w8" else ("qweight", "s1") + (("s1z",) if lin.mode == "chn" else ("s2_scales", "s2_zeros"))
            for a in attrs:
                t, pieces, o = getattr(lin, a), [], 0
                for sz in sizes:
                    if a in ("s2_scales", "s2_zeros"):
                        pieces.append(tp.shard_level2_columns(t[:, o:o + sz], r, n))
                    elif a in ("qweight", "weight"):
                        pieces.append(tp.shard_columns(t[o:o + sz], r, n))
                    else:
                        pieces.append(tp.shard_vector(t[o:o + sz], r, n))
                    o += sz
                out[a] = torch.cat(pieces, dim=1 if a in ("s2_scales", "s2_zeros") else 0).contiguous().to(dev)
            return out

        def row_parts(lin):
            out = {}
            if lin.mode == "w8":
                k = lin.K // n
                out["weight"] = lin.weight[:, r * k:(r + 1) * k].contiguous().to(dev)
                out["wscale"] = lin.wscale.to(dev)
            else:
                out["qweight"] = tp.shard_rows(lin.qweight, r, n).to(dev)
                out["s1"] = lin.s1.to(dev)
                if lin.mode == "chn":
                    out["s1z"] = lin.s1z.to(dev)
                else:
                    out["s2_scales"] = tp.shard_level2_rows(lin.s2_scales, r, n).to(dev)
                    out["s2_zeros"] = tp.shard_level2_rows(lin.s2_zeros, r, n).to(dev)
            return out

        def put(lin, parts):
            for a, t in parts.items():
                dst = getattr(lin, a)
                assert tuple(dst.shape) == tuple(t.shape), (a, dst.shape, t.shape)
                dst.copy_(t)

        cfg = self.cfg
        for mine, theirs in zip(self.layers, full.layers):
            put(mine["qkv"], col_parts(theirs["qkv"], (cfg.heads * D, cfg.kv_heads * D, cfg.kv_heads * D)))
            put(mine["gate_up"], col_parts(theirs["gate_up"], (cfg.intermediate, cfg.intermediate)))
            put(mine["o"], row_parts(theirs["o"]))
            put(mine["down"], row_parts(theirs["down"]))
            mine["ln1"].copy_(theirs["ln1"]); mine["ln2"].copy_(theirs["ln2"])
        self.norm_w.copy_(full.norm_w); self.embed.copy_(full.embed); self.lm_head.copy_(full.lm_head)
        # KV pages: [Hkv][64][D*bits/8] codes, then scales [Hkv][64], then zeros [Hkv][64]: this rank's kv heads
        Hf, Hl = full.Hkv, self.Hkv
        cb_f, cb_l = 64 * full.size_per_token, 64 * self.size_per_token
        for mine_p, full_p in zip(self.kpools + self.vpools, full.kpools + full.vpools):
            fp = full_p.to(dev)
            mine_p[:, :cb_l] = fp[:, :cb_f].reshape(-1, Hf, cb_f // Hf)[:, r * Hl:(r + 1) * Hl].reshape(-1, cb_l)
            meta_f = fp[:, cb_f:].reshape(-1, 2, Hf, 128)
            mine_p[:, cb_l:] = meta_f[:, :, r * Hl:(r + 1) * Hl].reshape(-1, 2 * Hl * 128)
        self.context_lens.copy_(full.context_lens)

    # ---------------------------------------------------------------------------------------------------------
    def _capture(self, key: tuple, body, warmup: int) -> torch.cuda.CUDAGraph:
        """Run body() `warmup` times eagerly on a side stream (allocates workspaces, sets kernel attributes), then capture it in a CUDA
        graph kept in graphs[key]."""
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(warmup):
                body()
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        g = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(g):
            body()
        self.graphs[key] = g
        return g

    def capture(self, warmup: int = 2, sample: bool = False, penalties: bool = False, logprobs: int = 0) -> None:
        """Warm up eagerly (allocates workspaces, sets kernel attributes) and capture the whole step in a CUDA graph.  sample=True: the step
        ends in sample_rows (see forward); each warm-up call and each replay advances s_offsets by one.  penalties / logprobs: see forward;
        each warm-up call and each replay appends one token to s_history.  The graph is kept under the key (sample, penalties, logprobs) of
        step and becomes self.graph."""
        self._graph_key = ("decode", bool(sample), bool(penalties), int(logprobs)) + self._sp_key()
        self.graph = self._capture(self._graph_key, lambda: self.tokens_out.copy_(self.forward(self.tokens_in, sample, penalties, logprobs)), warmup)

    def step(self, key: Optional[tuple] = None) -> None:
        """Replay the captured step: tokens_in -> tokens_out (both device resident).  key = (sample, penalties, logprobs) selects one of
        the captures; None replays the latest.  With shared_prefix, a capture made under another layout plan is not replayed: KeyError for
        a key, RuntimeError for None."""
        if key is None and self.shared_prefix and self.graph is not None and self._graph_key[4:] != self._sp_key():
            raise RuntimeError("the latest capture was made under another shared-prefix layout: capture again after fork / prefill")
        (self.graph if key is None else self.graphs[("decode", *key) + self._sp_key()]).replay()

    def weight_bytes_per_step(self) -> int:
        return sum(l.weight_bytes() for ly in self.layers for l in (ly["qkv"], ly["o"], ly["gate_up"], ly["down"]))

    def kv_bytes_per_step(self) -> int:
        """Algorithmic KV traffic (SURVEY.md 8d): codes + scale/zero of K and V for ctx tokens, + q in / o out."""
        B, D = self.batch, self.cfg.head_dim
        per_layer = B * self.Hkv * self.ctx * D * self.kv_bits // 8 * 2 + B * self.Hkv * self.ctx * 8 + 4 * B * self.Hq * D
        return per_layer * self.L
