"""Decode-step harness: the reference's per-layer operator sequence (python/pyhie/allspark/model/qwen_v15.py:206-379,
SURVEY.md §1) driven through the b200spark C ABI, with synthetic weights and CUDA-graph replay.

This is measurement/test scaffolding around the hot path (the reference's AsModel::GenerateContinueDecoder loop,
csrc/core/model/model.cpp:1212-1323, stays the real caller); it owns no numerics of its own: every tensor op is a
library kernel.

Graph per layer (reference order, with the fusions the C ABI offers):
  RMSNorm -> GemmA16Wx(QKV,+bias) -> [Rotary + cache append + Q gather] -> SpanAttention
  -> GemmA16Wx(o_proj) (+residual) -> RMSNorm -> GemmA16Wx(gate, SiLU) -> GemmA16Wx(up) -> MUL
  -> GemmA16Wx(down) (+residual);  final RMSNorm -> Gemm(lm_head, bf16) -> argmax.
"""
import os
from dataclasses import dataclass

import torch
import torch.distributed as dist

from . import _lib, ops, quantize as PQ, tp as TP
from ._lib import ACT_NONE, ACT_SILU, BIN_MUL, KV_FP8, KV_I8, KV_NONE, KV_U4


@dataclass
class ModelConfig:
    name: str
    hidden: int
    n_heads: int
    n_kv: int
    inter: int
    layers: int
    vocab: int
    head: int = 128
    rope_base: float = 1e6
    eps: float = 1e-6
    qkv_bias: bool = True
    qk_norm: bool = False  # Qwen3: per-head RMSNorm of the q and k heads before rotary (QKLayerNormNoBeta), head 128 only
    # a Hugging Face rope_scaling entry (ops.rope_table: linear, yarn, llama3), applied statically: one frequency table for
    # every position and sequence; None: the unscaled rotary (rope_base^(-2f / head)).  Head 128 only.
    rope_scaling: dict | None = None
    # the rotary covers the first rotary_dim dims of each q and k head (None: the whole head; GLM: half of it), paired NeoX
    # rotate-half ("neox": d with d + rotary_dim / 2) or GPT-J / ChatGLM style ("interleaved": 2i with 2i + 1, head 128 only)
    rotary_dim: int | None = None
    rope_style: str = "neox"


QWEN2_7B = ModelConfig("Qwen2-7B", 3584, 28, 4, 18944, 28, 152064)
LLAMA3_8B = ModelConfig("Llama-3-8B", 4096, 32, 8, 14336, 32, 128256, rope_base=5e5, eps=1e-5, qkv_bias=False)
QWEN2_72B = ModelConfig("Qwen2-72B", 8192, 64, 8, 29568, 80, 152064)
QWEN2_05B = ModelConfig("Qwen2-0.5B", 896, 14, 2, 4864, 24, 151936, head=64)   # config C0: the CPU-parity anchor
TINY = ModelConfig("tiny-2L", 512, 8, 2, 1024, 2, 1024)
# Qwen3 dense models (shapes of the published config.json files): no QKV bias, per-head Q/K norm, head_dim 128 carried
# explicitly — n_heads * head differs from hidden for 0.6B (16 x 128 = 2048 against 1024), so o_proj's K is not hidden
QWEN3_8B = ModelConfig("Qwen3-8B", 4096, 32, 8, 12288, 36, 151936, qkv_bias=False, qk_norm=True)
QWEN3_06B = ModelConfig("Qwen3-0.6B", 1024, 16, 8, 3072, 28, 151936, qkv_bias=False, qk_norm=True)  # full-depth parity anchor
# Long-context rotary scaling as the published model cards enable it.  Qwen2.5 / Qwen3 reach 131072 tokens with YaRN over
# their native 32768; a Qwen3 stack turns it on with dataclasses.replace(QWEN3_8B, rope_scaling=YARN_4X_32K).
YARN_4X_32K = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}
QWEN25_7B = ModelConfig("Qwen2.5-7B", 3584, 28, 4, 18944, 28, 152064, rope_scaling=YARN_4X_32K)
LLAMA31_8B = ModelConfig("Llama-3.1-8B", 4096, 32, 8, 14336, 32, 128256, rope_base=5e5, eps=1e-5, qkv_bias=False,
                         rope_scaling={"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                       "original_max_position_embeddings": 8192})
# GLM-4 / ChatGLM3 (shapes of the published config.json files): 2 kv heads, QKV bias, the interleaved rotary over half of
# each head.  The -chat long-context variants only raise rope_ratio, which multiplies the base: GLM-4-9B-chat's 500 is
# dataclasses.replace(GLM4_9B, rope_base=1e4 * 500).
GLM4_9B = ModelConfig("GLM-4-9B", 4096, 32, 2, 13696, 40, 151552, rope_base=1e4, eps=1.5625e-7, qkv_bias=True, rotary_dim=64,
                      rope_style="interleaved")
CHATGLM3_6B = ModelConfig("ChatGLM3-6B", 4096, 32, 2, 13696, 28, 65024, rope_base=1e4, eps=1e-5, qkv_bias=True, rotary_dim=64,
                          rope_style="interleaved")

KV_MODES = {"none": KV_NONE, "bf16": KV_NONE, "i8": KV_I8, "u4": KV_U4, "fp8": KV_FP8}


_DT = torch.bfloat16  # the model dtype FT while a DecodeStack is being built (DecodeStack(dtype=...): bf16 or fp16)


def synth_weight(K, N, gen, device, std=0.02):
    return (torch.randn(K, N, generator=gen, device=device, dtype=torch.float32) * std).to(_DT)


def _quantize(w, wbits, group, keep_ref):
    """IQ quantizer of a synthetic [K, N] weight: (q, scales, zeros, ref); wbits 16 keeps the weight dense (no scales or
    zeros).  ref: the dense fp32 (q - z) * s of the FULL matrix for the CPU oracle (keep_ref), else None."""
    if wbits == 4:
        q, s, z = PQ.quantize_a16w4(w, group)
    elif wbits == 8:
        q, s, z = PQ.quantize_a16w8(w, group)
    else:
        q, s, z = w, None, None
    ref = (PQ.dequantize(q, s, z, group, wbits, w.shape[1]) if wbits != 16 else w.float()).cpu() if keep_ref else None
    return q, s, z, ref


class QuantLinear:
    """One projection: synthetic bf16 weight -> IQ quantizer -> (TP shard) -> GemmWQ handle (keeps nothing but the handle).
    shard: None | ("cols", ranges) | ("rows", rank, tp)."""

    def __init__(self, K, N, wbits, group, gen, device, max_m, bias=False, keep_ref=False, shard=None):
        w = synth_weight(K, N, gen, device)
        b = (torch.randn(N, generator=gen, device=device) * 0.02).to(_DT) if bias else None
        q, s, z, self.ref = _quantize(w, wbits, group, keep_ref)
        if keep_ref:
            self.ref_bias = b.float().cpu() if b is not None else None
        if shard is not None:
            if shard[0] == "cols":
                q, s, z, b = TP.shard_cols(q, s, z, b, wbits, shard[1])
                N = sum(e - a for a, e in shard[1])
            else:
                q, s, z = TP.shard_rows(q, s, z, wbits, group, shard[1], shard[2])
                K = q.shape[0]
                if shard[1] != 0:
                    b = None  # a row-split bias is added once (rank 0)
        self.K, self.N, self.wbits = K, N, wbits
        self.op = ops.GemmWQ(K, N, wbits, group, max_m=max_m, dtype=_DT)
        self.op.prepare(q.contiguous(), s, z, b)

    def __call__(self, x, ws, **kw):
        return self.op(x, ws, **kw)


class SwiGLULinear:
    """gate_proj + up_proj as ONE weight stream with a fused silu(gate)*up epilogue (b2_gemm_wq_prepare_swiglu).
    Weights are drawn in the same order as two separate QuantLinear's (gate first) so both graphs see identical values."""

    def __init__(self, K, N, wbits, group, gen, device, max_m, keep_ref=False, shard=None):
        qs = []
        self.ref = []
        for _ in range(2):
            q, s, z, ref = _quantize(synth_weight(K, N, gen, device), wbits, group, keep_ref)
            if keep_ref:
                self.ref.append(ref)
            if shard is not None:
                q, s, z, _ = TP.shard_cols(q, s, z, None, wbits, shard[1])
            qs.append((q, s, z))
        if shard is not None:
            N = sum(e - a for a, e in shard[1])
        self.K, self.N = K, N
        self.op = ops.GemmWQ(K, N, wbits, group, max_m=max_m, pair=True, dtype=_DT)
        self.op.prepare_swiglu(*qs[0], *qs[1])

    def __call__(self, x, ws, **kw):
        return self.op(x, ws, **kw)


class _RefView:
    """Makes a SwiGLULinear look like the separate gate / up projections to the CPU oracle (decoder_ref.from_stack)."""

    def __init__(self, ref):
        self.ref, self.ref_bias = ref, None


class DecodeStack:
    def __init__(self, cfg, batch, max_len, wbits=4, group=-1, kv="none", span=128, seed=1234, device="cuda",
                 keep_ref=False, layers=None, tp_rank=0, tp_size=1, tp_group=None, fuse_swiglu=True,
                 collective=None, comm=None, dtype=torch.bfloat16, q_len=1, tree=False, logprobs=0, sample=False,
                 penalties=False, sampled_verify=False, ngram=None):
        """tp_size > 1: the reference's tensor-parallel layout (QKV/gate/up column split, o/down row split + all-reduce,
        vocab-split lm_head + B-element all-gather); every rank builds the SAME full synthetic weights from `seed` and
        keeps its shard, exactly like the reference splits an already-quantized checkpoint.  A rank reaches its peers through
        an initialised torch.distributed process group, or through a connected `comm` (collective "b2" / "fused"); a stack
        with neither is refused before any weight is built.
        q_len = T > 1: multi-token verify steps (speculative decoding).  Every step runs T rows per sequence: self.tokens
        [B, T] holds the last emitted token (column 0, written by the step itself) and T-1 drafts (filled by the caller);
        step() returns (pred [B, T], accepted [B]) and advances the lengths by the accepted counts on the device.
        tree=True (with q_len = T > 1): the T rows of a sequence are the nodes of a draft tree.  self.parents [B, T] int32
        (tree format: include/b200spark.h) is filled by the caller next to self.tokens before each step; the step appends
        and attends in tree form, accepts the longest greedy path and compacts the path's cache rows in every layer.
        step() returns (pred [B, T], accepted [B], path [B, T]); the emitted tokens are pred[b, path[b, :accepted[b]]].
        logprobs = N (0 <= N <= 10): the step also returns log-probabilities on the device (b2_logprobs; TP > 1: per-rank
        records, one all-gather, b2_logprobs_merge) in place of the argmax, with the same ids and launch count: self.tok_lp
        [B*T] fp32 (the logprob of each row's own argmax), self.top_ids [B*T, N] int64 and self.top_lp [B*T, N] fp32 (the N
        most likely tokens, argmax order).  Every row of a multi-token or tree step gets them; the logprob of an emitted token
        is tok_lp at its row: row b*T + u for the token pred[b, u] (u = path[b, j] in a tree).  N = 0 runs today's step.
        sample=True (q_len 1): the step draws next_ids with b2_sample in place of the argmax, with the same launch
        count.  The per-sequence parameters live on the device, [B] each: self.temperature (fp32, default 1.0), self.top_k
        (int32, 0 = no limit), self.top_p (fp32, 1.0), self.seeds and self.offsets (int64, 0); set_sampling() writes them in
        place, so a captured graph stays valid, and every step advances the offsets by 1.  With logprobs = N the step runs
        b2_sample, then b2_logprobs at the drawn ids (one launch more): tok_lp is the logprob of the sampled token under the
        model's distribution, before temperature and filtering (as the reference reports it), and top_ids / top_lp the N most
        likely tokens of that distribution.
        sample=True with tp_size > 1: every rank draws b2_sample's id of the whole row from its vocab shard, bit for bit
        (b2_sample_shard: six phases, each followed by an all-gather of small per-row records, then b2_sample_shard_merge)
        in place of argmax_shard, its two all-gathers and the merge.  The caller writes the same parameters on every rank.
        That is 9 launches more than the greedy TP step with collective "b2" or "fused" (7 kernels and 6 all-gathers in place
        of 4 launches) and 5 more with "nccl" (whose all-gathers are not counted).  With logprobs = N, b2_logprobs_shard at
        the drawn ids, the all-gather of its records and b2_logprobs_merge follow, as in the greedy TP step: 13 launches
        more than that step with "b2" / "fused", 7 with "nccl".
        penalties=True (q_len 1): the reference's logits processor runs on the lm_head's output (b2_penalize; each TP rank
        its vocab shard), so the argmax, b2_sample and b2_logprobs all see the processed row; the step then appends next_ids
        to a per-sequence token history on the device (one launch each).  set_history(b, ids, prompt_len) loads sequence
        b's tokens, set_penalties() writes the per-sequence parameters in place (neutral until written).  self.history and
        self.penalties are the views of the current batch; capture() leaves the history as it found it.
        sampled_verify=True (q_len = T > 1, chain or tree, one GPU): sampled speculative verification.  The step draws every
        row with b2_sample_tokens in place of the argmax (row b*T + u at sequence b's counter offsets[b] + depth(u), with
        sequence b's parameters, kept and written as for sample=True) and accepts along the draws with
        b2_spec_accept_sampled, which also advances offsets[b] by accepted[b]; the launch count is the greedy verify step's.
        step() returns what a verify step returns, the emitted tokens are pred[b, :accepted[b]] (pred[b, path[b, :accepted[b]]]
        in a tree), and they are exactly the tokens single-token sampling would draw from the same rows and seeds.  With
        logprobs = N, b2_logprobs runs at the drawn ids (one launch more): tok_lp at row b*T + u is the logprob of pred[b, u].
        ngram=(n_min, n_max, width) (q_len = T > 1, chain or tree, greedy or sampled_verify): the step drafts its own tokens
        on the device.  Before the embedding, b2_ngram_draft fills self.tokens[:, 1:] (and self.parents in a tree) from a
        per-sequence token history by n-gram (prompt-lookup) matching; width > 1 candidates make a draft tree and need
        tree=True.  After accept (and compaction) b2_history_append_tokens appends the step's emitted tokens to the history.
        Two launches more; the verify body is unchanged.  set_history(b, ids, prompt_len) loads sequence b's history and
        sets self.tokens[b, 0] = ids[-1], the last emitted token; self.n_draft [B] int32 holds the drafts each step filled.
        capture() leaves the history as it found it."""
        global _DT
        assert dtype in (torch.bfloat16, torch.float16) and (dtype == torch.bfloat16 or (tp_size == 1 and cfg.head == 128)), \
            "fp16: single GPU, head size 128 (the communicator and the head-64 kernels are bf16)"
        assert 1 <= q_len <= 16 and (q_len == 1 or (tp_size == 1 and cfg.head == 128)), \
            "multi-token steps: q_len <= 16, single GPU, head size 128"
        assert not tree or (q_len > 1 and tp_size == 1 and cfg.head == 128), "draft trees: q_len > 1, single GPU, head size 128"
        assert not cfg.qk_norm or cfg.head == 128, "per-head Q/K norm: head size 128"
        assert cfg.rope_scaling is None or cfg.head == 128, "rope scaling: head size 128"
        assert cfg.rope_style in ops.ROPE_STYLES, "rope_style: 'neox' or 'interleaved'"
        assert cfg.rope_style == "neox" or cfg.head == 128, "interleaved rotary: head size 128 (the head-64 append is NeoX only)"
        assert 0 <= logprobs <= ops._lib.MAX_TOP_LOGPROBS, "logprobs: 0 .. 10 alternatives"
        assert not sample or q_len == 1, "sample=True: single-token steps (q_len == 1); sampled verify steps: sampled_verify=True"
        assert not sampled_verify or (q_len > 1 and tp_size == 1 and not sample and not penalties), \
            "sampled_verify=True: multi-token or tree steps (q_len > 1) on one GPU (tp_size == 1), without sample=True, and " \
            "without penalties=True (the history is not kept per draft position)"
        assert not penalties or q_len == 1, \
            "penalties=True: single-token steps (q_len == 1); the history is not kept per draft position"
        if ngram is not None:
            assert q_len > 1, "ngram: drafting needs multi-token verify steps (q_len > 1)"
            n_min, n_max, width = ngram
            assert 1 <= n_min <= n_max <= 16, "ngram=(n_min, n_max, width): 1 <= n_min <= n_max <= 16"
            assert 1 <= width <= q_len - 1 and (width == 1 or tree), \
                "ngram=(n_min, n_max, width): 1 <= width <= q_len - 1, and width > 1 drafts a tree (tree=True)"
            ngram = (int(n_min), int(n_max), int(width))
        collective = collective or os.environ.get("B2_TP_COLLECTIVE", "b2")
        # a rank reaches its peers through a torch.distributed process group (the "nccl" collectives, and the handle
        # exchange that connects the communicator), or through a communicator the caller connected; refuse before any
        # weight is built rather than fail in the first exchange
        assert tp_size == 1 or (dist.is_available() and dist.is_initialized()) or (comm is not None and collective != "nccl"), \
            "tp_size > 1: initialise a torch.distributed process group (or pass a connected comm with collective 'b2' / " \
            "'fused') first; a stack without peers runs with tp_size == 1"
        self.logprobs, self.sample, self.pen, self.sv, self.ngram = logprobs, sample, penalties, sampled_verify, ngram
        self.dtype = _DT = dtype
        self.q_len, self.tree = q_len, tree
        rows = batch * q_len  # activation rows of a step
        self.cfg, self.B, self.max_len = cfg, batch, max_len
        self.tp_rank, self.tp, self.tp_group = tp_rank, tp_size, tp_group
        # tensor-parallel exchange: "fused" = all-reduce inside the row-parallel GEMV's epilogue (b2_gemm_wq_run_allreduce;
        # batches <= 16, else it degrades to "b2"), "b2" = GEMM + b2_allreduce (one-shot over NVLink peer memory, residual
        # fused), "nccl" = torch.distributed all_reduce + copy (the baseline the reference's AllReduceOp amounts to)
        self.collective = collective
        self.comm = comm
        self.fuse_swiglu = fuse_swiglu
        self.group_size, self.wbits = group, wbits
        self.device = device
        self.n_layers = layers if layers is not None else cfg.layers
        self.kv_mode = KV_MODES[kv]
        gen = torch.Generator(device=device).manual_seed(seed)
        H, nH, nG, I = cfg.hidden, cfg.n_heads, cfg.n_kv, cfg.inter
        hd = self.head = cfg.head
        tp, r = tp_size, tp_rank
        self.nH_l, self.nG_l, self.I_l = nH // tp, nG // tp, I // tp
        nHl, nGl = self.nH_l, self.nG_l
        col_qkv = ("cols", TP.col_ranges_qkv(nH, nG, r, tp)) if tp > 1 else None
        col_i = ("cols", TP.col_range_even(I, r, tp)) if tp > 1 else None
        row = ("rows", r, tp) if tp > 1 else None
        self.embed = synth_weight(cfg.vocab, H, gen, device, std=1.0)
        # the Q/K norm gammas come from their own generator, so a stack with qk_norm=False gets identical weights otherwise;
        # every rank keeps them whole (they are per head, shared by all heads)
        gen_qk = torch.Generator(device=device).manual_seed(seed + 1) if cfg.qk_norm else None
        self.layers = []
        for _ in range(self.n_layers):
            L = {}
            if cfg.qk_norm:
                L["qn"] = (1.0 + 0.1 * torch.randn(hd, generator=gen_qk, device=device)).to(_DT)
                L["kn"] = (1.0 + 0.1 * torch.randn(hd, generator=gen_qk, device=device)).to(_DT)
            L["g1"] = (1.0 + 0.1 * torch.randn(H, generator=gen, device=device)).to(_DT)
            L["qkv"] = QuantLinear(H, (nH + 2 * nG) * hd, wbits, group, gen, device, rows, bias=cfg.qkv_bias, keep_ref=keep_ref,
                                   shard=col_qkv)
            L["o"] = QuantLinear(nH * hd, H, wbits, group, gen, device, rows, keep_ref=keep_ref, shard=row)
            L["g2"] = (1.0 + 0.1 * torch.randn(H, generator=gen, device=device)).to(_DT)
            if fuse_swiglu:
                L["gateup"] = SwiGLULinear(H, I, wbits, group, gen, device, rows, keep_ref=keep_ref, shard=col_i)
                if keep_ref:
                    L["gate"], L["up"] = _RefView(L["gateup"].ref[0]), _RefView(L["gateup"].ref[1])
            else:
                L["gate"] = QuantLinear(H, I, wbits, group, gen, device, rows, keep_ref=keep_ref, shard=col_i)
                L["up"] = QuantLinear(H, I, wbits, group, gen, device, rows, keep_ref=keep_ref, shard=col_i)
            L["down"] = QuantLinear(I, H, wbits, group, gen, device, rows, keep_ref=keep_ref, shard=row)
            L["cache"] = ops.SpanCache(batch, max_len, nHl, nGl, span, self.kv_mode, device, head=hd, dtype=dtype)
            self.layers.append(L)
        self.gf = (1.0 + 0.1 * torch.randn(H, generator=gen, device=device)).to(_DT)
        self.vocab_l = cfg.vocab // tp
        self.lm_head = QuantLinear(H, cfg.vocab, 16, -1, gen, device, rows, keep_ref=keep_ref,
                                   shard=("cols", TP.col_range_even(cfg.vocab, r, tp)) if tp > 1 else None)
        self.attn = ops.SpanAttn(self.layers[0]["cache"].cfg, rows)
        self.ws = ops.Workspace(device)
        # rope scaling: one fp32 frequency table on the device, shared by every layer and sequence (every TP rank builds the
        # same one); without it the append computes base^(-2f / rotary_dim) itself, as before.  A pairing other than NeoX
        # rides as a third element, in both forms.
        rd = cfg.rotary_dim or hd
        self.rope = (cfg.rope_base, rd) if cfg.rope_scaling is None else ops.rope_table(cfg.rope_scaling, cfg.rope_base, rd, device)
        if cfg.rope_style != "neox":
            self.rope = tuple(self.rope) + (cfg.rope_style,)
        rec = ops.logprobs_partial_bytes(logprobs) if logprobs else 0  # bytes of one row's logprob record (TP > 1)
        if tp > 1 and self.collective != "nccl" and self.comm is None:  # the largest exchange: activations, or a record
            rec_max = max(rec, ops.sample_shard_record_bytes(1) if sample else 0)
            self.comm = ops.Comm(tp_rank, tp, max(batch * H * 2, 4096, batch * rec_max)).connect_group(tp_group)
        # The step state, declared once: every array a step reads or writes per sequence or per activation row.  Columns:
        # the layout for b sequences, dtype, initial value (None: uninitialised), whether this stack needs it, and whether a
        # step carries it to the next (capture() rewinds those after its warm-up step).  Layouts: per_seq(*s) is [b, *s];
        # per_row(*s) is [b * T, *s], a row per token; gathered(n, k) is [n, b * k], the layout an all-gather writes (n ranks)
        # and the per-tile row statistics take (n tiles).  Without a dtype, the layout makes an object for b sequences
        # that views a prefix of them itself (.view(b)).  self._<name> holds the construction batch's array and
        # self.<name> the current batch's view (set_batch); both are None when the stack does not need it.
        T, i32, i64, f32, u8 = q_len, torch.int32, torch.int64, torch.float32, torch.uint8
        per_seq = lambda *s: lambda b: (b, *s)
        per_row = lambda *s: lambda b: (b * T, *s)
        gathered = lambda n, k=1: lambda b: (n, b * k)
        drawn, greedy_tp, lp_tp = sample or sampled_verify, tp > 1 and not logprobs, tp > 1 and logprobs > 0
        handoff = self._norm_placement(rows) == "handoff"
        chain = (torch.arange(T) - 1).clamp_(min=0)  # the parents of a chain: a tree stack's drafts until the caller writes trees
        state = (
            ("lens_old", per_seq(), i32, 0, True, True),
            ("lens_new", per_seq(), i32, T, True, True),  # lens_old + q_len
            ("ids", per_seq(), i64, 0, True, False),
            ("next_ids", per_seq(), i64, 0, True, False),
            ("tokens", per_seq(T), i64, 0, T > 1, True),
            ("pred", per_seq(T), i64, 0, T > 1, False),
            ("accepted", per_seq(), i32, 0, T > 1, False),
            ("parents", per_seq(T), i32, chain, tree, False),
            ("path", per_seq(T), i32, 0, tree, False),
            ("temperature", per_seq(), f32, 1.0, drawn, False),
            ("top_k", per_seq(), i32, 0, drawn, False),
            ("top_p", per_seq(), f32, 1.0, drawn, False),
            ("seeds", per_seq(), i64, 0, drawn, False),
            ("offsets", per_seq(), i64, 0, drawn, True),
            ("history", lambda b: ops.TokenHistory(b, max_len, cfg.vocab, device), None, None, penalties or ngram is not None,
             True),
            ("penalties", lambda b: ops.Penalties(b, device), None, None, penalties, False),
            ("n_draft", per_seq(), i32, 0, ngram is not None, False),
            ("x", per_row(H), _DT, None, True, False),
            ("xn", per_row(H), _DT, None, True, False),
            ("qkv", per_row((nHl + 2 * nGl) * hd), _DT, None, True, False),
            ("q", per_row(nHl * hd), _DT, None, True, False),
            ("ao", per_row(nHl * hd), _DT, None, True, False),
            ("gate", per_row(self.I_l), _DT, None, True, False),
            ("up", per_row(self.I_l), _DT, None, True, False),
            ("logits", per_row(self.vocab_l), _DT, None, True, False),
            ("tok_lp", per_row(), f32, None, logprobs > 0, False),
            ("top_ids", per_row(logprobs), i64, None, logprobs > 0, False),
            ("top_lp", per_row(logprobs), f32, None, logprobs > 0, False),
            # per-tile row statistics of o_proj / down_proj ([tiles][R] per step) for the next norm
            ("ssq_o", gathered(self.layers[0]["o"].op.sumsq_parts(), T), f32, 0, handoff, False),
            ("ssq_d", gathered(self.layers[0]["down"].op.sumsq_parts(), T), f32, 0, handoff, False),
            ("part", per_row(H), _DT, None, tp > 1, False),  # row-split partial sums (all-reduced)
            # the vocab-split argmax: per-rank (max, argmax) pairs and their all-gathers
            ("loc_ids", per_seq(), i64, None, greedy_tp, False),
            ("loc_val", per_seq(), f32, None, greedy_tp, False),
            ("all_ids", gathered(tp), i64, None, greedy_tp, False),
            ("all_val", gathered(tp), f32, None, greedy_tp, False),
            # vocab-split logprobs: one record per row and rank (b2_logprobs_shard), all-gathered as bytes
            ("loc_rec", per_seq(rec), u8, None, lp_tp, False),
            ("all_rec", gathered(tp, rec), u8, None, lp_tp, False),
            # this rank's state and records of the vocab-split draw (b2_sample_shard)
            ("stp", lambda b: ops.sample_tp_buffers(b, tp, device), None, None, sample and tp > 1, False),
        )
        self.Bmax, self._layouts, self._carried = batch, {}, []
        for name, layout, dt, init, needed, carried in state:
            full = None
            if needed:
                if dt is None:
                    full = layout(batch)
                else:
                    full = torch.empty(layout(batch), dtype=dt, device=device)
                    if init is not None:
                        full.copy_(torch.as_tensor(init))
                self._layouts[name] = layout
                if carried:
                    self._carried.append(name)
            setattr(self, "_" + name, full)
            setattr(self, name, full)
        self.graph = None
        self.set_batch(batch)
        self.launches_per_step = 0

    def set_batch(self, b):
        """Run the next steps with the first `b` sequences only (b <= construction batch): every array of the step state is
        re-viewed (its first b sequences are a prefix of its storage); a captured graph is dropped.  bench.py measures batch
        64, 8 and 1 on ONE set of weights and caches this way."""
        assert 1 <= b <= self.Bmax
        self.B = b
        for name, layout in self._layouts.items():
            full = getattr(self, "_" + name)
            if isinstance(full, torch.Tensor):
                setattr(self, name, full.view(-1)[:full.numel() // self.Bmax * b].view(layout(b)))
            else:
                setattr(self, name, full.view(b))
        self.graph = None

    def set_sampling(self, temperature=None, top_k=None, top_p=None, seeds=None, offsets=None):
        """Write the sampling parameters of the current batch in place (a scalar or [B] values each; None keeps the value)."""
        assert self.sample or self.sv, "set_sampling: the stack was built with sample=False and sampled_verify=False"
        for k, v in (("temperature", temperature), ("top_k", top_k), ("top_p", top_p), ("seeds", seeds), ("offsets", offsets)):
            if v is not None:
                t = getattr(self, k)
                t.copy_(torch.as_tensor(v, dtype=t.dtype).expand(t.shape))

    def set_penalties(self, repetition=None, presence=None, frequency=None, no_repeat_ngram=None, min_length=None, eos_id=None,
                      suppress_repetition_in_generation=None):
        """Write the logits-processor parameters of the current batch in place (a scalar or [B] values each; None keeps the
        value).  Ranges as the reference's request checks: repetition in [0, 2], presence and frequency in [-2, 2]."""
        assert self.pen, "set_penalties: the stack was built with penalties=False"
        self.penalties.set(repetition, presence, frequency, no_repeat_ngram, min_length, eos_id, suppress_repetition_in_generation)

    def set_history(self, b, ids, prompt_len=None):
        """Load sequence b's tokens into its history (prompt first; prompt_len of them, all by default).  With ngram the last
        of them is also the last emitted token of the next step: tokens[b, 0] = ids[-1]."""
        assert self.pen or self.ngram, "set_history: the stack was built with penalties=False and without ngram"
        self._history.load(b, ids, prompt_len)
        ids = torch.as_tensor(ids).reshape(-1)
        if self.ngram and ids.numel():
            self._tokens[b, 0] = int(ids[-1])

    # ------------------------------------------------------------------ cache fill
    def set_context(self, ctx, seed=4321):
        """Fill every layer's cache with `ctx` tokens of N(0,1) rows through the prefill-side span writer
        (b2_span_context_copy: quantized spans carry realistic params, bytes identical to `ctx` appends), and set the
        sequence lengths."""
        gen = torch.Generator(device=self.device).manual_seed(seed)
        nG = self.nG_l
        kw, vw = nG * self.head, nG * self.head
        if self.head != 128:  # the prefill writer covers head 128; small heads go through the append kernel
            pos = torch.zeros(self.Bmax, dtype=torch.int32, device=self.device)
            width = (self.nH_l + 2 * nG) * self.head
            for t in range(ctx):
                rows = torch.randn(self.Bmax, width, generator=gen, device=self.device).to(self.dtype)
                for L in self.layers:
                    ops.cache_append(L["cache"], rows, pos, q_out=self._q)
                pos += 1
        for b in range(self.Bmax if self.head == 128 else 0):
            rows = torch.randn(ctx, kw + vw, generator=gen, device=self.device).to(self.dtype)
            for L in self.layers:
                ops.context_copy(L["cache"], "k", b, rows[:, :kw])
                ops.context_copy(L["cache"], "v", b, rows[:, kw:])
        self._lens_old.fill_(ctx)
        self._lens_new.fill_(ctx + self.q_len)
        torch.cuda.synchronize()

    # ------------------------------------------------------------------ one decode step (eager or captured)
    def _row_parallel(self, lin, inp):
        """o_proj / down_proj.  TP=1: residual fused in the GEMM epilogue.  TP>1: per-rank partial sums exchanged over NVLink
        (reference: AllReduceOp after o_proj and down_proj, allreduce_op.cpp:73-115 — here stream-ordered, no host sync);
        the residual is added once, after the sum, on every rank."""
        if self.tp == 1:
            lin(inp, self.ws, out=self.x, residual=self.x)
        elif self.collective == "nccl":
            lin(inp, self.ws, out=self.part, residual=self.x if self.tp_rank == 0 else None)
            dist.all_reduce(self.part, group=self.tp_group)
            self.x.copy_(self.part)
        elif self.collective != "fused" or not lin.op.run_allreduce(inp, self.ws, self.comm, out=self.x, residual=self.x):
            lin(inp, self.ws, out=self.part)  # "b2", and "fused" where the fused form does not cover the call
            self.comm.allreduce(self.part, out=self.x, residual=self.x)

    @property
    def collective_impl(self):
        return {"nccl": "nccl all_reduce + copy", "b2": "GEMM + b2_allreduce (one-shot, NVLink peer memory)",
                "fused": "all-reduce fused into the row-parallel GEMV epilogue (one-shot, NVLink peer memory)"}[self.collective]

    def _allreduce(self, t, out=None):
        """the exchange alone (collective_probe)"""
        if self.collective == "nccl":
            dist.all_reduce(t, group=self.tp_group)
            if out is not None:
                out.copy_(t)
        else:
            self.comm.allreduce(t, out=out if out is not None else t)

    def _gather(self, rec, all_rec):
        """all-gather this rank's records (opaque bytes, [rows, bytes]) into all_rec [tp, rows * bytes], in rank order"""
        if self.collective == "nccl":
            dist.all_gather_into_tensor(all_rec.view(-1), rec.view(-1), group=self.tp_group)
        else:
            self.comm.allgather(rec, all_rec)

    def _norm_placement(self, R):
        """Where a step of R activation rows runs its RMSNorms.
        "self": qkv and gate/up normalise their own input (b2_gemm_fuse, self-contained form): they stage bf16(x * gamma),
          collect sum x^2 in the same pass and scale their reduced tile by 1/rms, so two launches per layer disappear.
          Every CTA repeats the normalisation of its k-slice of every live row, so it pays at R <= 2 only.  It needs the
          mma.sync GEMV at R rows, which group sizes that are not a multiple of 64 never take.
        "handoff": o_proj / down_proj also write the next norm's input scaled by its gamma plus per-tile row statistics;
          qkv, gate/up and lm_head take that input and scale their result rows by 1/rms.  Only layer 0's first norm stays
          a stand-alone kernel (two launches per layer fewer).  It needs the wgmma GEMM (R >= 17; per-channel or int4
          weights) and a whole hidden state per rank (TP = 1).
        "standalone": b2_rmsnorm before each consumer, everywhere else (R 3..16, TP > 1 at R >= 17, ...)."""
        g = self.group_size
        if R <= 2 and (g == -1 or g % 64 == 0):
            return "self"
        if R >= 17 and self.tp == 1 and (g == -1 or self.wbits == 4):
            return "handoff"
        return "standalone"

    def _step_ops(self):
        cfg, ws = self.cfg, self.ws
        H = cfg.hidden
        T = self.q_len
        norm = self._norm_placement(self.B * T)
        # The flags choose the step's form, not which arrays were allocated: a stack built with tree, sampled_verify, ngram
        # or penalties may have the flag switched off and capture the other form (tools/spec_bench.py, penalty_bench.py).
        parents, path = (self.parents, self.path) if self.tree else (None, None)
        # the step form of append + attention: single token, chain of T tokens, or draft tree
        form = {} if T == 1 else {"q_len": T, "parents": parents}
        if self.ngram:  # this step's drafts, from the history the previous step extended
            ops.ngram_draft(self.history, self.tokens, parents, *self.ngram, n_draft=self.n_draft)
        ops.embedding(self.embed, self.ids if T == 1 else self.tokens.view(-1), out=self.x)
        for li, L in enumerate(self.layers):
            if norm == "self":
                L["qkv"](self.x, ws, out=self.qkv, norm_in=(None, L["g1"], H, cfg.eps))
            elif norm == "handoff" and li > 0:  # xn = bf16(x * g1) and the row statistics were written by the previous layer's down_proj
                L["qkv"](self.xn, ws, out=self.qkv, norm_in=(self.ssq_d, None, H, cfg.eps))
            else:
                ops.rmsnorm(self.x, L["g1"], cfg.eps, out=self.xn)
                L["qkv"](self.xn, ws, out=self.qkv)
            ops._cache_append(L["cache"], self.qkv, self.lens_old, q_out=self.q, rope=self.rope,
                              qk_norm=(L["qn"], L["kn"], cfg.eps) if cfg.qk_norm else None, **form)
            self.attn._run(self.q, L["cache"], self.lens_new, self.max_len, ws, out=self.ao, **form)
            if norm == "self":
                self._row_parallel(L["o"], self.ao)
                mlp_in, nin = self.x, (None, L["g2"], H, cfg.eps)
            elif norm == "handoff":
                L["o"](self.ao, ws, out=self.x, residual=self.x, sumsq_out=self.ssq_o, xg_out=(self.xn, L["g2"]))
                mlp_in, nin = self.xn, (self.ssq_o, None, H, cfg.eps)
            else:
                self._row_parallel(L["o"], self.ao)
                ops.rmsnorm(self.x, L["g2"], cfg.eps, out=self.xn)
                mlp_in, nin = self.xn, None
            if self.fuse_swiglu:
                L["gateup"](mlp_in, ws, out=self.gate, norm_in=nin)
            else:
                L["gate"](mlp_in, ws, out=self.gate, act=ACT_SILU, norm_in=nin)
                L["up"](mlp_in, ws, out=self.up, norm_in=nin)
                ops.binary(self.gate, self.up, BIN_MUL, out=self.gate)
            if norm == "handoff":
                g_next = self.layers[li + 1]["g1"] if li + 1 < len(self.layers) else self.gf
                L["down"](self.gate, ws, out=self.x, residual=self.x, sumsq_out=self.ssq_d, xg_out=(self.xn, g_next))
            else:
                self._row_parallel(L["down"], self.gate)
        if norm == "handoff":
            self.lm_head(self.xn, ws, out=self.logits, norm_in=(self.ssq_d, None, H, cfg.eps))
        else:
            ops.rmsnorm(self.x, self.gf, cfg.eps, out=self.xn)
            self.lm_head(self.xn, ws, out=self.logits)
        # the token choice: one id per row, drawn or the argmax, with the log-probabilities if asked for
        ids = self.next_ids if T == 1 else self.pred.view(-1)
        drawn = self.sample or self.sv
        if self.pen:  # the logits processor, in place on this rank's vocab shard
            ops.penalize(self.logits, self.history, self.penalties, self.tp_rank * self.vocab_l)
        if self.sv:  # row b*T + u at sequence b's counter offsets[b] + depth(u)
            ops.sample_tokens(self.logits, T, self.temperature, self.top_k, self.top_p, self.seeds, self.offsets, parents,
                              out=ids)
        elif self.sample and self.tp > 1:  # every rank draws the whole row's id from its shard by exchanging records
            ops.sample_tp(self.logits, self.tp_rank * self.vocab_l, cfg.vocab, self.temperature, self.top_k, self.top_p,
                          self.seeds, self.offsets, self._gather, self.tp, out=ids, bufs=self.stp)
        elif self.sample:
            ops.sample(self.logits, self.temperature, self.top_k, self.top_p, self.seeds, self.offsets, out=ids)
        if self.logprobs:  # at the drawn ids; greedy, the same launch writes the argmax ids
            lp = (self.tok_lp, self.top_ids, self.top_lp)
            tok_ids, out = (ids, (None, *lp)) if drawn else (None, (ids, *lp))
            if self.tp == 1:
                ops.logprobs(self.logits, self.logprobs, tok_ids=tok_ids, out=out)
            else:  # vocab-split: per-rank records, one all-gather of them, the merge
                ops.logprobs_shard(self.logits, self.logprobs, self.tp_rank * self.vocab_l, tok_ids=tok_ids, out=self.loc_rec)
                self._gather(self.loc_rec, self.all_rec)
                ops.logprobs_merge(self.all_rec, self.logprobs, out=out)
        elif not drawn and self.tp == 1:
            ops.argmax(self.logits, out=ids)
        elif not drawn:  # vocab-split lm_head: local (max, argmax) + B-element all-gathers instead of all-reducing the logits
            ops.argmax_shard(self.logits, self.tp_rank * self.vocab_l, self.loc_ids, self.loc_val)
            self._gather(self.loc_val, self.all_val)
            self._gather(self.loc_ids, self.all_ids)
            ops.argmax_merge(self.all_val, self.all_ids, out=ids)  # lowest rank on ties == lowest vocab id
        if T > 1:  # verification: accepted counts, next token, lengths (and the draw counters) stay on the device
            ops._spec_accept(self.accepted, self.next_ids, self.lens_old, self.lens_new, self.tokens, self.pred, path, parents,
                             self.offsets if self.sv else None)
            if self.tree:  # the accepted path's rows move to consecutive slots in every layer
                ops.cache_compact([L["cache"] for L in self.layers], self.lens_old, self.accepted, path, T)
        else:
            ops.lens_add(self.lens_old, 1)
            ops.lens_add(self.lens_new, 1)
        if self.pen or self.ngram:  # the step's emitted tokens join the history
            if T == 1:
                self.history.append(self.next_ids)
            else:
                self.history.append_tokens(self.pred, self.accepted, path)

    def _eager_step(self):
        """one step run eagerly; launches_per_step := the kernels it launched"""
        n = _lib.calls
        self._step_ops()
        self.launches_per_step = _lib.calls - n

    def step(self):
        """q_len 1: returns next_ids [B].  q_len > 1: one verify step, returns (pred [B, T], accepted [B]); the step's
        emitted tokens are pred[b, :accepted[b]].  Tree: (pred, accepted, path [B, T]), emitted pred[b, path[b, :accepted[b]]]."""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._eager_step()
        if self.tree:
            return self.pred, self.accepted, self.path
        return self.next_ids if self.q_len == 1 else (self.pred, self.accepted)

    def capture(self):
        """Warm up once eagerly (plans, workspace growth), rewind the state the step carries, then capture one step."""
        carried = [getattr(self, k) for k in self._carried]
        saved = [v.snapshot() if isinstance(v, ops.TokenHistory) else v.clone() for v in carried]
        self._eager_step()
        torch.cuda.synchronize()
        for v, s in zip(carried, saved):
            if isinstance(v, ops.TokenHistory):
                v.restore(s)
            else:
                v.copy_(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._step_ops()
        torch.cuda.synchronize()
        self.graph = g
        return g

    def collective_probe(self, reps, dist):
        """Time the decode step's collectives ALONE (TP > 1): the 2 x layers all-reduces of [B, hidden] bf16 + the lm_head
        all-gathers, back to back in one CUDA graph, `reps` replays -> ms per step.  No compute overlaps them here, so
        ms_per_step_alone / step time is an upper bound of the collective's share of the step."""
        assert self.tp > 1
        g = torch.cuda.CUDAGraph()
        def ops_():
            for _ in range(2 * len(self.layers)):
                self._allreduce(self.part)
            if self.logprobs:
                self._gather(self.loc_rec, self.all_rec)
            else:
                self._gather(self.loc_val, self.all_val)
                self._gather(self.loc_ids, self.all_ids)
        ops_()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            ops_()
        g.replay()
        torch.cuda.synchronize()
        dist.barrier(group=self.tp_group)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / reps], device=self.device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.tp_group)
        return {"ms_per_step_alone": round(float(t.item()), 4), "all_reduces_per_step": 2 * len(self.layers),
                "bytes_per_all_reduce": self.part.numel() * 2, "impl": self.collective_impl}

    # ------------------------------------------------------------------ accounting
    def algo_bytes_per_step(self, ctx):
        """SURVEY.md §8d: quantized projection weights + params + bf16 lm_head + KV of every sequence."""
        wbytes = 0
        for L in self.layers:
            for k in (("qkv", "o", "gateup", "down") if self.fuse_swiglu else ("qkv", "o", "gate", "up", "down")):
                wbytes += L[k].op.algo_bytes(0)
        wbytes += self.lm_head.op.algo_bytes(0)
        kv = self.attn.algo_bytes(self.B * (ctx + 1)) * len(self.layers)
        return wbytes, kv
