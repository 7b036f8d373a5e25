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
from dataclasses import dataclass

import torch

from . import ops, quantize as PQ, tp as TP
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


QWEN2_7B = ModelConfig("Qwen2-7B", 3584, 28, 4, 18944, 28, 152064)
LLAMA3_8B = ModelConfig("Llama-3-8B", 4096, 32, 8, 14336, 32, 128256, rope_base=5e5, eps=1e-5, qkv_bias=False)
QWEN2_72B = ModelConfig("Qwen2-72B", 8192, 64, 8, 29568, 80, 152064)
QWEN2_05B = ModelConfig("Qwen2-0.5B", 896, 14, 2, 4864, 24, 151936, head=64)   # config C0: the CPU-parity anchor
TINY = ModelConfig("tiny-2L", 512, 8, 2, 1024, 2, 1024)

KV_MODES = {"none": KV_NONE, "bf16": KV_NONE, "i8": KV_I8, "u4": KV_U4, "fp8": KV_FP8}


_DT = torch.bfloat16  # the model dtype FT while a DecodeStack is being built (DecodeStack(dtype=...): bf16 or fp16)


def synth_weight(K, N, gen, device, std=0.02):
    return (torch.randn(K, N, generator=gen, device=device, dtype=torch.float32) * std).to(_DT)


class QuantLinear:
    """One projection: synthetic bf16 weight -> IQ quantizer -> (TP shard) -> GemmWQ handle (keeps nothing but the handle).
    shard: None | ("cols", ranges) | ("rows", rank, tp)."""

    def __init__(self, K, N, wbits, group, gen, device, max_m, bias=False, keep_ref=False, shard=None):
        w = synth_weight(K, N, gen, device)
        b = (torch.randn(N, generator=gen, device=device) * 0.02).to(_DT) if bias else None
        if wbits == 4:
            q, s, z = PQ.quantize_a16w4(w, group)
        elif wbits == 8:
            q, s, z = PQ.quantize_a16w8(w, group)
        else:
            q, s, z = w, None, None
        self.ref = None
        if keep_ref:  # dense fp32 (q - z) * s of the FULL matrix for the CPU oracle
            self.ref = (PQ.dequantize(q, s, z, group, wbits, N) if wbits != 16 else w.float()).cpu()
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
            w = synth_weight(K, N, gen, device)
            if wbits == 4:
                q, s, z = PQ.quantize_a16w4(w, group)
            elif wbits == 8:
                q, s, z = PQ.quantize_a16w8(w, group)
            else:
                q, s, z = w, None, None
            if keep_ref:
                self.ref.append((PQ.dequantize(q, s, z, group, wbits, N) if wbits != 16 else w.float()).cpu())
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
                 collective=None, comm=None, dtype=torch.bfloat16, q_len=1, tree=False):
        """tp_size > 1: the reference's tensor-parallel layout (QKV/gate/up column split, o/down row split + all-reduce,
        vocab-split lm_head + B-element all-gather); every rank builds the SAME full synthetic weights from `seed` and
        keeps its shard, exactly like the reference splits an already-quantized checkpoint.
        q_len = T > 1: multi-token verify steps (speculative decoding).  Every step runs T rows per sequence: self.tokens
        [B, T] holds the last emitted token (column 0, written by the step itself) and T-1 drafts (filled by the caller);
        step() returns (pred [B, T], accepted [B]) and advances the lengths by the accepted counts on the device.
        tree=True (with q_len = T > 1): the T rows of a sequence are the nodes of a draft tree.  self.parents [B, T] int32
        (tree format: include/b200spark.h) is filled by the caller next to self.tokens before each step; the step appends
        and attends in tree form, accepts the longest greedy path and compacts the path's cache rows in every layer.
        step() returns (pred [B, T], accepted [B], path [B, T]); the emitted tokens are pred[b, path[b, :accepted[b]]]."""
        global _DT
        assert dtype in (torch.bfloat16, torch.float16) and (dtype == torch.bfloat16 or (tp_size == 1 and cfg.head == 128)), \
            "fp16: single GPU, head size 128 (the communicator and the head-64 kernels are bf16)"
        assert 1 <= q_len <= 16 and (q_len == 1 or (tp_size == 1 and cfg.head == 128)), \
            "multi-token steps: q_len <= 16, single GPU, head size 128"
        assert not tree or (q_len > 1 and tp_size == 1 and cfg.head == 128), "draft trees: q_len > 1, single GPU, head size 128"
        self.dtype = _DT = dtype
        self.q_len, self.tree = q_len, tree
        rows = batch * q_len  # activation rows of a step
        self.cfg, self.B, self.max_len = cfg, batch, max_len
        self.tp_rank, self.tp, self.tp_group = tp_rank, tp_size, tp_group
        # tensor-parallel exchange: "fused" = all-reduce inside the row-parallel GEMV's epilogue (b2_gemm_wq_run_allreduce;
        # batches <= 16, else it degrades to "b2"), "b2" = GEMM + b2_allreduce (one-shot over NVLink peer memory, residual
        # fused), "nccl" = torch.distributed all_reduce + copy (the baseline the reference's AllReduceOp amounts to)
        import os
        self.collective = collective or os.environ.get("B2_TP_COLLECTIVE", "b2")
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
        self.layers = []
        for _ in range(self.n_layers):
            L = {}
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
        self.rope = (cfg.rope_base, hd)
        # device-resident step state, allocated for the construction batch; set_batch() re-views it for a smaller batch
        self.Bmax = batch
        self._lens_old = torch.zeros(batch, dtype=torch.int32, device=device)
        self._lens_new = torch.full((batch,), q_len, dtype=torch.int32, device=device)  # lens_old + q_len
        self._ids = torch.zeros(batch, dtype=torch.int64, device=device)
        self._next_ids = torch.zeros(batch, dtype=torch.int64, device=device)
        if q_len > 1:
            self._tokens = torch.zeros(batch, q_len, dtype=torch.int64, device=device)
            self._pred = torch.zeros(batch, q_len, dtype=torch.int64, device=device)
            self._accepted = torch.zeros(batch, dtype=torch.int32, device=device)
        if tree:  # a chain until the caller writes its trees
            self._parents = (torch.arange(q_len, dtype=torch.int32, device=device) - 1).clamp_(min=0).repeat(batch, 1)
            self._path = torch.zeros(batch, q_len, dtype=torch.int32, device=device)
        bf = dict(dtype=_DT, device=device)
        self._bufs = dict(x=torch.empty(rows, H, **bf), xn=torch.empty(rows, H, **bf),
                          qkv=torch.empty(rows, (nHl + 2 * nGl) * hd, **bf), q=torch.empty(rows, nHl * hd, **bf),
                          ao=torch.empty(rows, nHl * hd, **bf), gate=torch.empty(rows, self.I_l, **bf),
                          up=torch.empty(rows, self.I_l, **bf), logits=torch.empty(rows, self.vocab_l, **bf))
        if tp > 1:
            if self.collective != "nccl" and self.comm is None:
                self.comm = ops.Comm(tp_rank, tp, max(batch * H * 2, 4096)).connect_group(tp_group)
            self._bufs["part"] = torch.empty(batch, H, **bf)             # row-split partial sums (all-reduced)
            self.loc_ids = torch.empty(batch, dtype=torch.int64, device=device)
            self.loc_val = torch.empty(batch, dtype=torch.float32, device=device)
            self.all_ids = torch.empty(tp, batch, dtype=torch.int64, device=device)
            self.all_val = torch.empty(tp, batch, dtype=torch.float32, device=device)
        self.graph = None
        self.set_batch(batch)
        if self._norm_placement(rows) == "handoff":  # per-tile row statistics of o_proj / down_proj, [tiles][R] per step
            self._ssq_o = torch.zeros(self.layers[0]["o"].op.sumsq_parts() * rows, dtype=torch.float32, device=device)
            self._ssq_d = torch.zeros(self.layers[0]["down"].op.sumsq_parts() * rows, dtype=torch.float32, device=device)
        self.launches_per_step = 0

    def set_batch(self, b):
        """Run the next steps with the first `b` sequences only (b <= construction batch): every step buffer, the length
        vectors and the span tables are re-viewed (row-major, so the first b rows are contiguous); a captured graph is
        dropped.  bench.py measures batch 64, 8 and 1 on ONE set of weights and caches this way."""
        assert 1 <= b <= self.Bmax
        self.B = b
        for k, v in self._bufs.items():
            setattr(self, k, v[:b * self.q_len])
        self.lens_old, self.lens_new = self._lens_old[:b], self._lens_new[:b]
        self.ids, self.next_ids = self._ids[:b], self._next_ids[:b]
        if self.q_len > 1:
            self.tokens, self.pred, self.accepted = self._tokens[:b], self._pred[:b], self._accepted[:b]
        if self.tree:
            self.parents, self.path = self._parents[:b], self._path[:b]
        self.graph = None

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
                    ops.cache_append(L["cache"], rows, pos, q_out=self._bufs["q"])
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
    def _row_parallel(self, lin, inp, n):
        """o_proj / down_proj.  TP=1: residual fused in the GEMM epilogue.  TP>1: per-rank partial sums exchanged over NVLink
        (reference: AllReduceOp after o_proj and down_proj, allreduce_op.cpp:73-115 — here stream-ordered, no host sync);
        the residual is added once, after the sum, on every rank."""
        if self.tp == 1:
            lin(inp, self.ws, out=self.x, residual=self.x)
            return n + 1
        if self.collective == "nccl":
            import torch.distributed as dist
            lin(inp, self.ws, out=self.part, residual=self.x if self.tp_rank == 0 else None)
            dist.all_reduce(self.part, group=self.tp_group)
            self.x.copy_(self.part)
            return n + 1
        if self.collective == "fused" and lin.op.run_allreduce(inp, self.ws, self.comm, out=self.x, residual=self.x):
            return n + 1
        lin(inp, self.ws, out=self.part)
        self.comm.allreduce(self.part, out=self.x, residual=self.x)
        return n + 2

    @property
    def collective_impl(self):
        return {"nccl": "nccl all_reduce + copy", "b2": "GEMM + b2_allreduce (one-shot, NVLink peer memory)",
                "fused": "all-reduce fused into the row-parallel GEMV epilogue (one-shot, NVLink peer memory)"}[self.collective]

    def _allreduce(self, t, out=None):
        """the exchange alone (collective_probe)"""
        if self.collective == "nccl":
            import torch.distributed as dist
            dist.all_reduce(t, group=self.tp_group)
            if out is not None:
                out.copy_(t)
        else:
            self.comm.allreduce(t, out=out if out is not None else t)

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
        R = self.B * T  # activation rows
        norm = self._norm_placement(R)
        if norm == "handoff":
            ssq_o = self._ssq_o[:self._ssq_o.numel() // self.Bmax * self.B].view(-1, R)
            ssq_d = self._ssq_d[:self._ssq_d.numel() // self.Bmax * self.B].view(-1, R)
        # the step form of append + attention: single token, chain of T tokens, or draft tree
        form = {} if T == 1 else {"q_len": T, "parents": self.parents if self.tree else None}
        n = 0
        ops.embedding(self.embed, self.ids if T == 1 else self.tokens.view(-1), out=self.x); n += 1
        for li, L in enumerate(self.layers):
            if norm == "self":
                L["qkv"](self.x, ws, out=self.qkv, norm_in=(None, L["g1"], H, cfg.eps)); n += 1
            elif norm == "handoff" and li > 0:  # xn = bf16(x * g1) and the row statistics were written by the previous layer's down_proj
                L["qkv"](self.xn, ws, out=self.qkv, norm_in=(ssq_d, None, H, cfg.eps)); n += 1
            else:
                ops.rmsnorm(self.x, L["g1"], cfg.eps, out=self.xn); n += 1
                L["qkv"](self.xn, ws, out=self.qkv); n += 1
            ops._cache_append(L["cache"], self.qkv, self.lens_old, q_out=self.q, rope=self.rope, **form); n += 1
            self.attn._run(self.q, L["cache"], self.lens_new, self.max_len, ws, out=self.ao, **form); n += 1
            if norm == "self":
                n = self._row_parallel(L["o"], self.ao, n)
                mlp_in, nin = self.x, (None, L["g2"], H, cfg.eps)
            elif norm == "handoff":
                L["o"](self.ao, ws, out=self.x, residual=self.x, sumsq_out=ssq_o, xg_out=(self.xn, L["g2"])); n += 1
                mlp_in, nin = self.xn, (ssq_o, None, H, cfg.eps)
            else:
                n = self._row_parallel(L["o"], self.ao, n)
                ops.rmsnorm(self.x, L["g2"], cfg.eps, out=self.xn); n += 1
                mlp_in, nin = self.xn, None
            if self.fuse_swiglu:
                L["gateup"](mlp_in, ws, out=self.gate, norm_in=nin); n += 1
            else:
                L["gate"](mlp_in, ws, out=self.gate, act=ACT_SILU, norm_in=nin); n += 1
                L["up"](mlp_in, ws, out=self.up, norm_in=nin); n += 1
                ops.binary(self.gate, self.up, BIN_MUL, out=self.gate); n += 1
            if norm == "handoff":
                g_next = self.layers[li + 1]["g1"] if li + 1 < len(self.layers) else self.gf
                L["down"](self.gate, ws, out=self.x, residual=self.x, sumsq_out=ssq_d, xg_out=(self.xn, g_next)); n += 1
            else:
                n = self._row_parallel(L["down"], self.gate, n)
        if norm == "handoff":
            self.lm_head(self.xn, ws, out=self.logits, norm_in=(ssq_d, None, H, cfg.eps)); n += 1
        else:
            ops.rmsnorm(self.x, self.gf, cfg.eps, out=self.xn); n += 1
            self.lm_head(self.xn, ws, out=self.logits); n += 1
        if T > 1:
            ops.argmax(self.logits, out=self.pred.view(-1)); n += 1
        elif self.tp == 1:
            ops.argmax(self.logits, out=self.next_ids); n += 1
        else:  # vocab-split lm_head: local (max, argmax) + B-element all-gather instead of all-reducing 152064 logits
            ops.argmax_shard(self.logits, self.tp_rank * self.vocab_l, self.loc_ids, self.loc_val); n += 1
            if self.collective == "nccl":
                import torch.distributed as dist
                dist.all_gather_into_tensor(self.all_val, self.loc_val, group=self.tp_group)
                dist.all_gather_into_tensor(self.all_ids, self.loc_ids, group=self.tp_group)
            else:
                self.comm.allgather(self.loc_val, self.all_val); n += 1
                self.comm.allgather(self.loc_ids, self.all_ids); n += 1
            ops.argmax_merge(self.all_val, self.all_ids, out=self.next_ids); n += 1  # lowest rank on ties == lowest vocab id
        if T > 1:  # greedy verification: accepted counts, next token and lengths stay on the device
            ops._spec_accept(self.accepted, self.next_ids, self.lens_old, self.lens_new, self.tokens, self.pred,
                             self.path if self.tree else None, self.parents if self.tree else None); n += 1
            if self.tree:  # the accepted path's rows move to consecutive slots in every layer
                ops.cache_compact([L["cache"] for L in self.layers], self.lens_old, self.accepted, self.path, T); n += 1
        else:
            ops.lens_add(self.lens_old, 1); n += 1
            ops.lens_add(self.lens_new, 1); n += 1
        # rows per launch above 16 rows: 64 on the wgmma path (per-channel int4/int8, bf16 lm_head), 16 for sub-channel
        # weights (mma.sync path); below, one launch takes all rows
        hchunks = (R + 63) // 64 if R > 16 else 1
        qchunks = ((R + 15) // 16 if (self.group_size != -1 and self.wbits != 4) else hchunks) if R > 16 else 1
        n += (qchunks - 1) * (4 if self.fuse_swiglu else 5) * len(self.layers) + (hchunks - 1)
        self.launches_per_step = n

    def step(self):
        """q_len 1: returns next_ids [B].  q_len > 1: one verify step, returns (pred [B, T], accepted [B]); the step's
        emitted tokens are pred[b, :accepted[b]].  Tree: (pred, accepted, path [B, T]), emitted pred[b, path[b, :accepted[b]]]."""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step_ops()
        if self.tree:
            return self.pred, self.accepted, self.path
        return self.next_ids if self.q_len == 1 else (self.pred, self.accepted)

    def capture(self):
        """Warm up once eagerly (plans, workspace growth), rewind the lengths, then capture one step."""
        lo, ln = self.lens_old.clone(), self.lens_new.clone()
        tk = self.tokens.clone() if self.q_len > 1 else None  # the accept kernel rewrites column 0
        self._step_ops()
        torch.cuda.synchronize()
        self.lens_old.copy_(lo); self.lens_new.copy_(ln)
        if tk is not None:
            self.tokens.copy_(tk)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._step_ops()
        self.lens_old.copy_(lo); self.lens_new.copy_(ln)
        if tk is not None:
            self.tokens.copy_(tk)
        torch.cuda.synchronize()
        self.graph = g
        return g

    def collective_probe(self, reps, dist):
        """Time the decode step's collectives ALONE (TP > 1): the 2 x layers all-reduces of [B, hidden] bf16 + the lm_head
        all-gathers, back to back in one CUDA graph, `reps` replays -> ms per step.  No compute overlaps them here, so
        ms_per_step_alone / step time is an upper bound of the collective's share of the step."""
        import torch.distributed as dist_
        assert self.tp > 1
        g = torch.cuda.CUDAGraph()
        def ops_():
            for _ in range(2 * len(self.layers)):
                self._allreduce(self.part)
            if self.collective == "nccl":
                dist_.all_gather_into_tensor(self.all_val, self.loc_val, group=self.tp_group)
                dist_.all_gather_into_tensor(self.all_ids, self.loc_ids, group=self.tp_group)
            else:
                self.comm.allgather(self.loc_val, self.all_val)
                self.comm.allgather(self.loc_ids, self.all_ids)
        ops_()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            ops_()
        g.replay()
        torch.cuda.synchronize()
        dist_.barrier(group=self.tp_group)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / reps], device=self.device)
        dist_.all_reduce(t, op=dist_.ReduceOp.MAX, group=self.tp_group)
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
