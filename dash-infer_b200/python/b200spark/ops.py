"""Torch-tensor front end over the C ABI (device memory + streams come from torch; compute does not).

Every call goes through include/b200spark.h on torch's current CUDA stream.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import (ACT_NONE, BIN_ADD, BIN_MUL, DT_BF16, DT_I8, DT_U8, KV_I8, KV_NONE, KV_U4, GemmDesc, GemmFuse, RopeCfg,
                   SpanCfg, check, lib)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class Workspace:
    """The shared 'workspace' tensor of the reference's TensorMap: one buffer reused by every op, grown on demand
    (AsTensor::SetShape semantics, csrc/core/tensor/tensor.cpp:721-746)."""

    def __init__(self, device="cuda"):
        self.device = device
        self.buf = torch.empty(256, dtype=torch.uint8, device=device)

    def reserve(self, nbytes):
        if self.buf.numel() < nbytes:
            self.buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
        return self.buf


def _ft(t):
    """B2 dtype code of a 16-bit tensor (the FT of the glue ops)"""
    return {torch.bfloat16: DT_BF16, torch.float16: _lib.DT_F16}[t.dtype]


class GemmWQ:
    """GemmA16W4 / GemmA16W8 / dense Gemm (wbits 16) handle."""

    def __init__(self, K, N, wbits, group_size=-1, max_m=64, signed=True, pair=False, dtype=torch.bfloat16):
        """pair=True: gate/up weight pair with a fused SwiGLU epilogue (N = intermediate size).
        dtype: the activation / output / scale type FT of the handle (bf16 or fp16)."""
        self.K, self.N, self.wbits, self.group_size, self.max_m, self.pair = K, N, wbits, group_size, max_m, pair
        self.dtype = dtype
        self.h = C.c_void_p()
        qtype = DT_U8 if wbits == 4 or not signed else DT_I8
        ft = {torch.bfloat16: DT_BF16, torch.float16: _lib.DT_F16}[dtype]
        d = GemmDesc(K, N, wbits, group_size if wbits != 16 else -1, ft, qtype, max_m, 1 if pair else 0)
        check(lib.b2_gemm_wq_create(C.byref(self.h), C.byref(d)), "b2_gemm_wq_create")
        self.bias = None

    def prepare(self, qdata, scales=None, zeros=None, bias=None):
        assert qdata.is_cuda and qdata.is_contiguous()
        if self.wbits != 16:
            assert scales.dtype == self.dtype and zeros.dtype == self.dtype
            scales, zeros = scales.contiguous(), zeros.contiguous()
        check(lib.b2_gemm_wq_prepare_weights(self.h, _ptr(qdata), _ptr(scales), _ptr(zeros), None, _stream()),
              "b2_gemm_wq_prepare_weights")
        self.bias = bias.contiguous() if bias is not None else None
        torch.cuda.current_stream().synchronize()  # the caller may free qdata right after
        return self

    def prepare_swiglu(self, qg, sg, zg, qu, su, zu):
        assert self.pair
        c = lambda t: t.contiguous() if t is not None else None
        qg, sg, zg, qu, su, zu = map(c, (qg, sg, zg, qu, su, zu))
        check(lib.b2_gemm_wq_prepare_swiglu(self.h, _ptr(qg), _ptr(sg), _ptr(zg), _ptr(qu), _ptr(su), _ptr(zu), _stream()),
              "b2_gemm_wq_prepare_swiglu")
        torch.cuda.current_stream().synchronize()
        return self

    def workspace_bytes(self, M):
        return lib.b2_gemm_wq_workspace_bytes(self.h, M)

    def algo_bytes(self, M):
        return lib.b2_gemm_wq_algo_bytes(self.h, M)

    def packed_bytes(self):
        return lib.b2_gemm_wq_packed_bytes(self.h)

    def sumsq_parts(self):
        return lib.b2_gemm_wq_sumsq_parts(self.h)

    def __call__(self, a, ws, out=None, act=ACT_NONE, alpha=1.0, residual=None, norm_in=None, sumsq_out=None, xg_out=None):
        """Fused RMSNorm (b2_gemm_fuse), two forms:
        M <= 16, self-contained: norm_in = (None, gamma [K], K, eps) — the GEMV normalises its own activations.
        M >= 17, hand-off on the wgmma path: the producer (o_proj / down_proj with residual) takes
        sumsq_out [sumsq_parts(), M] fp32 and xg_out = (xg [M, N], gamma_out [N]) and also writes xg = FT(out * gamma_out)
        and per-tile row sums of squares; the consumer takes a = xg and norm_in = (sumsq, None, hidden, eps).
        Any other combination fails with B2_ERR_UNSUPPORTED."""
        if self.pair:
            act = _lib.ACT_SWIGLU
        M = a.numel() // a.shape[-1]
        assert a.dtype == self.dtype and a.shape[-1] == self.K and a.stride(-1) == 1
        if out is None:
            out = torch.empty(*a.shape[:-1], self.N, dtype=self.dtype, device=a.device)
        wsb = ws.reserve(self.workspace_bytes(M))
        lda = a.stride(-2) if a.dim() > 1 else self.K
        ldc = out.stride(-2) if out.dim() > 1 else self.N
        if norm_in is None and sumsq_out is None and xg_out is None:
            check(lib.b2_gemm_wq_run(self.h, _ptr(a), lda, _ptr(out), ldc, M, _ptr(self.bias), _ptr(residual), act,
                                     float(alpha), _ptr(wsb), wsb.numel(), _stream()), "b2_gemm_wq_run")
            return out
        f = GemmFuse()
        if norm_in is not None:
            ss, gamma, hidden, eps = norm_in   # ss None: the GEMV takes the row statistics itself (hidden == K)
            f.norm_sumsq, f.norm_gamma = (ss.data_ptr() if ss is not None else None), (gamma.data_ptr() if gamma is not None else None)
            f.norm_parts, f.norm_hidden, f.norm_eps = (ss.shape[0] if ss is not None else 0), int(hidden), float(eps)
        if sumsq_out is not None:
            f.sumsq_out = sumsq_out.data_ptr()
        if xg_out is not None:  # (xg [M, N] bf16, gamma_out [N] bf16): the hand-off form of batches >= 17
            xg, g_out = xg_out
            f.xg_out, f.gamma_out, f.ldxg = xg.data_ptr(), g_out.data_ptr(), xg.stride(-2) if xg.dim() > 1 else self.N
        check(lib.b2_gemm_wq_run_fused(self.h, _ptr(a), lda, _ptr(out), ldc, M, _ptr(self.bias), _ptr(residual), act,
                                       float(alpha), _ptr(wsb), wsb.numel(), C.byref(f), _stream()), "b2_gemm_wq_run_fused")
        return out

    def run_fp8(self, q8, ws, out=None, act=ACT_NONE, alpha=1.0, residual=None):
        """fp8-e4m3 activations (a Fp8Act from quant_fp8) x int4 per-channel weights on the e4m3 wgmma kernel."""
        if self.pair:
            act = _lib.ACT_SWIGLU
        M = q8.y.shape[0]
        if out is None:
            out = torch.empty(M, self.N, dtype=torch.bfloat16, device=q8.y.device)
        wsb = ws.reserve(max(self.workspace_bytes(max(M, 17)), 16))
        check(lib.b2_gemm_wq_run_fp8(self.h, _ptr(q8.y), q8.y.stride(0), _ptr(q8.scale), _ptr(q8.tile_sums), _ptr(out), out.stride(0), M,
                                     _ptr(self.bias), _ptr(residual), act, float(alpha), _ptr(wsb), wsb.numel(), _stream()),
              "b2_gemm_wq_run_fp8")
        return out

    def run_allreduce(self, a, ws, comm, out, residual=None, alpha=1.0):
        """Row-parallel projection fused with its all-reduce over `comm` (b2_gemm_wq_run_allreduce).  Returns False when the
        configuration is not covered (M > 16, ...): the caller then runs the GEMM and b2_allreduce separately."""
        M = a.numel() // a.shape[-1]
        wsb = ws.reserve(self.workspace_bytes(M))
        st = lib.b2_gemm_wq_run_allreduce(self.h, _ptr(a), a.stride(-2) if a.dim() > 1 else self.K, _ptr(out),
                                          out.stride(-2) if out.dim() > 1 else self.N, M, _ptr(self.bias), _ptr(residual), float(alpha),
                                          _ptr(wsb), wsb.numel(), comm.h, _stream())
        if st == 6:  # B2_ERR_UNSUPPORTED
            return False
        check(st, "b2_gemm_wq_run_allreduce")
        return True

    def __del__(self):
        try:
            if self.h:
                lib.b2_gemm_wq_destroy(self.h)
                self.h = None
        except Exception:
            pass


class Comm:
    """Tensor-parallel communicator over NVLink peer memory (b2_comm_*).  `connect_group` exchanges the CUDA IPC handles
    over a torch.distributed process group (host side plumbing only); `connect_local` wires communicators that live in the
    same process (tests: two ranks on one GPU)."""

    def __init__(self, rank, nranks, max_bytes):
        self.rank, self.nranks, self.max_bytes = rank, nranks, int(max_bytes)
        self.h = C.c_void_p()
        check(lib.b2_comm_create(C.byref(self.h), rank, nranks, self.max_bytes), "b2_comm_create")

    def connect_group(self, group=None):
        import torch.distributed as dist
        buf = C.create_string_buffer(_lib.COMM_HANDLE_BYTES)
        check(lib.b2_comm_export(self.h, buf), "b2_comm_export")
        handles = [None] * self.nranks
        dist.all_gather_object(handles, bytes(buf.raw), group=group)
        allh = b"".join(handles)
        check(lib.b2_comm_connect(self.h, allh), "b2_comm_connect")
        dist.barrier(group=group)
        return self

    @staticmethod
    def connect_local(comms):
        n = len(comms)
        ptrs = (C.c_void_p * n)(*[lib.b2_comm_local_buffer(c.h) for c in comms])
        for c in comms:
            check(lib.b2_comm_connect_pointers(c.h, ptrs), "b2_comm_connect_pointers")
        return comms

    def allreduce(self, t, out=None, residual=None):
        out = t if out is None else out
        check(lib.b2_allreduce(self.h, _ptr(out), _ptr(t), _ptr(residual), t.numel(), DT_BF16, _stream()), "b2_allreduce")
        return out

    def allgather(self, t, out):
        check(lib.b2_allgather(self.h, _ptr(out), _ptr(t), t.numel() * t.element_size(), _stream()), "b2_allgather")
        return out

    def check_error(self):
        check(lib.b2_comm_error(self.h), "b2_comm_error (a peer did not arrive within B2_COMM_TIMEOUT_MS)")

    def __del__(self):
        try:
            if self.h:
                lib.b2_comm_destroy(self.h)
                self.h = None
        except Exception:
            pass


class SpanCache:
    """Test/bench stand-in for the reference's CacheSpanManager + SpannedVirtualCache: owns span pages for one
    layer's K and V of a batch and the device pointer tables [batch, max_spans] the kernels walk."""

    def __init__(self, batch, max_len, n_heads, n_groups, span_len=128, quant_mode=KV_NONE, device="cuda", pool=None, fill=0, head=128,
                 dtype=torch.bfloat16):
        """fill: byte the span pool is initialised with (the reference's span manager never zeroes frames; tests use
        0xFF = NaN patterns to prove no kernel consumes unwritten rows)."""
        self.batch, self.max_len = batch, max_len
        self.max_spans = (max_len + span_len - 1) // span_len
        self.head = head
        self.dtype = dtype  # FT of Q / the output / an unquantized cache
        self.cfg = SpanCfg({torch.bfloat16: DT_BF16, torch.float16: _lib.DT_F16}[dtype], quant_mode, n_heads, n_groups, head, span_len,
                           self.max_spans, 0)
        self.span_bytes = lib.b2_span_bytes(C.byref(self.cfg))
        assert self.span_bytes > 0, "bad span config"
        n = batch * self.max_spans
        stride = (self.span_bytes + 255) // 256 * 256
        self.stride = stride
        # pages deliberately handed out in a scrambled order: the kernels must not assume contiguity
        self.k_pool = torch.full((n * stride,), fill, dtype=torch.uint8, device=device)
        self.v_pool = torch.full((n * stride,), fill, dtype=torch.uint8, device=device)
        g = torch.Generator().manual_seed(99)
        perm_k = torch.randperm(n, generator=g)
        perm_v = torch.randperm(n, generator=g)
        self.k_tab = (self.k_pool.data_ptr() + perm_k * stride).to(torch.int64).reshape(batch, self.max_spans).to(device)
        self.v_tab = (self.v_pool.data_ptr() + perm_v * stride).to(torch.int64).reshape(batch, self.max_spans).to(device)
        self.perm_k, self.perm_v = perm_k.reshape(batch, -1), perm_v.reshape(batch, -1)

    def span_view(self, which, b, si):
        pool, perm = (self.k_pool, self.perm_k) if which == "k" else (self.v_pool, self.perm_v)
        off = int(perm[b, si]) * self.stride
        return pool[off: off + self.span_bytes]


def _cache_append(cache, qkv, old_lens, q_out=None, rope=None, q_len=None, parents=None):
    """Append one step's rows to the span cache (+ optional fused rotary).  q_len None: row b of qkv is sequence b, written at
    position old_lens[b].  q_len: row b*q_len + t is token t of sequence b, written at position old_lens[b] + t; with parents
    (int32 [B, q_len]) it is node t of sequence b's draft tree, written at slot old_lens[b] + t with rotary position
    old_lens[b] + depth(t)."""
    cfg = cache.cfg
    rows = qkv.shape[0]
    assert rows % (q_len or 1) == 0 and (parents is None or (q_len and parents.dtype == torch.int32 and parents.is_contiguous()))
    if q_out is None:
        q_out = torch.empty(rows, cfg.n_heads * cfg.head_size, dtype=qkv.dtype, device=qkv.device)
    r = RopeCfg(float(rope[0]), int(rope[1]), 0) if rope is not None else None
    head = (C.byref(cfg), _ptr(cache.k_tab), _ptr(cache.v_tab), _ptr(q_out), _ptr(qkv), _ptr(old_lens))
    tail = (C.byref(r) if r is not None else None, _stream())
    if q_len is None:
        check(lib.b2_span_cache_append(*head, rows, *tail), "b2_span_cache_append")
    elif parents is None:
        check(lib.b2_span_cache_append_tokens(*head, rows // q_len, int(q_len), *tail), "b2_span_cache_append_tokens")
    else:
        check(lib.b2_span_cache_append_tree(*head, _ptr(parents), rows // q_len, int(q_len), *tail), "b2_span_cache_append_tree")
    return q_out


def cache_append(cache, qkv, old_lens, q_out=None, rope=None):
    return _cache_append(cache, qkv, old_lens, q_out, rope)


def cache_append_tokens(cache, qkv, old_lens, q_len, q_out=None, rope=None):
    return _cache_append(cache, qkv, old_lens, q_out, rope, q_len)


def cache_append_tree(cache, qkv, old_lens, parents, q_len, q_out=None, rope=None):
    return _cache_append(cache, qkv, old_lens, q_out, rope, q_len, parents)


def _spec_accept(accepted, next_ids, old_lens, new_lens, tokens, pred, path=None, parents=None):
    """Greedy verification of a multi-token step (b2_spec_accept): tokens / pred int64 [B, T]; writes accepted (int32 [B]),
    next_ids (int64 [B] or None) and tokens[:, 0], advances old_lens by the accepted counts and sets new_lens = old_lens + T.
    With parents (int32 [B, T]) the step is a draft tree (b2_spec_accept_tree), which also writes path (int32 [B, T], the first
    accepted[b] entries)."""
    B, T = tokens.shape
    assert tokens.is_contiguous() and pred.is_contiguous() and pred.shape == tokens.shape
    if parents is None:
        check(lib.b2_spec_accept(_ptr(accepted), _ptr(next_ids), _ptr(old_lens), _ptr(new_lens), _ptr(tokens), _ptr(pred), B, T,
                                 _stream()), "b2_spec_accept")
        return accepted
    assert parents.dtype == torch.int32 and parents.is_contiguous() and parents.shape == tokens.shape
    assert path.dtype == torch.int32 and path.is_contiguous() and path.shape == tokens.shape
    check(lib.b2_spec_accept_tree(_ptr(accepted), _ptr(path), _ptr(next_ids), _ptr(old_lens), _ptr(new_lens), _ptr(tokens),
                                  _ptr(pred), _ptr(parents), B, T, _stream()), "b2_spec_accept_tree")
    return accepted, path


def spec_accept(accepted, next_ids, old_lens, new_lens, tokens, pred):
    return _spec_accept(accepted, next_ids, old_lens, new_lens, tokens, pred)


def spec_accept_tree(accepted, path, next_ids, old_lens, new_lens, tokens, pred, parents):
    return _spec_accept(accepted, next_ids, old_lens, new_lens, tokens, pred, path, parents)


_COMPACT_TABLES = {}


def compact_tables(caches):
    """Device arrays of the caches' K and V span-table pointers (one per layer), built once per set of tables.  The key is
    the tables' addresses, which are exactly what the arrays hold, so a cached entry is right for any caches at them."""
    key = tuple((c.k_tab.data_ptr(), c.v_tab.data_ptr()) for c in caches)
    if key not in _COMPACT_TABLES:
        dev = caches[0].k_tab.device
        _COMPACT_TABLES[key] = (torch.tensor([k for k, _ in key], dtype=torch.int64, device=dev),
                                torch.tensor([v for _, v in key], dtype=torch.int64, device=dev))
    return _COMPACT_TABLES[key]


def cache_compact(caches, old_lens, accepted, path, q_len):
    """After spec_accept_tree: move the accepted path's rows to consecutive slots in every cache (one per layer, all of one
    config) with one launch (b2_span_cache_compact).  Call compact_tables(caches) once before capturing a CUDA graph."""
    kt, vt = compact_tables(caches)
    B = accepted.shape[0]
    check(lib.b2_span_cache_compact(C.byref(caches[0].cfg), _ptr(kt), _ptr(vt), len(caches), _ptr(old_lens), _ptr(accepted),
                                    _ptr(path), B, int(q_len), _stream()), "b2_span_cache_compact")


def context_copy(cache, which, b, src, seq_len=None):
    """Prefill: write sequence b's K (which='k') or V ('v') rows src [seq, ..., n_groups*128 leading values per token] into its
    spans (b2_span_context_copy).  src may be a strided view (e.g. the K part of a fused qkv tensor)."""
    assert src.dtype == cache.dtype and src.stride(-1) == 1
    seq_len = src.shape[0] if seq_len is None else seq_len
    tab = cache.k_tab if which == "k" else cache.v_tab
    check(lib.b2_span_context_copy(C.byref(cache.cfg), C.c_void_p(tab.data_ptr() + b * cache.max_spans * 8), _ptr(src), src.stride(0),
                                   int(seq_len), _stream()), "b2_span_context_copy")


class SpanAttn:
    def __init__(self, cfg, max_batch):
        self.cfg = cfg
        self.h = C.c_void_p()
        check(lib.b2_span_attn_create(C.byref(self.h), C.byref(cfg), max_batch), "b2_span_attn_create")

    def workspace_bytes(self, batch, max_len):
        return lib.b2_span_attn_workspace_bytes(self.h, batch, max_len)

    def tokens_workspace_bytes(self, batch, q_len, max_len):
        return lib.b2_span_attn_tokens_workspace_bytes(self.h, batch, q_len, max_len)

    def _run(self, q, cache, new_lens, max_len, ws, out=None, scale=None, q_len=None, parents=None):
        """q_len None: q [batch, nH*128], row b attends to tokens 0 .. new_lens[b] - 1.  q_len: q [batch*q_len, nH*128], row
        b*q_len + t attends to tokens 0 .. new_lens[b] - q_len + t; with parents (int32 [batch, q_len], a draft tree) to the
        prefix (tokens < new_lens[b] - q_len) and to the slots new_lens[b] - q_len + j of t and its ancestors."""
        B = q.shape[0] // (q_len or 1)
        assert parents is None or (q_len and parents.dtype == torch.int32 and parents.is_contiguous())
        if out is None:
            out = torch.empty_like(q)
        if scale is None:
            scale = 1.0 / (self.cfg.head_size ** 0.5)
        wsb = ws.reserve(self.workspace_bytes(B, max_len) if q_len is None else self.tokens_workspace_bytes(B, q_len, max_len))
        head = (self.h, _ptr(out), _ptr(q), _ptr(cache.k_tab), _ptr(cache.v_tab), _ptr(new_lens))
        tail = (int(max_len), _ptr(wsb), wsb.numel(), float(scale), _stream())
        if q_len is None:
            check(lib.b2_span_attn_run(*head, B, *tail), "b2_span_attn_run")
        elif parents is None:
            check(lib.b2_span_attn_run_tokens(*head, B, int(q_len), *tail), "b2_span_attn_run_tokens")
        else:
            check(lib.b2_span_attn_run_tree(*head, _ptr(parents), B, int(q_len), *tail), "b2_span_attn_run_tree")
        return out

    def __call__(self, q, cache, new_lens, max_len, ws, out=None, scale=None):
        return self._run(q, cache, new_lens, max_len, ws, out, scale)

    def run_tokens(self, q, cache, new_lens, q_len, max_len, ws, out=None, scale=None):
        return self._run(q, cache, new_lens, max_len, ws, out, scale, q_len)

    def run_tree(self, q, cache, new_lens, parents, q_len, max_len, ws, out=None, scale=None):
        return self._run(q, cache, new_lens, max_len, ws, out, scale, q_len, parents)

    def algo_bytes(self, total_tokens):
        return lib.b2_span_attn_algo_bytes(C.byref(self.cfg), int(total_tokens))

    def __del__(self):
        try:
            if self.h:
                lib.b2_span_attn_destroy(self.h)
                self.h = None
        except Exception:
            pass


def rmsnorm(x, gamma, eps=1e-6, out=None):
    out = torch.empty_like(x) if out is None else out
    cols = x.shape[-1]
    check(lib.b2_rmsnorm_ft(_ptr(out), _ptr(x), _ptr(gamma), x.numel() // cols, cols, float(eps), _ft(x), _stream()), "b2_rmsnorm")
    return out


class Fp8Act:
    """fp8-e4m3 activations in the b2 layout: y uint8 [rows, cols] (k permuted inside groups of 8), scale fp32 [rows],
    tile_sums fp32 [rows, ceil(cols/64)]."""

    def __init__(self, rows, cols, device="cuda"):
        self.y = torch.empty(rows, (cols + 15) // 16 * 16, dtype=torch.uint8, device=device)
        self.scale = torch.empty(rows, dtype=torch.float32, device=device)
        self.tile_sums = torch.empty(rows, (cols + 63) // 64, dtype=torch.float32, device=device)
        self.cols = cols


def quant_fp8(x, gamma=None, eps=1e-6, out=None):
    """Per-token fp8 quantization (optionally fused with RMSNorm) for GemmWQ.run_fp8."""
    rows, cols = x.shape
    out = Fp8Act(rows, cols, x.device) if out is None else out
    check(lib.b2_quant_fp8(_ptr(out.y), out.y.stride(0), _ptr(out.scale), _ptr(out.tile_sums), _ptr(x), _ptr(gamma), rows, cols,
                           float(eps), _stream()), "b2_quant_fp8")
    return out


def rotary(qkv, pos, n_heads, n_groups, base=1e6, rotary_dim=128):
    if qkv.dtype != torch.bfloat16:  # b2_rotary is bf16 only (fp16 models rotate in the fused cache append)
        raise TypeError(f"rotary: qkv must be bfloat16, got {qkv.dtype}")
    r = RopeCfg(float(base), int(rotary_dim), 0)
    check(lib.b2_rotary(_ptr(qkv), _ptr(pos), qkv.shape[0], n_heads, n_groups, 128, C.byref(r), _stream()), "b2_rotary")
    return qkv


def binary(a, b, op, out=None):
    out = torch.empty_like(a) if out is None else out
    check(lib.b2_binary_ft(_ptr(out), _ptr(a), _ptr(b), a.numel(), op, _ft(a), _stream()), "b2_binary")
    return out


def embedding(table, ids, out=None):
    B, H = ids.numel(), table.shape[1]
    out = torch.empty(B, H, dtype=table.dtype, device=table.device) if out is None else out
    check(lib.b2_embedding(_ptr(out), _ptr(table), _ptr(ids), B, H, _stream()), "b2_embedding")
    return out


def argmax(logits, out=None):
    B, n = logits.shape
    out = torch.empty(B, dtype=torch.int64, device=logits.device) if out is None else out
    check(lib.b2_argmax_ft(_ptr(out), None, _ptr(logits), B, n, logits.stride(0), 0, _ft(logits), _stream()), "b2_argmax")
    return out


def argmax_shard(logits, id_offset, ids_out, vals_out):
    if logits.dtype != torch.bfloat16:  # b2_argmax_shard is bf16 only
        raise TypeError(f"argmax_shard: logits must be bfloat16, got {logits.dtype}")
    B, n = logits.shape
    check(lib.b2_argmax_shard(_ptr(ids_out), _ptr(vals_out), _ptr(logits), B, n, logits.stride(0), int(id_offset), _stream()),
          "b2_argmax_shard")
    return ids_out, vals_out


def argmax_merge(all_vals, all_ids, out):
    tp, B = all_vals.shape
    check(lib.b2_argmax_merge(_ptr(out), _ptr(all_vals), _ptr(all_ids), tp, B, _stream()), "b2_argmax_merge")
    return out


def lens_add(lens, delta):
    check(lib.b2_lens_add(_ptr(lens), lens.numel(), int(delta), _stream()), "b2_lens_add")
    return lens
