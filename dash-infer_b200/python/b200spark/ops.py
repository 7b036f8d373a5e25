"""Torch-tensor front end over the C ABI (device memory + streams come from torch; compute does not).

Every call goes through include/b200spark.h on torch's current CUDA stream.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import (ACT_NONE, BIN_ADD, BIN_MUL, DT_BF16, DT_I8, DT_U8, KV_I8, KV_NONE, KV_U4, GemmDesc, GemmFuse, PenaltyParams,
                   ROPE_INTERLEAVED, ROPE_NEOX, QkNorm, RopeCfg, RopeTable, SpanCfg, check, lib)


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

    def tc_cluster(self):
        return lib.b2_gemm_wq_tc_cluster(self.h)

    def launches(self, M):
        """Kernel launches of one call over M rows, as wq_gemm.cu dispatches them: one up to 16 rows; above, one per 64 rows
        on the wgmma kernel, or one per 16 rows on the mma.sync kernel that sub-channel int8 weights keep."""
        if M <= 16:
            return 1
        return -(-M // (16 if self.wbits == 8 and self.group_size != -1 else 64))

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
                                     float(alpha), _ptr(wsb), wsb.numel(), _stream()), "b2_gemm_wq_run", self.launches(M))
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
                                       float(alpha), _ptr(wsb), wsb.numel(), C.byref(f), _stream()), "b2_gemm_wq_run_fused",
              self.launches(M))
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


def _qk_norm(norm, dtype, device):
    """(q_gamma, k_gamma, eps) -> QkNorm; the gammas are [128] contiguous tensors of the model FT on the activations' device"""
    q_gamma, k_gamma, eps = norm
    for g in (q_gamma, k_gamma):
        assert g.shape == (128,) and g.dtype == dtype and g.is_contiguous() and g.device == device, \
            "qk_norm gammas: contiguous [128] tensors of the model dtype on the activations' device"
    return QkNorm(q_gamma.data_ptr(), k_gamma.data_ptr(), float(eps), 0)


def qk_rmsnorm(x, n_heads, n_groups, q_gamma, k_gamma, eps=1e-6, out=None):
    """QKLayerNormNoBeta (b2_qk_rmsnorm): x [rows, >= (n_heads + 2 n_groups) * 128] FT, row stride x.stride(0); the q and k
    heads of each row are RMS-normalised per head with q_gamma / k_gamma [128], the V heads copied.  out may be x."""
    out = torch.empty_strided(x.shape, x.stride(), dtype=x.dtype, device=x.device) if out is None else out
    assert x.dim() == 2 and x.stride(-1) == 1 and out.shape == x.shape and out.stride() == x.stride() and out.dtype == x.dtype
    nrm = _qk_norm((q_gamma, k_gamma, eps), x.dtype, x.device)
    check(lib.b2_qk_rmsnorm(_ptr(out), _ptr(x), x.shape[0], x.stride(0), int(n_heads), int(n_groups), 128, C.byref(nrm), _ft(x),
                            _stream()), "b2_qk_rmsnorm")
    return out


def rope_table(scaling, base, rotary_dim, device=None):
    """Inverse frequencies and attention factor of a Hugging Face `rope_scaling` entry: (inv_freq fp32 [rotary_dim / 2],
    attn_factor), for the table form of the rotary (b2_rope_table: rope=(inv_freq, attn_factor) in _cache_append,
    table=... in rotary).  Computed in fp64 and rounded to fp32 once.  With d = rotary_dim, f = 0 .. d/2 - 1 and
    theta_f = base^(-2f / d) (the unscaled frequencies):

    None, {"rope_type": "default"}: inv_f = theta_f, attn_factor 1.
    linear (factor s): inv_f = theta_f / s.
    yarn (factor s, original_max_position_embeddings L; beta_fast 32, beta_slow 1, attention_factor, mscale,
      mscale_all_dim, truncate optional, as in transformers' _compute_yarn_parameters):
        corr(r) = d ln(L / (2 pi r)) / (2 ln base);  low = floor(corr(beta_fast)), high = ceil(corr(beta_slow)) (no
        floor / ceil with truncate False), clamped to low >= 0, high <= d - 1;
        ramp_f = clamp((f - low) / (high - low), 0, 1) (high += 0.001 when high == low);  e_f = 1 - ramp_f;
        inv_f = (theta_f / s) (1 - e_f) + theta_f e_f
      so frequencies below low keep theta_f and those from high on are interpolated by s.  attn_factor = the dict's
      attention_factor, else mscale(s, mscale) / mscale(s, mscale_all_dim) when both are given, else mscale(s) with
      mscale(s, m=1) = 0.1 m ln(s) + 1 (1 for s <= 1).
    llama3 (factor s, low_freq_factor a, high_freq_factor c, original_max_position_embeddings L):
        wavelength w_f = 2 pi / theta_f;  w_f > L / a: inv_f = theta_f / s;  w_f < L / c: inv_f = theta_f;  between:
        g = (L / w_f - a) / (c - a), inv_f = (1 - g) theta_f / s + g theta_f.   attn_factor 1.
    Any other type (dynamic NTK among them) raises ValueError: the decode stack applies one static table to every
    position, and dynamic scaling would rotate cached keys and the current query with different frequencies."""
    import math
    d = int(rotary_dim)
    assert d > 0 and d % 2 == 0
    theta = float(base) ** (-torch.arange(0, d // 2, dtype=torch.float64) * 2.0 / d)
    sc = dict(scaling or {})
    kind = sc.get("rope_type", sc.get("type", "default"))
    af = 1.0
    if kind == "default":
        inv = theta
    elif kind == "linear":
        inv = theta / float(sc["factor"])
    elif kind == "yarn":
        s, L = float(sc["factor"]), float(sc["original_max_position_embeddings"])
        fast, slow = float(sc.get("beta_fast") or 32), float(sc.get("beta_slow") or 1)

        def corr(r):
            return d * math.log(L / (r * 2 * math.pi)) / (2 * math.log(base))

        low, high = corr(fast), corr(slow)
        if sc.get("truncate", True):
            low, high = math.floor(low), math.ceil(high)
        low, high = max(low, 0), min(high, d - 1)
        if low == high:
            high += 0.001
        ramp = ((torch.arange(d // 2, dtype=torch.float64) - low) / (high - low)).clamp(0, 1)
        e = 1 - ramp
        inv = (theta / s) * (1 - e) + theta * e

        def mscale(x, m=1.0):
            return 1.0 if x <= 1 else 0.1 * m * math.log(x) + 1.0

        if sc.get("attention_factor") is not None:
            af = float(sc["attention_factor"])
        elif sc.get("mscale") and sc.get("mscale_all_dim"):
            af = mscale(s, float(sc["mscale"])) / mscale(s, float(sc["mscale_all_dim"]))
        else:
            af = mscale(s)
    elif kind == "llama3":
        s, a, c = float(sc["factor"]), float(sc["low_freq_factor"]), float(sc["high_freq_factor"])
        L = float(sc["original_max_position_embeddings"])
        w = 2 * math.pi / theta
        g = (L / w - a) / (c - a)
        inv = torch.where(w > L / a, theta / s, torch.where(w < L / c, theta, (1 - g) * theta / s + g * theta))
    else:
        raise ValueError(f"rope_table: unsupported rope scaling type {kind!r} (default, linear, yarn, llama3)")
    inv = inv.to(torch.float32)
    return (inv.to(device) if device is not None else inv), float(af)


ROPE_STYLES = {"neox": ROPE_NEOX, "interleaved": ROPE_INTERLEAVED}


def rope_style(style):
    """b2_rope_cfg.style of "neox" / "interleaved" or of the int itself (ROPE_NEOX, ROPE_INTERLEAVED; others are passed on
    for the library to refuse)"""
    return ROPE_STYLES[style] if isinstance(style, str) else int(style)


def _rope_table(rope, rows, device):
    """(inv_freq, attn_factor[, style]) -> (RopeCfg, RopeTable): inv_freq fp32 [rotary_dim / 2] (one row shared by every
    sequence) or [rows, >= rotary_dim / 2] (row b for sequence b, stride inv_freq.stride(0)) on the activations' device;
    style: the pairing (rope_style), NeoX when left out"""
    inv, af = rope[:2]
    style = rope_style(rope[2]) if len(rope) > 2 else ROPE_NEOX
    assert inv.dtype == torch.float32 and inv.device == device and inv.stride(-1) == 1, \
        "rope table: fp32 inverse frequencies on the activations' device"
    if inv.dim() == 1:
        rd, stride = 2 * inv.shape[0], 0
    else:
        assert inv.dim() == 2 and inv.shape[0] == rows, "rope table: [rotary_dim / 2] or one row per sequence"
        rd, stride = 2 * inv.shape[1], inv.stride(0)
    return RopeCfg(0.0, int(rd), style), RopeTable(inv.data_ptr(), int(stride), float(af), 0)


def _cache_append(cache, qkv, old_lens, q_out=None, rope=None, q_len=None, parents=None, qk_norm=None):
    """Append one step's rows to the span cache (+ optional fused rotary).  q_len None: row b of qkv is sequence b, written at
    position old_lens[b].  q_len: row b*q_len + t is token t of sequence b, written at position old_lens[b] + t; with parents
    (int32 [B, q_len]) it is node t of sequence b's draft tree, written at slot old_lens[b] + t with rotary position
    old_lens[b] + depth(t).  qk_norm = (q_gamma, k_gamma, eps): the per-head Q/K RMSNorm before rotary
    (b2_span_cache_append_qknorm), every step form.  rope = (base, rotary_dim): the rotary with base^(-2f / rotary_dim);
    rope = (inv_freq tensor, attn_factor): the scaled rotary from a frequency table (rope_table; one row, or one row per
    sequence) in every step form, with or without qk_norm (b2_span_cache_append_rope_table).  Either tuple may carry a
    third element, the pairing style (rope_style: "neox" / "interleaved" or ROPE_NEOX / ROPE_INTERLEAVED); NeoX without
    it."""
    cfg = cache.cfg
    rows = qkv.shape[0]
    assert rows % (q_len or 1) == 0 and (parents is None or (q_len and parents.dtype == torch.int32 and parents.is_contiguous()))
    if q_out is None:
        q_out = torch.empty(rows, cfg.n_heads * cfg.head_size, dtype=qkv.dtype, device=qkv.device)
    head = (C.byref(cfg), _ptr(cache.k_tab), _ptr(cache.v_tab), _ptr(q_out), _ptr(qkv), _ptr(old_lens))
    if rope is not None and isinstance(rope[0], torch.Tensor):
        r, tab = _rope_table(rope, rows // (q_len or 1), qkv.device)
        nrm = _qk_norm(qk_norm, qkv.dtype, qkv.device) if qk_norm is not None else None
        check(lib.b2_span_cache_append_rope_table(*head, _ptr(parents), rows // (q_len or 1), int(q_len or 1), C.byref(r),
                                                  C.byref(tab), C.byref(nrm) if nrm is not None else None, _stream()),
              "b2_span_cache_append_rope_table")
        return q_out
    r = RopeCfg(float(rope[0]), int(rope[1]), rope_style(rope[2]) if len(rope) > 2 else ROPE_NEOX) if rope is not None else None
    tail = (C.byref(r) if r is not None else None, _stream())
    if qk_norm is not None:
        nrm = _qk_norm(qk_norm, qkv.dtype, qkv.device)
        check(lib.b2_span_cache_append_qknorm(*head, _ptr(parents), rows // (q_len or 1), int(q_len or 1), tail[0], C.byref(nrm),
                                              tail[1]), "b2_span_cache_append_qknorm")
    elif q_len is None:
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


def _spec_accept(accepted, next_ids, old_lens, new_lens, tokens, pred, path=None, parents=None, offsets=None):
    """Greedy verification of a multi-token step (b2_spec_accept): tokens / pred int64 [B, T]; writes accepted (int32 [B]),
    next_ids (int64 [B] or None) and tokens[:, 0], advances old_lens by the accepted counts and sets new_lens = old_lens + T.
    With parents (int32 [B, T]) the step is a draft tree (b2_spec_accept_tree), which also writes path (int32 [B, T], the first
    accepted[b] entries).  With offsets (int64 [B], the sequences' draw counters) pred holds sample_tokens' draws and the
    sampled form runs (b2_spec_accept_sampled): the same walk, then offsets += accepted."""
    B, T = tokens.shape
    assert tokens.is_contiguous() and pred.is_contiguous() and pred.shape == tokens.shape
    if parents is not None:
        assert parents.dtype == torch.int32 and parents.is_contiguous() and parents.shape == tokens.shape
        assert path.dtype == torch.int32 and path.is_contiguous() and path.shape == tokens.shape
    if offsets is not None:
        assert offsets.dtype == torch.int64 and offsets.is_contiguous() and tuple(offsets.shape) == (B,), \
            f"spec_accept: offsets must be [{B}] int64 contiguous"
        check(lib.b2_spec_accept_sampled(_ptr(accepted), _ptr(path), _ptr(next_ids), _ptr(old_lens), _ptr(new_lens),
                                         _ptr(tokens), _ptr(pred), _ptr(parents), _ptr(offsets), B, T, _stream()),
              "b2_spec_accept_sampled")
        return accepted if parents is None else (accepted, path)
    if parents is None:
        check(lib.b2_spec_accept(_ptr(accepted), _ptr(next_ids), _ptr(old_lens), _ptr(new_lens), _ptr(tokens), _ptr(pred), B, T,
                                 _stream()), "b2_spec_accept")
        return accepted
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


def rotary(qkv, pos, n_heads, n_groups, base=1e6, rotary_dim=128, table=None, style=ROPE_NEOX):
    """In-place rotary of the q and k heads of qkv [rows, (n_heads + 2 n_groups) * 128] at positions pos [rows], pairing
    style (rope_style: NeoX rotate-half by default, or "interleaved").  table = (inv_freq, attn_factor) (rope_table;
    [rotary_dim / 2], or [rows, >= rotary_dim / 2] with row b for qkv row b): the scaled form b2_rotary_table, bf16 or fp16,
    base and rotary_dim unused; otherwise b2_rotary, bf16 only."""
    if table is not None:
        r, tab = _rope_table(tuple(table[:2]) + (style,), qkv.shape[0], qkv.device)
        check(lib.b2_rotary_table(_ptr(qkv), _ptr(pos), qkv.shape[0], n_heads, n_groups, 128, C.byref(r), C.byref(tab), _ft(qkv),
                                  _stream()), "b2_rotary_table")
        return qkv
    if qkv.dtype != torch.bfloat16:  # b2_rotary is bf16 only (fp16 models rotate in the fused cache append)
        raise TypeError(f"rotary: qkv must be bfloat16, got {qkv.dtype}")
    r = RopeCfg(float(base), int(rotary_dim), rope_style(style))
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


def _lp_outputs(rows, n_top, device, out):
    """(ids [rows] int64, tok_lp [rows] fp32, top_ids [rows, n_top] int64 or None, top_lp [rows, n_top] fp32 or None)"""
    if out is not None:
        ids, tok_lp, top_ids, top_lp = out
    else:
        ids = torch.empty(rows, dtype=torch.int64, device=device)
        tok_lp = torch.empty(rows, dtype=torch.float32, device=device)
        top_ids = torch.empty(rows, n_top, dtype=torch.int64, device=device) if n_top else None
        top_lp = torch.empty(rows, n_top, dtype=torch.float32, device=device) if n_top else None
    for t, dt, shape in ((ids, torch.int64, (rows,)), (tok_lp, torch.float32, (rows,)), (top_ids, torch.int64, (rows, n_top)),
                         (top_lp, torch.float32, (rows, n_top))):
        assert t is None or (t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape), \
            f"logprobs outputs: {shape} {dt} contiguous"
    assert (top_ids is None) == (n_top == 0) and (top_lp is None) == (n_top == 0)
    return ids, tok_lp, top_ids, top_lp


def _tok_ids(tok_ids, rows):
    assert tok_ids is None or (tok_ids.dtype == torch.int64 and tok_ids.is_contiguous() and tok_ids.numel() == rows)
    return _ptr(tok_ids)


def logprobs(logits, n_top, tok_ids=None, out=None):
    """Log-probabilities of the rows of logits [rows, n] FT (b2_logprobs; any row stride): returns (ids, tok_lp, top_ids,
    top_lp) — the argmax ids (== argmax()), the logprob of tok_ids[r] (of the top-1 without tok_ids), and the top n_top
    (0 <= n_top <= 10) ids and logprobs in argmax order (None when n_top == 0).  out: the four tensors to write (ids or
    tok_lp may be None)."""
    rows, n = logits.shape
    assert logits.stride(-1) == 1
    ids, tok_lp, top_ids, top_lp = _lp_outputs(rows, n_top, logits.device, out)
    check(lib.b2_logprobs(_ptr(ids), _ptr(tok_lp), _ptr(top_ids), _ptr(top_lp), _tok_ids(tok_ids, rows), _ptr(logits), rows, n,
                          logits.stride(0), int(n_top), _ft(logits), _stream()), "b2_logprobs")
    return ids, tok_lp, top_ids, top_lp


def logprobs_partial_bytes(n_top):
    return lib.b2_logprobs_partial_bytes(int(n_top))


def logprobs_shard(logits, n_top, id_offset, tok_ids=None, out=None):
    """The vocab-split form's first half (b2_logprobs_shard): logits [rows, n] hold vocab ids id_offset .. id_offset + n - 1;
    returns the rows' partial records, uint8 [rows, logprobs_partial_bytes(n_top)] (opaque bytes for an all-gather)."""
    rows, n = logits.shape
    assert logits.stride(-1) == 1
    if out is None:
        out = torch.empty(rows, logprobs_partial_bytes(n_top), dtype=torch.uint8, device=logits.device)
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.numel() == rows * logprobs_partial_bytes(n_top)
    check(lib.b2_logprobs_shard(_ptr(out), _tok_ids(tok_ids, rows), _ptr(logits), rows, n, logits.stride(0), int(id_offset),
                                int(n_top), _ft(logits), _stream()), "b2_logprobs_shard")
    return out


def logprobs_merge(all_partials, n_top, out=None):
    """The second half (b2_logprobs_merge): all_partials uint8 [nranks, rows * bytes] (or [nranks, rows, bytes]), the ranks'
    records as all-gathered; returns logprobs()' outputs over the whole vocabulary."""
    nranks, rb = all_partials.shape[0], logprobs_partial_bytes(n_top)
    rows = all_partials[0].numel() // rb
    assert all_partials.dtype == torch.uint8 and all_partials.is_contiguous()
    assert rows > 0 and all_partials[0].numel() == rows * rb, "records of another n_top: %d bytes per rank" % all_partials[0].numel()
    ids, tok_lp, top_ids, top_lp = _lp_outputs(rows, n_top, all_partials.device, out)
    check(lib.b2_logprobs_merge(_ptr(ids), _ptr(tok_lp), _ptr(top_ids), _ptr(top_lp), _ptr(all_partials), nranks, rows, int(n_top),
                                _stream()), "b2_logprobs_merge")
    return ids, tok_lp, top_ids, top_lp


def _sampling_args(rows, B, out, temperature, top_k, top_p, seeds, offsets, what):
    for t, dt, name, n in ((out, torch.int64, "out", rows), (temperature, torch.float32, "temperature", B),
                           (top_k, torch.int32, "top_k", B), (top_p, torch.float32, "top_p", B), (seeds, torch.int64, "seeds", B),
                           (offsets, torch.int64, "offsets", B)):
        if t is None:  # no output (sample_shard)
            continue
        assert t.dtype == dt and t.is_contiguous() and tuple(t.shape) == (n,), f"{what}: {name} must be [{n}] {dt} contiguous"


def sample(logits, temperature, top_k, top_p, seeds, offsets, out=None):
    """A token drawn from each row of logits [rows, n] FT (b2_sample; any row stride): temperature, top_p fp32 [rows], top_k
    int32 [rows], seeds, offsets int64 [rows] (read as uint64 bits), all on the device.  Advances offsets by 1 in place and
    returns the ids, int64 [rows] (out, if given).  The contract, step by step: include/b200spark.h."""
    rows, n = logits.shape
    assert logits.stride(-1) == 1
    out = torch.empty(rows, dtype=torch.int64, device=logits.device) if out is None else out
    _sampling_args(rows, rows, out, temperature, top_k, top_p, seeds, offsets, "sample")
    check(lib.b2_sample(_ptr(out), _ptr(logits), rows, n, logits.stride(0), _ptr(temperature), _ptr(top_k), _ptr(top_p),
                        _ptr(seeds), _ptr(offsets), _ft(logits), _stream()), "b2_sample")
    return out


def sample_tokens(logits, q_len, temperature, top_k, top_p, seeds, offsets, parents=None, out=None):
    """The draws of a verify step (b2_sample_tokens): logits [B * q_len, n] FT (any row stride), row b*q_len + t = draft node
    t of sequence b, drawn with sequence b's parameters (temperature, top_k, top_p, seeds, offsets: [B], as for sample()) at
    counter offsets[b] + depth(t) (t for a chain; parents int32 [B, q_len] for a draft tree).  The offsets are only read.
    Returns the ids, int64 [B * q_len] (out, if given)."""
    rows, n = logits.shape
    assert logits.stride(-1) == 1 and q_len >= 1 and rows % q_len == 0, "sample_tokens: logits rows = B * q_len"
    B = rows // q_len
    out = torch.empty(rows, dtype=torch.int64, device=logits.device) if out is None else out
    _sampling_args(rows, B, out, temperature, top_k, top_p, seeds, offsets, "sample_tokens")
    assert parents is None or (parents.dtype == torch.int32 and parents.is_contiguous() and tuple(parents.shape) == (B, q_len)), \
        f"sample_tokens: parents must be [{B}, {q_len}] int32 contiguous"
    check(lib.b2_sample_tokens(_ptr(out), _ptr(logits), B, q_len, _ptr(parents), n, logits.stride(0), _ptr(temperature),
                               _ptr(top_k), _ptr(top_p), _ptr(seeds), _ptr(offsets), _ft(logits), _stream()), "b2_sample_tokens")
    return out


def sample_shard_record_bytes(phase):
    return lib.b2_sample_shard_record_bytes(int(phase))


def sample_shard_state_bytes():
    return lib.b2_sample_shard_state_bytes()


def sample_shard(phase, logits, id_offset, n_total, temperature, top_k, top_p, seeds, offsets, state, all_records=None,
                 out=None, nranks=None):
    """One phase of sampling under tensor parallelism (b2_sample_shard) on this rank's shard: logits [rows, n] FT hold
    columns id_offset .. id_offset + n - 1 of rows of n_total columns; the sampling parameters are sample()'s, the same on
    every rank; state uint8 [rows, sample_shard_state_bytes()] is this rank's own.  all_records: the previous phase's
    records of every rank as all-gathered, uint8 [nranks, rows * bytes] (None for phase 0).  Returns this phase's records,
    uint8 [rows, sample_shard_record_bytes(phase)] (out, if given)."""
    rows, n = logits.shape
    assert logits.stride(-1) == 1
    assert 0 <= phase < _lib.SAMPLE_SHARD_PHASES and (all_records is None) == (phase == 0)
    _sampling_args(rows, rows, None, temperature, top_k, top_p, seeds, offsets, "sample_shard")
    assert state.dtype == torch.uint8 and state.is_contiguous() and state.numel() == rows * sample_shard_state_bytes()
    if all_records is not None:
        nranks = all_records.shape[0]
        rb = sample_shard_record_bytes(phase - 1)
        assert all_records.dtype == torch.uint8 and all_records.is_contiguous() and all_records.numel() == nranks * rows * rb, \
            f"sample_shard: all_records must be [nranks, {rows} * {rb}] uint8 contiguous (phase {phase - 1}'s records)"
    rb = sample_shard_record_bytes(phase)
    out = torch.empty(rows, rb, dtype=torch.uint8, device=logits.device) if out is None else out
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.numel() == rows * rb
    check(lib.b2_sample_shard(int(phase), _ptr(out), _ptr(state), _ptr(all_records), int(nranks or 1), _ptr(logits), rows, n,
                              logits.stride(0), int(id_offset), int(n_total), _ptr(temperature), _ptr(top_k), _ptr(top_p),
                              _ptr(seeds), _ptr(offsets), _ft(logits), _stream()), "b2_sample_shard")
    return out


def sample_shard_merge(all_records, state, offsets, out=None):
    """The end of sampling under tensor parallelism (b2_sample_shard_merge): all_records uint8 [nranks, rows * 8], the last
    phase's records as all-gathered; state and offsets this rank's.  Advances offsets by 1 in place and returns the ids,
    int64 [rows] (out, if given): b2_sample's ids of the whole rows, the same on every rank."""
    nranks, rows = all_records.shape[0], offsets.numel()
    assert all_records.dtype == torch.uint8 and all_records.is_contiguous()
    assert all_records.numel() == nranks * rows * sample_shard_record_bytes(_lib.SAMPLE_SHARD_PHASES - 1)
    assert state.dtype == torch.uint8 and state.numel() == rows * sample_shard_state_bytes()
    assert offsets.dtype == torch.int64 and offsets.is_contiguous()
    out = torch.empty(rows, dtype=torch.int64, device=offsets.device) if out is None else out
    assert out.dtype == torch.int64 and out.is_contiguous() and out.numel() == rows
    check(lib.b2_sample_shard_merge(_ptr(out), _ptr(all_records), _ptr(state), nranks, rows, _ptr(offsets), _stream()),
          "b2_sample_shard_merge")
    return out


class _SampleTPBuffers(dict):
    def view(self, rows):
        """the buffers of the first `rows` rows, sharing the storage (DecodeStack.set_batch)"""
        n = self["state"].shape[0]
        return _SampleTPBuffers(state=self["state"][:rows], rec=[r[:rows] for r in self["rec"]],
                                all=[a.view(-1)[:a.numel() // n * rows].view(a.shape[0], -1) for a in self["all"]])


def sample_tp_buffers(rows, nranks, device="cuda"):
    """The buffers of sample_tp() for `rows` rows and `nranks` ranks: this rank's state, each phase's own records and
    their all-gathered form ([nranks, rows * bytes], the layout an all-gather writes).  view(r) gives the first r rows'."""
    P = _lib.SAMPLE_SHARD_PHASES
    u8 = dict(dtype=torch.uint8, device=device)
    return _SampleTPBuffers(state=torch.empty(rows, sample_shard_state_bytes(), **u8),
                            rec=[torch.empty(rows, sample_shard_record_bytes(p), **u8) for p in range(P)],
                            all=[torch.empty(nranks, rows * sample_shard_record_bytes(p), **u8) for p in range(P)])


def sample_tp(logits_shard, id_offset, n_total, temperature, top_k, top_p, seeds, offsets, exchange, nranks, out=None,
              bufs=None):
    """sample() of the whole rows under tensor parallelism, on one rank: every phase of b2_sample_shard, each followed by
    exchange(record, all_records) (the all-gather of this rank's records into all_records [nranks, rows * bytes] in rank
    order: Comm.allgather, torch.distributed.all_gather_into_tensor, ...), then the merge.  Every rank calls it with its
    own shard and the same parameters; every rank returns the same ids (out, if given), b2_sample's ids of the
    concatenated rows, and advances its offsets by 1.  The launch sequence is static, so a CUDA graph can capture it.
    bufs: sample_tp_buffers(rows, nranks), kept by a caller that captures graphs."""
    rows = logits_shard.shape[0]
    bufs = sample_tp_buffers(rows, nranks, logits_shard.device) if bufs is None else bufs
    prev = None
    for p in range(_lib.SAMPLE_SHARD_PHASES):
        sample_shard(p, logits_shard, id_offset, n_total, temperature, top_k, top_p, seeds, offsets, bufs["state"], prev,
                     out=bufs["rec"][p], nranks=nranks)
        exchange(bufs["rec"][p], bufs["all"][p])
        prev = bufs["all"][p]
    return sample_shard_merge(prev, bufs["state"], offsets, out=out)


def lens_add(lens, delta):
    check(lib.b2_lens_add(_ptr(lens), lens.numel(), int(delta), _stream()), "b2_lens_add")
    return lens


class TokenHistory:
    """The per-sequence token history of the logits processor (b2_token_history), on the device: `rows` slots of at most
    max_len tokens each over a vocabulary of `vocab` ids.  tokens [rows, max_len], len / prompt_len / n_distinct [rows],
    table [rows, vocab] (bit 30: in the prompt, bits 0..29: generated count) and distinct [rows, max_len], all int32.
    view(b) shares the storage with the first b slots (DecodeStack.set_batch)."""

    _FIELDS = ("tokens", "len", "prompt_len", "table", "distinct", "n_distinct")

    def __init__(self, rows, max_len, vocab, device="cuda"):
        assert rows >= 1 and 1 <= max_len < 2 ** 30 and vocab >= 1
        self.rows, self.max_len, self.vocab = rows, max_len, vocab
        z = lambda *shape: torch.zeros(*shape, dtype=torch.int32, device=device)
        self.tokens, self.len, self.prompt_len = z(rows, max_len), z(rows), z(rows)
        self.table, self.distinct, self.n_distinct = z(rows, vocab), z(rows, max_len), z(rows)
        self.c = _lib.TokenHistory(*(t.data_ptr() for t in (self.tokens, self.len, self.prompt_len, self.table, self.distinct,
                                                              self.n_distinct)), max_len, vocab)

    def view(self, rows):
        assert 1 <= rows
        v = object.__new__(TokenHistory)
        v.__dict__.update(self.__dict__)
        v.rows = rows
        for k in self._FIELDS:
            setattr(v, k, getattr(self, k)[:rows])
        return v

    def load(self, slot, ids, prompt_len=None):
        """Slot `slot` := ids (the prompt first; prompt_len of them, all by default), after clearing its previous tokens."""
        ids = torch.as_tensor(ids, dtype=torch.int32).reshape(-1).to(self.tokens.device)
        n = ids.numel()
        prompt_len = n if prompt_len is None else int(prompt_len)
        assert 0 <= slot < self.rows, f"history slot {slot} outside [0, {self.rows})"
        assert n <= self.max_len and 0 <= prompt_len <= n, f"history: {n} tokens (max {self.max_len}), prompt {prompt_len}"
        assert n == 0 or (int(ids.min()) >= 0 and int(ids.max()) < self.vocab), f"history: token ids outside [0, {self.vocab})"
        check(lib.b2_history_load(C.byref(self.c), int(slot), _ptr(ids), n, prompt_len, _stream()), "b2_history_load")
        return self

    def reset(self, slot):
        return self.load(slot, [], 0)

    def append(self, ids):
        """Append ids[r] (int64 [rows], on the device) to slot r, for the first ids.numel() slots."""
        assert ids.dtype == torch.int64 and ids.is_contiguous() and ids.numel() <= self.rows
        check(lib.b2_history_append(C.byref(self.c), _ptr(ids), ids.numel(), _stream()), "b2_history_append")
        return self

    def append_tokens(self, pred, accepted, path=None):
        """Append the emitted tokens of a verify step to slot b, for the first pred.shape[0] slots (b2_history_append_tokens):
        pred[b, path[b, i]] (chain, path None: pred[b, i]) for i < accepted[b].  pred int64 [B, T], accepted int32 [B], path
        int32 [B, T], on the device."""
        B, T = pred.shape
        assert pred.dtype == torch.int64 and pred.is_contiguous() and B <= self.rows
        assert accepted.dtype == torch.int32 and accepted.is_contiguous() and tuple(accepted.shape) == (B,)
        assert path is None or (path.dtype == torch.int32 and path.is_contiguous() and path.shape == pred.shape)
        check(lib.b2_history_append_tokens(C.byref(self.c), _ptr(pred), _ptr(accepted), _ptr(path), B, T, _stream()),
              "b2_history_append_tokens")
        return self

    def snapshot(self):
        return [getattr(self, k).clone() for k in self._FIELDS]

    def restore(self, snap):
        for k, s in zip(self._FIELDS, snap):
            getattr(self, k).copy_(s)


def ngram_draft(history, tokens, parents, n_min, n_max, width, n_draft=None):
    """N-gram (prompt-lookup) drafts of a verify step from the token history (b2_ngram_draft), written in place: tokens int64
    [B, T] (column 0, the last emitted token, is read; columns 1.. get the drafts), parents int32 [B, T] for a draft tree
    (None: a chain, width 1), n_draft int32 [B] (optional) = the drafts filled per sequence.  Slot b of history is
    sequence b.  The contract (matching, periodic continuation, trie numbering, padding): include/b200spark.h."""
    B, T = tokens.shape
    assert tokens.dtype == torch.int64 and tokens.is_contiguous() and B <= history.rows
    assert parents is None or (parents.dtype == torch.int32 and parents.is_contiguous() and parents.shape == tokens.shape)
    assert n_draft is None or (n_draft.dtype == torch.int32 and n_draft.is_contiguous() and tuple(n_draft.shape) == (B,))
    check(lib.b2_ngram_draft(_ptr(tokens), _ptr(parents), _ptr(n_draft), C.byref(history.c), B, T, int(n_min), int(n_max),
                             int(width), _stream()), "b2_ngram_draft")
    return tokens


class Penalties:
    """Per-row parameters of b2_penalize, device arrays [rows]: repetition, presence, frequency (fp32), no_repeat_ngram,
    min_length, eos_id, suppress (int32).  They start neutral (1, 0, 0, 0, 0, -1, 0), which changes nothing."""

    FLOAT = ("repetition", "presence", "frequency")
    INT = ("no_repeat_ngram", "min_length", "eos_id", "suppress")

    def __init__(self, rows, device="cuda"):
        self.rows = rows
        self.repetition = torch.ones(rows, dtype=torch.float32, device=device)
        self.presence = torch.zeros(rows, dtype=torch.float32, device=device)
        self.frequency = torch.zeros(rows, dtype=torch.float32, device=device)
        for k in self.INT:
            setattr(self, k, torch.zeros(rows, dtype=torch.int32, device=device))
        self.eos_id.fill_(-1)

    def view(self, rows):
        v = object.__new__(Penalties)
        v.rows = rows
        for k in self.FLOAT + self.INT:
            setattr(v, k, getattr(self, k)[:rows])
        return v

    def set(self, repetition=None, presence=None, frequency=None, no_repeat_ngram=None, min_length=None, eos_id=None,
            suppress_repetition_in_generation=None):
        """Write parameters in place (a scalar or [rows] values each; None keeps the value).  The ranges are the reference's
        request checks (as_engine.cpp): repetition in [0, 2], presence and frequency in [-2, 2]; n-gram size and min-length
        >= 0."""
        vals = dict(repetition=repetition, presence=presence, frequency=frequency, no_repeat_ngram=no_repeat_ngram,
                    min_length=min_length, eos_id=eos_id, suppress=suppress_repetition_in_generation)
        lim = dict(repetition=(0.0, 2.0), presence=(-2.0, 2.0), frequency=(-2.0, 2.0), no_repeat_ngram=(0, 2 ** 31 - 1),
                   min_length=(0, 2 ** 31 - 1), eos_id=(-2 ** 31, 2 ** 31 - 1), suppress=(0, 1))
        for k, v in vals.items():
            if v is None:
                continue
            t = getattr(self, k)
            h = torch.as_tensor(v, dtype=torch.float64).expand(t.shape)
            lo, hi = lim[k]
            if not bool(((h >= lo) & (h <= hi)).all()):
                raise ValueError(f"penalties: {k} must lie in [{lo}, {hi}]")
            if k in self.INT and not bool((h == h.round()).all()):
                raise ValueError(f"penalties: {k} must be an integer")
            t.copy_(h.to(t.dtype))
        return self

    def c(self):
        return PenaltyParams(*(getattr(self, k).data_ptr() for k in self.FLOAT + self.INT), None)


def penalize(logits, history, params, id_offset=0):
    """The logits processor (b2_penalize), in place on logits [rows, n] FT (any row stride), which hold vocabulary ids
    [id_offset, id_offset + n): row r reads history slot r and params row r.  Returns logits."""
    rows, n = logits.shape
    assert logits.stride(-1) == 1
    assert rows <= history.rows and rows <= params.rows, "penalize: more rows than history slots or parameter rows"
    check(lib.b2_penalize(_ptr(logits), rows, n, logits.stride(0), int(id_offset), C.byref(history.c), C.byref(params.c()),
                          _ft(logits), _stream()), "b2_penalize")
    return logits


def penalize_tokens(logits, history, params, tokens, parents=None, id_offset=0):
    """The logits processor of a verify step (b2_penalize_tokens), in place on logits [B * T, n] FT (any row stride), which
    hold vocabulary ids [id_offset, id_offset + n): row b*T + t = draft node t of sequence b, processed as b2_penalize
    would process it with history slot b followed by the drafts on the path from the root to t (tokens int64 [B, T], the
    step's token array; parents int32 [B, T] for a draft tree, None for a chain).  Params row b is sequence b's; the
    history is only read.  Returns logits."""
    rows, n = logits.shape
    B, T = tokens.shape
    assert logits.stride(-1) == 1 and rows == B * T, f"penalize_tokens: logits rows must be B * T = {B * T}"
    assert tokens.dtype == torch.int64 and tokens.is_contiguous()
    assert parents is None or (parents.dtype == torch.int32 and parents.is_contiguous() and parents.shape == tokens.shape), \
        f"penalize_tokens: parents must be [{B}, {T}] int32 contiguous"
    assert B <= history.rows and B <= params.rows, "penalize_tokens: more sequences than history slots or parameter rows"
    check(lib.b2_penalize_tokens(_ptr(logits), B, T, _ptr(parents), _ptr(tokens), n, logits.stride(0), int(id_offset),
                                 C.byref(history.c), C.byref(params.c()), _ft(logits), _stream()), "b2_penalize_tokens")
    return logits
