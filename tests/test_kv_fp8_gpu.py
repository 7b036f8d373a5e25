"""GPU: the fp8-e4m3 KV cache (B2_KV_FP8) — append, prefill writer, fused rotary, attention, decode stack and the C++ operator.

Contract (tests/kv_fp8_ref.py): the span bytes are bit-identical to the CPU quantizer (IEEE fp32 scale and reciprocal,
round-to-nearest-even e4m3, saturating).  Attention on the device's own cache bytes is within 2e-3 abs (+ the output type's
rounding) of fp64 attention on the dequantized cache, like the other modes (tests/test_attn_gpu.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import kv_fp8_ref as F8
from oracle import kvcache_ref as KV

pytestmark = pytest.mark.gpu

FP8 = F8.QUANT_FP8
ALPHA = 1.0 / np.sqrt(128)


def _fill(mode, rows, lens, nH, nG, span, max_len, dtype=torch.bfloat16, fill=0):
    """Append rows [T, B, (nH + 2 nG) * 128] (fp32, rounded to dtype here) token by token with the product append kernel.
    Sequences already at their final length keep re-writing position lens[b] (beyond their length)."""
    from b200spark import ops
    T, B = rows.shape[0], rows.shape[1]
    cache = ops.SpanCache(B, max_len, nH, nG, span, mode, fill=fill, dtype=dtype)
    dev = torch.from_numpy(rows).to(dtype).cuda()
    for t in range(T):
        pos = torch.tensor([min(t, lens[b]) for b in range(B)], dtype=torch.int32, device="cuda")
        ops.cache_append(cache, dev[t], pos)
    torch.cuda.synchronize()
    return cache


def _rows(rng, T, B, nH, nG, dtype=torch.bfloat16):
    x = rng.standard_normal((T, B, (nH + 2 * nG) * 128)).astype(np.float32)
    return torch.from_numpy(x).to(dtype).float().numpy()


def _mirror_device(cache, lens, nG, span):
    """SpanCacheFp8Ref holding the device's own span bytes (attention parity on identical cache contents)."""
    k, v = F8.SpanCacheFp8Ref(span, nG), F8.SpanCacheFp8Ref(span, nG)
    for ref, which in ((k, "k"), (v, "v")):
        for b in range(len(lens)):
            ref.add_sequence()
            ref.spans[b] = [cache.span_view(which, b, si).cpu().numpy().copy() for si in range((lens[b] + span - 1) // span)]
    return k, v


def _attend(cache, q, lens, max_len, dtype):
    from b200spark import ops
    B = len(lens)
    attn = ops.SpanAttn(cache.cfg, B)
    new_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    qd = torch.from_numpy(q.reshape(B, -1)).to(dtype).cuda()
    out = attn(qd, cache, new_lens, max_len, ops.Workspace())
    out2 = attn(qd, cache, new_lens, max_len, ops.Workspace())
    torch.cuda.synchronize()
    assert out.dtype == dtype and torch.equal(out, out2)  # deterministic, counters re-armed
    return out.float().cpu().numpy().reshape(B, -1, 128)


def _check(got, ref, dtype):
    # 2e-3 abs + the rounding of the stored output / fp16 probabilities (bf16 2^-7, fp16 2^-9 relative envelope)
    rel = 2.0 ** -9 if dtype == torch.float16 else 2.0 ** -7
    assert np.isfinite(got).all()
    assert np.all(np.abs(got - ref) <= 2e-3 + rel * np.abs(ref)), float(np.abs(got - ref).max())


def _span_rows(buf, nG, span):
    codes = buf[:nG * span * 128].reshape(nG, span, 128)
    prm = buf[nG * span * 128:].view(np.float32).reshape(nG, span, 2)
    return codes, prm


# ---------------------------------------------------------------------------------------------------------------- writers
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("span", [16, 128])
def test_append_bit_exact(dtype, span):
    B, nH, nG = 3, 8, 2
    lens = [37, 5, 130]
    rows = _rows(np.random.default_rng(span + (dtype == torch.float16)), max(lens), B, nH, nG, dtype)
    cache = _fill(FP8, rows, lens, nH, nG, span, 140, dtype)
    for b in range(B):
        for si in range((lens[b] + span - 1) // span):
            n = min(span, lens[b] - si * span)
            for which, lo in (("k", nH), ("v", nH + nG)):
                x = rows[si * span: si * span + n, b].reshape(n, nH + 2 * nG, 128)[:, lo:lo + nG].transpose(1, 0, 2)
                q, _, s = F8.quant_rows(x)
                codes, prm = _span_rows(cache.span_view(which, b, si).cpu().numpy(), nG, span)
                assert np.array_equal(codes[:, :n], q), (b, si, which)
                assert np.array_equal(prm[:, :n, 1], s), (b, si, which)
                assert not prm[:, :n, 0].view(np.uint32).any()  # zero slot: +0.0
                assert not np.isin(codes[:, :n], [0x7F, 0xFF]).any()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_context_copy_matches_oracle_and_append(dtype):
    """Prefill writer on strided K / V views of a fused qkv tensor: bit-identical to the CPU quantizer and to what appends of
    the same rows write."""
    from b200spark import ops
    nH, nG, span, T = 8, 2, 16, 45
    W = (nH + 2 * nG) * 128
    rows = _rows(np.random.default_rng(7), T, 1, nH, nG, dtype)
    qkv = torch.from_numpy(rows[:, 0]).to(dtype).cuda()
    pre = ops.SpanCache(1, 64, nH, nG, span, FP8, fill=0xFF, dtype=dtype)
    ops.context_copy(pre, "k", 0, qkv[:, nH * 128:])
    ops.context_copy(pre, "v", 0, qkv[:, (nH + nG) * 128:])
    app = _fill(FP8, rows, [T], nH, nG, span, 64, dtype, fill=0xFF)
    assert qkv[:, nH * 128:].stride(0) == W
    for si in range((T + span - 1) // span):
        n = min(span, T - si * span)
        for which, lo in (("k", nH), ("v", nH + nG)):
            x = rows[si * span: si * span + n, 0].reshape(n, nH + 2 * nG, 128)[:, lo:lo + nG].transpose(1, 0, 2)
            q, _, s = F8.quant_rows(x)
            pc, pp = _span_rows(pre.span_view(which, 0, si).cpu().numpy(), nG, span)
            ac, ap = _span_rows(app.span_view(which, 0, si).cpu().numpy(), nG, span)
            assert np.array_equal(pc[:, :n], q) and np.array_equal(pp[:, :n, 1], s), (si, which)
            assert np.array_equal(pc[:, :n], ac[:, :n]) and np.array_equal(pp[:, :n], ap[:, :n]), (si, which)
            assert not pp[:, :n, 0].view(np.uint32).any()
            if n < span:  # rows >= seq_len are left untouched
                assert (pc[:, n:] == 0xFF).all()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fused_rope_append(dtype):
    """The fp8 bytes of a fused-rotary append are the CPU quantization of the rows an unquantized cache stores with the same
    rotary."""
    nH, nG, span = 8, 2, 128
    lens = [5, 130]
    rows = _rows(np.random.default_rng(11), 1, 2, nH, nG, dtype)
    pos = torch.tensor(lens, dtype=torch.int32, device="cuda")
    from b200spark import ops
    dev = torch.from_numpy(rows[0]).to(dtype).cuda()
    plain = ops.SpanCache(2, 256, nH, nG, span, KV.QUANT_NONE, dtype=dtype)
    f8 = ops.SpanCache(2, 256, nH, nG, span, FP8, dtype=dtype)
    q0 = ops.cache_append(plain, dev, pos, rope=(1e6, 128))
    q1 = ops.cache_append(f8, dev, pos, rope=(1e6, 128))
    torch.cuda.synchronize()
    assert torch.equal(q0, q1)
    for b, p in enumerate(lens):
        si, r = p // span, p % span
        for which in ("k", "v"):
            stored = plain.span_view(which, b, si).cpu()[:nG * span * 256].view(dtype).reshape(nG, span, 128)[:, r].float().numpy()
            q, _, s = F8.quant_rows(stored)
            codes, prm = _span_rows(f8.span_view(which, b, si).cpu().numpy(), nG, span)
            assert np.array_equal(codes[:, r], q) and np.array_equal(prm[:, r, 1], s), (b, which)


# -------------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("span", [16, 32, 64, 128])
@pytest.mark.parametrize("nH,nG", [(8, 2), (7, 1), (28, 4), (16, 1)])
def test_attention_small(nH, nG, span, dtype):
    lens = [1, 63, 64, 65, 200]
    B = len(lens)
    rows = _rows(np.random.default_rng(span * 7 + nH), max(lens), B, nH, nG, dtype)
    cache = _fill(FP8, rows, lens, nH, nG, span, 256, dtype)
    kref, vref = _mirror_device(cache, lens, nG, span)
    q = np.stack([rows[lens[b] - 1, b, :nH * 128] for b in range(B)]).reshape(B, nH, 128)
    got = _attend(cache, q, lens, 256, dtype)
    _check(got, KV.attention_ref(q, kref, vref, lens, nH, ALPHA), dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_attention_long_ragged(dtype):
    """Ragged lengths up to 2049 (split-KV partials and their merge), Qwen2-7B head geometry."""
    nH, nG, span = 28, 4, 128
    lens = [2048, 2049, 777, 1]
    B = len(lens)
    rows = _rows(np.random.default_rng(5), max(lens), B, nH, nG, dtype)
    cache = _fill(FP8, rows, lens, nH, nG, span, 2176, dtype)
    kref, vref = _mirror_device(cache, lens, nG, span)
    q = np.stack([rows[lens[b] - 1, b, :nH * 128] for b in range(B)]).reshape(B, nH, 128)
    _check(_attend(cache, q, lens, 2176, dtype), KV.attention_ref(q, kref, vref, lens, nH, ALPHA), dtype)


def test_attention_ctx_32768():
    """One sequence of 32768 tokens: ~130 split-KV pieces per kv-head, merged in two levels."""
    from b200spark import ops
    nH, nG, span, L = 28, 4, 128, 32768
    rng = np.random.default_rng(77)
    cache = ops.SpanCache(1, L, nH, nG, span, FP8)
    rows = torch.from_numpy(rng.standard_normal((L, (nH + 2 * nG) * 128)).astype(np.float32)).to(torch.bfloat16)
    rows_d = rows.cuda()
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    for t in range(L):
        ops.cache_append(cache, rows_d[t:t + 1], pos)
        ops.lens_add(pos, 1)
    torch.cuda.synchronize()
    kref, vref = _mirror_device(cache, [L], nG, span)
    q = rows[L - 1, :nH * 128].float().numpy().reshape(1, nH, 128)
    _check(_attend(cache, q, [L], L, torch.bfloat16), KV.attention_ref(q, kref, vref, [L], nH, ALPHA), torch.bfloat16)


def test_attention_merge_paths(monkeypatch):
    """At 2048 tokens and batch 1 a (sequence, kv-head) is split into more than 16 pieces and merged in two levels;
    B2_ATTN_MAX_PIECES=4 forces the direct merge of 4 pieces.  Both agree with the oracle."""
    from b200spark import ops
    nH, nG, span, L = 28, 4, 128, 2048
    rows = _rows(np.random.default_rng(21), L, 1, nH, nG)
    cache = _fill(FP8, rows, [L], nH, nG, span, 2176)
    kref, vref = _mirror_device(cache, [L], nG, span)
    q = rows[L - 1, 0, :nH * 128].reshape(1, nH, 128)
    ref = KV.attention_ref(q, kref, vref, [L], nH, ALPHA)
    tree = _attend(cache, q, [L], 2176, torch.bfloat16)
    monkeypatch.setenv("B2_ATTN_MAX_PIECES", "4")
    capped = _attend(cache, q, [L], 2176, torch.bfloat16)
    for got in (tree, capped):
        _check(got, ref, torch.bfloat16)


@pytest.mark.parametrize("L", [1, 37, 129, 191])
def test_attention_ignores_unwritten_span_memory(L):
    """0xFF is an e4m3 NaN.  The pool is filled with it before appending; odd lengths leave unwritten rows inside the last
    64-token tile and the last 16-byte parameter chunk.  The tile loader zero-fills dead rows, so nothing reaches P V."""
    nH, nG, span = 28, 4, 32
    lens = [L, L, L]
    rows = _rows(np.random.default_rng(1000 + L), L, 3, nH, nG)
    cache = _fill(FP8, rows, lens, nH, nG, span, 256, fill=0xFF)
    kref, vref = _mirror_device(cache, lens, nG, span)
    q = np.stack([rows[L - 1, b, :nH * 128] for b in range(3)]).reshape(3, nH, 128)
    _check(_attend(cache, q, lens, 256, torch.bfloat16), KV.attention_ref(q, kref, vref, lens, nH, ALPHA), torch.bfloat16)


def _price(rows, lens, nH, nG, span, max_len):
    """Relative Frobenius error of the fp8 and the int8 cache's attention output against a bf16 cache of the same rows."""
    B = len(lens)
    q = np.stack([rows[lens[b] - 1, b, :nH * 128] for b in range(B)]).reshape(B, nH, 128)
    out = {m: _attend(_fill(m, rows, lens, nH, nG, span, max_len), q, lens, max_len, torch.bfloat16)
           for m in (KV.QUANT_NONE, KV.QUANT_I8, FP8)}
    base = out[KV.QUANT_NONE].astype(np.float64)
    return {m: float(np.linalg.norm(out[m] - base) / np.linalg.norm(base)) for m in (KV.QUANT_I8, FP8)}


def test_accuracy_price_against_bf16_cache():
    """N(0,1) rows: int8's per-row step (range / 255) beats e4m3's 2^-4 relative precision.  Rows with one key channel at
    64 sigma (a common key outlier): int8's step grows with the outlier and the small channels are lost, fp8 keeps them."""
    nH, nG, span = 28, 4, 64
    lens = [1024, 517, 64]
    rows = _rows(np.random.default_rng(3), max(lens), len(lens), nH, nG)
    plain = _price(rows, lens, nH, nG, span, 1088)
    out = rows.reshape(rows.shape[0], rows.shape[1], nH + 2 * nG, 128).copy()
    out[:, :, nH:nH + nG, 5] = 64.0  # channel 5 of every key row (bf16-exact)
    outl = _price(out.reshape(rows.shape), lens, nH, nG, span, 1088)
    print("relative Frobenius error vs a bf16 cache: N(0,1) rows fp8 %.3e i8 %.3e; 64-sigma key channel fp8 %.3e i8 %.3e"
          % (plain[FP8], plain[KV.QUANT_I8], outl[FP8], outl[KV.QUANT_I8]))
    # measured on an H100 (seeded rows): N(0,1) fp8 3.59e-2, i8 8.65e-3; 64-sigma key channel fp8 3.67e-2, i8 7.69e-2
    assert plain[FP8] <= 4e-2
    assert outl[FP8] <= 4e-2
    assert outl[FP8] < outl[KV.QUANT_I8]


# ---------------------------------------------------------------------------------------------------------- decode stack
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_decode_stack_fp8_kv(dtype):
    """Tiny 2-layer DecodeStack(kv="fp8") against the decoder oracle reading fp8-dequantized rows: the u4 logit tolerance
    (4e-2 of the logit range: a 1-ulp difference upstream can move a code by one e4m3 step), the greedy token whenever the
    oracle's top-2 margin exceeds twice the bound; a captured graph replays exactly what eager steps compute."""
    from b200spark import model
    B, steps = 2, 6
    st = model.DecodeStack(model.TINY, B, 64, wbits=4, group=-1, kv="fp8", span=16, keep_ref=True, dtype=dtype)
    ref = F8.decoder_ref(st)
    ref.reset(B)
    ids = torch.tensor([3, 777], dtype=torch.int64)
    for t in range(steps):
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        torch.cuda.synchronize()
        glog = st.logits.float().cpu()
        rlog, rnext = ref.step(ids, [t] * B)
        tol = 4e-2 * rlog.abs().max().item()
        err = (glog - rlog).abs().max().item()
        assert err <= tol, (t, err, tol)
        assert torch.equal(nxt, torch.argmax(glog, dim=-1))
        top2 = torch.topk(rlog, 2, dim=-1).values
        for b in range(B):
            if (top2[b, 0] - top2[b, 1]).item() > 2 * tol:
                assert nxt[b].item() == rnext[b].item(), (t, b)
        ids = nxt
    # graph replay == eager
    a = model.DecodeStack(model.TINY, 3, 64, wbits=4, kv="fp8", span=16, seed=7, dtype=dtype)
    g = model.DecodeStack(model.TINY, 3, 64, wbits=4, kv="fp8", span=16, seed=7, dtype=dtype)
    g.capture()
    ids = torch.tensor([1, 2, 3], dtype=torch.int64, device="cuda")
    for t in range(5):
        a.ids.copy_(ids); g.ids.copy_(ids)
        na = a.step().clone()
        ng = g.step().clone()
        torch.cuda.synchronize()
        assert torch.equal(a.logits, g.logits), t
        assert torch.equal(na, ng)
        ids = na


# ------------------------------------------------------------------------------------------------------ C++ operator
def test_span_attention_operator_fp8_cache():
    """DecOptMQA with AsCacheQuantFP8 spans on layer 2 of a 3-layer cache, 40 decode steps with span 16.  The op's spans are
    not reachable from here, so the oracle attends over its own quantization of the same rows — bit-identical to the
    device's (test_append_bit_exact), hence the plain attention tolerance."""
    import b200spark  # noqa: F401  (loads libb200spark.so with RTLD_GLOBAL first)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = C.CDLL(os.path.join(root, "dash-infer_b200", "lib", "liballspark_b200.so"))
    lib.as_test_span_attn.restype = C.c_int
    lib.as_test_span_attn.argtypes = [C.c_int] * 9 + [C.c_void_p, C.c_void_p]
    B, nH, nG, span, steps = 3, 8, 2, 16, 40
    W, OW = (nH + 2 * nG) * 128, nH * 128
    rng = np.random.default_rng(8)
    qkv = torch.from_numpy(rng.standard_normal((steps, B, W)).astype(np.float32)).to(torch.bfloat16)
    qn = qkv.contiguous().view(torch.int16).numpy()
    out = np.zeros((steps, B, OW), np.int16)
    rc = lib.as_test_span_attn(B, steps, nH, nG, span, FP8, 256, 3, 2, qn.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    got = torch.from_numpy(out).view(torch.bfloat16).float().numpy().reshape(steps, B, nH, 128)
    kref, vref = F8.SpanCacheFp8Ref(span, nG), F8.SpanCacheFp8Ref(span, nG)
    for _ in range(B):
        kref.add_sequence(); vref.add_sequence()
    x = qkv.float().numpy().reshape(steps, B, nH + 2 * nG, 128)
    for t in range(steps):
        for b in range(B):
            kref.append(b, t, x[t, b, nH:nH + nG]); vref.append(b, t, x[t, b, nH + nG:])
        if t in (0, 1, span - 1, span, steps - 1):
            _check(got[t], KV.attention_ref(x[t, :, :nH], kref, vref, [t + 1] * B, nH, ALPHA), torch.bfloat16)
