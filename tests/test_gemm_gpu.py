"""GPU parity: weight-only GEMV/GEMM through the C ABI vs the fp32 math oracle.

Tolerance: max_i min(abs, rel) <= 2e-2 (bf16) — the reference's own metric (tests/cpp/test_common.h.in:82-110) at a
tighter bound than its 5e-1 (operator_gemm_lowp_test.cpp:650-651).  Shapes follow the reference sweep
(M in {1,3,17,31,...}, odd N) plus the Qwen2-7B projections."""
import numpy as np
import pytest
import torch

from oracle import quant_ref as Q

pytestmark = pytest.mark.gpu
TOL = 2e-2


def _mk(K, N, M, seed, ft=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(K, N, generator=g) * 0.02).to(ft)
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(ft)
    return w, a


def _run(wbits, K, N, M, group, act=0, use_bias=False, use_res=False, alpha=1.0, seed=0, signed=True, ft=torch.bfloat16):
    from b200spark import ops, quantize as PQ
    w, a = _mk(K, N, M, seed, ft)
    g = torch.Generator().manual_seed(seed + 1)
    bias = (torch.randn(N, generator=g) * 0.02).to(ft) if use_bias else None
    res = (torch.randn(M, N, generator=g) * 0.1).to(ft) if use_res else None
    dev = "cuda"
    if wbits == 4:
        qd, s, z = PQ.quantize_a16w4(w, group)
        qu = Q.unpack_u4x2(qd.numpy(), N)
    elif wbits == 8:
        qd, s, z = PQ.quantize_a16w8(w, group, signed=signed)
        qu = qd.numpy()
    else:
        qd, s, z = w, None, None
    op = ops.GemmWQ(K, N, wbits, group, max_m=max(M, 1), signed=signed, dtype=ft)
    op.prepare(qd.to(dev), s.to(dev) if s is not None else None, z.to(dev) if z is not None else None,
               bias.to(dev) if bias is not None else None)
    ws = ops.Workspace()
    out = op(a.to(dev), ws, act=act, alpha=alpha, residual=res.to(dev) if res is not None else None)
    torch.cuda.synchronize()
    out2 = op(a.to(dev), ws, act=act, alpha=alpha, residual=res.to(dev) if res is not None else None)  # re-armed counters
    torch.cuda.synchronize()
    assert torch.equal(out, out2), "not deterministic / split-K counters not re-armed"
    a32 = a.float().numpy()
    if wbits == 16:
        ref = alpha * (a32.astype(np.float64) @ w.float().numpy().astype(np.float64))
        if bias is not None:
            ref = ref + bias.float().numpy()[None, :]
        ref = Q.activation(ref.astype(np.float32), act)
    else:
        ref = Q.gemm_wq_math(a32, qu, s.float().numpy(), z.float().numpy(), group,
                             bias.float().numpy() if bias is not None else None, act, alpha)
    if res is not None:
        ref = ref + res.float().numpy()
    got = out.float().cpu().numpy()
    err = Q.err_min_abs_rel(ref, got)
    assert err <= TOL, f"err {err}"
    return err


@pytest.mark.parametrize("M", [1, 2, 3, 8, 9, 16, 17, 31, 32, 33, 64])
@pytest.mark.parametrize("wbits", [4, 8, 16])
def test_small_shapes_all_m(wbits, M):
    _run(wbits, 512, 256, M, -1, seed=M)


@pytest.mark.parametrize("wbits,group", [(4, 128), (4, 64), (8, 128), (8, 256)])
@pytest.mark.parametrize("M", [1, 5, 16, 32])
def test_subchannel(wbits, group, M):
    _run(wbits, 1024, 384, M, group, seed=7)


@pytest.mark.parametrize("wbits", [4, 8])
def test_odd_shapes(wbits):
    # N not a multiple of 128 / odd N (packed nibble tail), K not a multiple of 64 (K % 8 == 0 required)
    _run(wbits, 520, 130, 3, -1, seed=3)
    _run(wbits, 328, 77, 1, -1, seed=4)
    _run(wbits, 200, 48, 4, 64, seed=5)  # K padded to the group: tail group sees zero activations


def test_uint8_weights():
    _run(8, 512, 256, 4, -1, signed=False, seed=11)


@pytest.mark.parametrize("act", [0, 2, 3, 4, 5])  # the lowp launchers implement none/gelu_erf/gelu_tanh/relu/silu
def test_bias_activation(act):
    _run(4, 512, 256, 3, -1, act=act, use_bias=True, seed=20 + act)


def test_alpha_residual():
    _run(4, 512, 256, 5, -1, act=5, use_bias=True, use_res=True, alpha=0.5, seed=31)
    _run(8, 512, 256, 1, 128, use_res=True, seed=32)


@pytest.mark.parametrize("K,N", [(3584, 4608), (3584, 3584), (3584, 18944), (18944, 3584)])
@pytest.mark.parametrize("M", [1, 8])
def test_qwen2_7b_projections_w4(K, N, M):
    _run(4, K, N, M, -1, use_bias=(N == 4608), seed=K % 97 + M)


def test_qwen2_7b_w8_and_g128():
    _run(8, 3584, 3584, 1, -1, seed=41)
    _run(4, 4096, 6144, 32, 128, seed=42)  # Llama-3-8B QKV, GPTQ g128, batch 32


def test_dense_bf16_tcgen05_multiwave():
    """bf16 weights on the wgmma path (lm_head shape class): more n-groups than SMs, ragged N tail, M 17..64."""
    _run(16, 3584, 19000, 64, -1, seed=71)
    _run(16, 1024, 4100, 23, -1, seed=72, use_bias=True, act=5)


def test_tcgen05_persistent_units():
    """More (n-group, k-split) units than SMs: every CTA walks several units (ring phases, accumulator and the parked tile
    carry over; the next unit's weights are prefetched during the epilogue)."""
    _run(4, 1024, 128 * 300 + 50, 33, -1, seed=73, use_res=True)
    _run(8, 512, 128 * 450, 64, -1, seed=74, use_bias=True)
    _run(16, 1024, 128 * 400 + 8, 64, -1, seed=75)


def test_forced_split_paths(monkeypatch):
    monkeypatch.setenv("B2_GEMV2", "0")  # the split-K kernel (still used for fused norm / all-reduce epilogues and tiny N)
    monkeypatch.setenv("B2_GEMM_FORCE_SPLIT", "1")
    _run(4, 1024, 256, 2, -1, seed=51)
    monkeypatch.setenv("B2_GEMM_FORCE_SPLIT", "7")
    _run(4, 1024, 256, 2, -1, seed=52)
    _run(8, 1024, 256, 9, 128, seed=53)


def test_linearity_full_size():
    """Size-independent property at a full-size projection: f(a1 + a2) == f(a1) + f(a2) within bf16 rounding,
    and f(0) == bias exactly."""
    from b200spark import ops, quantize as PQ
    K, N = 3584, 18944
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
    qd, s, z = PQ.quantize_a16w4(w.cuda(), -1)
    op = ops.GemmWQ(K, N, 4, -1, max_m=8).prepare(qd, s, z)
    ws = ops.Workspace()
    a1 = (torch.rand(4, K, generator=g) - 0.5).to(torch.bfloat16).cuda()
    a2 = torch.zeros_like(a1)
    a2[:, ::2] = 0.25
    s12 = (a1.float() + a2.float()).to(torch.bfloat16)
    exact = (s12.float() == a1.float() + a2.float()).all().item()
    y1, y2, y12 = op(a1, ws).float(), op(a2, ws).float(), op(s12, ws).float()
    y0 = op(torch.zeros_like(a1), ws).float()
    assert torch.count_nonzero(y0) == 0
    if exact:
        assert (y12 - (y1 + y2)).abs().max().item() <= 2e-2 * max(1.0, y12.abs().max().item())


@pytest.mark.parametrize("wbits,group,M", [(4, -1, 1), (4, -1, 8), (4, -1, 64), (8, -1, 3), (4, 128, 5), (8, -1, 33), (16, -1, 2), (16, -1, 40)])
def test_fused_swiglu_pair(wbits, group, M):
    """gate/up pair image + SwiGLU epilogue == silu(A.Wg) * (A.Wu) of the fp32 oracle (one rounding instead of three)."""
    from b200spark import ops, quantize as PQ
    K, N = 1024, 704  # N not a multiple of 64: exercises the padded tail tile
    g = torch.Generator().manual_seed(M * 7 + wbits)
    wg = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
    wu = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(torch.bfloat16)
    outs, refs = [], []
    sets = []
    for w in (wg, wu):
        if wbits == 4:
            q, s, z = PQ.quantize_a16w4(w, group); qu = Q.unpack_u4x2(q.numpy(), N)
        elif wbits == 8:
            q, s, z = PQ.quantize_a16w8(w, group); qu = q.numpy()
        else:
            q, s, z, qu = w, None, None, None
        sets.append((q, s, z))
        if wbits == 16:
            refs.append(a.float().numpy().astype(np.float64) @ w.float().numpy().astype(np.float64))
        else:
            refs.append(Q.gemm_wq_math(a.float().numpy(), qu, s.float().numpy(), z.float().numpy(), group).astype(np.float64))
    dev = lambda t: t.cuda() if t is not None else None
    op = ops.GemmWQ(K, N, wbits, group, max_m=M, pair=True)
    op.prepare_swiglu(*[dev(t) for t in sets[0]], *[dev(t) for t in sets[1]])
    ws = ops.Workspace()
    out = op(a.cuda(), ws)
    out2 = op(a.cuda(), ws)
    torch.cuda.synchronize()
    assert out.shape == (M, N) and torch.equal(out, out2)
    ref = (refs[0] / (1.0 + np.exp(-refs[0]))) * refs[1]
    assert Q.err_min_abs_rel(ref.astype(np.float32), out.float().cpu().numpy()) <= TOL


@pytest.mark.parametrize("M", [1, 16])
def test_fuse_fields_outside_both_norm_forms_are_unsupported(M):
    """On the split-K GEMV's batches a b2_gemm_fuse is the self-contained form (norm_gamma alone) or nothing: norm_sumsq
    with norm_gamma, and sumsq_out alone, return B2_ERR_UNSUPPORTED before any launch and leave the output untouched."""
    from b200spark import ops, quantize as PQ
    from b200spark._lib import B2Error
    K, N = 1024, 640
    g = torch.Generator().manual_seed(M)
    q, s, z = PQ.quantize_a16w4((torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16), -1)
    op = ops.GemmWQ(K, N, 4, -1, max_m=M).prepare(q.cuda(), s.cuda(), z.cuda())
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    gamma = torch.ones(K, dtype=torch.bfloat16, device="cuda")
    ssq = torch.ones(op.sumsq_parts(), M, dtype=torch.float32, device="cuda")
    ws = ops.Workspace()
    out = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(B2Error, match="B2_ERR_UNSUPPORTED"):
        op(a, ws, out=out, norm_in=(ssq, gamma, K, 1e-6))
    with pytest.raises(B2Error, match="B2_ERR_UNSUPPORTED"):
        op(a, ws, out=out, sumsq_out=ssq)
    torch.cuda.synchronize()
    assert torch.count_nonzero(out) == 0 and torch.equal(ssq, torch.ones_like(ssq))


@pytest.mark.parametrize("wbits,group,M", [(4, -1, 17), (4, -1, 64), (8, -1, 33), (4, 128, 40), (16, -1, 64), (4, -1, 100)])
def test_tcgen05_rmsnorm_handoff(wbits, group, M):
    """Batches >= 17: the producer GEMM (+residual) also writes xg = bf16(C * gamma) and per-tile row statistics; the consumer
    takes A = xg and scales its result rows by 1/rms.  Producer: C bit-identical to the plain call, xg and the statistics
    follow the stored bf16 values.  Consumer (plain and gate/up SwiGLU pair): against fp64 RMSNorm -> GEMM math and against
    the two-kernel path (b2_rmsnorm, then the plain GEMM)."""
    from b200spark import ops, quantize as PQ
    H, N2 = 3584, 1280
    g = torch.Generator().manual_seed(wbits * 10 + M)
    d = lambda t: t.cuda() if t is not None else None

    def quant(w, K, N):
        if wbits == 4:
            q, s, z = PQ.quantize_a16w4(w, group); qu = Q.unpack_u4x2(q.numpy(), N)
        elif wbits == 8:
            q, s, z = PQ.quantize_a16w8(w, group); qu = q.numpy()
        else:
            return (w, None, None), w.float().numpy().astype(np.float64)
        gs = K if group == -1 else group
        sc = np.repeat(s.float().numpy().astype(np.float64), gs, axis=0)[:K]
        zz = np.repeat(z.float().numpy().astype(np.float64), gs, axis=0)[:K]
        return (q, s, z), (qu.astype(np.float64) - zz) * sc

    mk = lambda k, n: (torch.randn(k, n, generator=g) * 0.02).to(torch.bfloat16)
    (qp, sp, zp), _ = quant(mk(H, H), H, H)
    prod = ops.GemmWQ(H, H, wbits, group, max_m=M).prepare(d(qp), d(sp), d(zp))
    a = (torch.rand(M, H, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    res = (torch.randn(M, H, generator=g) * 2.0).to(torch.bfloat16).cuda()
    gamma = (1 + 0.2 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
    eps = 1e-6
    ws = ops.Workspace()
    ssq = torch.zeros(prod.sumsq_parts(), M, dtype=torch.float32, device="cuda")
    xg = torch.empty(M, H, dtype=torch.bfloat16, device="cuda")
    x = prod(a, ws, residual=res, sumsq_out=ssq, xg_out=(xg, gamma))
    x_plain = prod(a, ws, residual=res)
    torch.cuda.synchronize()
    assert torch.equal(x, x_plain)
    assert torch.equal(xg, (x.float() * gamma.float()).to(torch.bfloat16))
    assert torch.allclose(ssq.sum(0), x.float().pow(2).sum(-1), rtol=1e-5)

    x64 = x.float().cpu().numpy().astype(np.float64)
    xn = x64 / np.sqrt((x64 ** 2).mean(-1, keepdims=True) + eps) * gamma.float().cpu().numpy().astype(np.float64)
    for pair in (False, True):
        sets, deq = [], []
        for _ in range(2 if pair else 1):
            t, wd = quant(mk(H, N2), H, N2)
            sets.append(t); deq.append(wd)
        cons = ops.GemmWQ(H, N2, wbits, group, max_m=M, pair=pair)
        if pair:
            cons.prepare_swiglu(*[d(t) for t in sets[0]], *[d(t) for t in sets[1]])
        else:
            cons.prepare(*[d(t) for t in sets[0]])
        y = cons(xg, ws, norm_in=(ssq, None, H, eps))
        y2 = cons(xg, ws, norm_in=(ssq, None, H, eps))
        y_two = cons(ops.rmsnorm(x, gamma, eps), ws)
        torch.cuda.synchronize()
        assert torch.equal(y, y2)
        outs = [xn @ w for w in deq]
        ref = ((outs[0] / (1.0 + np.exp(-outs[0]))) * outs[1] if pair else outs[0]).astype(np.float32)
        e_h = Q.err_min_abs_rel(ref, y.float().cpu().numpy())
        e_two = Q.err_min_abs_rel(ref, y_two.float().cpu().numpy())
        assert e_h <= (2 * TOL if pair else TOL), (e_h, e_two)
        assert e_h <= 2.0 * e_two + 2e-3, (e_h, e_two)


# ---------------------------------------------------------------------------------------------------------------------
# fp16 activations (the reference dispatches FLOAT16 first: gemm_a16w4_gpu.cpp:31-38, and most of its lowp tests are fp16:
# tests/cpp/operator/cuda/operator_gemm_lowp_test.cpp:469-471).  Same kernels, the 16-bit type is a template parameter;
# the exact-integer dequantisation uses 128 + q (fp16 has three more mantissa bits than bf16's 16 + q).
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 3, 8, 16, 17, 31, 33, 64])
@pytest.mark.parametrize("wbits,group", [(4, -1), (8, -1), (16, -1), (4, 128), (8, 64)])
def test_fp16_all_paths(wbits, group, M):
    """split-K GEMV (M <= 16), wgmma (M >= 17; sub-channel int8 stays on the mma.sync kernel), odd N, bias + residual"""
    _run(wbits, 1024, 1023, M, group, use_bias=True, use_res=True, seed=wbits + M, ft=torch.float16)


@pytest.mark.parametrize("K,N,M", [(3584, 4608, 1), (3584, 3584, 8), (18944, 3584, 16), (3584, 18944, 64), (18944, 3584, 64), (3584, 4608, 32)])
def test_fp16_qwen2_7b_projections(K, N, M):
    _run(4, K, N, M, -1, use_bias=(N == 4608), use_res=(N == 3584), seed=K % 89 + M, ft=torch.float16)
    if M in (8, 64):
        _run(8, K, N, M, -1, seed=K % 83 + M, signed=(M == 8), ft=torch.float16)


@pytest.mark.parametrize("wbits,group,M", [(4, -1, 4), (4, -1, 64), (4, 128, 40), (8, -1, 20)])
def test_fp16_swiglu_pair(wbits, group, M):
    from b200spark import ops, quantize as PQ
    K, N = 2048, 2944
    g = torch.Generator().manual_seed(M * 3 + wbits)
    ws_, refs = [], []
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(torch.float16)
    for _ in range(2):
        w = (torch.randn(K, N, generator=g) * 0.02).to(torch.float16)
        if wbits == 4:
            q, s, z = PQ.quantize_a16w4(w, group); qu = Q.unpack_u4x2(q.numpy(), N)
        else:
            q, s, z = PQ.quantize_a16w8(w, group); qu = q.numpy()
        ws_.append((q, s, z))
        refs.append(Q.gemm_wq_math(a.float().numpy(), qu, s.float().numpy(), z.float().numpy(), group).astype(np.float64))
    op = ops.GemmWQ(K, N, wbits, group, max_m=M, pair=True, dtype=torch.float16)
    op.prepare_swiglu(*[t.cuda() for t in ws_[0]], *[t.cuda() for t in ws_[1]])
    out = op(a.cuda(), ops.Workspace())
    torch.cuda.synchronize()
    assert out.dtype == torch.float16
    ref = (refs[0] / (1.0 + np.exp(-refs[0]))) * refs[1]
    assert Q.err_min_abs_rel(ref.astype(np.float32), out.float().cpu().numpy()) <= TOL


@pytest.mark.parametrize("ft", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("group,K,M", [(32, 1024, 1), (40, 1000, 5), (72, 2048, 16), (200, 1000, 33), (136, 4096, 100), (96, 3584, 64)])
def test_general_group_sizes_w4(group, K, M, ft):
    """Group sizes that do not divide the 64-k tile (the reference's dequantize + cuBLAS test draws any multiple of 8 in
    [64, 512]: operator_gemm_lowp_test.cpp:893-903; gemm_a16w4.cpp:57-63 accepts >= 32): int4, on the wgmma kernel at
    every batch, the (scale, zero) looked up per 8-k word of the weight image."""
    _run(4, K, 1023, M, group, use_bias=True, use_res=(M > 16), seed=group + M, ft=ft)


@pytest.mark.parametrize("group,ft", [(-1, torch.bfloat16), (128, torch.bfloat16), (96, torch.bfloat16), (128, torch.float16)])
def test_wgmma_two_ctas_per_sm_persistent(group, ft):
    """More than 2 x (SM count) n-groups: the int4 GEMM of batches >= 17 runs two CTAs per SM, each walking several
    (n-group, k-split) units — per-channel, sub-channel, a group size that does not divide the 64-k tile, bf16 and fp16."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    _run(4, 512, (2 * sms + 6) * 128, 40, group, use_res=True, seed=17, ft=ft)


@pytest.mark.parametrize("wbits,group,M,N", [(4, -1, 1, 5117), (4, -1, 7, 5120), (8, -1, 16, 5117), (4, 128, 9, 5118), (16, -1, 3, 5117)])
def test_cluster_split_k_epilogue(monkeypatch, wbits, group, M, N):
    """Shapes wide enough for the thread-block-cluster split-K (the k-slices of a tile meet in distributed shared memory and
    every CTA finishes its share of the tile): bias + activation + residual + alpha, odd N (scalar tail, unaligned rows), and
    the same call with clusters disabled (workspace + ticket split-K) as a second opinion."""
    monkeypatch.setenv("B2_GEMV2", "0")  # bf16 weights: stay on the split-K kernel
    e1 = _run(wbits, 2048, N, M, group, act=1, use_bias=True, use_res=True, alpha=0.5, seed=N + M)
    monkeypatch.setenv("B2_GEMM_CLUSTER", "0")
    e0 = _run(wbits, 2048, N, M, group, act=1, use_bias=True, use_res=True, alpha=0.5, seed=N + M)
    assert abs(e1 - e0) <= 1e-2


@pytest.mark.parametrize("wbits,group,M,K,N,pair", [(4, -1, 1, 3584, 4608, False), (4, -1, 8, 3584, 4608, False),
                                                   (4, -1, 16, 3584, 18944, True), (4, 128, 5, 1024, 704, False),
                                                   (8, -1, 3, 1024, 640, False), (16, -1, 2, 1024, 640, False),
                                                   (4, 128, 16, 4096, 1024, True), (4, -1, 1, 3584, 18944, True)])
def test_self_contained_rmsnorm(wbits, group, M, K, N, pair):
    """norm_in=(None, gamma, K, eps): the GEMV normalises its own activations — bf16(x*gamma) staged, sum x^2 collected in
    the same pass (per split-K slice, summed by the reducer), 1/rms applied to the fp32 tile.  Checked against the fp64
    RMSNorm -> GEMM math and against the two-kernel path (b2_rmsnorm, then the plain GEMV)."""
    from b200spark import ops, quantize as PQ
    g = torch.Generator().manual_seed(wbits * 100 + M + K)
    x = (torch.randn(M, K, generator=g) * 3.0).to(torch.bfloat16)       # residual-stream scale, not unit rows
    gamma = (1 + 0.2 * torch.randn(K, generator=g)).to(torch.bfloat16)
    eps = 1e-6
    ws_list, deq = [], []
    for _ in range(2 if pair else 1):
        w = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
        if wbits == 4:
            q, s, z = PQ.quantize_a16w4(w, group); qu = Q.unpack_u4x2(q.numpy(), N)
        elif wbits == 8:
            q, s, z = PQ.quantize_a16w8(w, group); qu = q.numpy()
        else:
            q, s, z, qu = w, None, None, None
        ws_list.append((q, s, z))
        if wbits == 16:
            deq.append(w.float().numpy().astype(np.float64))
        else:
            gs = K if group == -1 else group
            sc = np.repeat(s.float().numpy().astype(np.float64), gs, axis=0)[:K]
            zz = np.repeat(z.float().numpy().astype(np.float64), gs, axis=0)[:K]
            deq.append((qu.astype(np.float64) - zz) * sc)
    d = lambda t: t.cuda() if t is not None else None
    op = ops.GemmWQ(K, N, wbits, group, max_m=M, pair=pair)
    if pair:
        op.prepare_swiglu(*[d(t) for t in ws_list[0]], *[d(t) for t in ws_list[1]])
    else:
        op.prepare(*[d(t) for t in ws_list[0]])
    ws = ops.Workspace()
    xd, gd = x.cuda(), gamma.cuda()
    y = op(xd, ws, norm_in=(None, gd, K, eps))
    y2 = op(xd, ws, norm_in=(None, gd, K, eps))
    y_two = op(ops.rmsnorm(xd, gd, eps), ws)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
    x64 = x.float().numpy().astype(np.float64)
    xn = x64 / np.sqrt((x64 ** 2).mean(-1, keepdims=True) + eps) * gamma.float().numpy().astype(np.float64)
    outs = [xn @ w for w in deq]
    ref = (outs[0] / (1.0 + np.exp(-outs[0]))) * outs[1] if pair else outs[0]
    e_self = Q.err_min_abs_rel(ref.astype(np.float32), y.float().cpu().numpy())
    e_two = Q.err_min_abs_rel(ref.astype(np.float32), y_two.float().cpu().numpy())
    # the SwiGLU product carries the rounding of both of its factors: twice the single-GEMM bound
    assert e_self <= (2 * TOL if pair else TOL), (e_self, e_two)
    assert e_self <= 2.0 * e_two + 2e-3, (e_self, e_two)   # no worse than the two-kernel path beyond rounding noise


# ---------------------------------------------------------------------------------------------------------------------
# The launches bench.py actually times (VERDICT r1: "the bench runs it unchecked"): wgmma path at M in {17, 32, 64}
# on every Qwen2-7B projection shape, int4 and int8, plus the fused gate/up pair and the Qwen2-72B TP=8 shard shapes.
# ---------------------------------------------------------------------------------------------------------------------
QWEN7B = [(3584, 4608), (3584, 3584), (3584, 18944), (18944, 3584)]


@pytest.mark.parametrize("K,N", QWEN7B)
@pytest.mark.parametrize("M", [17, 32, 64])
def test_qwen2_7b_projections_w4_tcgen05(K, N, M):
    _run(4, K, N, M, -1, use_bias=(N == 4608), use_res=(N == 3584), seed=K % 89 + M)


@pytest.mark.parametrize("K,N", QWEN7B)
@pytest.mark.parametrize("M", [17, 64])
def test_qwen2_7b_projections_w8_tcgen05(K, N, M):
    _run(8, K, N, M, -1, use_bias=(N == 4608), use_res=(N == 3584), seed=K % 83 + M)


def _pair_case(wbits, K, N, M, group, seed):
    from b200spark import ops, quantize as PQ
    g = torch.Generator().manual_seed(seed)
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(torch.bfloat16)
    sets, refs = [], []
    for _ in range(2):
        w = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
        if wbits == 16:
            sets.append((w.cuda(), None, None))
            refs.append(a.float().numpy().astype(np.float64) @ w.float().numpy().astype(np.float64))
            continue
        if wbits == 4:
            q, s, z = PQ.quantize_a16w4(w, group); qu = Q.unpack_u4x2(q.numpy(), N)
        else:
            q, s, z = PQ.quantize_a16w8(w, group); qu = q.numpy()
        sets.append((q.cuda(), s.cuda(), z.cuda()))
        refs.append(Q.gemm_wq_math(a.float().numpy(), qu, s.float().numpy(), z.float().numpy(), group).astype(np.float64))
    op = ops.GemmWQ(K, N, wbits, group, max_m=M, pair=True)
    op.prepare_swiglu(*sets[0], *sets[1])
    ws = ops.Workspace()
    out = op(a.cuda(), ws)
    out2 = op(a.cuda(), ws)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    ref = (refs[0] / (1.0 + np.exp(-refs[0]))) * refs[1]
    err = Q.err_min_abs_rel(ref.astype(np.float32), out.float().cpu().numpy())
    assert err <= TOL, err


@pytest.mark.parametrize("wbits", [4, 8])
@pytest.mark.parametrize("M", [1, 8, 64])
def test_qwen2_7b_gate_up_swiglu_pair_full_size(wbits, M):
    """The single largest launch of the decode step: gate+up 3584 x (2 x 18944) with the SwiGLU epilogue (persistent units)."""
    _pair_case(wbits, 3584, 18944, M, -1, seed=100 + M + wbits)


@pytest.mark.parametrize("M", [16, 64])
def test_qwen2_72b_tp8_shard_shapes(M):
    """Per-rank shapes of config C4 at TP=8 (Qwen2-72B: hidden 8192, 64/8 heads, inter 29568): column-split QKV and gate/up,
    row-split o_proj / down_proj (K = 1024 / 3696: neither is a multiple of 256, the k-tiles-per-stage of the int4 path)."""
    _run(4, 8192, (64 + 16) // 8 * 128, M, -1, use_bias=True, seed=200 + M)      # qkv shard   [8192, 1280]
    _run(4, 64 // 8 * 128, 8192, M, -1, use_res=True, seed=201 + M)              # o shard     [1024, 8192]
    _run(4, 29568 // 8, 8192, M, -1, use_res=True, seed=202 + M)                 # down shard  [3696, 8192]
    _pair_case(4, 8192, 29568 // 8, M, -1, seed=203 + M)                         # gate/up shard pair


def test_llama3_8b_g128_full_size_m32():
    """Config C3 shapes (Llama-3-8B GPTQ-style g128, batch 32): QKV / o / down, sub-channel weights at M > 16, and the
    verdict's pair case (4, 4096, 14336 x 2, 32, 128)."""
    _run(4, 4096, 4096, 32, 128, use_res=True, seed=301)
    _run(4, 14336, 4096, 32, 128, use_res=True, seed=302)
    _pair_case(4, 4096, 14336, 32, 128, seed=303)


def test_mixed_group_sizes_share_a_kernel():
    """ADVICE r1: two handles of the same kernel instantiation with different group sizes (g128 needs more shared memory
    per activation chunk than g256): planning the second must not lower the first one's shared-memory opt-in."""
    from b200spark import ops, quantize as PQ
    g = torch.Generator().manual_seed(9)
    K, N, M = 2048, 256, 4
    hs = []
    for group in (512, 64):  # large-smem plan first, then a smaller one
        w = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
        q, s, z = PQ.quantize_a16w4(w, group)
        op = ops.GemmWQ(K, N, 4, group, max_m=M).prepare(q.cuda(), s.cuda(), z.cuda())
        hs.append((op, Q.unpack_u4x2(q.numpy(), N), s, z, group))
    ws = ops.Workspace()
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(torch.bfloat16)
    for _ in range(2):      # plan A, plan B, then launch A again
        for op, qu, s, z, group in hs:
            out = op(a.cuda(), ws)
            torch.cuda.synchronize()
            ref = Q.gemm_wq_math(a.float().numpy(), qu, s.float().numpy(), z.float().numpy(), group)
            assert Q.err_min_abs_rel(ref, out.float().cpu().numpy()) <= TOL


@pytest.mark.parametrize("cb", [16, 32, 64, 128])
def test_gemv2_every_channel_block(monkeypatch, cb):
    """The no-split-K GEMV of dense bf16 weights with its channel block forced to 16 / 32 / 64 / 128 (8 / 4 / 2 / 1 k-slices
    per CTA): M 1 / 3 / 8 / 11 / 16 (MT 1 and 2), ragged N and K, bias / activation / residual, and the gate/up pair image
    (needs >= 32: 16 gate + 16 up rows per CTA)."""
    monkeypatch.setenv("B2_GEMV2_CB", str(cb))
    _run(16, 1024, 640, 1, -1, seed=1, use_bias=True, use_res=True)
    _run(16, 520, 130, 3, -1, seed=2)                      # K % 64 != 0, ragged N
    _run(16, 1024, 384, 8, -1, seed=3, act=5)
    _run(16, 512, 256, 16, -1, seed=4, use_bias=True)
    _run(16, 520, 130, 11, -1, seed=5, act=5, use_bias=True, use_res=True, alpha=0.5)  # MT = 2 with 5 dead rows
    if cb >= 32:
        _pair_case(16, 1024, 704, 1, -1, seed=8)
        _pair_case(16, 1024, 704, 16, -1, seed=9)


def test_gemv2_matches_split_k_kernel(monkeypatch):
    """Both decompositions stream the same image: results agree to fp32 summation order (then one bf16 rounding).  Dense bf16
    weights at a shape the default policy sends to the no-split-K GEMV (296 n-groups: 128-channel blocks)."""
    from b200spark import ops
    K, N, M = 3584, 37888, 8
    g = torch.Generator().manual_seed(12)
    w = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    op = ops.GemmWQ(K, N, 16, -1, max_m=M).prepare(w.cuda())
    ws = ops.Workspace()
    monkeypatch.setenv("B2_GEMV2", "1")
    y2 = op(a, ws).float()
    monkeypatch.setenv("B2_GEMV2", "0")
    y1 = op(a, ws).float()
    torch.cuda.synchronize()
    assert (y1 - y2).abs().max().item() <= 2.0 ** -7 * y1.abs().max().item()
    assert (y1 != y2).float().mean().item() < 0.02
