"""GPU: fp8-e4m3 activations x int4 weights on the e4m3 wgmma kernel (SURVEY.md §8 f3; BASELINE config "GPTQ-int4, fp8
activations").  Beyond the reference (its FP8 op is per-tensor A8W8 via cuBLASLt, gemm_fp8_a8w8_gpu.cpp:325-395), so the
contract is stated here:
  * b2_quant_fp8 is checked bit for bit against a torch restatement (per-token scale = amax / 448, round-to-nearest-even e4m3);
  * b2_gemm_wq_run_fp8 is checked against fp64 arithmetic ON THE QUANTIZED ACTIVATIONS: products e4m3 x int4 are exact and the
    accumulation is fp32, so the tolerance is the GEMM tolerance (min(abs, rel) <= 2e-2, observed ~4e-3 = bf16 output rounding);
  * the accuracy price of fp8 activations vs bf16 activations is measured and bounded (relative Frobenius error <= 4 %)."""
import numpy as np
import pytest
import torch

from oracle import quant_ref as Q

pytestmark = pytest.mark.gpu
PERM = [0, 2, 4, 6, 1, 3, 5, 7]


def _decode(fp8act, cols):
    """b2 fp8 activation layout -> float32 [rows, cols] of the quantized values (natural k order)."""
    y = fp8act.y[:, :cols].contiguous().view(torch.float8_e4m3fn).float().cpu()
    rows = y.shape[0]
    g = y.reshape(rows, -1, 8)
    nat = torch.empty_like(g)
    for j, k in enumerate(PERM):
        nat[:, :, k] = g[:, :, j]
    return nat.reshape(rows, -1)


@pytest.mark.parametrize("rows,cols,norm", [(1, 3584, False), (64, 3584, False), (5, 1088, False), (33, 18944, False), (7, 4096, True)])
def test_quant_fp8_bit_exact(rows, cols, norm):
    from b200spark import ops
    g = torch.Generator().manual_seed(rows + cols)
    x = (torch.randn(rows, cols, generator=g) * 1.7).to(torch.bfloat16).cuda()
    gamma = (1 + 0.1 * torch.randn(cols, generator=g)).to(torch.bfloat16).cuda() if norm else None
    q8 = ops.quant_fp8(x, gamma, 1e-6)
    torch.cuda.synchronize()
    xn = ops.rmsnorm(x, gamma, 1e-6) if norm else x
    xf = xn.float().cpu().numpy()
    # IEEE fp32 like the kernel (torch's GPU division by a scalar multiplies by the reciprocal instead)
    sc = (np.maximum(np.abs(xf).max(axis=1), np.float32(1e-12)) / np.float32(448)).astype(np.float32)
    assert np.array_equal(q8.scale.cpu().numpy(), sc)
    rs = (np.float32(1) / sc).astype(np.float32)
    exp = torch.from_numpy((xf * rs[:, None]).astype(np.float32)).to(torch.float8_e4m3fn).float()
    got = _decode(q8, cols)
    assert torch.equal(got, exp)
    ts = got.reshape(rows, -1, 64).sum(-1) if cols % 64 == 0 else torch.stack([got[:, i:i + 64].sum(-1) for i in range(0, cols, 64)], 1)
    assert torch.equal(q8.tile_sums.cpu(), ts)


def _case(K, N, M, seed, use_bias=False, use_res=False, act=0, pair=False):
    from b200spark import ops, quantize as PQ
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g)).to(torch.bfloat16).cuda()
    bias = (torch.randn(N, generator=g) * 0.02).to(torch.bfloat16) if use_bias else None
    res = (torch.randn(M, N, generator=g) * 0.1).to(torch.bfloat16) if use_res else None
    sets, deq = [], []
    for _ in range(2 if pair else 1):
        w = (torch.randn(K, N, generator=g) * 0.02).to(torch.bfloat16)
        q, s, z = PQ.quantize_a16w4(w, -1)
        sets.append((q.cuda(), s.cuda(), z.cuda()))
        qu = Q.unpack_u4x2(q.numpy(), N).astype(np.float64)
        deq.append((qu - z.float().numpy().astype(np.float64)) * s.float().numpy().astype(np.float64))
    op = ops.GemmWQ(K, N, 4, -1, max_m=M, pair=pair)
    if pair:
        op.prepare_swiglu(*sets[0], *sets[1])
    else:
        op.prepare(*sets[0], bias.cuda() if bias is not None else None)
    ws = ops.Workspace()
    q8 = ops.quant_fp8(a)
    out = op.run_fp8(q8, ws, act=act, residual=res.cuda() if res is not None else None)
    out2 = op.run_fp8(q8, ws, act=act, residual=res.cuda() if res is not None else None)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    aq = _decode(q8, K).numpy().astype(np.float64) * q8.scale.cpu().numpy().astype(np.float64)[:, None]
    if pair:
        gte, up = aq @ deq[0], aq @ deq[1]
        ref = gte / (1.0 + np.exp(-gte)) * up
    else:
        ref = aq @ deq[0]
        if bias is not None:
            ref = ref + bias.float().numpy()[None]
        ref = Q.activation(ref.astype(np.float32), act).astype(np.float64)
        if res is not None:
            ref = ref + res.float().numpy()
    got = out.float().cpu().numpy()
    err = Q.err_min_abs_rel(ref.astype(np.float32), got)
    assert err <= 2e-2, err
    # what fp8 activations cost against bf16 activations (same weights)
    ref16 = a.float().cpu().numpy().astype(np.float64) @ deq[0]
    if not pair and act == 0 and not use_bias and not use_res:
        rel = np.linalg.norm(got - ref16) / np.linalg.norm(ref16)
        print("fp8 vs bf16 activations: relative Frobenius error %.4f (K=%d N=%d M=%d)" % (rel, K, N, M))
        assert rel <= 4e-2, rel
    return err


@pytest.mark.parametrize("M", [1, 5, 17, 32, 64])
def test_fp8_gemm_small(M):
    _case(1024, 384, M, seed=M)


def test_fp8_gemm_odd_k_tiles_and_ragged_n():
    _case(1088, 130, 9, seed=11)          # 17 k-tiles: the last fp8 activation tile is half empty; ragged N
    _case(3648, 640, 64, seed=12, use_bias=True, act=5, use_res=True)   # 57 tiles, split-K with odd boundaries


@pytest.mark.parametrize("K,N", [(3584, 4608), (3584, 3584), (18944, 3584)])
@pytest.mark.parametrize("M", [32, 64])
def test_fp8_gemm_qwen2_7b_projections(K, N, M):
    _case(K, N, M, seed=K % 97 + M, use_bias=(N == 4608), use_res=(N == 3584))


def test_fp8_gemm_gate_up_pair_and_llama_shapes():
    _case(3584, 18944, 64, seed=21, pair=True)     # persistent units + SwiGLU epilogue
    _case(4096, 6144, 32, seed=22)                 # Llama-3-8B QKV at the C3 batch
    _case(14336, 4096, 32, seed=23, use_res=True)  # Llama-3-8B down_proj


def test_fp8_rejects_what_it_does_not_cover():
    from b200spark import ops, quantize as PQ
    from b200spark._lib import B2Error
    g = torch.Generator().manual_seed(1)
    w = (torch.randn(512, 256, generator=g) * 0.02).to(torch.bfloat16)
    q, s, z = PQ.quantize_a16w8(w, -1)
    op8 = ops.GemmWQ(512, 256, 8, -1, max_m=4).prepare(q.cuda(), s.cuda(), z.cuda())
    q4, s4, z4 = PQ.quantize_a16w4(w, 128)
    opg = ops.GemmWQ(512, 256, 4, 128, max_m=4).prepare(q4.cuda(), s4.cuda(), z4.cuda())
    q8 = ops.quant_fp8(torch.randn(4, 512).to(torch.bfloat16).cuda())
    for op in (op8, opg):
        with pytest.raises(B2Error):
            op.run_fp8(q8, ops.Workspace())
