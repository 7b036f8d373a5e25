"""GPU: the split-K of the batch 17-64 wgmma GEMM inside thread-block clusters (the S k-slices of an n-group sum their
partial tiles through distributed shared memory, each finishing its share of the rows) against the workspace path
(B2_GEMM_TC_CLUSTER=0: partial tiles to global memory, the last slice to arrive sums and finishes the tile).  Both add the
slices from +0 in slice order, so on random inputs every output — C, the RMSNorm hand-off's xg_out and sumsq_out, the
SwiGLU pair's — must be the same bit for bit, over a repeated launch and a CUDA-graph replay.  Covers S = 2, 3, 4 and 6,
int4 / grouped int4 / int8 / bf16 weights, bf16 and fp16 activations, fp8 activations, bias, residual, every epilogue form
and N not a multiple of 128."""
import pytest
import torch

import tc_schedule as TS

pytestmark = pytest.mark.gpu

# (id, wbits, group, K, N, pair, dtype, epilogue): S = min(132 // NG, KT // 4, 6) k-slices on a 132-SM H100
SHAPES = [
    ("w4-S2", 4, -1, 1024, 6400, False, torch.bfloat16, "res"),        # NG 50
    ("w4-S3-n4600", 4, -1, 3584, 4600, False, torch.bfloat16, "handoff"),  # NG 36 (the qkv shape), N % 128 = 120
    ("w4-S4", 4, -1, 3584, 3584, False, torch.bfloat16, "handoff"),     # NG 28 (the o_proj shape)
    ("w4-S6", 4, -1, 1536, 1290, False, torch.bfloat16, "bias"),        # NG 11, N % 4 = 2: the generic epilogue
    ("w4g128-S4", 4, 128, 3584, 3584, False, torch.bfloat16, "res"),
    ("w4g128-S3-fp16", 4, 128, 2048, 4608, False, torch.float16, "res"),
    ("w4-S4-fp16", 4, -1, 1024, 3584, False, torch.float16, "handoff"),
    ("w8-S3", 8, -1, 2048, 4608, False, torch.bfloat16, "bias"),
    ("w8-S2-fp16", 8, -1, 1024, 6400, False, torch.float16, "silu"),
    ("w16-S4", 16, -1, 1024, 3584, False, torch.bfloat16, "res"),
    ("w16-S3-n4600", 16, -1, 1024, 4600, False, torch.bfloat16, "handoff"),
    ("pair-S3", 4, -1, 3584, 2200, True, torch.bfloat16, "swiglu"),     # NG 35 pair n-groups
    ("pair-S2-fp16", 4, -1, 1024, 3200, True, torch.float16, "swiglu"),  # NG 50
]


def _weights(wbits, group, K, N, dt, g):
    if wbits == 16:
        return ((torch.rand(K, N, device="cuda", generator=g) - 0.5) * 0.1).to(dt), None, None
    G = 1 if group == -1 else K // group
    if wbits == 4:
        q = torch.randint(0, 256, (K, (N + 1) // 2), dtype=torch.uint8, device="cuda", generator=g)
        zr = 15
    else:
        q = torch.randint(-128, 128, (K, N), dtype=torch.int8, device="cuda", generator=g)
        zr = 8
    s = (torch.rand(G, N, device="cuda", generator=g) * 1e-2 + 1e-3).to(dt)
    z = torch.randint(0, zr + 1, (G, N), device="cuda", generator=g).to(dt)
    return q, s, z


def _handle(wbits, group, K, N, pair, dt, M, seed, bias=False):
    from b200spark import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    op = ops.GemmWQ(K, N, wbits, group, max_m=M, pair=pair, dtype=dt)
    if pair:
        return op.prepare_swiglu(*_weights(wbits, group, K, N, dt, g), *_weights(wbits, group, K, N, dt, g))
    b = (torch.rand(N, device="cuda", generator=g) - 0.5).to(dt) if bias else None
    return op.prepare(*_weights(wbits, group, K, N, dt, g), bias=b)


def _graph(fn):
    gr, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(gr, stream=s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    return gr


def _run_both(make, run, monkeypatch):
    """run(op) -> tuple of output tensors, for the cluster plan and the workspace plan; each checked over a second launch
    and a graph replay.  Returns (cluster size of the first plan, outputs of both)."""
    got, sizes = [], []
    for knob in (None, "0"):
        if knob:
            monkeypatch.setenv("B2_GEMM_TC_CLUSTER", knob)
        op = make()
        sizes.append(op.tc_cluster())
        first = run(op)
        again = run(op)
        replayed = []
        gr = _graph(lambda: replayed.extend(run(op)))
        gr.replay()
        torch.cuda.synchronize()
        for a, b, c in zip(first, again, replayed):
            assert torch.equal(a, b) and torch.equal(a, c), "repeat / replay differs"
        got.append(first)
        monkeypatch.delenv("B2_GEMM_TC_CLUSTER", raising=False)
    assert sizes[1] == 1, sizes
    return sizes[0], got


@pytest.mark.parametrize("M", [17, 32, 33, 64, 80])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s[0])
def test_cluster_split_matches_workspace_split(shape, M, monkeypatch):
    from b200spark import _lib, ops
    name, wbits, group, K, N, pair, dt, epi = shape
    NG = (N + 63) // 64 if pair else (N + 127) // 128
    pl = TS.plan(NG, (K + 63) // 64, torch.cuda.get_device_properties(0).multi_processor_count)
    assert pl.rounds == 0 and pl.S > 1, pl
    g = torch.Generator(device="cuda").manual_seed(M)
    A = ((torch.rand(M, K, device="cuda", generator=g) - 0.5) * 2).to(dt)
    res = ((torch.rand(M, N, device="cuda", generator=g) - 0.5) * 4).to(dt)
    gamma = (torch.rand(N, device="cuda", generator=g) + 0.5).to(dt)

    def run(op):
        out = torch.full((M, N), float("nan"), dtype=dt, device="cuda")
        if epi == "handoff":
            ssq = torch.full((op.sumsq_parts(), M), -1.0, dtype=torch.float32, device="cuda")
            xg = torch.full((M, N), float("nan"), dtype=dt, device="cuda")
            op(A, ops.Workspace(), out=out, residual=res, sumsq_out=ssq, xg_out=(xg, gamma))
            return out, xg, ssq
        act = _lib.ACT_SILU if epi == "silu" else _lib.ACT_NONE
        op(A, ops.Workspace(), out=out, act=act, residual=res if epi in ("res", "bias") else None)
        return (out,)

    S, (cl, gl) = _run_both(lambda: _handle(wbits, group, K, N, pair, dt, M, 7, epi in ("bias", "silu")), run, monkeypatch)
    if pl.S <= 4:  # every GPC of an H100 holds four clusters of up to 4 CTAs: these must run as clusters
        assert S == pl.S, (name, S, pl.S)
    assert S in (1, pl.S)
    for a, b in zip(cl, gl):
        assert torch.equal(a, b), f"{name} M={M}: cluster split != workspace split"
    assert not torch.isnan(cl[0].float()).any()
    if epi == "handoff":
        assert bool((cl[2] >= 0).all())


@pytest.mark.parametrize("M", [17, 64])
def test_fp8_activations_cluster_split(M, monkeypatch):
    """The e4m3 instantiation (b2_gemm_wq_run_fp8) takes the same cluster split."""
    from b200spark import ops
    K, N = 3584, 4608
    g = torch.Generator(device="cuda").manual_seed(M)
    x = ((torch.rand(M, K, device="cuda", generator=g) - 0.5) * 2).to(torch.bfloat16)
    q8 = ops.quant_fp8(x)
    res = ((torch.rand(M, N, device="cuda", generator=g) - 0.5) * 4).to(torch.bfloat16)

    def run(op):
        return (op.run_fp8(q8, ops.Workspace(), residual=res),)

    S, (cl, gl) = _run_both(lambda: _handle(4, -1, K, N, False, torch.bfloat16, M, 11), run, monkeypatch)
    assert S == 3, S
    assert torch.equal(cl[0], gl[0])
