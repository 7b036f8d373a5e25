"""GPU: the weight-only GEMM kernels on exact-arithmetic inputs (tests/gemm_exact.py), every output element held to one
rounding of the restated arithmetic instead of the 2e-2 of the random-data tests.

  * weight read-back: A is a block of one-hot rows, so out[m, n] is the dequantized weight (k_m, n) itself (SwiGLU pairs:
    silu(w_gate) w_up) — every k of small shapes, and every tile / chunk / word / nibble / group start / the K tail of large
    ones, read through the packed image and the (scale, zero) look-up of each kernel;
  * dyadic GEMMs: full-rank dyadic A with bias, alpha, activations 0-6 and residual, on every kernel path;
  * call forms: strided A and C views, the output inside a guard frame that must stay untouched, in-place residual
    (out is residual) bit-identical to the out-of-place call, two runs and a CUDA-graph replay bit-identical.
Each case names the kernel it must reach; every kernel name the profiler shows (template arguments included) must be one the
host dispatch copied in gemm_exact.launches() predicts, and the GEMV split form is read off the handle's workspace size."""
import numpy as np
import pytest
import torch

import gemm_exact as X

pytestmark = pytest.mark.gpu
SENTINEL = -0x5A5B  # int16 bit pattern of the guard frame (a NaN-free, unlikely value in both FTs)
GUARD = 3           # guard rows above / below and columns right of the output


def _dt(case):
    return torch.float16 if case.ft == "fp16" else torch.bfloat16


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _setenv(monkeypatch, gc):
    for k, v in gc.env.items():
        monkeypatch.setenv(k, v)


def _handle(gc, inp):
    from b200spark import ops
    c = gc.case
    dt = _dt(c)
    op = ops.GemmWQ(c.K, c.N, c.wbits, c.group, max_m=max(gc.M, 1), signed=c.signed, pair=c.pair, dtype=dt)

    def dev(wt):
        q = torch.from_numpy(np.ascontiguousarray(X.pack_qdata(c, wt)))
        if c.wbits == 16:
            return (q.to(dt).cuda(), None, None)
        return (q.cuda(), torch.from_numpy(wt.s).to(dt).cuda(), torch.from_numpy(wt.z).to(dt).cuda())
    if c.pair:
        op.prepare_swiglu(*dev(inp["wt"]), *dev(inp["wt2"]))
    else:
        bias = inp.get("bias")
        op.prepare(*dev(inp["wt"]), torch.from_numpy(bias).to(dt).cuda() if bias is not None else None)
    return op


def _kernels(fn):
    """Names of the weight-only GEMM kernels fn launches (None if the profiler shows no kernel names here)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):  # one retry: a profiling session now and then delivers no kernel records
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if "wq_g" in e.name]
        if names:
            return names
    return None


def _assert_path(gc, names, M=None, a8=False):
    want = X.launches(gc.case, gc.M if M is None else M, gc.env, _sms(), a8=a8)
    assert {l["path"] for l in want} == {gc.path}, f"{gc.id}: the dispatch sends it to {want}, not {gc.path}"
    if names is None:
        return "dispatch copy"
    # the profiler may drop some of a call's kernel records (seen after many profiling sessions in one process), so the check
    # is that every kernel it does show is one the dispatch predicts
    got = {n[n.index("wq_g"):n.index(">") + 1] for n in names}
    assert got <= {l["kernel"] for l in want}, f"{gc.id}: ran {sorted(got)}, expected {[l['kernel'] for l in want]}"
    return "profiler"


def _gemv_split(gc, op, inp, monkeypatch):
    """The split form the GEMV plan chose, read off the handle's workspace size (16 bytes: no workspace, i.e. S = 1 or the
    cluster split; else the partial tiles of S k-slices): forced and global splits must have S > 1; a 'cluster' case must
    have S > 1 with clusters disabled and need no workspace with them, which leaves only the cluster split."""
    rows = min(gc.M, X.GEMV_MAX_M)
    mp = 8 << X.mt_index_for(rows)
    per_slice = gc.case.NG * mp * (X.KBN + 1) * 4
    ws = op.workspace_bytes(gc.M)
    S = (ws - 16) // per_slice if ws > 16 else 1
    forced = int(gc.env.get("B2_GEMM_FORCE_SPLIT", 0))
    if forced:
        assert S == forced, (gc.id, S)
        return f"split=forced S={S}"
    if gc.env.get("B2_GEMM_CLUSTER") == "0":
        assert S > 1, (gc.id, S)
        return f"split=global S={S}"
    if "cluster" in gc.id:
        monkeypatch.setenv("B2_GEMM_CLUSTER", "0")
        twin = _handle(gc, inp)
        S0 = (twin.workspace_bytes(gc.M) - 16) // per_slice     # planned now, while clusters are off
        monkeypatch.delenv("B2_GEMM_CLUSTER")
        assert S0 > 1 and ws == 16, (gc.id, S0, ws)
        return f"split=cluster (global S={S0})"
    return f"split={'none/cluster' if ws == 16 else f'global S={S}'}"


class Framed:
    """A [M, N] view inside a buffer with GUARD rows above and below, ld = N + pad columns, an element offset `off` into the
    row (off odd: a view that is not 4-byte aligned) and every cell outside the view set to SENTINEL."""

    def __init__(self, M, N, dt, pad=0, off=0):
        self.ld = N + pad
        self.buf = torch.full(((M + 2 * GUARD) * self.ld + GUARD + off,), SENTINEL, dtype=torch.int16, device="cuda")
        self.off = GUARD * self.ld + off
        self.M, self.N = M, N
        self.view = self.buf.view(dt)[self.off:self.off + M * self.ld].view(M, self.ld)[:, :N]

    def fill(self, t):
        self.view.copy_(t)
        return self

    def guards_intact(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        idx = self.off + torch.arange(self.M, device="cuda")[:, None] * self.ld + torch.arange(self.N, device="cuda")[None, :]
        mask[idx.reshape(-1)] = False
        return bool((self.buf[mask] == SENTINEL).all())


def _acts(A, dt, pad):
    """A as a view with lda = K + pad (16-byte aligned rows)."""
    M, K = A.shape
    buf = torch.zeros(M, K + pad, dtype=dt, device="cuda")
    buf[:, :K] = torch.from_numpy(A).to(dt)
    return buf[:, :K]


# ------------------------------------------------------------------------------------------------------------ read-back
@pytest.mark.parametrize("gc", X.READBACK_CASES, ids=lambda g: g.id)
def test_weight_readback(gc, monkeypatch):
    _setenv(monkeypatch, gc)
    from b200spark import ops
    c = gc.case
    dt = _dt(c)
    inp = dict(wt=X.make_weights(c, X._seed(gc)), wt2=X.make_weights(c, X._seed(gc) + 1) if c.pair else None)
    op = _handle(gc, inp)
    W = X.path_weights(c, inp["wt"], gc.path)
    W2 = X.path_weights(c, inp["wt2"], gc.path) if c.pair else None
    ks = X.readback_ks(gc)
    nl = (len(ks) + gc.M - 1) // gc.M
    ks_all = (ks * (nl * gc.M // len(ks) + 1))[:nl * gc.M]          # the last launch is filled up with ks from the start
    order = np.random.default_rng(len(ks)).permutation(gc.M)          # one-hot rows in permuted order inside a launch
    ks_all = [ks_all[l * gc.M + order[i]] for l in range(nl) for i in range(gc.M)]
    A = torch.from_numpy(X.onehot_acts(ks_all, c.K)).to(dt).cuda()
    fr = Framed(nl * gc.M, c.N, dt, GUARD)
    out = fr.view
    ws = ops.Workspace()
    how = _assert_path(gc, _kernels(lambda: op(A[:gc.M], ws, out=out[:gc.M])))
    for l in range(nl):
        op(A[l * gc.M:(l + 1) * gc.M], ws, out=out[l * gc.M:(l + 1) * gc.M])
    torch.cuda.synchronize()
    assert fr.guards_intact(), f"{gc.id}: a write outside [M, N]"
    got = out.double().cpu().numpy()
    rows = np.asarray(ks_all)
    if c.pair:
        y, E = X.expected(np.eye(c.K)[rows], W, W2=W2)
    else:
        y, E = W[rows], np.zeros((len(rows), c.N))
    bad, dev = X.check(got, y, E, c.ft)
    assert not bad.any(), (f"{gc.id}: {int(bad.sum())} of {bad.size} weights read back wrong, first (m, k, n): "
                           f"{[(int(m), ks_all[m], int(n)) for m, n in np.argwhere(bad)[:8]]}")
    print(f"READBACK {gc.id} path={gc.path} via={how} k={len(ks)} elements={got.size} worst={dev.max():.3f}")


# ------------------------------------------------------------------------------------------------------------ dyadic GEMMs
@pytest.mark.parametrize("i", range(len(X.DYADIC_CASES)), ids=lambda i: X.DYADIC_CASES[i].id)
def test_dyadic_gemm(i, monkeypatch):
    gc = X.DYADIC_CASES[i]
    _setenv(monkeypatch, gc)
    from b200spark import ops
    c = gc.case
    dt = _dt(c)
    inp = X.dyadic_inputs(gc)
    X.case_precondition(gc, inp)
    y, E = X.restate(gc, inp)
    op = _handle(gc, inp)
    pa, pc, off = X.call_form(i)
    A = _acts(inp["A"], dt, pa)
    ws = ops.Workspace()
    fr = Framed(gc.M, c.N, dt, pc, off)
    res = None
    if inp["res"] is not None:
        rf = Framed(gc.M, c.N, dt, pc, off).fill(torch.from_numpy(inp["res"]).to(dt))
        res = rf.view
    run = lambda out, r: op(A, ws, out=out, act=gc.act, alpha=gc.alpha, residual=r)
    how = _assert_path(gc, _kernels(lambda: run(fr.view, res)))
    split = _gemv_split(gc, op, inp, monkeypatch) if gc.path == "gemv" else ""
    first = fr.view.clone()
    run(fr.view, res)                                    # a second run: split-K counters re-armed, deterministic
    torch.cuda.synchronize()
    assert torch.equal(fr.view, first), f"{gc.id}: second run differs"
    assert fr.guards_intact(), f"{gc.id}: a write outside [M, N]"
    got = first.double().cpu().numpy()
    bad, dev = X.check(got, y, E, c.ft)
    assert not bad.any(), (f"{gc.id}: {int(bad.sum())} of {bad.size} elements off their bound, first (m, n): "
                           f"{np.argwhere(bad)[:8].tolist()}, dev {dev[bad][:8]}")
    if res is not None:                                  # in place: out is residual
        run(rf.view, rf.view)
        torch.cuda.synchronize()
        assert torch.equal(rf.view, first), f"{gc.id}: in-place residual differs from the out-of-place call"
        assert rf.guards_intact()
        rf.fill(torch.from_numpy(inp["res"]).to(dt))
    # CUDA graph replay (the handle's plan and workspace already exist)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    fr2 = Framed(gc.M, c.N, dt, pc, off)
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            run(fr2.view, res)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(fr2.view, first), f"{gc.id}: graph replay differs"
    assert fr2.guards_intact()
    print(f"DYADIC {gc.id} path={gc.path} via={how} {split} form={(pa, pc, off)} elements={got.size} "
          f"exact={int((E == 0).sum())} worst={dev.max():.3f}")


# ------------------------------------------------------------------------------------------------------------ wgmma split-K
@pytest.mark.parametrize("gc", [g for g in X.DYADIC_CASES if g.id in ("tc-w4-m17", "tc-w4-q72-down", "tc-w8-m64", "tc-g128-m32")],
                         ids=lambda g: g.id)
def test_tc_split_k_matches_one_slice(gc, monkeypatch):
    """tc_S > 1 (partials in the workspace, fixed-order reduction by the last CTA) against tc_S = 1: bit-identical on exact
    inputs, and both equal to the restatement."""
    from b200spark import ops
    c = gc.case
    assert X.tc_split(c, _sms()) > 1, "the default plan must split K here"
    inp = X.dyadic_inputs(gc)
    dt = _dt(c)
    A = _acts(inp["A"], dt, 0)
    # the residual is read with the output's row stride
    res = Framed(gc.M, c.N, dt, GUARD).fill(torch.from_numpy(inp["res"]).to(dt)).view if inp["res"] is not None else None
    outs, frames = [], []
    for env in ({}, {"B2_GEMM_TC_MAX_SPLIT": "1"}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        op = _handle(gc, inp)
        fr = Framed(gc.M, c.N, dt, GUARD)
        frames.append(fr)
        outs.append(op(A, ops.Workspace(), out=fr.view, act=gc.act, alpha=gc.alpha, residual=res))
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    assert all(fr.guards_intact() for fr in frames)
    y, E = X.restate(gc, inp)
    bad, _ = X.check(outs[0].double().cpu().numpy(), y, E, c.ft)
    assert not bad.any()


# ------------------------------------------------------------------------------------------------------------ RMSNorm hand-off
@pytest.mark.parametrize("M", [17, 64])
def test_rmsnorm_handoff_producer_exact(M):
    """Producer form at M >= 17 (xg_out, sumsq_out): C is rn(y) exactly, xg = rn(C * gamma) of the stored values, and the
    per-tile statistics are the sums of squares of the stored values (fp32 sums of exact squares: a relative 2^-20)."""
    from b200spark import ops
    gc = X.GpuCase("handoff", X.Case(4, 1024, 1280), M, "tc", res=True)
    inp = X.dyadic_inputs(gc)
    X.case_precondition(gc, inp)
    y, E = X.restate(gc, inp)
    op = _handle(gc, inp)
    A = _acts(inp["A"], torch.bfloat16, 0)
    res = Framed(M, 1280, torch.bfloat16, 4).fill(torch.from_numpy(inp["res"]).to(torch.bfloat16)).view  # output's row stride
    gamma = torch.from_numpy(X.make_vec(1280, 5, 2.0 ** -4, 32)).to(torch.bfloat16).cuda()
    ssq = torch.zeros(op.sumsq_parts(), M, dtype=torch.float32, device="cuda")
    xg = torch.empty(M, 1280, dtype=torch.bfloat16, device="cuda")
    fr = Framed(M, 1280, torch.bfloat16, 4)
    out = op(A, ops.Workspace(), out=fr.view, residual=res, sumsq_out=ssq, xg_out=(xg, gamma))
    torch.cuda.synchronize()
    assert fr.guards_intact()
    got = out.double().cpu().numpy()
    bad, _ = X.check(got, y, E, "bf16")
    assert not bad.any()
    g64 = gamma.double().cpu().numpy()
    assert np.array_equal(xg.double().cpu().numpy(), X.rn_ft((got * g64[None, :]).astype(np.float32).astype(np.float64), "bf16"))
    tiles = (got ** 2).reshape(M, -1, 128).sum(-1).T
    assert np.allclose(ssq.double().cpu().numpy(), tiles, rtol=2.0 ** -20, atol=0)


# ------------------------------------------------------------------------------------------------------------ fp8 activations
@pytest.mark.parametrize("gc", X.FP8_CASES, ids=lambda g: g.id)
def test_fp8_activations(gc):
    """b2_gemm_wq_run_fp8: the device quantizer against its bit-exact restatement, then the e4m3 wgmma GEMM against the
    fp32 restatement of gemm_exact.restate_fp8 (exact activations: bit for bit), a guard frame, a second run and a graph
    replay.  rb-* cases read every weight back through one-hot rows."""
    from b200spark import ops
    c = gc.case
    if gc.id.startswith("rb-"):
        ks = X.readback_ks(gc)
        nl = (len(ks) + gc.M - 1) // gc.M
        ks_all = (ks * (nl * gc.M // len(ks) + 1))[:nl * gc.M]
        order = np.random.default_rng(len(ks)).permutation(gc.M)
        ks_all = [ks_all[l * gc.M + order[i]] for l in range(nl) for i in range(gc.M)]
        inp = dict(wt=X.fp8_weights(c, X._seed(gc)), wt2=None, A=X.onehot_acts(ks_all, c.K), bias=None, res=None)
    else:
        inp = X.dyadic_inputs(gc)
        nl = 1
    X.case_precondition(gc, inp)
    y, E = X.restate(gc, inp, sms=_sms())
    op = _handle(gc, inp)
    x = torch.from_numpy(inp["A"]).to(torch.bfloat16).cuda()
    q8 = ops.quant_fp8(x)
    torch.cuda.synchronize()
    y8, sc, ts = X.quant_fp8(inp["A"])
    assert np.array_equal(q8.scale.cpu().numpy(), sc) and np.array_equal(q8.tile_sums.cpu().numpy(), ts)
    perm = [0, 2, 4, 6, 1, 3, 5, 7]   # k order inside each group of 8 in the fp8 activation layout
    dec = q8.y[:, :c.K].contiguous().view(torch.float8_e4m3fn).double().cpu().numpy().reshape(x.shape[0], -1, 8)
    nat = np.empty_like(dec)
    nat[:, :, perm] = dec
    assert np.array_equal(nat.reshape(x.shape[0], -1), y8)
    ws = ops.Workspace()
    fr = Framed(nl * gc.M, c.N, torch.bfloat16, 4)
    rf = Framed(gc.M, c.N, torch.bfloat16, 4).fill(torch.from_numpy(inp["res"]).to(torch.bfloat16)) if gc.res else None
    res = rf.view if rf is not None else None

    def sub(l):
        s8 = ops.Fp8Act(gc.M, c.K)
        s8.y, s8.scale, s8.tile_sums = q8.y[l * gc.M:(l + 1) * gc.M], q8.scale[l * gc.M:(l + 1) * gc.M], q8.tile_sums[l * gc.M:(l + 1) * gc.M]
        return s8
    parts = [sub(l) for l in range(nl)]
    run = lambda l, out: op.run_fp8(parts[l], ws, out=out, act=gc.act, alpha=gc.alpha, residual=res)
    how = _assert_path(gc, _kernels(lambda: run(0, fr.view[:gc.M])), a8=True)
    for l in range(nl):
        run(l, fr.view[l * gc.M:(l + 1) * gc.M])
    torch.cuda.synchronize()
    assert fr.guards_intact(), f"{gc.id}: a write outside [M, N]"
    first = fr.view.clone()
    got = first.double().cpu().numpy()
    bad, dev = X.check(got, y, E, "bf16")
    assert not bad.any(), (f"{gc.id}: {int(bad.sum())} of {bad.size} elements off their bound, first (m, n): "
                           f"{np.argwhere(bad)[:8].tolist()}, dev {dev[bad][:8]}")
    if nl == 1:
        run(0, fr.view)
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        fr2 = Framed(gc.M, c.N, torch.bfloat16, 4)
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                run(0, fr2.view)
        torch.cuda.current_stream().wait_stream(s)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(fr.view, first) and torch.equal(fr2.view, first) and fr2.guards_intact()
    print(f"FP8 {gc.id} path={gc.path} via={how} elements={got.size} exact={int((E == 0).sum())} worst={dev.max():.3f}")
