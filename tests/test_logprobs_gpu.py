"""GPU: b2_logprobs, b2_logprobs_shard + b2_logprobs_merge and DecodeStack(logprobs=N) against fp64 log_softmax within the
bound of tests/logprobs_ref.py, with ids bit-exact against b2_argmax and the argmax order."""
import os
import socket

import numpy as np
import pytest
import torch

import glue_ref as G
import logprobs_ref as P

pytestmark = pytest.mark.gpu


def _batch(n, rows, pad, dt, seed):
    """[rows, n + pad] fp32 exact in dt: row r of kind r % 14 (ARGMAX_KINDS, then LP_KINDS), PAD_PLANTS in the padding"""
    rng = np.random.default_rng(seed)
    kinds = G.ARGMAX_KINDS + P.LP_KINDS
    x = np.empty((rows, n + pad), np.float32)
    for r in range(rows):
        k = kinds[r % len(kinds)]
        x[r, :n] = G.ft_values(G.argmax_row(k, n, rng), dt) if k in G.ARGMAX_KINDS else P.lp_row(k, n, dt, rng)
        for j in range(pad):
            x[r, n + j] = G.PAD_PLANTS[(r + j) % len(G.PAD_PLANTS)]
    return x


def _check(out, x, n, n_top, exact, bound, tok_ids=None, argmax_ids=None, want=None):
    """worst ratio to the bound of top_lp and tok_lp; ids asserted exact.  want: P.top_order(x, n, 10), if computed"""
    ids, tlp, tids, tlps = out
    want = P.top_order(x, n, max(n_top, 1)) if want is None else want
    ids = ids.cpu().numpy()
    assert np.array_equal(ids, want[:, 0])
    if argmax_ids is not None:
        assert np.array_equal(ids, argmax_ids)
    worst = 0.0
    if n_top:
        tids, tlps = tids.cpu().numpy(), tlps.cpu().numpy()
        assert np.array_equal(tids, want[:, :n_top])
        assert np.array_equal(tids[:, 0], ids)
        worst = P.lp_ratio(tlps, P.gather(exact, tids), P.gather(bound, tids))
    tok = want[:, 0] if tok_ids is None else tok_ids.cpu().numpy()
    ok = (tok >= 0) & (tok < n)
    te = np.where(ok, P.gather(exact, np.where(ok, tok, 0)[:, None])[:, 0], np.nan)
    tb = np.where(ok, P.gather(bound, np.where(ok, tok, 0)[:, None])[:, 0], 0.0)
    tlp = tlp.cpu().numpy()
    assert np.isnan(tlp[~ok]).all()
    return max(worst, P.lp_ratio(tlp, te, tb))


@pytest.mark.parametrize("n", G.ARGMAX_N)
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_logprobs_sweep(dt, n):
    """rows 1 / 64 / 65 of every kind, ld = n + 5 with PAD_PLANTS in the padding, n_top 0 / 1 / 5 / 10, with and without
    token ids (some out of range)"""
    from b200spark import ops
    ft = G.FTS[dt]
    x = _batch(n, 65, 5, ft, seed=n + 17)
    lg = G.to_ft(x, ft).cuda()
    exact, bound = P.lp_bound(x, n)
    rng = np.random.default_rng(n)
    tok = torch.from_numpy(rng.integers(-2, n + 2, 65)).cuda()
    want = P.top_order(x, n, P.MAX_TOP)
    worst = 0.0
    for rows in G.ARGMAX_BATCH:
        view = lg[:rows, :n]
        am = ops.argmax(view).cpu().numpy()
        for n_top in P.N_TOPS:
            out = ops.logprobs(view, n_top)
            worst = max(worst, _check(out, x[:rows], n, n_top, exact[:rows], bound[:rows], None, am, want[:rows]))
            out = ops.logprobs(view, n_top, tok_ids=tok[:rows])
            worst = max(worst, _check(out, x[:rows], n, n_top, exact[:rows], bound[:rows], tok[:rows], am, want[:rows]))
    assert worst <= 1.0, worst


@pytest.mark.parametrize("tp", [2, 4, 8])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_shard_merge(dt, tp):
    """shards of the whole row (strided views, id_offset = the shard start) + the merge of the stacked records: ids equal
    the whole-row form, logprobs within the merge bound; one shard + the merge is b2_logprobs bit for bit"""
    from b200spark import ops
    ft = G.FTS[dt]
    n = 151936
    rng = np.random.default_rng(tp)
    x = np.stack([G.ft_values(G.tp_row(k, n, tp, rng), ft) for k in G.TP_KINDS]
                 + [P.lp_row(k, n, ft, rng) for k in P.LP_KINDS])
    B = x.shape[0]
    lg = G.to_ft(x, ft).cuda()
    shards = G.shard_bounds(n, tp)
    exact, bound = P.lp_bound(x, n, shards)
    tok = torch.from_numpy(rng.integers(0, n, B)).cuda()
    tok[0] = n  # out of range on every shard: NaN
    want = P.top_order(x, n, P.MAX_TOP)
    for n_top in P.N_TOPS:
        rb = ops.logprobs_partial_bytes(n_top)
        allp = torch.empty(tp, B * rb, dtype=torch.uint8, device="cuda")
        for r, (s, e) in enumerate(shards):
            ops.logprobs_shard(lg[:, s:e], n_top, s, tok_ids=tok, out=allp[r].view(B, rb))
        merged = ops.logprobs_merge(allp, n_top)
        whole = ops.logprobs(lg, n_top, tok_ids=tok)
        assert torch.equal(merged[0], whole[0])
        if n_top:
            assert torch.equal(merged[2], whole[2])
        assert _check(merged, x, n, n_top, exact, bound, tok, want=want) <= 1.0
        one = ops.logprobs_merge(ops.logprobs_shard(lg, n_top, 0, tok_ids=tok)[None].reshape(1, -1), n_top)
        for a, b in zip(one, whole):
            if a is not None:
                assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                   b.view(torch.int32) if b.dtype == torch.float32 else b)


def test_graph_replay_and_repeatability():
    """a CUDA-graph replay equals the eager call bit for bit, and two eager runs are bitwise equal"""
    from b200spark import ops
    x = _batch(152064, 64, 0, torch.bfloat16, seed=3)
    lg = G.to_ft(x, torch.bfloat16).cuda()
    outs = [ops.logprobs(lg, 10) for _ in range(2)]
    gout = tuple(torch.empty_like(t) for t in outs[0])
    ops.logprobs(lg, 10, out=gout)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.logprobs(lg, 10, out=gout)
    for t in gout:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b, c in zip(outs[0], outs[1], gout):
        bits = (lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t)
        assert torch.equal(bits(a), bits(b)) and torch.equal(bits(a), bits(c))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B,T,tree", [(1, 1, False), (3, 1, False), (17, 1, False), (64, 1, False), (1, 4, False),
                                      (3, 4, False), (17, 4, False), (64, 4, False), (3, 4, True)])
def test_decode_stack_logprobs(dtype, B, T, tree):
    """DecodeStack(TINY, logprobs=10): the step's ids equal b2_argmax of its own logits, top_lp / tok_lp lie within the
    bound of fp64 log_softmax of those logits; the step keeps the launch count of a logprobs=0 stack, whose step is
    unchanged; the graph replay gives the eager results"""
    from b200spark import model, ops
    kw = dict(wbits=4, span=16, seed=11, dtype=dtype, q_len=T, tree=tree)
    st = model.DecodeStack(model.TINY, B, 64, logprobs=10, **kw)
    base = model.DecodeStack(model.TINY, B, 64, **kw)
    g = torch.Generator().manual_seed(B * 31 + T)
    for s in (st, base):
        if T == 1:
            s.ids.copy_(torch.randint(0, model.TINY.vocab, (B,), generator=g).cuda())
        else:
            s.tokens.copy_(torch.randint(0, model.TINY.vocab, (B, T), generator=g).cuda())
        g = torch.Generator().manual_seed(B * 31 + T)
        if tree:
            s.parents.copy_(torch.tensor([0, 0, 0, 1], dtype=torch.int32).repeat(B, 1).cuda())
    for step in range(2):
        a = st.step()
        b = base.step()
        torch.cuda.synchronize()
        ids = (a if T == 1 else a[0]).reshape(-1)
        assert torch.equal(st.logits, base.logits)
        assert torch.equal(ids, (b if T == 1 else b[0]).reshape(-1))
        assert torch.equal(ids, ops.argmax(st.logits))
        x = st.logits.float().cpu().numpy()
        exact, bound = P.lp_bound(x, x.shape[1])
        worst = _check((ids, st.tok_lp, st.top_ids, st.top_lp), x, x.shape[1], 10, exact, bound)
        assert worst <= 1.0, (step, worst)
    assert st.launches_per_step == base.launches_per_step
    # graph replay from the same state as an eager step
    snap = [t.clone() for t in (st.lens_old, st.lens_new)] + ([st.tokens.clone()] if T > 1 else [st.ids.clone()])
    st._step_ops()
    torch.cuda.synchronize()
    eager = [t.clone() for t in (st.tok_lp, st.top_ids, st.top_lp)]
    st.lens_old.copy_(snap[0]); st.lens_new.copy_(snap[1])
    (st.tokens if T > 1 else st.ids).copy_(snap[2])
    st.capture()
    st.step()
    torch.cuda.synchronize()
    for e, t in zip(eager, (st.tok_lp, st.top_ids, st.top_lp)):
        assert torch.equal(e, t)


def test_launch_count_unchanged_without_logprobs():
    """logprobs=0 runs today's step: the launch counts the step had before logprobs existed"""
    from b200spark import model
    for B, T in ((1, 1), (17, 1), (64, 1), (3, 4)):
        st = model.DecodeStack(model.TINY, B, 64, wbits=4, span=16, q_len=T)
        lp = model.DecodeStack(model.TINY, B, 64, wbits=4, span=16, q_len=T, logprobs=10)
        st.step(); lp.step()
        torch.cuda.synchronize()
        assert st.launches_per_step == lp.launches_per_step > 0


# ---------------------------------------------------------------- 2 GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret, collective):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, "dash-infer_b200", "python"))
    import torch.distributed as dist
    from b200spark import model
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    B = 3
    st = model.DecodeStack(model.TINY, B, 64, wbits=4, span=16, seed=7, tp_rank=rank, tp_size=world, collective=collective,
                           logprobs=10)
    one = model.DecodeStack(model.TINY, B, 64, wbits=4, span=16, seed=7, logprobs=10)
    st.capture()
    ids = torch.tensor([1, 2, 3], dtype=torch.int64, device="cuda")
    ok, worst = True, 0.0
    for _ in range(4):
        st.ids.copy_(ids); one.ids.copy_(ids)
        n_tp = st.step().clone(); n_one = one.step().clone()
        torch.cuda.synchronize()
        full = one.logits.float()
        worst = max(worst, ((st.top_lp - one.top_lp).abs().max() / one.top_lp.abs().max()).item())
        top2 = torch.topk(full, 2, dim=-1).values
        for b in range(B):
            if (top2[b, 0] - top2[b, 1]).item() > 0.04 * full.abs().max().item():
                ok = ok and n_tp[b].item() == n_one[b].item() and st.top_ids[b, 0].item() == one.top_ids[b, 0].item()
        ids = n_one
    if st.comm is not None:
        st.comm.check_error()
    ret[rank] = (ok, worst)
    dist.barrier()
    os._exit(0)  # graphs hold captured collectives: leave without tearing the communicators down


@pytest.mark.parametrize("collective", ["b2", "nccl"])
def test_tp2_logprobs_match_single_gpu(collective):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, ret, collective)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    for r in range(2):
        ok, worst = ret[r]
        assert worst < 2e-2, worst
        assert ok
