"""GPU: GLM-shaped decode stacks (interleaved rotary over half of each 128-dim head, QKV bias, up to 16 q heads per kv head)
against the oracle that rotates the GLM way (tests/glm_ref.py: ref_from_stack), under the rules of test_qwen3_gpu.py:
tiny stacks in five weight / KV modes at both norm placements and in fp16, chain and tree verify steps, the same launches
and graph kernel nodes as the NeoX stack, GLM-4-9B layers, and TP = 2 against one GPU."""
import dataclasses
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import glm_ref as R
from oracle import kvcache_ref as KV
from test_stack_launches_gpu import graph_kernels, recorded_step

pytestmark = pytest.mark.gpu

KVM = {"none": KV.QUANT_NONE, "i8": KV.QUANT_I8, "u4": KV.QUANT_U4}


def _tiny(n_kv=1, **kw):
    """16 q heads x 128 over n_kv kv heads (16 per group at n_kv = 1, the attention kernel's limit), rotary over 64 dims"""
    from b200spark import model
    return model.ModelConfig("tiny-glm", 512, 16, n_kv, 1024, 2, 1024, rope_base=1e4, eps=1e-5, qkv_bias=True, rotary_dim=64,
                             rope_style="interleaved", **kw)


def _run_against_oracle(st, ref, B, steps, ids, tol_scale, capture_at=None):
    ref.reset(B)
    for t in range(steps):
        if capture_at == t:
            st.capture()
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        torch.cuda.synchronize()
        glog = st.logits.float().cpu()
        rlog, rnext = ref.step(ids, [t] * B)
        tol = tol_scale * rlog.abs().max().item()
        err = (glog - rlog).abs().max().item()
        assert err <= tol, (t, err, tol)
        assert torch.equal(nxt, torch.argmax(glog, dim=-1))
        top2 = torch.topk(rlog, 2, dim=-1).values
        for b in range(B):
            if (top2[b, 0] - top2[b, 1]).item() > 2 * tol:
                assert nxt[b].item() == rnext[b].item(), (t, b)
        ids = nxt
    assert st.lens_old.cpu().tolist() == [steps] * B


@pytest.mark.parametrize("wbits,group,kv,n_kv", [(4, -1, "none", 1), (8, -1, "none", 2), (4, 128, "none", 2), (8, -1, "i8", 1),
                                                 (4, -1, "u4", 2)])
@pytest.mark.parametrize("B", [2, 20])
def test_tiny_glm_logits_and_tokens(wbits, group, kv, n_kv, B):
    """eager for 3 steps, then a captured graph; B = 2 runs the self-contained GEMV norms, B = 20 the hand-off form"""
    from b200spark import model
    st = model.DecodeStack(_tiny(n_kv), B, 64, wbits=wbits, group=group, kv=kv, span=16, keep_ref=True)
    ref = R.ref_from_stack(st, KVM[kv])
    ids = (torch.arange(B, dtype=torch.int64) * 37 + 3) % 1024
    _run_against_oracle(st, ref, B, 6, ids, 4e-2 if kv == "u4" else 1e-2, capture_at=3)


@pytest.mark.parametrize("B", [2, 20])
def test_tiny_glm_fp16(B):
    from b200spark import model
    st = model.DecodeStack(_tiny(2), B, 64, wbits=4, span=16, keep_ref=True, dtype=torch.float16)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    ids = (torch.arange(B, dtype=torch.int64) * 53 + 1) % 1024
    _run_against_oracle(st, ref, B, 5, ids, 1e-2, capture_at=3)


def test_oracle_with_the_neox_pairing_is_farther():
    """the oracle that pairs NeoX-style over the same 64 dims is at least twice as far from the stack as the GLM oracle: the
    agreement above comes from the pairing, not from a tolerance that would accept the other one"""
    from b200spark import model
    B = 3
    st = model.DecodeStack(_tiny(2), B, 64, wbits=8, group=-1, kv="none", span=16, keep_ref=True)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    other = R.ref_from_stack(st, KV.QUANT_NONE)
    other.rope_il = False
    ref.reset(B); other.reset(B)
    ids = (torch.arange(B, dtype=torch.int64) * 37 + 3) % 1024
    e_ref = e_other = 0.0
    for t in range(12):
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        torch.cuda.synchronize()
        glog = st.logits.float().cpu()
        rlog, _ = ref.step(ids, [t] * B)
        olog, _ = other.step(ids, [t] * B)
        mx = rlog.abs().max().item()
        e_ref = max(e_ref, (glog - rlog).abs().max().item() / mx)
        e_other = max(e_other, (glog - olog).abs().max().item() / mx)
        ids = nxt
    print("tiny GLM stack: worst |logit error| / range against the GLM oracle %.2e, against the NeoX-paired one %.2e"
          % (e_ref, e_other))
    assert e_ref <= 1e-2 and e_other >= 2 * e_ref, (e_ref, e_other)


def test_launches_and_graph_kernels_equal_the_neox_stack():
    """the pairing rides in the append: the same launches per step and the same kernel nodes in the captured graph as the
    same stack with rope_style="neox", at every norm placement, and different logits"""
    from b200spark import model
    cfg = _tiny(2)
    for B in (1, 5, 20):
        il = model.DecodeStack(cfg, B, 64, wbits=4, span=16, seed=9)
        nx = model.DecodeStack(dataclasses.replace(cfg, rope_style="neox"), B, 64, wbits=4, span=16, seed=9)
        for t in range(3):
            for st in (il, nx):
                st.ids.fill_(5 + 70 * t)
                st.step()
        torch.cuda.synchronize()
        assert il.launches_per_step == nx.launches_per_step, B
        assert torch.equal(il.embed, nx.embed)
        assert not torch.equal(il.logits, nx.logits)
        n_il, n_nx = len(graph_kernels(recorded_step(il))), len(graph_kernels(recorded_step(nx)))
        assert n_il == n_nx == il.launches_per_step, (B, n_il, n_nx)
    big = model.DecodeStack(model.GLM4_9B, 1, 16, wbits=4, span=16, layers=1)
    big_nx = model.DecodeStack(dataclasses.replace(model.GLM4_9B, rope_style="neox"), 1, 16, wbits=4, span=16, layers=1)
    big.step(); big_nx.step()
    torch.cuda.synchronize()
    assert big.launches_per_step == big_nx.launches_per_step
    print("GLM-4-9B (1 layer, batch 1) launches per step:", big.launches_per_step)


def _greedy(cfg, B, steps, first, **kw):
    from b200spark import model
    st = model.DecodeStack(cfg, B, 64, **kw)
    ids, logits, cur = [], [], first.cuda()
    for _ in range(steps):
        st.ids.copy_(cur)
        cur = st.step().clone()
        ids.append(cur.cpu())
        logits.append(st.logits.float().cpu().clone())
    return torch.stack(ids, 1), logits


@pytest.mark.parametrize("tree", [False, True])
def test_verify_steps_accept_the_models_own_continuation(tree):
    """chain and tree verify steps of T = 4 whose drafts are the single-token stack's greedy continuation: wherever the
    single-token logits decide the tokens, all T are accepted and the emitted tokens are the single steps' tokens"""
    from b200spark import model
    cfg, B, T, rounds = _tiny(2), 4, 4, 3
    kw = dict(wbits=4, kv="none", span=16, seed=77)
    first = torch.tensor([3, 41, 97, 500], dtype=torch.int64)
    ref_ids, ref_logits = _greedy(cfg, B, T * (rounds + 2), first, **kw)
    st = model.DecodeStack(cfg, B, 64, q_len=T, tree=tree, **kw)
    st.tokens[:, 0] = first.cuda()
    done, live, checked_all = [0] * B, [True] * B, 0
    for r in range(rounds):
        for b in range(B):
            st.tokens[b, 1:] = ref_ids[b, done[b]:done[b] + T - 1].cuda()
        out = st.step()
        pred, acc = out[0].cpu(), out[1].cpu()
        logits = st.logits.float().cpu().view(B, T, -1)
        for b in range(B):
            n_ok = 0
            for t in range(T):
                if not live[b]:
                    break
                rl = ref_logits[done[b] + t][b]
                err = (logits[b, t] - rl).abs().max().item()
                assert err <= 1e-2 * rl.abs().max().item(), (r, b, t, err)
                top2 = torch.topk(rl, 2).values
                if (top2[0] - top2[1]).item() <= 2 * err:
                    live[b] = False
                    break
                assert pred[b, t].item() == ref_ids[b, done[b] + t].item(), (r, b, t)
                n_ok += 1
            if n_ok == T:
                assert acc[b].item() == T, (r, b, acc)
                if tree:
                    assert out[2][b].cpu().tolist() == list(range(T))
            checked_all += n_ok
            done[b] += int(acc[b])
    assert st.lens_old.cpu().tolist() == done
    assert checked_all >= 2 * T, checked_all


@pytest.mark.parametrize("B", [1, 64])
def test_glm4_9b_layer(B):
    """one full-width GLM-4-9B layer (hidden 4096, 32 q heads over 2 kv heads, inter 13696, int4 per-channel) + final norm +
    the 151552-wide lm_head, from a cache of 300 tokens (B = 1) or an empty one, three steps against the GLM oracle"""
    from b200spark import model
    cfg, steps = model.GLM4_9B, 3
    ctx = 300 if B == 1 else 0
    st = model.DecodeStack(cfg, B, ctx + 32, wbits=4, group=-1, kv="none", span=128, keep_ref=True, layers=1)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    ref.reset(B)
    if ctx:
        st.set_context(ctx)
        gen = torch.Generator(device="cuda").manual_seed(4321)  # set_context's draws, in its order
        kw = st.nG_l * st.head
        for b in range(B):
            rows = torch.randn(ctx, 2 * kw, generator=gen, device="cuda").to(st.dtype).float().cpu()
            ref.k[0][b] = list(rows[:, :kw].reshape(ctx, st.nG_l, st.head).unbind(0))
            ref.v[0][b] = list(rows[:, kw:].reshape(ctx, st.nG_l, st.head).unbind(0))
    ids = torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321), dtype=torch.int64)
    for t in range(steps):
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        torch.cuda.synchronize()
        glog = st.logits.float().cpu()
        rlog, rnext = ref.step(ids, [ctx + t] * B)
        mx = rlog.abs().max().item()
        tol = 1e-2 * mx + 2.0 ** (np.floor(np.log2(mx)) - 7)
        err = (glog - rlog).abs().max().item()
        assert err <= tol, (t, err, tol)
        assert torch.equal(nxt, torch.argmax(glog, dim=-1))
        top2 = torch.topk(rlog, 2, dim=-1).values
        for b in range(B):
            if (top2[b, 0] - top2[b, 1]).item() > 2 * tol:
                assert nxt[b].item() == rnext[b].item(), (t, b)
        ids = nxt
    assert st.lens_old.cpu().tolist() == [ctx + steps] * B


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tp_worker(rank, world, port, ret):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, "dash-infer_b200", "python"))
    import torch.distributed as dist
    from b200spark import model
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    B, steps = 3, 6
    cfg = _tiny(2)  # one kv head per rank
    st = model.DecodeStack(cfg, B, 64, wbits=4, group=-1, span=16, seed=7, tp_rank=rank, tp_size=world)
    one = model.DecodeStack(cfg, B, 64, wbits=4, group=-1, span=16, seed=7)
    st.capture()
    ids = torch.tensor([1, 2, 3], dtype=torch.int64, device="cuda")
    same = 0
    for _ in range(steps):
        st.ids.copy_(ids); one.ids.copy_(ids)
        a = st.step().clone(); nxt = one.step().clone()
        torch.cuda.synchronize()
        same += int(torch.equal(a, nxt))
        ids = nxt
    if st.comm is not None:
        st.comm.check_error()
    ret[rank] = same
    dist.barrier()
    os._exit(0)


def test_tp2_glm_emits_the_single_gpu_tokens():
    """TP = 2 (per-channel weights, one kv head per rank) emits the TP = 1 greedy tokens at every step"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    for r in range(2):
        assert ret[r] == 6, ret[r]
