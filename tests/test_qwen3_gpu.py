"""GPU: Qwen3-shaped decode stacks (per-head Q/K RMSNorm fused into the span-cache append, no QKV bias, n_heads * 128 !=
hidden) against the oracle with the norm (tests/qk_norm_ref.py: ref_from_stack), under the rules of test_model_gpu.py."""
import dataclasses
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import qk_norm_ref as R
from oracle import kvcache_ref as KV

pytestmark = pytest.mark.gpu


def _tiny():
    """8 q heads x 128 = 1024 against hidden 512: o_proj's K is not the hidden size"""
    from b200spark import model
    return model.ModelConfig("tiny-qwen3", 512, 8, 2, 1024, 2, 1024, qkv_bias=False, qk_norm=True)


KVM = {"none": KV.QUANT_NONE, "i8": KV.QUANT_I8, "u4": KV.QUANT_U4}


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


@pytest.mark.parametrize("wbits,group,kv", [(4, -1, "none"), (8, -1, "none"), (4, 128, "none"), (8, -1, "i8"), (4, -1, "u4")])
@pytest.mark.parametrize("B", [2, 20])
def test_tiny_qwen3_logits_and_tokens(wbits, group, kv, B):
    """eager for 3 steps, then a captured graph; B = 2 runs the self-contained GEMV norms, B = 20 the hand-off form"""
    from b200spark import model
    st = model.DecodeStack(_tiny(), B, 64, wbits=wbits, group=group, kv=kv, span=16, keep_ref=True)
    ref = R.ref_from_stack(st, KVM[kv])
    ids = (torch.arange(B, dtype=torch.int64) * 37 + 3) % 1024
    _run_against_oracle(st, ref, B, 6, ids, 4e-2 if kv == "u4" else 1e-2, capture_at=3)


@pytest.mark.parametrize("B", [2, 5, 20])
def test_tiny_qwen3_fp16(B):
    """fp16 at every norm placement (self at B <= 2, stand-alone at 5, hand-off at 20), eager then a captured graph"""
    from b200spark import model
    st = model.DecodeStack(_tiny(), B, 64, wbits=4, span=16, keep_ref=True, dtype=torch.float16)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    ids = (torch.arange(B, dtype=torch.int64) * 53 + 1) % 1024
    _run_against_oracle(st, ref, B, 5, ids, 1e-2, capture_at=3)


def test_launches_and_weights_equal_with_and_without_the_norm():
    """the norm rides in the append: same launches per step at every placement (self / stand-alone / hand-off), apart from
    the gammas the same weights, and the norm changes the result"""
    from b200spark import model
    cfg = _tiny()
    for B in (1, 5, 20):
        on = model.DecodeStack(cfg, B, 64, wbits=4, span=16, seed=9)
        off = model.DecodeStack(dataclasses.replace(cfg, qk_norm=False), B, 64, wbits=4, span=16, seed=9)
        for t in range(2):  # two different tokens: with one token, or one token twice, attention returns its V row
            for st in (on, off):
                st.ids.fill_(5 + 70 * t)
                st.step()
        torch.cuda.synchronize()
        assert on.launches_per_step == off.launches_per_step, B
        assert torch.equal(on.embed, off.embed) and torch.equal(on.layers[1]["g2"], off.layers[1]["g2"])
        assert not torch.equal(on.logits, off.logits)
    big = model.DecodeStack(model.QWEN3_8B, 1, 16, wbits=4, span=16, layers=1)
    big_off = model.DecodeStack(dataclasses.replace(model.QWEN3_8B, qk_norm=False), 1, 16, wbits=4, span=16, layers=1)
    big.step(); big_off.step()
    torch.cuda.synchronize()
    assert big.launches_per_step == big_off.launches_per_step
    print("Qwen3-8B (1 layer, batch 1) launches per step:", big.launches_per_step)


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
    single-token logits decide the tokens (top-2 margin above twice the logit difference), all T are accepted and the
    emitted tokens are the single steps' tokens"""
    from b200spark import model
    cfg, B, T, rounds = _tiny(), 2, 4, 3
    kw = dict(wbits=4, kv="none", span=16, seed=77)
    first = torch.tensor([3, 41], dtype=torch.int64)
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
def test_full_width_qwen3_8b_layer_and_lm_head(B):
    """one full-width Qwen3-8B layer (hidden 4096, 32/8 heads, inter 12288, int4 per-channel: qkv N = 6144, o K = 4096,
    gate/up 2 x 12288, down K = 12288) + final norm + the 151936-wide lm_head, three steps from an empty cache, against the
    oracle with the norm (the tolerance of test_full_width_qwen2_7b_layer_and_lm_head)"""
    from b200spark import model
    steps = 3
    st = model.DecodeStack(model.QWEN3_8B, B, 32, wbits=4, group=-1, kv="none", span=16, keep_ref=True, layers=1)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    ref.reset(B)
    ids = torch.randint(0, model.QWEN3_8B.vocab, (B,), generator=torch.Generator().manual_seed(4321), dtype=torch.int64)
    for t in range(steps):
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        torch.cuda.synchronize()
        glog = st.logits.float().cpu()
        rlog, rnext = ref.step(ids, [t] * B)
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


def test_qwen3_0p6b_bf16_decode_parity():
    """Qwen3-0.6B shapes (hidden 1024, 16 q heads / 8 kv heads of 128: o_proj K 2048, inter 3072, 28 layers), bf16 weights,
    batch 1, decoded to length 128, under the rule of test_config_c0_qwen2_0p5b_bf16_decode_parity: at most 1.5x as far from
    the exact graph as the rounded oracle (or 1e-2 of the range), and the exact path's token wherever its top-2 margin
    exceeds twice that bound"""
    from b200spark import model
    B, T = 1, 128
    st = model.DecodeStack(model.QWEN3_06B, B, T + 8, wbits=16, group=-1, kv="none", span=16, keep_ref=True)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    exact = R.ref_from_stack(st, KV.QUANT_NONE, exact=True)
    ref.reset(B); exact.reset(B)
    ids = torch.tensor([1234], dtype=torch.int64)
    worst_g = worst_r = 0.0
    for t in range(T):
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        rlog, _ = ref.step(ids, [t] * B)
        elog, enext = exact.step(ids, [t] * B)
        if t < 8 or t % 16 == 15 or t == T - 1:
            torch.cuda.synchronize()
            glog = st.logits.float().cpu()
            mx = elog.abs().max().item()
            eg, er = (glog - elog).abs().max().item(), (rlog - elog).abs().max().item()
            worst_g, worst_r = max(worst_g, eg / mx), max(worst_r, er / mx)
            bound = max(1.5 * er, 1e-2 * mx)
            assert eg <= bound, (t, eg, er, mx)
            top2 = torch.topk(elog, 2, dim=-1).values
            if (top2[0, 0] - top2[0, 1]).item() > 2 * bound:
                assert nxt[0].item() == enext[0].item(), t
        ids = enext
    assert st.lens_old.cpu().tolist() == [T]
    print("Qwen3-0.6B: worst |logit error| / range vs the exact graph: b200spark %.2e, rounded oracle %.2e" % (worst_g, worst_r))


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
    B, steps = 3, 5
    cfg = _tiny()
    st = model.DecodeStack(cfg, B, 64, wbits=4, span=16, seed=7, tp_rank=rank, tp_size=world)
    one = model.DecodeStack(cfg, B, 64, wbits=4, span=16, seed=7)
    st.capture()
    ids = torch.tensor([1, 2, 3], dtype=torch.int64, device="cuda")
    worst = 0.0
    for _ in range(steps):
        st.ids.copy_(ids); one.ids.copy_(ids)
        st.step(); nxt = one.step().clone()
        torch.cuda.synchronize()
        full = one.logits.float()
        worst = max(worst, ((st.logits.float() - full[:, rank * st.vocab_l:(rank + 1) * st.vocab_l]).abs().max()
                            / full.abs().max()).item())
        ids = nxt
    if st.comm is not None:
        st.comm.check_error()
    ret[rank] = worst
    dist.barrier()
    os._exit(0)


def test_tp2_qwen3_matches_single_gpu():
    """the gammas are replicated on every rank: a TP = 2 Qwen3 stack gives the single-GPU stack's logits (within bf16
    partial-sum rounding)"""
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
        assert ret[r] < 2e-2, ret[r]
