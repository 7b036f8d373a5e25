"""GPU: decode stacks with a rope_scaling entry (one static frequency table on the device, passed to every layer's append)
against the oracle that rotates with that table in fp64 (tests/rope_scaling_ref.py: ref_from_stack), under the rules of
test_qwen3_gpu.py: a tiny YaRN stack (a native context of 8, so nearly every frequency is scaled) in five weight / KV modes,
fp16, with the Q/K norm, CUDA-graph replay and chain / tree verify steps, and farther from the unscaled oracle than from
the table oracle; a Qwen2.5-7B layer decoding past 32768 tokens; a Llama-3.1-8B layer; the same launches per step with and
without scaling."""
import dataclasses

import numpy as np
import pytest
import torch

import qk_norm_ref as QR
import rope_scaling_ref as R
from oracle import kvcache_ref as KV

pytestmark = pytest.mark.gpu

# YaRN over a native context of 8: the correction dims clamp to 0 .. 2, so all but the first two frequencies are divided by
# the factor and the tiny stack's rotary differs from the unscaled one at every position (the scaling is static: the table
# does not depend on the position)
YARN8 = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 8}
KVM = {"none": KV.QUANT_NONE, "i8": KV.QUANT_I8, "u4": KV.QUANT_U4}


def _tiny(**kw):
    from b200spark import model
    return model.ModelConfig("tiny-yarn", 512, 8, 2, 1024, 2, 1024, rope_scaling=YARN8, **kw)


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
def test_tiny_yarn_logits_and_tokens(wbits, group, kv):
    """12 steps, eager then a captured graph"""
    from b200spark import model
    B = 3
    st = model.DecodeStack(_tiny(), B, 64, wbits=wbits, group=group, kv=kv, span=16, keep_ref=True)
    ref = R.ref_from_stack(st, KVM[kv])
    ids = (torch.arange(B, dtype=torch.int64) * 37 + 3) % 1024
    _run_against_oracle(st, ref, B, 12, ids, 4e-2 if kv == "u4" else 1e-2, capture_at=6)


@pytest.mark.parametrize("qk_norm", [False, True])
def test_tiny_yarn_fp16_and_qk_norm(qk_norm):
    from b200spark import model
    B = 2
    st = model.DecodeStack(_tiny(qkv_bias=not qk_norm, qk_norm=qk_norm), B, 64, wbits=4, span=16, keep_ref=True,
                           dtype=torch.float16)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    ids = (torch.arange(B, dtype=torch.int64) * 53 + 1) % 1024
    _run_against_oracle(st, ref, B, 10, ids, 1e-2, capture_at=5)


def test_oracle_without_the_table_is_farther():
    """the oracle that ignores rope_scaling (the base frequencies) is at least twice as far from the scaled stack as the
    oracle with the table, over 12 steps: the agreement above comes from the table, not from a tolerance that would accept
    the unscaled rotary too"""
    from b200spark import model
    B = 3
    st = model.DecodeStack(_tiny(), B, 64, wbits=8, group=-1, kv="none", span=16, keep_ref=True)
    ref = R.ref_from_stack(st, KV.QUANT_NONE)
    plain = QR.ref_from_stack(st, KV.QUANT_NONE)  # rotates with cfg.rope_base, as if rope_scaling were None
    ref.reset(B); plain.reset(B)
    ids = (torch.arange(B, dtype=torch.int64) * 37 + 3) % 1024
    e_ref = e_plain = 0.0
    for t in range(12):
        st.ids.copy_(ids.cuda())
        nxt = st.step().cpu()
        torch.cuda.synchronize()
        glog = st.logits.float().cpu()
        rlog, _ = ref.step(ids, [t] * B)
        plog, _ = plain.step(ids, [t] * B)
        mx = rlog.abs().max().item()
        e_ref = max(e_ref, (glog - rlog).abs().max().item() / mx)
        e_plain = max(e_plain, (glog - plog).abs().max().item() / mx)
        ids = nxt
    print("tiny YaRN stack: worst |logit error| / range against the table oracle %.2e, against the unscaled one %.2e"
          % (e_ref, e_plain))
    assert e_ref <= 1e-2 and e_plain >= 2 * e_ref, (e_ref, e_plain)


def test_scaling_changes_the_result_but_not_the_launches():
    """the same weights, different logits and the same launches per step with and without scaling (the table rides in the
    append)"""
    from b200spark import model
    cfg = _tiny()
    for B in (1, 5, 20):
        on = model.DecodeStack(cfg, B, 64, wbits=4, span=16, seed=9)
        off = model.DecodeStack(dataclasses.replace(cfg, rope_scaling=None), B, 64, wbits=4, span=16, seed=9)
        for t in range(12):
            for st in (on, off):
                st.ids.fill_(5 + 70 * t)
                st.step()
        torch.cuda.synchronize()
        assert on.launches_per_step == off.launches_per_step, B
        assert torch.equal(on.embed, off.embed)
        assert not torch.equal(on.logits, off.logits)
    for cfg in (model.QWEN25_7B, model.LLAMA31_8B):
        big = model.DecodeStack(cfg, 1, 16, wbits=4, span=16, layers=1)
        big_off = model.DecodeStack(dataclasses.replace(cfg, rope_scaling=None), 1, 16, wbits=4, span=16, layers=1)
        big.step(); big_off.step()
        torch.cuda.synchronize()
        assert big.launches_per_step == big_off.launches_per_step
        print("%s (1 layer, batch 1) launches per step: %d" % (cfg.name, big.launches_per_step))


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
    """chain and tree verify steps of T = 4 over the scaled rotary: where the single-token logits decide the tokens, all T
    drafts of the model's own continuation are accepted and the emitted tokens are the single steps' tokens"""
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


def _full_width_layer(cfg, B, ctx, steps):
    """one full-width layer + final norm + lm_head, int4 per-channel, from a cache of ctx tokens (the prefill writer's
    N(0,1) rows, mirrored into the oracle), `steps` steps against the oracle with the table"""
    from b200spark import model
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


def test_qwen25_7b_layer_past_the_native_context():
    """a Qwen2.5-7B layer (YaRN x4 over 32768) at batch 1 decoding positions 32800 .. 32802"""
    from b200spark import model
    _full_width_layer(model.QWEN25_7B, 1, 32800, 3)


@pytest.mark.parametrize("B", [1, 64])
def test_llama31_8b_layer(B):
    """a Llama-3.1-8B layer (llama3 scaling, factor 8 over 8192) from an empty cache and past 8192 tokens"""
    from b200spark import model
    _full_width_layer(model.LLAMA31_8B, B, 0 if B == 64 else 8300, 3)
