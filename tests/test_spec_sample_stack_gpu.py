"""GPU: DecodeStack(q_len=T, sampled_verify=True) on model.TINY, chains and trees.

Every verify step's draws equal b2_sample on that step's own logits rows at offsets_before[b] + depth(t); the accepted
counts, paths, lengths and offsets follow the CPU walk; at temperature 0 the stack equals a greedy q_len = T twin; graph
replay equals eager steps; with logprobs the reported logprobs are those of the drawn tokens.  (Stream equality against
a single-token stack is a kernel-level test: verify rows pass the GEMMs at M = B*T, so their logits differ by rounding.)"""
import numpy as np
import pytest
import torch

import spec_sample_ref as SS

pytestmark = pytest.mark.gpu

B, T = 3, 6
PAR = [0, 0, 1, 0, 3, 4]  # two branches below the root


def _stack(sv=True, tree=False, dtype=torch.bfloat16, wbits=4, kv="none", logprobs=0):
    from b200spark import model
    st = model.DecodeStack(model.TINY, B, 64, wbits=wbits, kv=kv, span=16, seed=11, q_len=T, tree=tree, dtype=dtype,
                           sampled_verify=sv, logprobs=logprobs)
    if tree:
        st.parents.copy_(torch.tensor([PAR] * B, dtype=torch.int32))
    st.tokens[:, 0] = torch.arange(B, dtype=torch.int64, device="cuda") * 5 + 1
    return st


def _drafts(i, prev):
    """drafts of step i: the previous step's draws of nodes 1.. (often right for a peaked continuation), else fixed ids"""
    rng = np.random.default_rng(i)
    d = rng.integers(0, 200, (B, T - 1))
    if prev is not None and i % 2:
        d[:] = prev[:, 1:]
    return torch.from_numpy(d).cuda()


def _run(st, steps, graph=False, check=None):
    outs, prev = [], None
    for i in range(steps):
        st.tokens[:, 1:] = _drafts(i, prev)
        if graph and st.graph is None:
            st.capture()
        tk, off, lo = st.tokens.clone(), st.offsets.clone() if st.sv else None, st.lens_old.clone()
        res = st.step()
        torch.cuda.synchronize()
        if check is not None:
            check(st, res, tk, off, lo)
        prev = res[0].cpu().numpy()
        outs.append([r.clone() for r in res] + [st.logits.clone()] + ([st.offsets.clone()] if st.sv else []))
    return outs


def _check_step(st, res, tk, off, lo):
    """the draws equal b2_sample on the step's own rows; the walk, the lengths and the offsets follow the restatement"""
    from b200spark import ops
    pred, acc = res[0].cpu().numpy(), res[1].cpu().numpy()
    par = np.asarray([PAR] * B) if st.tree else None
    ctr = SS.counters(off.cpu().numpy().view(np.uint64), par, B, T).reshape(-1)
    idx = torch.arange(B, device="cuda").repeat_interleave(T)
    want = ops.sample(st.logits, st.temperature[idx].contiguous(), st.top_k[idx].contiguous(), st.top_p[idx].contiguous(),
                      st.seeds[idx].contiguous(), torch.from_numpy(ctr.view(np.int64).copy()).cuda())
    assert np.array_equal(pred.reshape(-1), want.cpu().numpy())
    n, paths, nxt = SS.accept(tk.cpu().numpy(), pred, par)
    assert np.array_equal(acc, n) and np.array_equal(st.tokens[:, 0].cpu().numpy(), nxt)
    if st.tree:
        path = res[2].cpu().numpy()
        assert all(list(path[b, :n[b]]) == paths[b] for b in range(B))
    assert np.array_equal(st.lens_old.cpu().numpy(), lo.cpu().numpy() + n)
    assert np.array_equal(st.lens_new.cpu().numpy(), lo.cpu().numpy() + n + T)
    assert np.array_equal(st.offsets.cpu().numpy().view(np.uint64), SS.advance(off.cpu().numpy().view(np.uint64), n, T))


MODES = [(torch.bfloat16, 4, "none"), (torch.bfloat16, 8, "i8"), (torch.bfloat16, 4, "u4"), (torch.float16, 4, "fp8"),
         (torch.float16, 4, "none")]


@pytest.mark.parametrize("dtype,wbits,kv", MODES)
@pytest.mark.parametrize("tree", [False, True])
def test_steps_follow_the_kernels(dtype, wbits, kv, tree):
    st = _stack(tree=tree, dtype=dtype, wbits=wbits, kv=kv)
    st.set_sampling(temperature=[0.7, 1.0, 0.0], top_k=[50, 0, 0], top_p=[0.9, 1.0, 1.0], seeds=[3, 1 << 40, 7],
                    offsets=[0, 2 ** 32 - 2, 100])
    _run(st, 8, check=_check_step)
    assert st.lens_old.min().item() >= 8


@pytest.mark.parametrize("tree", [False, True])
def test_temperature_zero_equals_greedy_twin(tree):
    """t = 0 everywhere: pred, accepted, path and logits equal a greedy q_len = T stack bit for bit, same launch count"""
    st, twin = _stack(tree=tree), _stack(sv=False, tree=tree)
    st.set_sampling(temperature=0.0, offsets=5)
    a, b = _run(st, 6), _run(twin, 6)
    for x, y in zip(a, b):
        for u, v in zip(x, y):  # the sampled stack's extra entry (offsets) is left over by zip
            assert torch.equal(u, v)
    assert st.launches_per_step == twin.launches_per_step > 0
    assert st.offsets.cpu().tolist() == (5 + st.lens_old.cpu()).tolist()


@pytest.mark.parametrize("tree", [False, True])
def test_graph_replay_equals_eager(tree):
    outs = []
    for graph in (False, True):
        st = _stack(tree=tree)
        st.set_sampling(temperature=[0.8, 1.2, 0.6], top_k=[0, 40, 5], top_p=[0.95, 1.0, 0.8], seeds=[11, 12, 13], offsets=1)
        outs.append(_run(st, 6, graph=graph))
    for x, y in zip(*outs):
        for u, v in zip(x, y):
            assert torch.equal(u, v)


@pytest.mark.parametrize("tree", [False, True])
def test_logprobs_of_the_draws(tree):
    """logprobs=4: tok_lp and the top lists equal ops.logprobs(st.logits, 4, tok_ids=pred) bit for bit; one launch more
    than the greedy verify step"""
    from b200spark import ops
    st = _stack(tree=tree, logprobs=4)
    st.set_sampling(temperature=1.0, top_p=0.95, seeds=[1, 2, 3])

    def check(st, res, tk, off, lo):
        _, tlp, tids, tlps = ops.logprobs(st.logits, 4, tok_ids=res[0].reshape(-1).contiguous())
        torch.cuda.synchronize()
        assert torch.equal(st.tok_lp.view(torch.int32), tlp.view(torch.int32))
        assert torch.equal(st.top_ids, tids) and torch.equal(st.top_lp.view(torch.int32), tlps.view(torch.int32))

    _run(st, 3, check=check)
    greedy = _stack(sv=False, tree=tree)
    _run(greedy, 1)
    assert st.launches_per_step == greedy.launches_per_step + 1
