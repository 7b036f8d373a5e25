"""GPU: DecodeStack(q_len=T, ngram=...) against a twin on the same weights, caches and seeds without `ngram`, into which the
test writes the restatement's drafts (tests/ngram_ref.py) computed from a host copy of the history.  Chains and trees,
greedy and sampled verification, bf16 and fp16: every output of every step is bit-identical, so the drafter is the only
difference.  Graph replay equals eager steps, capture() keeps the history, set_batch works, and a stack without `ngram`
runs the launches it ran before."""
import numpy as np
import pytest
import torch

import ngram_ref as N
import penalty_ref as P

pytestmark = pytest.mark.gpu

B, MAX_LEN, VOCAB = 4, 160, 1024


def _stack(T, tree, sv, dtype, ngram):
    from b200spark import model
    return model.DecodeStack(model.TINY, B, MAX_LEN, wbits=4, span=16, seed=11, q_len=T, tree=tree, sampled_verify=sv,
                             dtype=dtype, ngram=ngram)


def _prompts():
    """sequences 0 and 1 repeat a random segment (long n-gram matches), 2 is random, 3 is one token"""
    rng = np.random.default_rng(23)
    seg = rng.integers(0, VOCAB, 7).tolist()
    return [seg * 4, rng.integers(0, VOCAB, 3).tolist() + seg * 3, rng.integers(0, VOCAB, 30).tolist(), [17]]


def _setup(st, tw, sv, ref):
    for b, ids in enumerate(_prompts()):
        st.set_history(b, ids)
        ref.load(b, ids)
        tw.tokens[b, 0] = ids[-1]
    if sv:
        for s in (st, tw):
            s.set_sampling(temperature=0.8, top_k=40, top_p=0.9, seeds=torch.arange(B) * 1000 + 3, offsets=5)


def _outputs(s, tree):
    out = [s.pred, s.accepted, s.next_ids, s.tokens, s.lens_old, s.lens_new, s.logits.view(torch.int16)]
    if tree:
        out += [s.path, s.parents]
    if s.sv:
        out.append(s.offsets)
    return [t.clone() for t in out]


def _run_twins(T, tree, sv, dtype, width, steps=6):
    ngram = (1, 3, width)
    st, tw = _stack(T, tree, sv, dtype, ngram), _stack(T, tree, sv, dtype, None)
    ref = P.History(B, MAX_LEN, VOCAB)
    _setup(st, tw, sv, ref)
    for step in range(steps):
        toks, pars, nd = N.draft_batch(ref.tokens, tw.tokens[:, 0].tolist(), T, 1, 3, width, tree)
        tw.tokens.copy_(torch.tensor(toks))
        if tree:
            tw.parents.copy_(torch.tensor(pars, dtype=torch.int32))
        st.step()
        tw.step()
        torch.cuda.synchronize()
        assert st.n_draft.tolist() == nd, step
        for i, (x, y) in enumerate(zip(_outputs(st, tree), _outputs(tw, tree))):
            assert torch.equal(x, y), (T, tree, sv, dtype, step, i)
        N.append_tokens(ref, tw.pred.tolist(), tw.accepted.tolist(), tw.path.tolist() if tree else None)
    h = st.history
    assert h.len.tolist() == [len(t) for t in ref.tokens]
    assert [h.tokens[b, :len(ref.tokens[b])].tolist() for b in range(B)] == ref.tokens
    assert st.launches_per_step == tw.launches_per_step + 2


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("sv", [False, True])
@pytest.mark.parametrize("form", [(4, False, 1), (8, False, 1), (8, True, 1), (8, True, 3), (16, True, 5)])
def test_stack_equals_twin_with_host_drafts(form, sv, dtype):
    T, tree, width = form
    _run_twins(T, tree, sv, dtype, width)


def test_without_ngram_launches_are_unchanged():
    """a stack without ngram runs the launches it ran before: TINY, R = 16 rows, standalone norms"""
    for tree, n in ((False, 21), (True, 22)):
        st = _stack(4, tree, False, torch.bfloat16, None)
        st.step()
        assert st.launches_per_step == n, tree


@pytest.mark.parametrize("tree", [False, True])
def test_graph_replay_equals_eager(tree):
    width = 3 if tree else 1
    ngram = (1, 3, width)
    eager, graph = _stack(8, tree, False, torch.bfloat16, ngram), _stack(8, tree, False, torch.bfloat16, ngram)
    for s in (eager, graph):
        for b, ids in enumerate(_prompts()):
            s.set_history(b, ids)
    torch.cuda.synchronize()
    before = [t.clone() for t in graph.history.snapshot()]
    graph.capture()
    assert all(torch.equal(x, y) for x, y in zip(before, graph.history.snapshot())), "capture() changed the history"
    for step in range(6):  # each replay drafts from the history the previous replay extended
        eager.step()
        graph.step()
        torch.cuda.synchronize()
        for i, (x, y) in enumerate(zip(_outputs(eager, tree), _outputs(graph, tree))):
            assert torch.equal(x, y), (tree, step, i)
        assert torch.equal(eager.n_draft, graph.n_draft)
    assert all(torch.equal(x, y) for x, y in zip(eager.history.snapshot(), graph.history.snapshot()))


def test_set_batch():
    """set_batch(2): drafts and appends for the first two sequences only, eager and replayed"""
    st, tw = _stack(8, True, False, torch.bfloat16, (1, 3, 2)), _stack(8, True, False, torch.bfloat16, None)
    ref = P.History(B, MAX_LEN, VOCAB)
    _setup(st, tw, False, ref)
    st.set_batch(2)
    tw.set_batch(2)
    assert st.history.rows == 2 and st.n_draft.numel() == 2
    for graph in (False, True):
        if graph:
            st.capture()
            tw.capture()
        for _ in range(2):
            toks, pars, nd = N.draft_batch(ref.tokens[:2], tw.tokens[:, 0].tolist(), 8, 1, 3, 2, True)
            tw.tokens.copy_(torch.tensor(toks))
            tw.parents.copy_(torch.tensor(pars, dtype=torch.int32))
            st.step()
            tw.step()
            torch.cuda.synchronize()
            assert st.n_draft.tolist() == nd
            for i, (x, y) in enumerate(zip(_outputs(st, True), _outputs(tw, True))):
                assert torch.equal(x, y), (graph, i)
            N.append_tokens(ref, tw.pred.tolist(), tw.accepted.tolist(), tw.path.tolist())
    lens = [len(t) for t in _prompts()]
    assert st._history.len.tolist()[2:] == lens[2:]
    assert st._history.len.tolist()[:2] == [len(t) for t in ref.tokens[:2]]
