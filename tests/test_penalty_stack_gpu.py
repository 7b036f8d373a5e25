"""GPU: DecodeStack(penalties=True).  The processed logits of every step equal the restatement (tests/penalty_ref.py)
applied to the raw logits of an identical stack without penalties, and the emitted ids follow the processed row (argmax,
b2_sample); neutral parameters change nothing; graph replay equals eager steps; capture() and set_batch keep the history
right."""
import numpy as np
import pytest
import torch

import penalty_ref as P

pytestmark = pytest.mark.gpu

B, MAX_LEN = 4, 64


def _stack(penalties, sample=False, logprobs=0):
    from b200spark import model
    return model.DecodeStack(model.TINY, B, MAX_LEN, wbits=4, span=16, seed=11, sample=sample, logprobs=logprobs,
                             penalties=penalties)


def _prompts():
    rng = np.random.default_rng(17)
    return [rng.integers(0, 1024, 10) for _ in range(B)], [10, 6, 10, 0]


def _load(st, ref=None):
    prompts, plens = _prompts()
    for b in range(B):
        st.set_history(b, prompts[b], plens[b])
        if ref is not None:
            ref.load(b, prompts[b], plens[b])


REAL = dict(repetition=[1.3, 1.05, 2.0, 0.5], presence=[0.5, -0.5, 2.0, 0.0], frequency=[0.4, 1.0, -2.0, 0.25],
            no_repeat_ngram=[2, 0, 1, 3], min_length=[13, 0, 11, 14], eos_id=[5, -1, 17, 1023],
            suppress_repetition_in_generation=[0, 1, 0, 1])


def _ref_params(rows):
    return dict(repetition=REAL["repetition"][:rows], presence=REAL["presence"][:rows], frequency=REAL["frequency"][:rows],
                no_repeat_ngram=REAL["no_repeat_ngram"][:rows], min_length=REAL["min_length"][:rows],
                eos_id=REAL["eos_id"][:rows], suppress=REAL["suppress_repetition_in_generation"][:rows])


def _ids0(rows=B):
    return torch.arange(rows, dtype=torch.int64, device="cuda") * 7 + 1


def test_neutral_parameters_change_nothing():
    """greedy, sampled and logprobs steps: ids, logits and logprobs equal penalties=False bit for bit, two launches more"""
    for kw in (dict(), dict(sample=True), dict(logprobs=3), dict(sample=True, logprobs=2)):
        st, base = _stack(True, **kw), _stack(False, **kw)
        _load(st)
        if kw.get("sample"):
            for s in (st, base):
                s.set_sampling(temperature=0.9, top_k=40, top_p=0.95, seeds=torch.arange(B) * 7 + 1, offsets=0)
        st.ids.copy_(_ids0())
        base.ids.copy_(_ids0())
        for _ in range(6):
            a, b = st.step().clone(), base.step().clone()
            torch.cuda.synchronize()
            assert torch.equal(a, b), kw
            assert torch.equal(st.logits.view(torch.int16), base.logits.view(torch.int16)), kw
            if kw.get("logprobs"):
                assert torch.equal(st.tok_lp.view(torch.int32), base.tok_lp.view(torch.int32))
                assert torch.equal(st.top_ids, base.top_ids)
            st.ids.copy_(a)
            base.ids.copy_(b)
        assert st.launches_per_step == base.launches_per_step + 2, kw
        assert st.history.len.tolist() == [16, 16, 16, 16]


def _run_checked(sample):
    from b200spark import ops
    st, raw = _stack(True, sample=sample), _stack(False, sample=sample)
    ref = P.History(B, MAX_LEN, 1024)
    _load(st, ref)
    st.set_penalties(**REAL)
    if sample:
        st.set_sampling(temperature=0.8, top_k=50, top_p=0.9, seeds=torch.arange(B) * 1000 + 3, offsets=0)
    st.ids.copy_(_ids0())
    raw.ids.copy_(_ids0())
    seq = []
    for step in range(8):
        before = st.offsets.clone() if sample else None
        ids = st.step().clone()
        raw.step()
        torch.cuda.synchronize()
        tok, lens, plens = ref.arrays()
        x = raw.logits.double().cpu().numpy()
        want, alt = P.penalize(x, tok, lens, plens, _ref_params(B), "bf16")
        got = st.logits.double().cpu().numpy()
        assert np.all(P.same(got, want) | P.same(got, alt)), step
        if sample:  # b2_sample on the processed row, with the step's draw counters
            assert torch.equal(ids, ops.sample(st.logits, st.temperature, st.top_k, st.top_p, st.seeds, before))
        else:
            assert torch.equal(ids, torch.argmax(st.logits.float(), dim=1))
        ref.append(ids.tolist())
        seq.append(ids)
        st.ids.copy_(ids)
        raw.ids.copy_(ids)
    h = st.history
    assert h.len.tolist() == [len(t) for t in ref.tokens]
    assert [h.tokens[b, :len(ref.tokens[b])].tolist() for b in range(B)] == ref.tokens
    return torch.stack(seq)


def test_real_parameters_greedy():
    seq = _run_checked(sample=False)
    assert seq.shape == (8, B)


def test_real_parameters_sampled():
    _run_checked(sample=True)


def _state(h):
    return [t.clone() for t in h.snapshot()]


def _equal_states(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_graph_replay_equals_eager_and_capture_keeps_the_history():
    eager, graph = _stack(True), _stack(True)
    for st in (eager, graph):
        _load(st)
        st.set_penalties(**REAL)
        st.ids.copy_(_ids0())
    torch.cuda.synchronize()
    before = _state(graph.history)
    graph.capture()
    assert _equal_states(before, graph.history.snapshot())
    for step in range(8):
        a, b = eager.step().clone(), graph.step().clone()
        torch.cuda.synchronize()
        assert torch.equal(a, b), step
        assert torch.equal(eager.logits.view(torch.int16), graph.logits.view(torch.int16)), step
        eager.ids.copy_(a)
        graph.ids.copy_(b)
    assert _equal_states(eager.history.snapshot(), graph.history.snapshot())
    # the parameters are read at every replay
    for st in (eager, graph):
        st.set_penalties(repetition=2.0, no_repeat_ngram=1)
    a, b = eager.step().clone(), graph.step().clone()
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(eager.logits.view(torch.int16), graph.logits.view(torch.int16))


def test_set_batch():
    """set_batch(2): the step processes and appends for the first two sequences only"""
    st, raw = _stack(True), _stack(False)
    ref = P.History(B, MAX_LEN, 1024)
    _load(st, ref)
    st.set_penalties(**REAL)
    st.set_batch(2)
    raw.set_batch(2)
    assert st.history.rows == 2 and st.penalties.repetition.numel() == 2
    st.ids.copy_(_ids0(2))
    raw.ids.copy_(_ids0(2))
    for graph in (False, True):
        if graph:
            st.capture()
            raw.capture()
        ids = st.step().clone()
        raw.step()
        torch.cuda.synchronize()
        tok, lens, plens = ref.arrays()
        want, alt = P.penalize(raw.logits.double().cpu().numpy(), tok[:2], lens[:2], plens[:2], _ref_params(2), "bf16")
        got = st.logits.double().cpu().numpy()
        assert np.all(P.same(got, want) | P.same(got, alt))
        ref.append(ids.tolist())
        st.ids.copy_(ids)
        raw.ids.copy_(ids)
    assert st._history.len.tolist() == [12, 12, 10, 10]


def test_multi_token_steps_are_refused():
    from b200spark import model
    with pytest.raises(AssertionError, match="penalties"):
        model.DecodeStack(model.TINY, 2, 64, wbits=4, span=16, q_len=4, penalties=True)
