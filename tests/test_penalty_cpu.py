"""CPU: the restatement of b2_penalize and of the token history (tests/penalty_ref.py), the ctypes mirrors of the new
structs, and the argument checks of the entry points, without a GPU.

Each restated bug of penalty_ref.BUGS changes an output on the constructed cases, so the GPU comparison against the
restatement would catch it in the kernel."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import penalty_ref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B2_ERR_PARAM = 3


def cases():
    """(name, ft, x, tokens, lens, prompt_lens, params, id_offset) over small rows"""
    out = []
    n = 48
    base = np.array([((i * 7) % 23 - 11) * 0.375 for i in range(n)], np.float64)
    base[20] = 0.0
    base[21] = -0.0
    for ft in ("bf16", "fp16"):
        x = P.rn(np.stack([base, -base, base * 3.3, base + 0.7]), ft)
        # row 0: prompt [3 5 3 9], generated [9 3 6]; row 1: no prompt, generated with duplicates and -0 (id 21); row 2:
        # prompt only, with a 0 logit (id 20) under repetition 0; row 3: a repeating bigram and id 47 (the last column)
        hist = [[3, 5, 3, 9, 9, 3, 6], [7, 7, 21, 1, 6], [2, 4, 20, 5], [10, 11, 12, 10, 11, 47, 10]]
        prompt = [4, 0, 4, 2]
        tok = np.full((4, 8), -1, np.int64)
        for r, h in enumerate(hist):
            tok[r, :len(h)] = h
        lens = np.array([len(h) for h in hist])
        params = dict(repetition=[1.05, 2.0, 0.0, 1.3], presence=[0.5, -0.75, 2.0, 0.25], frequency=[0.25, 1.5, -2.0, 0.5],
                      no_repeat_ngram=[2, 1, 0, 2], min_length=[7, 6, 3, 8], eos_id=[40, 47, 0, 47], suppress=[1, 0, 0, 1])
        out.append(("mixed", ft, x, tok, lens, np.array(prompt), params, 0))
        shard = x[:, 4:40]  # vocab ids 4 .. 39 of the same rows
        out.append(("shard", ft, shard, tok, lens, np.array(prompt), params, 4))
        # the same with suppress cleared and min_length exactly L, L + 1
        p2 = dict(params, suppress=[0, 0, 0, 0], min_length=[8, 5, 5, 7])
        out.append(("nosup", ft, x, tok, lens, np.array(prompt), p2, 0))
        # n-gram of 3 with matches at the first and last admissible j: tokens a b c ... a b c ... a b
        tk = np.array([[1, 2, 3, 4, 1, 2, 30, 1, 2] + [-1] * 3], np.int64)
        p3 = dict(repetition=[1.0], presence=[0.0], frequency=[0.0], no_repeat_ngram=[3], min_length=[0], eos_id=[-1],
                  suppress=[0])
        out.append(("ngram3", ft, x[:1], tk, np.array([9]), np.array([2]), p3, 0))
    return out


def run(case, bugs=()):
    _, ft, x, tok, lens, prompt, params, off = case
    return P.penalize(x, tok, lens, prompt, params, ft, off, bugs)


def test_neutral_parameters_change_nothing():
    for name, ft, x, tok, lens, prompt, params, off in cases():
        out, alt = P.penalize(x, tok, lens, prompt, P.neutral(x.shape[0]), ft, off)
        assert np.all(P.same(out, x)), name


def test_ban_constants():
    assert P.bits(P.rn(P.BAN, "bf16"), "bf16") == 0xCE6E
    assert P.bits(P.rn(P.BAN, "fp16"), "fp16") == 0xFC00


def test_known_values():
    """a few entries by hand: bf16 row 0 of the mixed case"""
    case = cases()[0]
    x = case[2]
    out, _ = run(case)
    R = P.rn(1.05, "bf16")[()]                    # 1.046875
    assert R == 1.046875
    # id 3: prompt + one generated occurrence, suppress set: repetition (generated), then 1 * 0.25 + 0.5
    v = P.rn(x[0, 3] / R if x[0, 3] >= 0 else x[0, 3] * R, "bf16")[()]
    assert out[0, 3] == P.rn(v - P.rn(0.75, "bf16"), "bf16")[()]
    # id 5: prompt only, suppress set: no repetition, no penalty
    assert out[0, 5] == x[0, 5]
    # the last token 6 occurs nowhere before: no n-gram ban; min_length 7 == L: no ban of eos 40
    assert out[0, 40] == x[0, 40]
    # row 3 ends in 10, and 10 was followed by 11 twice: 11 is banned; L = 7 < min_length 8 bans eos 47
    assert out[3, 11] == out[3, 47] == P.rn(P.BAN, "bf16")
    assert out[3, 12] != P.rn(P.BAN, "bf16")


@pytest.mark.parametrize("bug", P.BUGS)
def test_each_bug_changes_an_output(bug):
    changed = 0
    for case in cases():
        out, alt = run(case)
        bad, _ = run(case, bugs=(bug,))
        changed += int(np.sum(~(P.same(bad, out) | P.same(bad, alt))))
    assert changed > 0, bug


def test_history_appends_equal_one_load():
    rng = np.random.default_rng(1)
    h1, h2 = P.History(3, 40, 100), P.History(3, 40, 100)
    seqs = [rng.integers(0, 100, 30) for _ in range(3)]
    for r in range(3):
        h1.load(r, seqs[r][:10])
        h2.load(r, seqs[r][:30], prompt_len=10)
    for j in range(10, 30):
        h1.append([s[j] for s in seqs])
    assert h1.tokens == h2.tokens and h1.prompt == h2.prompt
    assert all(h1.table(r) == h2.table(r) for r in range(3))
    # a reload leaves no trace; a full slot takes no more tokens; an id outside the vocabulary is -1 and counted nowhere
    h1.load(1, [5, 5], 1)
    assert h1.table(1) == {5: P.IN_PROMPT | 1} and h1.tokens[1] == [5, 5]
    h1.reset(2)
    assert h1.tokens[2] == [] and h1.table(2) == {}
    h1.load(0, list(range(40)))
    h1.append([7, 200, -3])
    assert len(h1.tokens[0]) == 40 and h1.tokens[1][-1] == -1 and h1.tokens[2] == [-1] and h1.table(2) == {}


def test_struct_layouts_match_the_header(tmp_path):
    from b200spark import _lib
    structs = {"b2_token_history": _lib.TokenHistory, "b2_penalty_params": _lib.PenaltyParams}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200spark.h"', 'int main(void) {']
    for cname, cls in structs.items():
        lines.append('  printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('  printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(out["%s.%s" % (cname, fname)]) == getattr(cls, fname).offset, (cname, fname)


def test_argument_checks_without_gpu():
    """every bad argument returns B2_ERR_PARAM before any launch (fake, never dereferenced pointers)"""
    from b200spark import _lib
    lib = _lib.lib
    p = 0x1000
    h = _lib.TokenHistory(p, p, p, p, p, p, 16, 100)
    prm = _lib.PenaltyParams(p, p, p, p, p, p, p, None)
    ok = lambda **kw: dict(dict(logits=p, rows=2, n=100, ld=100, off=0, h=h, prm=prm, ft=_lib.DT_BF16), **kw)
    call = lambda a: lib.b2_penalize(a["logits"], a["rows"], a["n"], a["ld"], a["off"], C.byref(a["h"]), C.byref(a["prm"]),
                                     a["ft"], None)
    for bad in (dict(logits=None), dict(rows=-1), dict(n=0), dict(ld=99), dict(off=-1), dict(off=1), dict(ft=_lib.DT_F32),
                dict(h=_lib.TokenHistory(p, p, p, None, p, p, 16, 100)), dict(h=_lib.TokenHistory(p, p, p, p, p, p, 0, 100)),
                dict(h=_lib.TokenHistory(p, p, p, p, p, p, 1 << 30, 100)),
                dict(prm=_lib.PenaltyParams(p, p, p, p, p, None, p, None))):
        assert call(ok(**bad)) == B2_ERR_PARAM, bad
    assert call(ok(rows=0)) == 0  # nothing to do, nothing launched
    assert lib.b2_history_load(C.byref(h), 0, p, 17, 0, None) == B2_ERR_PARAM      # more than max_len
    assert lib.b2_history_load(C.byref(h), 0, p, 4, 5, None) == B2_ERR_PARAM       # prompt longer than the ids
    assert lib.b2_history_load(C.byref(h), -1, p, 4, 4, None) == B2_ERR_PARAM
    assert lib.b2_history_load(C.byref(h), 0, None, 4, 4, None) == B2_ERR_PARAM
    assert lib.b2_history_append(C.byref(h), None, 2, None) == B2_ERR_PARAM
    assert lib.b2_history_append(C.byref(h), p, -1, None) == B2_ERR_PARAM
    assert lib.b2_history_append(C.byref(h), p, 0, None) == 0


def test_parameter_ranges_are_checked_on_the_host():
    from b200spark import ops
    pen = ops.Penalties(2, device="cpu")
    pen.set(repetition=[1.05, 2.0], presence=-2.0, frequency=2.0, no_repeat_ngram=3, min_length=[0, 5], eos_id=[151643, -1],
            suppress_repetition_in_generation=1)
    assert pen.repetition.tolist() == [np.float32(1.05), 2.0] and pen.no_repeat_ngram.tolist() == [3, 3]
    assert pen.eos_id.tolist() == [151643, -1] and pen.suppress.tolist() == [1, 1]
    for bad in (dict(repetition=2.5), dict(repetition=-0.1), dict(repetition=float("nan")), dict(presence=2.01),
                dict(frequency=-3.0), dict(no_repeat_ngram=-1), dict(min_length=1.5), dict(no_repeat_ngram=[1, -2])):
        with pytest.raises(ValueError):
            pen.set(**bad)
    assert pen.repetition.tolist() == [np.float32(1.05), 2.0]  # a refused call writes nothing of that parameter


def test_history_front_end_checks():
    from b200spark import ops
    h = ops.TokenHistory(2, 8, 50, device="cpu")
    for args in ((0, list(range(9))), (0, [1, 2, 50]), (0, [-1]), (2, [1]), (0, [1, 2], 3)):
        with pytest.raises(AssertionError):
            h.load(*args)
    v = h.view(1)
    assert v.rows == 1 and v.table.shape == (1, 50) and v.table.data_ptr() == h.table.data_ptr()
