"""CPU: the per-head Q/K RMSNorm restatement (tests/qk_norm_ref.py) on hand-computed rows, the sharpness of its bounds
against restated bugs, the C-ABI struct mirror and the argument checks that return before touching a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import glue_ref as G
import qk_norm_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_restatement_on_hand_computed_rows(dt):
    dt = G.FTS[dt]
    one = np.ones(128, np.float32)
    x = np.stack([one, 2 * one, np.where(np.arange(128) == 5, 8.0, 0.0).astype(np.float32)])
    y = R.head_norm(x, one, 1e-6, dt)
    assert np.all(y[0] == 1.0) and np.all(y[1] == 1.0)  # rs = 1 / sqrt(1 + 1e-6), 1 / sqrt(4 + 1e-6): both round to 1
    # one 8 among zeros: mean 0.5, y = 8 sqrt(2) = 11.3137..., nearest bf16 and fp16 value 11.3125
    assert y[2, 5] == 11.3125 and np.count_nonzero(y[2]) == 1
    g = np.full(128, 0.75, np.float32)
    assert np.all(R.head_norm(x[1:2], g, 1e-6, dt) == 0.75)
    # the restatement is one of its own candidates
    xe, ge = R.exact_batch(64, dt, np.random.default_rng(0))
    assert len(R.exact_rows_failing(R.head_norm(xe, ge, 1e-6, dt), xe, ge, 1e-6, dt)) == 0


def _composed(x, pos, nH, nG, qg, kg, eps, dt, bug=None):
    """norm then rotary on the q and k heads (the fused append's value), and the rotary contract against the restated norm"""
    rows = x.shape[0]
    heads = nH + nG
    n = R.qk_rows(x, nH, nG, qg, kg, eps, dt).reshape(rows, -1, 128)[:, :heads]
    p = np.repeat(pos, heads)
    Y, D = R.rope_after(n.reshape(-1, 128), p, 1e6, 128)
    if bug == "after_rotary":
        r = G.rope_kernel32(x.reshape(rows, -1, 128)[:, :heads].reshape(-1, 128), p, 1e6, 128, dt).reshape(rows, -1)
        r = np.concatenate([r, x[:, heads * 128:]], 1)
        y = R.qk_rows(r, nH, nG, qg, kg, eps, dt).reshape(rows, -1, 128)[:, :heads].reshape(-1, 128)
    else:
        src = n if bug is None else R.qk_rows(x, nH, nG, qg, kg, eps, dt, rounded=False).reshape(rows, -1, 128)[:, :heads]
        y = G.rope_kernel32(src.reshape(-1, 128).astype(np.float32), p, 1e6, 128, dt)
    return float(G.rope_ratio(y, Y, D, dt).max())


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_bounds_are_sharp(dt):
    """the correct restatement stays inside each bound; every restated bug misses one by >= 4 bounds on some case"""
    dt = G.FTS[dt]
    rng = np.random.default_rng(1)
    nH, nG, eps = 4, 2, 1e-6
    qg, kg = R.gammas(dt, rng)
    cases = [R.realistic_rows(16, (nH + 2 * nG) * 128, dt, rng, kind, s) for kind in R.ROW_KINDS for s in (-12, 0, 6)]
    pos = rng.integers(1, 2048, 16)
    worst = {}
    for bug in [None] + R.BUGS:
        if bug in ("after_rotary", "no_round"):
            worst[bug] = max(_composed(x, pos, nH, nG, qg, kg, eps, dt, bug) for x in cases)
        else:
            worst[bug] = max(float(R.ratio(R.qk_rows(x, nH, nG, qg, kg, eps, dt, bug), R.exact(x, nH, nG, qg, kg, eps), dt).max())
                             for x in cases)
    worst["composed"] = max(_composed(x, pos, nH, nG, qg, kg, eps, dt) for x in cases)
    assert worst[None] <= 1.0 and worst["composed"] <= 1.0, worst
    for bug in R.BUGS:
        assert worst[bug] >= 4.0, (bug, worst[bug])


def test_qk_norm_struct_matches_the_header(tmp_path):
    from b200spark import _lib
    fields = [f for f, _ in _lib.QkNorm._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200spark.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(b2_qk_norm));']
    lines += ['  printf("%s %%zu\\n", offsetof(b2_qk_norm, %s));' % (f, f) for f in fields]
    lines += ['  return 0;', '}']
    src, exe = tmp_path / "qk.c", tmp_path / "qk"
    src.write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(_lib.QkNorm)
    for f in fields:
        assert int(out[f]) == getattr(_lib.QkNorm, f).offset, f


def test_argument_checks_without_gpu():
    """checks that return before any device access (fake, never dereferenced addresses)"""
    from b200spark import _lib
    lib = _lib.lib
    buf, g = C.c_void_p(0x10000), C.c_void_p(0x20000)
    nrm = _lib.QkNorm(g.value, g.value, 1e-6, 0)
    W = (4 + 2 * 2) * 128
    run = lambda y=buf, x=buf, rows=2, ld=W, head=128, norm=C.byref(nrm), ft=_lib.DT_BF16: lib.b2_qk_rmsnorm(
        y, x, rows, ld, 4, 2, head, norm, ft, None)
    assert run(norm=None) == 3
    assert lib.b2_qk_rmsnorm(buf, buf, 2, W, 4, 2, 128, C.byref(_lib.QkNorm(None, g.value, 1e-6, 0)), _lib.DT_BF16, None) == 3
    assert run(y=None) == 3 and run(rows=0) == 3
    assert run(ld=W - 4) == 3
    assert run(head=64) == 6 and run(ft=_lib.DT_F32) == 6
    assert run(x=C.c_void_p(0x10002)) == 6 and run(ld=W + 2) == 6
    assert lib.b2_qk_rmsnorm(buf, buf, 2, W, 4, 2, 128, C.byref(_lib.QkNorm(0x20002, g.value, 1e-6, 0)), _lib.DT_BF16, None) == 6
    # fused append: NULL norm, head 64 and a misaligned gamma are refused before launch
    cfg = _lib.SpanCfg(_lib.DT_BF16, 0, 4, 2, 128, 16, 4, 0)
    app = lambda cfg=cfg, norm=C.byref(nrm), q_len=1: lib.b2_span_cache_append_qknorm(
        C.byref(cfg), buf, buf, buf, buf, buf, None, 2, q_len, None, norm, None)
    assert app(norm=None) == 3
    assert app(cfg=_lib.SpanCfg(_lib.DT_BF16, 0, 4, 2, 64, 16, 4, 0)) == 6
    assert app(norm=C.byref(_lib.QkNorm(0x20004, g.value, 1e-6, 0))) == 6
    assert app(q_len=17) == 4
