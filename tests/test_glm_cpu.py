"""CPU: the GLM rotary (interleaved pairs over half the head): the reference's half_inner kernel and both inverse-frequency
formulas restated (tests/glm_ref.py) against an fp64 Hugging Face-style GLM rotary within glue_ref's NeoX bound, the
permutation identity on the library's arithmetic, the b2_rope_cfg layout, the style checks of every entry point without a
GPU, and the model configs."""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest
import torch

import glm_ref as R
import glue_ref as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(rng, dt, n=len(G.ROPE_POS), heads=3):
    return G.ft_values(rng.standard_normal((n, heads, R.HEAD)) * 2, dt)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("invfreq_type,ratio", [(1, 1.0), (2, 1.0), (1, 500.0), (2, 500.0)])
def test_reference_kernel_meets_the_fp64_bound(invfreq_type, ratio, dt):
    ft = G.FTS[dt]
    rng = np.random.default_rng(invfreq_type * 7 + int(ratio))
    x = _rows(rng, ft)
    pos = np.array(G.ROPE_POS)[:, None]
    y = R.half_inner32(x, pos, R.invfreq(invfreq_type, 1e4, ratio), ft)
    Y, D = R.glm64(x, pos, R.theta64(invfreq_type, 1e4, ratio), 64)
    assert G.rope_ratio(y, Y, D, ft).max() <= 1.0
    assert np.array_equal(y[..., 64:], x[..., 64:])
    # the NeoX pairing over the same 64 dims is far outside the bound: the bound tells the pairings apart
    Yn, _ = G.rope_neox64(x, pos, 1e4 * (ratio if invfreq_type == 2 else 1.0), 64)
    assert G.rope_ratio(G.rn(Yn, ft), Y, D, ft).max() >= 4.0


def test_invfreq_formulas():
    """type 1 divides the frequencies by rope_ratio, type 2 raises the base; at rope_ratio 1 they agree"""
    assert np.array_equal(R.invfreq(1, 1e4, 1.0), R.invfreq(2, 1e4, 1.0))
    assert R.invfreq(1, 1e4, 1.0)[0] == 1.0 and R.invfreq(2, 1e4, 500.0)[0] == 1.0
    assert R.invfreq(1, 1e4, 500.0)[0] == np.float32(1 / 500)
    i = 5
    assert R.invfreq(2, 1e4, 500.0)[i] == np.float32((5e6) ** (-2 * i / 64))
    assert R.invfreq(1, 1e4, 1.0).shape == (32,)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("rd", [128, 64])
def test_interleaved_equals_neox_of_the_permuted_rows(rd, dt):
    """the library's arithmetic written pair by pair equals, bit for bit, its NeoX arithmetic on P x permuted back"""
    ft = G.FTS[dt]
    rng = np.random.default_rng(rd)
    x = _rows(rng, ft)
    pos = np.array(G.ROPE_POS)[:, None]
    for base in G.ROPE_BASES:
        y = R.il_kernel32(x, pos, base, rd, ft)
        yn = R.apply_p_inv(G.rope_kernel32(R.apply_p(x, rd), pos, base, rd, ft), rd)
        assert np.array_equal(y, yn), base
        # and within the NeoX bound of the interleaved formula
        Y, D = R.il_formula(x, pos, base, rd)
        assert G.rope_ratio(y, Y, D, ft).max() <= 1.0
    p = R.perm(64)
    assert p[:4].tolist() == [0, 2, 4, 6] and p[32:34].tolist() == [1, 3] and p[64:].tolist() == list(range(64, 128))
    assert np.array_equal(R.apply_p_inv(R.apply_p(x, 64), 64), x)


def test_rope_cfg_layout_is_unchanged(tmp_path):
    """b2_rope_cfg keeps its 12 bytes: base, rotary_dim, and the former reserved word as style"""
    from b200spark import _lib
    cls = _lib.RopeCfg
    assert [f for f, _ in cls._fields_] == ["base", "rotary_dim", "style"]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200spark.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(b2_rope_cfg));',
             '  printf("neox %d\\n", B2_ROPE_NEOX);', '  printf("il %d\\n", B2_ROPE_INTERLEAVED);']
    lines += ['  printf("%s %%zu\\n", offsetof(b2_rope_cfg, %s));' % (f, f) for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(cls) == 12
    assert [int(out[f]) for f, _ in cls._fields_] == [0, 4, 8]
    assert (int(out["neox"]), int(out["il"])) == (_lib.ROPE_NEOX, _lib.ROPE_INTERLEAVED) == (0, 1)


def test_style_checks_without_gpu():
    """style outside {0, 1}: B2_ERR_PARAM at every entry point that takes a b2_rope_cfg; style 1 on the head-64 append:
    B2_ERR_UNSUPPORTED; all before any device access (fake device pointers are never touched)"""
    from b200spark import _lib
    lib = _lib.lib
    P, BAD = 3, 6
    A = 1 << 20
    cfg = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_NONE, 8, 2, 128, 16, 4, 0)
    cfg64 = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_NONE, 8, 2, 64, 16, 4, 0)
    tab = _lib.RopeTable(A, 0, 1.0, 0)
    nrm = _lib.QkNorm(A, A, 1e-6, 0)
    calls = {
        "append": lambda r: lib.b2_span_cache_append(C.byref(cfg), A, A, A, A, A, 1, C.byref(r), None),
        "tokens": lambda r: lib.b2_span_cache_append_tokens(C.byref(cfg), A, A, A, A, A, 1, 2, C.byref(r), None),
        "tree": lambda r: lib.b2_span_cache_append_tree(C.byref(cfg), A, A, A, A, A, A, 1, 2, C.byref(r), None),
        "qknorm": lambda r: lib.b2_span_cache_append_qknorm(C.byref(cfg), A, A, A, A, A, None, 1, 1, C.byref(r), C.byref(nrm),
                                                            None),
        "rope_table": lambda r: lib.b2_span_cache_append_rope_table(C.byref(cfg), A, A, A, A, A, None, 1, 1, C.byref(r),
                                                                    C.byref(tab), None, None),
        "rotary": lambda r: lib.b2_rotary(A, A, 1, 8, 2, 128, C.byref(r), None),
        "rotary_table": lambda r: lib.b2_rotary_table(A, A, 1, 8, 2, 128, C.byref(r), C.byref(tab), _lib.DT_BF16, None),
    }
    for name, call in calls.items():
        for style in (2, -1, 7):
            assert call(_lib.RopeCfg(1e4, 64, style)) == P, (name, style)
        assert call(_lib.RopeCfg(1e4, 96, 1)) == BAD, name  # rotary_dim stays 64 or 128
    assert lib.b2_span_cache_append(C.byref(cfg64), A, A, A, A, A, 1, C.byref(_lib.RopeCfg(1e4, 64, 1)), None) == BAD
    assert lib.b2_span_cache_append(C.byref(cfg64), A, A, A, A, A, 1, C.byref(_lib.RopeCfg(1e4, 64, 2)), None) == P


def test_configs_and_refusals():
    from b200spark import model, ops
    g = model.GLM4_9B
    assert (g.hidden, g.n_heads, g.n_kv, g.inter, g.layers, g.vocab) == (4096, 32, 2, 13696, 40, 151552)
    assert (g.rope_base, g.eps, g.qkv_bias, g.rotary_dim, g.rope_style, g.head) == (1e4, 1.5625e-7, True, 64, "interleaved", 128)
    c = model.CHATGLM3_6B
    assert dataclasses.replace(c, name=g.name, layers=40, vocab=151552, eps=g.eps) == g
    assert (c.layers, c.vocab, c.eps) == (28, 65024, 1e-5)
    assert g.n_heads // g.n_kv == 16  # the most q heads per kv head the attention kernel takes
    assert model.QWEN2_7B.rotary_dim is None and model.QWEN2_7B.rope_style == "neox"
    assert ops.rope_style("neox") == 0 and ops.rope_style("interleaved") == 1 and ops.rope_style(1) == 1
    tiny64 = model.ModelConfig("tiny-64", 512, 8, 2, 1024, 2, 1024, head=64, rope_style="interleaved")
    with pytest.raises(AssertionError, match="interleaved rotary: head size 128"):
        model.DecodeStack(tiny64, 1, 16, device="cpu")
    with pytest.raises(AssertionError, match="rope_style"):
        model.DecodeStack(dataclasses.replace(g, rope_style="gptj"), 1, 16, device="cpu")


def test_oracle_rotary_pairs():
    """the oracle's GLM rotary on a unit vector: only the pair (2i, 2i+1) at frequency i moves; dims >= 64 stay"""
    from b200spark import model
    ref = R.GlmRopeMixin()
    ref.rope_dim, ref.rope_il, ref.rope_af = 64, True, 1.0
    ref.rope_theta = torch.tensor(1e4, dtype=torch.float64) ** (-torch.arange(32, dtype=torch.float64) * 2.0 / 64)
    x = torch.zeros(1, 128)
    x[0, 6] = 1.0
    x[0, 100] = 3.0
    y = ref._rope(x, 5.0)
    ang = 5.0 * 1e4 ** (-3 * 2.0 / 64)
    assert y[0, 6].item() == pytest.approx(np.cos(ang), abs=1e-6) and y[0, 7].item() == pytest.approx(np.sin(ang), abs=1e-6)
    assert torch.count_nonzero(y[0, :64]).item() == 2 and y[0, 100].item() == 3.0
    assert model.GLM4_9B.rope_style == "interleaved"


def test_interleaved_kernels_add_no_local_memory():
    """The interleaved kernels (48 appends, 48 table appends, b2_rotary's and b2_rotary_table's two) keep the 32-byte frame of
    sincosf's slow-path range reduction that their NeoX counterparts carry: the pairing adds no spilled state."""
    import re
    import shutil
    cuobjdump = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    lib = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
    out = subprocess.run([cuobjdump, "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = int(re.search(r"STACK:(\d+)", line).group(1))
            cur = None
    kinds = {k: {n: s for n, s in usage.items() if k in n}
             for k in ("cache_append_il_kernel", "cache_append_table_il_kernel", "rotary_il_kernel", "rotary_table_il_kernel")}
    assert [len(v) for v in kinds.values()] == [48, 48, 1, 2], {k: len(v) for k, v in kinds.items()}
    assert all(s == 32 for v in kinds.values() for s in v.values()), kinds
