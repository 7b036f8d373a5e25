"""CPU: the scaled-rotary tables (ops.rope_table) against an independent fp64 restatement and known answers, the table
form's arithmetic against its bound and five wrong kernels against it, the b2_rope_table layout against the header, the
argument checks of the new entry points, and the local memory of the table kernels (cuobjdump)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import glue_ref as G
import rope_scaling_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = {"default": (1e6, None), "linear": R.LINEAR, "qwen25": R.QWEN25, "qwen3": R.QWEN3, "llama31": R.LLAMA31,
         "tiny_yarn": R.TINY_YARN}


@pytest.mark.parametrize("rd", [128, 64])
@pytest.mark.parametrize("kind", list(TYPES))
def test_table_matches_fp64_restatement(kind, rd):
    from b200spark import ops
    base, sc = TYPES[kind]
    inv, af = ops.rope_table(sc, base, rd)
    ref, raf = R.inv_ref(sc, base, rd)
    assert inv.dtype == torch.float32 and inv.shape == (rd // 2,)
    got = inv.numpy()
    # both round an fp64 value to fp32 once; the fp64 values may differ in their last bits, so allow one fp32 ulp
    assert np.all(np.abs(got.astype(np.float64) - ref) <= np.spacing(ref)), kind
    assert np.mean(got == ref) >= 0.95, kind
    assert af == pytest.approx(raf, rel=1e-15)


def test_known_answers():
    from b200spark import model, ops
    base, sc = R.QWEN25
    assert R.yarn_dims(sc, base, 128) == (23, 40)
    inv, af = ops.rope_table(sc, base, 128)
    plain, _ = ops.rope_table(None, base, 128)
    assert np.float32(af) == np.float32(1.1386294)
    assert torch.equal(inv[:23], plain[:23])
    assert torch.equal(inv[40:], (plain[40:].double() / 4).float())
    assert torch.all(inv[24:40] < plain[24:40]) and torch.all(inv[24:40] > plain[24:40] / 4)  # the ramp between
    base, sc = R.LLAMA31
    inv, af = ops.rope_table(sc, base, 128)
    plain, _ = ops.rope_table(None, base, 128)
    assert inv[0].item() == 1.0 and af == 1.0
    # wavelength 2 pi / theta_f >= 8192 / 4 from f = 29 on: 64 - 29 = 35 frequencies change
    wl = 2 * np.pi * base ** (np.arange(64) * 2 / 128)
    assert int(np.sum(wl >= 2048)) == 35
    assert int((inv != plain).sum()) == 35
    # the model configs carry these entries; Qwen3 turns YaRN on through the same dict
    assert model.QWEN25_7B.rope_scaling == R.QWEN25[1]
    assert model.LLAMA31_8B.rope_scaling == R.LLAMA31[1] and model.LLAMA31_8B.rope_base == 5e5
    assert model.QWEN2_7B.rope_scaling is None and model.QWEN3_8B.rope_scaling is None
    with pytest.raises(ValueError):
        ops.rope_table({"rope_type": "dynamic", "factor": 2.0}, 1e6, 128)


def _case(rd, per_seq, rng):
    """4 sequences x 3 tree nodes (depths 0, 1, 1 at slots 0, 1, 2) at far positions, 2 q + 1 k heads; per_seq: every
    sequence its own table (YaRN factors 2 .. 5), else one shared Qwen2.5 table"""
    from b200spark import ops
    B, T = 4, 3
    old = np.array([0, 4095, 32767, 131071])
    depth = [0, 1, 1]
    pos = np.array([o + depth[t] for o in old for t in range(T)])
    slots = np.array([o + t for o in old for t in range(T)])
    seq = np.repeat(np.arange(B), T)
    if per_seq:
        tabs = [ops.rope_table(dict(R.QWEN25[1], factor=2.0 + b), 1e6, rd) for b in range(B)]
        inv = np.stack([t[0].numpy() for t in tabs])  # the rows differ; one attn_factor for all of them
        af = tabs[1][1]
    else:
        inv, af = ops.rope_table(R.QWEN25[1], 1e6, rd)
        inv = inv.numpy()[None]
    x = G.ft_values(rng.standard_normal((B * T, 3, 128)) * 2, torch.bfloat16)
    return x, pos, slots, seq, inv, af


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("rd", [128, 64])
def test_restatement_within_bound_and_bugs_rejected(rd, dt):
    ft = G.FTS[dt]
    rng = np.random.default_rng(rd)
    for per_seq in (False, True):
        x, pos, slots, seq, inv, af = _case(rd, per_seq, rng)
        y = R.table_kernel32(x, pos, inv, af, 2, rd, ft, seq=seq)
        Y, D = R.table_formula(x, pos, inv, af, 2, rd, seq=seq)
        assert R.ratio(y, Y, D, ft).max() <= 1.0
        assert np.array_equal(y[..., rd:], x[..., rd:])
        for bug in R.BUGS:
            if bug == "neighbour_row" and not per_seq:
                continue
            yb = G.rn(R.table_formula(x, pos, inv, af, 2, rd, seq=seq, slots=slots, bug=bug)[0], ft)
            worst = R.ratio(yb, Y, D, ft).max()
            assert worst >= 4.0, (bug, per_seq, worst)


def test_struct_layout_matches_the_header(tmp_path):
    from b200spark import _lib
    cls, cname = _lib.RopeTable, "b2_rope_table"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200spark.h"', 'int main(void) {',
             '  printf("size %%zu\\n", sizeof(%s));' % cname]
    lines += ['  printf("%s %%zu\\n", offsetof(%s, %s));' % (f, cname, f) for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(cls) == 24
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f


def test_argument_checks_without_gpu():
    """every check runs before any device access: fake device pointers are never touched"""
    from b200spark import _lib
    lib = _lib.lib
    P, BAD = 3, 6  # B2_ERR_PARAM, B2_ERR_UNSUPPORTED
    A = 1 << 20  # a 16-byte aligned fake address
    cfg = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_NONE, 8, 2, 128, 16, 4, 0)
    rope = _lib.RopeCfg(0.0, 128, 0)
    good = _lib.RopeTable(A, 0, 1.0, 0)

    def app(table, rope_=rope, cfg_=cfg, norm=None, q_len=1):
        return lib.b2_span_cache_append_rope_table(C.byref(cfg_), A, A, A, A, A, None, 1, q_len,
                                                   C.byref(rope_) if rope_ is not None else None,
                                                   C.byref(table) if table is not None else None,
                                                   C.byref(norm) if norm is not None else None, None)

    def rot(table, rope_=rope, head=128, ft=_lib.DT_BF16):
        return lib.b2_rotary_table(A, A, 1, 8, 2, head, C.byref(rope_) if rope_ is not None else None,
                                   C.byref(table) if table is not None else None, ft, None)

    for call in (app, rot):
        assert call(None) == P
        assert call(good, rope_=None) == P
        assert call(_lib.RopeTable(0, 0, 1.0, 0)) == P
        assert call(_lib.RopeTable(A, -4, 1.0, 0)) == P
        assert call(_lib.RopeTable(A, 32, 1.0, 0)) == P           # 0 < stride < rotary_dim / 2
        assert call(_lib.RopeTable(A + 4, 0, 1.0, 0)) == BAD      # 16-byte alignment
        assert call(_lib.RopeTable(A, 66, 1.0, 0)) == BAD         # rows would lose it
        assert call(good, rope_=_lib.RopeCfg(0.0, 96, 0)) == BAD  # rotary_dim 128 or 64
    cfg64 = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_NONE, 8, 2, 64, 16, 4, 0)
    assert app(good, cfg_=cfg64, rope_=_lib.RopeCfg(0.0, 64, 0)) == BAD   # head 64
    assert app(good, q_len=17) == 4                                      # B2_ERR_LIMIT, as the other appends
    assert app(good, norm=_lib.QkNorm(0, A, 1e-6, 0)) == P
    assert app(good, norm=_lib.QkNorm(A + 2, A, 1e-6, 0)) == BAD
    assert rot(good, head=64) == BAD
    assert rot(good, ft=_lib.DT_F32) == BAD


CUOBJDUMP = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
_APPEND = re.compile(r"cache_append_(table_)?kernelILi(\d)ELb([01])ELb([01])ELb([01])ELb([01])EE")


@pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")
def test_table_kernels_add_no_local_memory():
    """The appends carry sincosf's slow-path range reduction in a 32-byte frame; the 48 table-form instantiations keep
    exactly that frame (no table state is spilled), and the stand-alone table rotary has the same frame as b2_rotary."""
    lib = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = int(re.search(r"STACK:(\d+)", line).group(1))
            cur = None
    table = {m.groups()[1:]: s for n, s in usage.items() for m in [_APPEND.search(n)] if m and m.group(1)}
    assert len(table) == 48, len(table)
    assert all(s == 32 for s in table.values()), {k: s for k, s in table.items() if s != 32}
    rot = {n: s for n, s in usage.items() if "rotary_table_kernel" in n}
    plain = [s for n, s in usage.items() if "rotary_kernel" in n and "table" not in n]
    assert len(rot) == 2 and len(plain) == 1 and all(s == plain[0] for s in rot.values()), (rot, plain)
