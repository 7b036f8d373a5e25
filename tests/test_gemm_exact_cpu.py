"""CPU checks of tests/gemm_exact.py, the restatement behind test_gemm_exact_gpu.py: it agrees with plain fp64 dequantized
arithmetic, its exactness precondition holds for every GPU case, every GPU case reaches the kernel it names, and each of a
list of plausible kernel bugs, applied to the restatement, would miss the GPU assertions by at least TEETH bounds."""
import numpy as np
import pytest

import gemm_exact as X
from oracle import quant_ref as Q

TEETH = 4.0
CASES = {g.id: g for g in X.DYADIC_CASES + X.READBACK_CASES}


def _inputs(gc):
    return X.dyadic_inputs(gc)


@pytest.mark.parametrize("gid", ["gemv-w4-pc-m16-fp16", "gemv-w8-u8-m4", "gemv-w4-g64-m9", "gemv-w8-g128-m17", "gemv2-cb16",
                                 "tc-w8-m20-fp16", "tc-g40-m1", "tc-g72-m17", "tc-g200-m40-fp16", "pair-gemv-w4"])
def test_restatement_matches_fp64_dequant(gid):
    """Per channel and sub-channel on the mma.sync kernels the restatement IS fp64 A @ dequant(W); the wgmma GROUPED weights
    are one FT rounding per weight away from it."""
    gc = CASES[gid]
    c = gc.case
    inp = _inputs(gc)
    for wt in [inp["wt"]] + ([inp["wt2"]] if c.pair else []):
        if c.wbits == 16:
            ref = wt.w
        else:
            ref = Q.dequant(wt.q.astype(np.float64), wt.s.astype(np.float32), wt.z.astype(np.float32), c.group).astype(np.float64)
        W = X.path_weights(c, wt, gc.path)
        if gc.path == "tc" and c.grouped:
            assert np.all(np.abs(W - ref) <= 0.5 * X.ulp_ft(ref, c.ft))
            assert np.all(np.abs(inp["A"] @ W - inp["A"] @ ref) <= np.abs(inp["A"]) @ (0.5 * X.ulp_ft(ref, c.ft)))
        else:
            assert np.array_equal(W, ref)


@pytest.mark.parametrize("gc", X.DYADIC_CASES + [g for g in X.FP8_CASES if not g.id.startswith("rb-")], ids=lambda g: g.id)
def test_precondition_holds_for_every_gpu_case(gc):
    worst = X.case_precondition(gc, _inputs(gc))
    assert 0 < worst < 1


def test_precondition_refuses_inexact_inputs():
    c = X.Case(8, 4096, 64, ft="fp16")
    wt = X.make_weights(c, 1)
    with pytest.raises(ValueError):
        X.precondition(c, wt, X.make_acts(2, 4096, J=4, seed=1), "gemv", unit_a=2.0 ** -3)


def _facts(gc):
    ls = X.launches(gc.case, gc.M, gc.env, a8=gc.a8)
    c = gc.case
    f = {(l["path"], gc.case.wbits) for l in ls}
    for l in ls:
        if l["path"] == "gemv":
            f |= {("gemv-mt", l["mt"]), ("gemv-split", l["split"]), ("gemv-grouped", c.grouped), ("gemv-ft", c.ft)}
            if c.grouped and c.group in (64, 128, 256):
                f.add(("gemv-g", c.group))
        if l["path"] == "gemv2":
            f.add(("gemv2-cb", l["cb"]))
        if l["path"] == "tc8":
            f |= {("tc8-m", gc.M), ("tc8-odd-tiles", gc.case.KT % 2 == 1), ("tc8-split", l["S"] > 1), ("tc8-multi", l["multi"])}
        if l["path"] == "tc":
            f |= {("tc-nm", l["nm"]), ("tc-multi", l["multi"]), ("tc-split", l["S"] > 1), ("tc-ft", c.ft)}
            if c.grouped:
                f.add(("tc-grouped", "group_k" if c.group_k else "group_tiles"))
            if c.group_k and gc.M == 1:
                f.add(("tc-group_k-m1",))
    if len(ls) > 1 and ls[0]["path"] == "tc":
        f.add(("tc-tail", ls[-1]["rows"]))
    if len(ls) > 1 and ls[0]["path"] == "gemv" and c.wbits == 8 and c.grouped:
        f.add(("gemv-w8-sub-passes", gc.M))
    if c.pair:
        f.add(("pair", ls[0]["path"]))
    return f


def test_dispatch_covers_every_path():
    """Every GPU case reaches the path it names (on an H100 with 132 SMs; the GPU test re-derives it from the device), and
    together the cases cover every row of the path table."""
    seen = set()
    for gc in X.DYADIC_CASES + X.READBACK_CASES + X.FP8_CASES:
        ls = X.launches(gc.case, gc.M, gc.env, a8=gc.a8)
        assert {l["path"] for l in ls} == {gc.path}, (gc.id, ls)
        seen |= _facts(gc)
    need = {("gemv", 4), ("gemv", 8), ("gemv", 16), ("gemv-mt", 1), ("gemv-mt", 2), ("gemv-ft", "fp16"), ("gemv-grouped", True),
            ("gemv-g", 64), ("gemv-g", 128), ("gemv-g", 256),
            ("gemv-split", "forced"), ("gemv-split", "global"), ("gemv-split", "planned"),
            ("gemv-w8-sub-passes", 17), ("gemv-w8-sub-passes", 33), ("gemv-w8-sub-passes", 40),
            *[("gemv2-cb", cb) for cb in (16, 32, 64, 128)],
            ("tc", 4), ("tc", 8), ("tc", 16), ("tc-nm", 32), ("tc-nm", 64), ("tc-multi", True), ("tc-multi", False),
            ("tc-split", True), ("tc-split", False), ("tc-ft", "fp16"), ("tc-grouped", "group_tiles"), ("tc-grouped", "group_k"),
            ("tc-group_k-m1",), *[("tc-tail", r) for r in (1, 8, 16, 32, 64)],
            ("pair", "gemv"), ("pair", "gemv2"), ("pair", "tc"), ("pair", "tc8"),
            ("tc8-m", 1), ("tc8-m", 17), ("tc8-m", 64), ("tc8-odd-tiles", True), ("tc8-split", True), ("tc8-multi", True)}
    assert need <= seen, sorted(need - seen, key=str)
    # the two wgmma epilogues: the vectorised one (no activation, 8-byte aligned rows, N % 4 == 0) and the generic one
    forms = [(gc, X.call_form(i)) for i, gc in enumerate(X.DYADIC_CASES)]
    vec = [gc.id for gc, (pa, pc, off) in forms if gc.path == "tc" and not gc.case.pair and gc.act == 0 and gc.case.N % 4 == 0
           and (gc.case.N + pc) % 4 == 0 and off == 0]
    gen = [gc.id for gc, (pa, pc, off) in forms if gc.path == "tc" and not gc.case.pair and (gc.act != 0 or gc.case.N % 4 or (gc.case.N + pc) % 4 or off)]
    assert vec and any(CASES[g].res for g in vec), vec
    assert any(CASES[g].res for g in gen) and any(CASES[g].case.N % 4 for g in gen) and any(f[2] for g2, f in forms if g2.id in gen), gen


# ------------------------------------------------------------------------------------------------------------ teeth
def _readback_y(gc, W):
    ks = X.readback_ks(gc)
    return W[ks], np.zeros((len(ks), gc.case.N))


def mut_nibble_swap():
    gc = CASES["rb-gemv-w4-pc"]
    wt = X.make_weights(gc.case, X._seed(gc))
    y, E = _readback_y(gc, X.path_weights(gc.case, wt, gc.path))
    q = wt.q.copy()
    n2 = gc.case.N // 2 * 2
    q[:, 0:n2:2], q[:, 1:n2:2] = wt.q[:, 1:n2:2], wt.q[:, 0:n2:2]      # low and high nibble of each byte
    ym, _ = _readback_y(gc, X.dequant_exact(gc.case, X.Weights(q=q, s=wt.s, z=wt.z)))
    return gc, y, E, ym


def mut_group_boundary():
    out = []
    for gid in ("rb-tc-g40", "rb-tc-g72-fp16"):
        gc = CASES[gid]
        c = gc.case
        wt = X.make_weights(c, X._seed(gc))
        y, E = _readback_y(gc, X.path_weights(c, wt, gc.path))
        k = np.arange(c.K)
        gm = np.minimum(np.maximum(k - 8, 0) // c.group, c.G - 1)       # each group starts one 8-k word later
        ym, _ = _readback_y(gc, X.dequant_tc_grouped(c, wt, gidx=gm))
        out.append((gc, y, E, ym))
    return out


def mut_drop_tail_word():
    gc = CASES["rb-tc-w4-pc"]
    c = gc.case
    assert c.K % 64
    wt = X.make_weights(c, X._seed(gc))
    W = X.path_weights(c, wt, gc.path)
    y, E = _readback_y(gc, W)
    Wm = W.copy()
    Wm[c.K - 8:] = 0
    ym, _ = _readback_y(gc, Wm)
    return gc, y, E, ym


def mut_neighbour_zero():
    out = []
    for gid, sh in (("gemv-w4-pc-m16-fp16", 1), ("tc-g72-m17", -1)):
        gc = CASES[gid]
        inp = _inputs(gc)
        y, E = X.restate(gc, inp)
        wt = inp["wt"]
        wm = X.Weights(q=wt.q, s=wt.s, z=np.roll(wt.z, sh, axis=1))
        Wm = X.dequant_tc_grouped(gc.case, wm) if gc.path == "tc" and gc.case.grouped else X.dequant_exact(gc.case, wm)
        ym, _ = X.restate(gc, inp, W=Wm)
        out.append((gc, y, E, ym))
    return out


def mut_swap_gate_up():
    out = []
    for gid in ("pair-gemv-w4", "pair-tc-w8", "pair-gemv2"):
        gc = CASES[gid]
        inp = _inputs(gc)
        y, E = X.restate(gc, inp)
        Wg, Wu = X.path_weights(gc.case, inp["wt"], gc.path), X.path_weights(gc.case, inp["wt2"], gc.path)
        ym, _ = X.restate(gc, inp, W=Wu, W2=Wg)
        out.append((gc, y, E, ym))
    return out


def mut_round_partials():
    gc = CASES["tc-w4-m17"]
    c = gc.case
    S = X.tc_split(c)
    assert S > 1
    inp = _inputs(gc)
    y, E = X.restate(gc, inp)
    W = X.path_weights(c, inp["wt"], gc.path)
    v = np.zeros((gc.M, c.N))
    for kt0, kt1 in X.tc_slices(c, S):
        k0, k1 = kt0 * 64, min(kt1 * 64, c.K)
        v += X.rn_ft(inp["A"][:, k0:k1] @ W[k0:k1], "bf16")
    ym = gc.alpha * v + (inp["bias"][None, :] if inp["bias"] is not None else 0)
    return gc, y, E, ym


def mut_residual_first():
    gc = CASES["gemv-w4-pc-m8-act"]
    inp = _inputs(gc)
    y, E = X.restate(gc, inp)
    ym, _ = X.restate(gc, inp, res_first=True)
    return gc, y, E, ym


def mut_row_swap():
    gc = CASES["tc-w4-m128"]
    inp = _inputs(gc)
    y, E = X.restate(gc, inp)
    perm = np.arange(gc.M)
    for b in range(0, gc.M, 64):
        perm[b:b + 32], perm[b + 32:b + 64] = np.arange(b + 32, b + 64), np.arange(b, b + 32)
    return gc, y, E, y[perm]


def mut_fp8_tile_sums():
    """The zero-point term of the fp8 path read from the next 64-k tile's sum."""
    gc = {g.id: g for g in X.FP8_CASES}["fp8-m64"]
    inp = _inputs(gc)
    y, E = X.restate(gc, inp)
    ym, _ = X.restate(gc, inp, ts_shift=1)
    return gc, y, E, ym


def mut_fp8_high_codes():
    """nib4_to_e4m3 without its second table: codes 8..15 become q & 7."""
    gc = {g.id: g for g in X.FP8_CASES}["rb-fp8-m17"]
    c = gc.case
    wt = X.fp8_weights(c, X._seed(gc))
    ks = X.readback_ks(gc)
    x = X.onehot_acts(ks, c.K)
    S = X.tc_split(c)
    y, E = X.restate_fp8(c, wt, x, S)
    ym, _ = X.restate_fp8(c, wt, x, S, q=wt.q & 7)
    return gc, y, E, ym


MUTATIONS = {"fp8_tile_sums": mut_fp8_tile_sums, "fp8_high_codes": mut_fp8_high_codes, "nibble_swap": mut_nibble_swap, "group_boundary": mut_group_boundary, "drop_tail_word": mut_drop_tail_word,
             "neighbour_zero": mut_neighbour_zero, "swap_gate_up": mut_swap_gate_up, "round_partials": mut_round_partials,
             "residual_first": mut_residual_first, "row_swap": mut_row_swap}


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_mutation_has_teeth(name):
    """The mutated restatement misses the honest bound by >= TEETH bounds on at least one element of every case that
    targets it: a kernel with that bug fails its GPU case."""
    res = MUTATIONS[name]()
    for gc, y, E, ym in (res if isinstance(res, list) else [res]):
        t = X.teeth(y, E, ym, gc.case.ft)
        print(f"TEETH {name} {gc.id}: {t:.1f} bounds")
        assert t >= TEETH, (name, gc.id, t)
