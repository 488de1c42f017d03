"""Exact-answer tests of fused attention: fsb_sdpa_fwd, fsb_sdpa_bwd and the bias path of fsb_attn_decode.

The kernels compute softmax in base 2: P = ex2(s * sc - m), sc = fp32(scale * log2 e). The inputs of tests/exact_inputs.py
make every score an integer multiple of 256 and pass the scale for which sc is exactly 1, so for every key tied at the row
maximum the argument of ex2 is 0 and P = 1, and for every other key it is <= -256 and P is exactly 0 (below fp32's smallest
subnormal). The row sum l is then the number of winners; with 1, 2 or 4 winners and integer V, O is their exact mean, and
it is compared with the fp64 reference bit for bit. One key wrongly admitted or dropped does not nudge O by 1/n: it replaces
the winner. Rows that by construction have another winner count (the uniform mean of the bias-selector tests) are held to
1 bf16 ulp of fp64. lse: bit-equal to max + log2(l) in base 2 on the exact rows (both terms are exact fp32 numbers), and
|lse ln2 - ref| <= 1e-5 max(1, |ref|) on every row.

Backward: with 2- and 4-way ties P is 1/2 or 1/4 and V, dO, K, Q are small integers chosen so that dP, delta and dS = P (dP -
delta) are integers of at most 8 bits: the bf16 roundings of P and dS inside the kernel are exact, dV and the sums behind dQ
and dK are exact in fp32, and the only roundings left are the fp32 product with `scale` and the bf16 store, which the
reference repeats. The gradients are held to 2^-18 max|grad| of that reference, and bit-equality, which additionally needs
ex2.approx(-1) == 0.5 and ex2.approx(-2) == 0.25 exactly, is asserted separately (it holds on the H100).

Gradient buffers are views of NaN-filled packed buffers with guard rows and guard head slots (tests/guards.py).
"""
import math

import pytest
import torch

import exact_inputs as X
from guards import Guarded, assert_ulp_close, bits

pytestmark = pytest.mark.gpu

from fsb200 import ops  # noqa: E402

DEV = "cuda"
BF16 = torch.bfloat16
SCALE = X.LN2_SCALE
EDGES = (0, 1, 63, 64, 127)        # mask edges are placed at these residues mod 128 (and so on both sides of 64 too)


def _packed_in(B, S, H, D, parts):
    """The fp64 tensors `parts` ([B, S, H, D] each) as bf16 slots of one packed [B, S, H, len(parts), D] buffer."""
    buf = torch.stack([p.to(BF16) for p in parts], dim=3).to(DEV).contiguous()
    return [buf[:, :, :, i] for i in range(len(parts))]


def _packed_out(B, S, H, D):
    pad = 2
    buf = torch.full((B * S + 2 * pad, H, 3, D), float("nan"), dtype=BF16, device=DEV)
    return Guarded(buf, lambda t: t[pad:pad + B * S].view(B, S, H, 3, D)[:, :, :, 1])


def _diff(got, want):
    bad = (bits(got.contiguous()) != bits(want.contiguous())).nonzero()
    i = tuple(int(v) for v in bad[0])
    return f"{len(bad)}/{got.numel()} elements differ; first at [b, s, h, d] = {i}: got {got[i].item()!r}, want {want[i].item()!r}"


def _check_fwd(out, lse, ref, what, exact_counts=(1, 2, 4)):
    """O bit-equal to bf16(ref) on rows with 1, 2 or 4 winners, within 1 bf16 ulp elsewhere; O = 0 and lse = +inf on rows
    without a permitted key; lse (base 2) bit-equal to max + log2(l) on the exact rows and to 1e-5 relative everywhere."""
    live = ref["live"]                                                        # [B, H, Sq]
    live_q = live.permute(0, 2, 1)
    assert not torch.isnan(out.float()).any() and not torch.isnan(lse).any(), f"{what}: NaN in O or lse"
    assert not out[~live_q].float().abs().gt(0).any(), f"{what}: O of a row without keys is not exactly 0"
    assert torch.isposinf(lse[~live]).all(), f"{what}: lse of a row without keys is not +inf"
    exact = torch.zeros_like(live)
    for c in exact_counts:
        exact |= ref["nwin"] == c
    exact = (exact & live).permute(0, 2, 1)
    want = X.bf16_of(ref["O"])
    if not torch.equal(bits(out[exact]), bits(want[exact])):
        sel = exact[..., None].expand_as(out)
        g, w = torch.where(sel, out, torch.zeros_like(out)), torch.where(sel, want, torch.zeros_like(want))
        raise AssertionError(f"{what}: O {_diff(g, w)}")
    rest = live_q & ~exact
    if rest.any():
        # floor: the reference's own fp64 noise (weights 1 / n are not dyadic) where the true mean is exactly 0
        assert_ulp_close(out[rest], ref["O"][rest], f"{what}: O of the rows with a uniform mean", floor=2.0 ** -40)
    # 1, 2 or 4 winners: the maximum is an exact fp32 number and log2(l) is 0, 1 or 2, so lse (base 2) is exact. At the
    # scores of the ramp and tie cases (up to 2^20) this is the only comparison fine enough to see l.
    ex = exact.permute(0, 2, 1)
    if not torch.equal(lse[ex], ref["lse2"][ex].float()):
        bad = (lse != ref["lse2"].float()) & ex
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: lse (base 2) differs on {int(bad.sum())} rows; first at [b, h, q] = {i}: got "
                             f"{lse[i].item()!r}, want {ref['lse2'][i].item()!r} with {int(ref['nwin'][i])} winners")
    got = lse[live].double() * math.log(2.0)
    lerr = (got - ref["lse"][live]).abs()
    tol = 1e-5 * ref["lse"][live].abs().clamp_min(1.0)
    assert bool((lerr <= tol).all()), f"{what}: lse off by {lerr.max().item():.3g}"
    return int(exact.sum()), int(rest.sum())


def _check_bwd(q, k, v, out, dout, lse, ref, causal, mask, what, rel=None, drel_prior=None):
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    dq, dk, dv = _packed_out(B, Sq, H, D), _packed_out(B, Sk, H, D), _packed_out(B, Sk, H, D)
    drel = None if rel is None else drel_prior.float().to(DEV).clone()
    ops.sdpa_bwd(q, k, v, out, dout, lse, SCALE, causal, dq.view, dk.view, dv.view, kv_mask=mask, rel_bias=rel,
                 drel_bias=drel)
    inexact = []
    for name, g in (("dq", dq), ("dk", dk), ("dv", dv)):
        g.check(f"{what} {name}")
        want = X.bf16_of(ref["d" + name[1].upper()])
        err = (g.view.double() - want.double()).abs().max().item()
        tol = 2.0 ** -18 * max(want.double().abs().max().item(), 2.0 ** -100)
        assert err <= tol, f"{what} {name}: max err {err:.4g} beyond 2^-18 max|grad| = {tol:.4g}; {_diff(g.view, want)}"
        if not torch.equal(bits(g.view.contiguous()), bits(want.contiguous())):
            inexact.append(name)
    if mask is not None:
        dead = ~mask.bool()
        for name, g in (("dk", dk), ("dv", dv)):
            assert not g.view[dead].float().abs().gt(0).any(), f"{what}: {name} of a masked key is not exactly 0"
    if drel is not None:
        want = ref["drel"]
        err = (drel.double() - want).abs().max().item()
        tol = 2.0 ** -18 * max(want.abs().max().item(), 1.0)
        bad = ((drel.double() - want).abs() > tol).nonzero()
        assert err <= tol, f"{what} drel: max err {err:.4g} (tol {tol:.4g}); first at [head, offset index] = " \
                           f"{bad[0].tolist()} of {len(bad)}"
        if not torch.equal(drel, want.float()):
            inexact.append("drel")
    # ex2.approx.ftz(-1) and (-2) are exactly 0.5 and 0.25 on the H100, so the recomputed P and with it every gradient
    # is bit-exact. PTX does not promise that; on hardware where it fails only this assertion may be relaxed.
    assert not inexact, f"{what}: within 2^-18 but not bit-equal: {inexact}"


def _run(score, Sq, D, causal, mask, what, negative_q=False, bwd=False, vstep=1, cache=False, exact_counts=(1, 2, 4)):
    """score [B, Skv, H]. Self-attention operands share one packed QKV buffer; with cache=True (or Sq != Skv) K and V are
    separate contiguous caches and Q is slot 0 of a packed projection."""
    B, Skv, H = score.shape
    q_vec, K = X.keys_for_scores(score, D)
    Q = X.queries(B, Sq, H, D, q_vec)
    V = X.value_codes(B, Skv, H, D, step=vstep)
    if Sq == Skv and not cache:
        q, k, v = _packed_in(B, Sq, H, D, [Q, K, V])
    else:
        q = _packed_in(B, Sq, H, D, [Q, Q, Q])[0]
        k, v = K.to(BF16).to(DEV), V.to(BF16).to(DEV)
    mask_d = None if mask is None else mask.to(DEV)
    dO = X.sparse_pm1(B, Sq, H, D, seed=Sq + D) if bwd else None
    ref = X.attention_ref(Q.to(DEV), K.to(DEV), V.to(DEV), SCALE, causal, mask_d, dO=None if dO is None else dO.to(DEV))
    out, lse = ops.sdpa_fwd(q, k, v, SCALE, causal, kv_mask=mask_d)
    n_exact, n_rest = _check_fwd(out, lse, ref, what, exact_counts)
    assert n_rest == 0, f"{what}: {n_rest} rows of this construction have a winner count outside {exact_counts}"
    if bwd:
        _check_bwd(q, k, v, out, dO.to(BF16).to(DEV), lse, ref, causal, mask_d, what)
    return ref


# ------------------------------------------------------------------------------------------------------------- C.1 ramps
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("S", [129, 1024, 2048 + 77])
def test_ramp_causal_with_padding(S, D):
    """Strict ramps (increasing for even b + h, decreasing for odd: the winner is the last / the first key a row may see)
    under causal, with per batch row: no padding; right padding; left padding whose first rows see no key at all; for every
    placement of the padding edge in EDGES. A leak of key i + 1 into row i replaces O[i] by V[i + 1]. With the backward (three
    edges for S <= 1024, one at S = 2048 + 77, where the dKV kernel skips up to 16 key tiles): P is one-hot, so dV is an exact
    scatter of dO rows and dQ = dK = 0."""
    B, H = 4, 2
    for e in EDGES:
        hi = (S - 1) // 128 * 128 - 128 + e if S > 256 else 64 + (e % 64)
        lo = 128 + e if S > 256 else e % 64 + 1
        mask = X.padding_mask(B, S, [(0, S - 1), (0, hi), (lo, S - 1), (lo + 64 if S > 256 else lo, hi)])
        _run(X.ramp_scores(B, S, H), S, D, True, mask, f"causal ramp S={S} D={D} edge {e}",
             bwd=e in (0, 63, 64) if S <= 1024 else e == 64)


@pytest.mark.parametrize("D", [64, 128])
def test_ramp_key_padding_and_ragged_tail(D):
    """Not causal: the mask alone decides, with both of its edges at every residue in EDGES; ramps below zero, so that a
    key of the zero-filled tail past Skv (score 0) or a masked key would beat every real key if it were admitted."""
    for S in (1024, 2048 + 77, 129):
        B, H = len(EDGES), 2
        top = (S - 1) // 128 * 128
        edges = [(min(128 + e, S // 2) if S > 256 else e % 64, (top - 128 + e if S > 256 else 64 + e % 64)) for e in EDGES]
        edges[0] = (edges[0][0], S - 1)                                  # one row reaches the ragged end of the last tile
        mask = X.padding_mask(B, S, edges)
        _run(X.ramp_scores(B, S, H, negative=True), S, D, False, mask, f"padding ramp S={S} D={D}", bwd=S == 1024)
    _run(X.ramp_scores(2, 2048 + 77, 2, negative=True), 2048 + 77, D, False, None, f"ragged tail, no mask D={D}")


@pytest.mark.parametrize("D", [64, 128])
def test_ramp_cross_attention_and_kv_cache_decode(D):
    """Sq != Skv, and the decode form (Sq 1 and 3 against separate K / V caches whose mask hides left padding and the
    unwritten tail): not causal, negative ramps."""
    _run(X.ramp_scores(2, 333, 2, negative=True), 200, D, False, None, f"cross 200x333 D={D}", bwd=True)
    _run(X.ramp_scores(2, 200, 2, negative=True), 333, D, False, X.padding_mask(2, 200, [(1, 128), (64, 199)]),
         f"cross 333x200 D={D}", bwd=True)
    for Sq in (1, 3):
        for Skv in (37, 129, 2048 + 77):
            filled = max(1, Skv - Skv // 4)
            mask = X.padding_mask(3, Skv, [(0, filled - 1), (1, filled - 1), (min(Skv // 3, filled - 1), filled - 1)])
            _run(X.ramp_scores(3, Skv, 4, negative=True), Sq, D, False, mask, f"decode Sq={Sq} Skv={Skv} D={D}", cache=True)


# ---------------------------------------------------------------------------------------------------- C.2 / D ties
def _tie_sets(S):
    """Peak placements: (name, [(key, level)]). Keys sit in the first and last 128-key step, in adjacent steps, and on both
    sides of multiples of 64 and 128."""
    last = S - 1
    return [("pair first+last step", [(5, 1), (last - 3, 1)]),
            ("pair adjacent steps", [(127, 1), (128, 1)]),
            ("pair across a 64 edge", [(63, 1), (64, 1)]),
            ("larger maximum later", [(1, 1), (65, 1), (last - 64, 2), (last, 2)]),
            ("larger maximum earlier", [(0, 2), (S // 2, 2), (last - 1, 1), (last, 1)])]


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", [200, 1024])
def test_ties_across_tiles(S, causal, D):
    """Two winners in different key steps, with the larger maximum arriving earlier or later: O is their exact mean, lse =
    m + 1. Under causal every row sees zero, one or two keys of the top level it can see (never three), so every row is
    exact. Forward and backward (V in steps of 16 and sparse +-1 dO keep dS within 8 bits)."""
    for name, peaks in _tie_sets(S):
        ref = _run(X.peaks_on_ramp(2, S, 2, peaks), S, D, causal, None, f"ties {name} S={S} causal={causal} D={D}", bwd=True,
                   vstep=16)
        assert int((ref["nwin"] == 2).sum()) > 0


@pytest.mark.parametrize("D", [64, 128])
def test_four_way_ties_with_padding(D):
    """Four winners spread over first, adjacent and last steps; not causal; padding hides two of them in one batch row and
    all four in another (which falls back to the ramp's single winner)."""
    S = 1024
    peaks = [(3, 1), (127, 1), (128, 1), (S - 2, 1)]
    mask = X.padding_mask(3, S, [(0, S - 1), (64, S - 64), (4, 126)])
    ref = _run(X.peaks_on_ramp(3, S, 2, peaks), S, D, False, mask, f"4-way ties D={D}", bwd=True, vstep=16)
    assert sorted(ref["nwin"].unique().tolist()) == [1, 2, 4]


# --------------------------------------------------------------------------------------- C.3 relative-position bias
def _selector_case(Sq, Skv, D, deltas, causal, mask, what, bwd=False, B=2):
    H = len(deltas)
    rel = X.selector_bias(H, Sq, Skv, deltas).to(DEV)
    g = torch.Generator().manual_seed(Sq + Skv)
    Q = torch.zeros(B, Sq, H, D, dtype=torch.float64)
    K = torch.randint(-3, 4, (B, Skv, H, D), generator=g).double()
    V = X.value_codes(B, Skv, H, D, step=16 if bwd else 1)
    if Sq == Skv:
        q, k, v = _packed_in(B, Sq, H, D, [Q, K, V])
    else:
        q, k, v = (t.to(BF16).to(DEV) for t in (Q, K, V))
    mask_d = None if mask is None else mask.to(DEV)
    dO = X.sparse_pm1(B, Sq, H, D, seed=7) if bwd else None
    prior = torch.full((H, Sq + Skv - 1), 0.25, dtype=torch.float64, device=DEV) if bwd else None
    ref = X.attention_ref(Q.to(DEV), K.to(DEV), V.to(DEV), SCALE, causal, mask_d, rel=rel,
                          dO=None if dO is None else dO.to(DEV), drel_prior=prior)
    out, lse = ops.sdpa_fwd(q, k, v, SCALE, causal, kv_mask=mask_d, rel_bias=rel)
    n_exact, n_rest = _check_fwd(out, lse, ref, what)
    assert n_exact > 0
    # the selected key, spelled out: O[b, i, h] == V[b, i + delta, h] wherever that key exists and is permitted
    for h, dl in enumerate(deltas):
        if isinstance(dl, int):
            i = torch.arange(Sq)
            j = i + dl
            ok = (j >= 0) & (j < Skv) & ((j <= i) if causal else torch.ones_like(i, dtype=torch.bool))
            for b in range(B):
                okb = ok if mask is None else ok & mask[b, j.clamp(0, Skv - 1)].bool()
                got, want = out[b, i[okb], h].cpu(), V[b, j[okb], h].to(BF16)
                assert torch.equal(got, want), f"{what}: head {h} (offset {dl}) batch {b}: O[i] != V[i + {dl}] at rows " \
                                               f"{i[okb][(got != want).any(-1)][:8].tolist()}"
    if bwd:
        assert n_rest == 0, f"{what}: {n_rest} rows average all their keys; the backward is exact only for 1, 2 or 4 winners"
        _check_bwd(q, k, v, out, dO.to(BF16).to(DEV), lse, ref, causal, mask_d, what, rel=rel, drel_prior=prior)
    return ref


@pytest.mark.parametrize("D", [64, 128])
def test_rel_bias_selects_one_offset(D):
    """q = 0 and a bias that is 0 except at one offset per head: row i must return V[i + offset] bit for bit; a bias vector
    read one entry off returns the neighbouring key's V. Offsets at the ends of the vector, around +-128 and inside; with and
    without causal / padding; and with Sq != Skv. Rows whose selected key does not exist or is masked get the uniform mean
    over their permitted keys (1 bf16 ulp of fp64)."""
    S = 300
    deltas = [-(S - 1), -128, -127, -65, -1, 0, 1, 37, 127, 128, S - 1]
    _selector_case(S, S, D, deltas, False, None, f"selector S={S} D={D}")
    _selector_case(S, S, D, deltas, True, None, f"selector causal S={S} D={D}")
    _selector_case(S, S, D, deltas, False, X.padding_mask(2, S, [(0, S - 1), (63, 256)]), f"selector padded S={S} D={D}")
    _selector_case(130, 391, D, [-129, -1, 0, 1, 128, 261, 390], False, None, f"selector 130x391 D={D}")
    _selector_case(391, 130, D, [-390, -128, 0, 64, 129], False, None, f"selector 391x130 D={D}")


@pytest.mark.parametrize("causal,masked", [(True, False), (False, True)])
def test_rel_bias_gradient_exact(causal, masked):
    """B = 18 (16 batch splits in the bias-gradient reduction, two holding two batches), Sq = Skv = 200. Each head selects
    two offsets, so rows that can see both keys tie two ways: dS = +-(dO . (V_a - V_b)) / 4, an integer, on two diagonals
    and exactly 0 on all others. Every one of the Sq + Skv - 1 entries of drel, accumulated onto 0.25, must match."""
    S = 200
    mask = None
    if masked:
        mask = torch.ones(18, S, dtype=torch.uint8)
        for b in range(18):
            mask[b, S - 3 * b - 1:] = 0
    # every row keeps at least one of its two selected keys permitted (a row with neither would average all its keys:
    # P = 1 / n, not a dyadic number)
    deltas = [(-64, -1), (-130, 0)] if causal else [(-63, 64), (-90, 50)]
    ref = _selector_case(S, S, 64, deltas, causal, mask, f"drel causal={causal} masked={masked}", bwd=True, B=18)
    assert int((ref["drel"] != 0.25).sum()) == 2 * len(deltas), "each selected diagonal carries a non-zero gradient"


# --------------------------------------------------------------------------------------------- C.3 decode bias selector
@pytest.mark.parametrize("D", [64, 128])
def test_decode_bias_selects_one_offset(D):
    """fsb_attn_decode reads the bias with sdpa_fwd's convention at seq_q = seq_kv = cap, for the query at slot kv_len - 1:
    with q = 0 and the selector bias, the step at length n must return V[n - 1 + offset]. kv_len walks across the chunk
    boundaries of the split plan (multiples of 64 keys up to the capacity)."""
    B, H, cap = 2, 4, 1100
    deltas = [0, -1, -64, -300]
    rel = X.selector_bias(H, cap, cap, deltas).to(DEV)
    V = X.value_codes(B, cap, H, D)
    g = torch.Generator().manual_seed(D)
    kc = torch.randint(-3, 4, (B, cap, H, D), generator=g).to(BF16).to(DEV)
    vc = V.to(BF16).to(DEV)
    q = torch.zeros(B, H, D, dtype=BF16, device=DEV)
    mask = torch.ones(B, cap, dtype=torch.uint8, device=DEV)
    lens = sorted({1, 2, 63, 64, 65, 127, 128, 129, 301, 512, 513, 1024, 1025, cap - 1, cap})
    for n in lens:
        kv_len = torch.tensor([n], dtype=torch.int32, device=DEV)
        out, lse = ops.attn_decode(q, kc, vc, kv_len, SCALE, kv_mask=mask, rel_bias=rel)
        for h, dl in enumerate(deltas):
            j = n - 1 + dl
            if j >= 0:
                want = V[:, j, h].to(BF16)
                assert torch.equal(out[:, h].cpu(), want), f"decode D={D} kv_len={n} head {h}: O != V[{j}] (offset {dl})"
                assert abs(lse[0, h].item() * math.log(2.0) - X.SELECT) <= 1e-5 * X.SELECT
            else:   # the selected slot does not exist: uniform mean over the n live keys
                want = V[:, :n, h].mean(1)
                assert_ulp_close(out[:, h].cpu(), want, f"decode D={D} kv_len={n} head {h} uniform mean", floor=2.0 ** -40)
