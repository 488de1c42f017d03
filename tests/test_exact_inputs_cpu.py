"""CPU proof that the constructions of tests/exact_inputs.py are what they claim: every operand exactly a bf16 value (or an
int8 / int4 code times a power-of-two scale), every partial sum in any order below the stated budget, the expected output
representable in the output type, and the attention winner sets as documented. The GPU tests compare kernels bit for bit
against these references; this file keeps the references honest without a device."""
import math

import numpy as np
import torch

import exact_inputs as X
import int4_ref


def _abs_sum(A, B):
    """sum_k |A||B|: an upper bound of every partial sum in every order."""
    return (A.abs() @ B.abs()).max().item()


def test_int_operands_budget_and_representability():
    for K in (8, 16, 56, 64, 72, 200, 4096 + 8, 6144, 8192):
        A, B = X.int_operands(33, 40, K, seed=K)
        a = X.int_amax(K)
        assert K * a * a < X.BUDGET and (a == 15 or K * (a + 1) ** 2 >= X.BUDGET)
        assert X.is_bf16(A) and X.is_bf16(B) and _abs_sum(A, B) < X.BUDGET
        assert A.min() < 0 < A.max() and (A == 0).any() and (B == 0).any()
        exact = A @ B
        assert torch.equal(exact, exact.round()) and torch.equal(exact.float().double(), exact)
        # fp32 accumulation in a shuffled order and in 7 splits gives the same bits as fp64
        perm = torch.randperm(K, generator=torch.Generator().manual_seed(K))
        acc = torch.zeros(33, 40, dtype=torch.float32)
        for chunk in perm.chunk(7):
            part = torch.zeros(33, 40, dtype=torch.float32)
            for k in chunk.tolist()[:64]:
                part += A[:, k, None].float() * B[None, k, :].float()
            acc += part
        sub = torch.cat([c[:64] for c in perm.chunk(7)])
        assert torch.equal(acc.double(), A[:, sub] @ B[sub])
    assert X.is_bf16(X.int_vector(100, 1, amax=200)) and X.is_bf16(X.int_vector(100, 1, amax=64) * 3 + 1)
    # an accumulated bf16 D: old (<= 200) + product + bias stays an integer below 2^24 -> one rounding
    assert X.BUDGET + 5000 + 64 * 3 + 1 < 2 ** 24


def test_position_code_names_the_block():
    for M, N, K in ((264, 392, 456), (136, 264, 4096 + 8), (8, 768, 8192), (384, 256, 6144)):
        A, B = X.position_coded(M, N, K)
        nb = (K + 63) // 64
        assert X.is_bf16(A) and X.is_bf16(B)
        want = A @ B
        assert want.max() < 2 ** 24 and torch.equal(want, want.round())
        # A: one 1 per row and k-block; B: column n is non-zero exactly on the k-blocks of its window; all blocks covered
        per_block = torch.stack([A[:, 64 * b:64 * (b + 1)].sum(1) for b in range(nb)], 1)
        assert torch.equal(per_block, torch.ones(M, nb, dtype=torch.float64))
        covered = torch.zeros(nb, dtype=torch.bool)
        nzb = torch.stack([(B[64 * b:64 * (b + 1)] != 0).all(0) for b in range(nb)], 1)          # [N, nb]
        anyb = torch.stack([(B[64 * b:64 * (b + 1)] != 0).any(0) for b in range(nb)], 1)
        for n in range(N):
            w0 = X.position_window_start(n, K)
            inside = torch.zeros(nb, dtype=torch.bool)
            inside[w0:w0 + X.POS_FIELDS] = True
            assert torch.equal(nzb[n], inside) and torch.equal(anyb[n], inside)
            covered |= inside
        assert covered.all()
        assert X.position_decode(want.long(), want.long()) is None
        # drop one k-block of B: the decoder names exactly that block for the first row that looks at it
        blk = nb // 2
        B2 = B.clone()
        B2[64 * blk:64 * (blk + 1)] = 0
        m, n, fields, count = X.position_decode((A @ B2).long(), want.long())
        assert count > 0 and [X.position_window_start(n, K) + f for f, g, w in fields] == [blk]
        assert fields[0][1] == 0 and 1 <= fields[0][2] <= 7
        # count it twice: the same block is named (its digit, or its digit and a carry into the next)
        m, n, fields, count = X.position_decode((A @ (B + (B - B2))).long(), want.long())
        assert X.position_window_start(n, K) + fields[0][0] == blk


def test_copy_gemm_inputs():
    Bb = X.normal_bf16_patterns(200, 392, seed=3)
    e = (Bb.view(torch.int16).to(torch.int32) >> 7) & 0xFF
    assert e.min() == 1 and e.max() == 254 and torch.isfinite(Bb.float()).all() and (Bb.float() != 0).all()
    A, sel = X.row_selector(264, 200, seed=1)
    assert torch.equal(A.sum(1), torch.ones(264, dtype=torch.float64)) and X.is_bf16(A)
    # the fp64 product IS the gather (0 * finite = 0, 1 * x = x)
    assert torch.equal((A @ Bb.double()), Bb.double()[sel])


def test_gelu_sweep_covers_every_value_with_an_exact_bias_split():
    Xv, base = X.gelu_sweep_values()
    assert Xv.shape[0] == 64 and X.is_bf16(Xv) and X.is_bf16(base)
    vals = set(Xv.to(torch.bfloat16).view(torch.int16).reshape(-1).tolist())
    want = {int(np.array(p, dtype=np.uint16).view(np.int16)) for s in (0, 0x8000) for p in range(s | 0x80, (s | 0x4300) + 1)}
    assert want | {0} == vals
    assert Xv.abs().max() == 128.0 and Xv.abs()[Xv != 0].min() == 2.0 ** -126
    diff = Xv - base[None, :]
    assert X.is_bf16(diff), "x - base must be a bf16 value for the bias variant"
    assert torch.equal((diff.float() + base.float()[None, :]).double(), Xv), "(x - base) + base must be exact in fp32"
    # references: erfc form agrees with the erf form where that one is accurate, and keeps the tail
    x = torch.tensor([-8.0, -3.0, -0.5, 0.0, 0.5, 3.0], dtype=torch.float64)
    assert torch.allclose(X.gelu_erf(x)[2:], 0.5 * x[2:] * (1 + torch.special.erf(x[2:] / math.sqrt(2))), rtol=1e-14, atol=0)
    assert -1e-14 < X.gelu_erf(x)[0].item() < -1e-15
    naive = 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    assert torch.allclose(X.gelu_tanh(x)[1:], naive[1:], rtol=1e-12, atol=0) and X.gelu_tanh(x)[0] < 0


def test_weight_only_operands():
    for qmax, (m, n, k) in ((127, (7, 200, 384)), (127, (8, 264, 5120)), (127, (2, 136, 13824)), (7, (33, 264, 5120)),
                            (7, (2, 136, 13824)), (7, (5, 200, 384))):
        A, Q = X.wq_int_operands(m, n, k, qmax, seed=k)
        assert X.is_bf16(A) and Q.dtype == torch.int8 and Q.min() == -qmax and Q.max() == qmax
        assert set(range(-qmax, qmax + 1)) <= set(Q[0].tolist()), "every code value occurs"
        assert _abs_sum(A, Q.double().t()) < X.BUDGET
        if k == 13824 and qmax == 127:   # the sparse form: exactly one non-zero in every 16-wide k-step of every row
            assert torch.equal((A.view(m, k // 16, 16) != 0).sum(-1), torch.ones(m, k // 16, dtype=torch.int64))
        else:
            assert (A != 0).float().mean() > 0.45
        if qmax == 127:
            s = X.w8_scales(n, 1)
            assert torch.equal(torch.log2(s), torch.log2(s).round()) and s.dtype == torch.float32
            exact = X.w8_exact(A, Q, s)
        else:
            s = X.w4_scales(n, k // 128, 1)
            e = torch.log2(s.float())
            assert s.dtype == torch.bfloat16 and torch.equal(e, e.round()) and e.min() >= -4 and e.max() <= -1
            assert (e[:, 1:] != e[:, :-1]).all(), "neighbouring groups differ, so a slipped group boundary changes the result"
            exact = X.w4_exact(A, Q, s)
            # W^ = q * s is exactly what the format's dequantiser gives, and the packed layout round-trips
            W = int4_ref.dequantize(Q.numpy(), s.float().numpy())
            assert np.array_equal(W.astype(np.float64), (Q.double() * s.double().repeat_interleave(128, 1)).numpy())
            assert np.array_equal(int4_ref.unpack(int4_ref.pack(Q.numpy())), Q.numpy())
            # partial sums are multiples of 2^-4 below 2^19: 23 bits
            assert (A.abs() @ (Q.double().abs() * s.double().repeat_interleave(128, 1)).t()).max() < 2 ** 19
            assert torch.equal(exact * 16, (exact * 16).round())
        assert torch.equal(exact.float().double(), exact), "the exact result fits fp32, so bf16(exact) is one rounding"


def test_attention_scale_and_key_encoding():
    assert X.kernel_log2_scale(X.LN2_SCALE) == 1.0, "the kernels' base-2 factor fp32(scale * log2 e) must be exactly 1"
    assert abs(X.LN2_SCALE - math.log(2)) < 1e-7
    assert float(np.float32(X.SELECT) * X.LOG2E_F32) + 2.0 == float(np.float32(np.float32(X.SELECT) * X.LOG2E_F32) +
                                                                     np.float32(2.0)), "bias height + log2(4) is exact in fp32"
    for D in (64, 128):
        for score in (X.ramp_scores(3, 2048 + 77, 4), X.ramp_scores(3, 2048 + 77, 4, negative=True),
                      X.peaks_on_ramp(2, 1024, 2, [(0, 2), (512, 2), (1022, 1), (1023, 1)])):
            q, K = X.keys_for_scores(score, D)
            assert X.is_bf16(K) and X.is_bf16(q)
            assert torch.equal(K @ q, score.double()) and torch.equal(K.float() @ q.float(), score.float())
            assert score.abs().max() < 2 ** 23 and (score % X.GAP == 0).all()
            Q = X.queries(3, 5, score.shape[2], D, q)
            assert X.is_bf16(Q) and torch.equal(torch.einsum("bqhd,bkhd->bhqk", Q[:score.shape[0]], K),
                                                score.double().permute(0, 2, 1)[:, :, None, :].expand(-1, -1, 5, -1))
    neg = X.ramp_scores(2, 300, 2, negative=True)
    assert neg.max() <= -X.GAP, "a zero-filled key (score 0) would beat every real key"
    s = X.ramp_scores(2, 300, 2)
    gaps = (s[:, 1:] - s[:, :-1]).abs()
    assert gaps.min() >= X.GAP and (s[0, 1:, 0] > s[0, :-1, 0]).all() and (s[0, 1:, 1] < s[0, :-1, 1]).all()
    assert 2.0 ** -X.GAP < 2.0 ** -149 / 2, "a weight one gap below the maximum is not representable in fp32"
    for step in (1, 16):
        V = X.value_codes(2, 300, 2, 64, step)
        assert X.is_bf16(V) and V.abs().max() == 7 * step and (V[:, 1:] != V[:, :-1]).float().mean() > 0.8
    dO = X.sparse_pm1(2, 50, 2, 64, seed=1)
    assert torch.equal(dO.abs().sum(-1), torch.full((2, 50, 2), 4.0, dtype=torch.float64))


def _ref_case(score, Sq, causal, mask, vstep=1, bwd=False, D=64):
    B, Skv, H = score.shape
    q, K = X.keys_for_scores(score, D)
    Q = X.queries(B, Sq, H, D, q)
    V = X.value_codes(B, Skv, H, D, vstep)
    dO = X.sparse_pm1(B, Sq, H, D, seed=3) if bwd else None
    return X.attention_ref(Q, K, V, X.LN2_SCALE, causal, mask, dO=dO), V, dO, K, Q


def test_attention_ramp_winner_sets():
    """Increasing ramp: the winner is the last permitted key; decreasing: the first. Under causal that is key min(i, hi) /
    key lo; rows before lo see nothing."""
    S = 300
    mask = X.padding_mask(4, S, [(0, S - 1), (0, 191), (129, S - 1), (64, 255)])
    ref, V, _, _, _ = _ref_case(X.ramp_scores(4, S, 2), S, True, mask)
    P = ref["P"]
    assert set(P.unique().tolist()) == {0.0, 1.0}
    i = torch.arange(S)
    for b, (lo, hi) in enumerate([(0, S - 1), (0, 191), (129, S - 1), (64, 255)]):
        for h in range(2):
            live = i >= lo
            assert torch.equal(ref["live"][b, h], live)
            win = torch.minimum(i, torch.tensor(hi)) if (b + h) % 2 == 0 else torch.full_like(i, lo)
            assert torch.equal(P[b, h].argmax(-1)[live], win[live])
            assert torch.equal(ref["O"][b, live, h], V[b, win[live], h])
            assert torch.isinf(ref["lse"][b, h][~live]).all() and not ref["O"][b, ~live, h].any()
    # not causal, negative ramp, ragged: winners are the mask's edges
    ref, V, _, _, _ = _ref_case(X.ramp_scores(2, 333, 2, negative=True), 200, False, X.padding_mask(2, 333, [(1, 300), (64, 332)]))
    assert ref["P"][0, 0].argmax(-1).unique().tolist() == [300] and ref["P"][0, 1].argmax(-1).unique().tolist() == [1]
    assert ref["P"][1, 0].argmax(-1).unique().tolist() == [64] and ref["P"][1, 1].argmax(-1).unique().tolist() == [332]


def test_attention_ties_are_dyadic_and_gradients_fit_eight_bits():
    S = 200
    for causal in (False, True):
        for peaks in ([(5, 1), (196, 1)], [(1, 1), (65, 1), (135, 2), (199, 2)], [(0, 2), (100, 2), (198, 1), (199, 1)]):
            ref, V, dO, K, Q = _ref_case(X.peaks_on_ramp(2, S, 2, peaks), S, causal, None, vstep=16, bwd=True)
            assert set(ref["nwin"].unique().tolist()) <= {1, 2} and (ref["nwin"] == 2).any()
            assert set(ref["P"].unique().tolist()) <= {0.0, 0.5, 1.0}
            _dyadic_checks(ref)
    mask = X.padding_mask(3, 1024, [(0, 1023), (64, 960), (4, 126)])
    ref, *_ = _ref_case(X.peaks_on_ramp(3, 1024, 2, [(3, 1), (127, 1), (128, 1), (1022, 1)]), 1024, False, mask, vstep=16, bwd=True)
    assert sorted(ref["nwin"].unique().tolist()) == [1, 2, 4]
    _dyadic_checks(ref)


def _dyadic_checks(ref):
    assert X.is_bf16(ref["O"]), "the exact mean is a bf16 value, so delta = dO . O is computed from exact operands"
    dS = ref["dS"]
    assert torch.equal(dS, dS.round()) and X.is_bf16(dS), "dS is an integer of at most 8 bits: its bf16 rounding is exact"
    for name in ("dQ", "dK", "dV"):
        g = ref[name] / (1.0 if name == "dV" else float(np.float32(X.LN2_SCALE)))
        assert (g * 4 - (g * 4).round()).abs().max() < 1e-9 and g.abs().max() < X.BUDGET, name
    assert ref["dS"].abs().max() > 0


def test_selector_bias_winners_and_exact_diagonals():
    S, H = 200, 2
    for causal, deltas, mask in ((True, [(-64, -1), (-130, 0)], None),
                                 (False, [(-63, 64), (-90, 50)], torch.ones(18, S, dtype=torch.uint8))):
        B = 18
        if mask is not None:
            for b in range(B):
                mask[b, S - 3 * b - 1:] = 0
        rel = X.selector_bias(H, S, S, deltas)
        assert (rel != 0).sum() == 4 and set(rel.unique().tolist()) == {0.0, X.SELECT}
        Q = torch.zeros(B, S, H, 64, dtype=torch.float64)
        K = torch.randint(-3, 4, (B, S, H, 64), generator=torch.Generator().manual_seed(1)).double()
        V = X.value_codes(B, S, H, 64, 16)
        dO = X.sparse_pm1(B, S, H, 64, seed=7)
        prior = torch.full((H, 2 * S - 1), 0.25, dtype=torch.float64)
        ref = X.attention_ref(Q, K, V, X.LN2_SCALE, causal, mask, rel=rel, dO=dO, drel_prior=prior)
        assert set(ref["nwin"][ref["live"]].unique().tolist()) <= {1, 2}, "every row keeps one or two selected keys"
        _dyadic_checks(ref)
        nz = (ref["drel"] != 0.25).nonzero()
        assert sorted(nz[:, 1].tolist()) == sorted(d + S - 1 for dl in deltas for d in dl)
        assert torch.equal(ref["drel"].float().double(), ref["drel"])
    # single offsets: row i selects key i + delta
    rel = X.selector_bias(3, 130, 391, [-129, 0, 390])
    V = X.value_codes(1, 391, 3, 64)
    ref = X.attention_ref(torch.zeros(1, 130, 3, 64, dtype=torch.float64), V, V, X.LN2_SCALE, False, None, rel=rel)
    assert torch.equal(ref["O"][0, 129, 0], V[0, 0, 0]) and torch.equal(ref["O"][0, :, 1], V[0, :130, 1])
    assert torch.equal(ref["O"][0, 0, 2], V[0, 390, 2]) and int(ref["nwin"][0, 2, 1]) == 391
