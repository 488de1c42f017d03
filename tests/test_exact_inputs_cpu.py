"""CPU proof that the constructions of tests/exact_inputs.py are what they claim: every operand exactly a bf16 value (or an
int8 / int4 code times a power-of-two scale), every partial sum in any order below the stated budget, the expected output
representable in the output type, and the attention winner sets as documented. The GPU tests compare kernels bit for bit
against these references; this file keeps the references honest without a device."""
import math

import numpy as np
import pytest
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


# ================================================================================ the training step's looping kernels
def _f32(x):
    return np.float32(x)


@pytest.mark.parametrize("V,S,shift,ignore", [(50264, 1024, 1, lambda t: t % 5 == 3), (32600, 512, 0, lambda t: t % 4 >= 2),
                                              (21128, 128, 1, lambda t: t % 9 == 4)])
def test_xent_rows_are_exact(V, S, shift, ignore):
    rows = {50264: 32768, 32600: 16384, 21128: 3200}[V]
    t = torch.arange(rows)
    d = X.xent_rows(t, V, S, shift, ignore=ignore)
    # every row: 2^j distinct live columns; dead labels are dead and live labels live; special columns are used
    assert max(X.xent_strides(V)) * (2 ** X.XENT_MAX_J + 1) <= V
    valid = d["valid"]
    lab = d["label"]
    assert bool((lab[~valid] == -100).all()) and bool(((lab[valid] >= 0) & (lab[valid] < V)).all())
    live_lab = X.xent_is_live(lab, d["base"], d["stride"], d["n_live"], V) & valid
    kind = (t // 7) % 4
    assert bool(live_lab[valid & (kind <= 1)].all()) and not bool(live_lab[valid & (kind == 3)].any())
    assert live_lab[valid].any() and (~live_lab[valid]).any()
    sp = set(X.xent_special_columns(V))
    assert {0, V - 1} <= set(d["base"].tolist()) and {0, V - 1} <= set(lab[valid & live_lab].tolist())
    assert len(sp & set(lab[valid & ~live_lab].tolist())) >= len(sp) // 2, "dead labels on the special columns"
    labels = X.xent_labels_array(d, S, shift, V)
    s = t % S
    read = s + shift < S
    assert torch.equal(labels[(t + shift)[read]], lab[read]), "labels[t + shift] is row t's label"
    n_valid = int(valid.sum())
    if V == 32600:
        assert n_valid == 8192
    else:
        assert n_valid & (n_valid - 1) != 0
    # logits of a spread of rows: bf16 values, 2^j at the maximum, the rest >= 128 below; exp of the gap flushes to 0
    pick = torch.cat([torch.arange(0, 600), torch.arange(rows - 300, rows), torch.randperm(rows)[:300]])
    x, live, dd = X.xent_logits(pick, V, lambda tt: X.xent_rows(tt, V, S, shift, ignore=ignore))
    assert X.is_bf16(x)
    assert torch.equal(live.sum(1), dd["n_live"])
    mx = x.max(1).values
    assert torch.equal(mx, dd["M"].float()) and set(dd["M"].tolist()) >= {-80, 80, 2048 + 128 * 7}
    assert bool(((x[~live] <= (mx[:, None].expand_as(x))[~live] - X.XENT_GAP)).all())
    assert _f32(-X.XENT_GAP) * X.LOG2E_F32 < -126, "ex2.approx.ftz of the scaled gap is below 2^-126: exactly 0"
    for c in X.xent_special_columns(V):
        assert live[:, c].any(), f"special column {c} is live in some row"


def test_xent_gradient_and_loss_references():
    for gs, nv in ((1.0, 26214), (1.0, 8192), (3.0, 2791)):
        sc = X.xent_grad_scale_f32(gs, nv)
        assert sc == float(np.float32(gs) / np.float32(nv))
        for j in range(X.XENT_MAX_J + 1):
            p = 2.0 ** -j
            for v in (p, p - 1, -1.0, 0.0):
                assert float(_f32(v)) == v, "p - onehot is exact in fp32 before the one product"
    M, j = torch.tensor([-80, 80, 2944]), torch.tensor([0, 6, 3])
    lab = torch.tensor([-80, -64, 2944 - 256])
    ref = X.xent_row_loss_exact(M, j, lab)
    assert torch.allclose(ref, torch.tensor([0.0, 144 + 6 * math.log(2), 256 + 3 * math.log(2)], dtype=torch.float64))
    # the kernel's fp32 chain, with logf off by one ulp, stays inside the bound
    for m, jj, lb in zip(M.tolist(), j.tolist(), lab.tolist()):
        lg = np.float32(math.log(2.0 ** jj))
        lg = np.nextafter(lg, np.float32(np.inf))
        got = float(np.float32(np.float32(m) + lg) - np.float32(lb))
        r = m + jj * math.log(2) - lb
        assert abs(got - r) <= float(X.xent_row_loss_bound(torch.tensor(m), torch.tensor(jj), torch.tensor(r)))


def test_adamw_trajectory_is_exact_in_fp32():
    """The kernel's fp32 operations with beta1 = beta2 = eps = wd = 0 on the coded gradients, simulated in numpy fp32 over
    every exponent class and the grad scales used, give m = g, v = g^2 and the closed-form master, bit for bit."""
    i = torch.cat([torch.arange(0, 5000), torch.arange(2 ** 29 - 2000, 2 ** 29 + 4), torch.tensor([124_445_183])])
    p = X.adam_p0(i).numpy()
    assert np.array_equal(p.astype(np.float64), X.adam_p0(i).double().numpy())
    lr = np.float32(X.ADAM_LR)
    for s, gs in enumerate((2.0 ** -3, 1.0, 4.0, 1.0)):
        g16 = X.adam_grad(i, s)
        assert X.is_bf16(g16.double())
        gj = g16.numpy().astype(np.float32) * np.float32(gs)
        m = np.float32(0) * np.float32(5) + np.float32(1) * gj
        v = np.float32(0) * np.float32(5) + np.float32(1) * gj * gj
        assert np.all(np.abs(v) >= np.float32(2.0 ** -126)) and np.all(np.isfinite(v))
        denom = np.sqrt(v) / np.float32(1) + np.float32(0)
        p = p * np.float32(1) - (lr / np.float32(1)) * (m / denom)
        assert np.array_equal(m, gj) and np.array_equal(v, gj * gj) and np.array_equal(denom, np.abs(gj))
        assert np.array_equal(p, X.adam_master(i, s + 1).numpy())
    # the exponent names the element class: every class occurs among any 121 neighbours
    assert len(set(X.adam_exponent(torch.arange(7, 7 + X.ADAM_EXP_SPAN)).tolist())) == X.ADAM_EXP_SPAN


def test_sumsq_fields_and_count():
    threads = 8 * 132 * 256
    n = 124_445_184
    nvec = n // 4
    R = -(-nvec // threads)
    seen = []
    for lo in range(0, R, X.SUMSQ_FIELDS):
        pos = X.sumsq_field_positions(lo, R, threads, nvec)
        vals = [X.sumsq_field_value(f) for _, _, f in pos]
        assert all(X.is_bf16(torch.tensor([v], dtype=torch.float64)) for v in vals)
        for p, r, f in pos:
            assert p < n and (p // 4) // threads == r and p % 4 == r % 4
        sq = [v * v for v in vals]
        # partial sums in any order, on top of 0 or 2: dyadic multiples of 2^-22 below 4 (24 bits): exact in fp32
        total = sum(sq) + 2.0
        assert total < 4 and all((x * 2 ** 22).is_integer() for x in sq)
        perm = np.random.default_rng(lo).permutation(len(sq))
        acc = np.float32(2.0)
        for k in perm:
            acc = np.float32(acc + np.float32(sq[k]))
        assert float(acc) == total
        # a lost field clears exactly its bit
        code = round((total - 2.0 - sq[-1]) * 2 ** 22)
        assert [f for _, _, f in pos if not (code >> (2 * f)) & 1] == [pos[-1][2]]
        seen += [r for _, r, _ in pos]
    assert seen == list(range(R))
    i = torch.arange(0, 64 * 1000 + 37)
    x = X.sumsq_count_pattern(i)
    assert int((x != 0).sum()) == X.sumsq_count(len(i)) and set(x.unique().tolist()) == {-1.0, 0.0, 1.0}
    assert set((i[x != 0] % 4).tolist()) == {0, 1, 2, 3}
    assert X.sumsq_count(n) + 3 < 2 ** 24


@pytest.mark.parametrize("rows,cols", [(32768, 768), (32768, 3072), (16384, 2048), (16384, 8192), (32, 786432),
                                       (8, 98304), (777, 1032)])
def test_colsum_windows_cover_every_row(rows, cols):
    ns, rps = X.colsum_plan(rows, cols, 132)
    covered = torch.zeros(rows, dtype=torch.bool)
    for p in range(X.colsum_passes(rows, cols, rps)):
        rr, strip, win = X.colsum_focus(rows, cols, rps, p)
        ok = rr >= 0
        covered[rr[ok]] = True
        assert bool(((rr[ok] // rps) == strip[:, None].expand_as(rr)[ok]).all()), "a window stays inside its strip"
        if cols <= 8192:
            x, want = X.colsum_matrix(rows, cols, rr)
            assert X.is_bf16(x.double()) and torch.equal(x.double().sum(0), want)
            assert want.max() < 2 ** X.COLSUM_BITS and (want + 500).max() < 2 ** 24
            # drop one row: the decoder names it
            c = int(ok.sum(1).argmax())
            k = int(ok[c].nonzero()[-1])
            lost, extra = X.colsum_missing_rows(want[c] - 2 ** k, want[c], rr[c])
            assert lost == [int(rr[c, k])] and extra == []
    assert covered.all(), "every row is watched by some column in some pass"


def test_embedding_bwd_runs_are_exact():
    T, V, h, big = 32768, 50264, 768, 50256
    ids, short_ids, lens = X.embedding_bwd_ids(T, V, big, seed=1)
    n_big = int((ids == big).sum())
    assert n_big == T // 2 and int(lens.sum()) == T - n_big and int(lens.max()) == X.EMB_CODED_MAX
    assert len(set(short_ids.tolist())) == len(short_ids) and big not in set(short_ids.tolist())
    srt = torch.sort(ids, stable=True).values
    assert int(srt[0]) == 0 and int(srt[-1]) == V - 1
    occ = X.occurrence_index(ids)
    assert int(occ[ids == big].max()) == n_big - 1
    for sid, ln in list(zip(short_ids.tolist(), lens.tolist()))[:50]:
        assert sorted(occ[ids == sid].tolist()) == list(range(ln))
    dout = X.embedding_bwd_dout(ids, occ, h, big, seed=2)
    old = X.embedding_bwd_old(V, h, big, n_big, short_ids, seed=3)
    assert X.is_bf16(dout) and X.is_bf16(old)
    # per id and column: sum |terms| + |old| < 2^24, so any order of fp32 additions is exact
    absum = old.abs().index_add(0, ids, dout.abs())
    assert absum.max() < 2 ** 24
    want = old.index_add(0, ids, dout)
    touched = torch.unique(ids)
    coded = torch.cat([short_ids])
    assert X.is_bf16(want[coded]), "short runs: old + run sum is a bf16 integer, so a lost bit shows"
    nb = -(-n_big // X.EMB_BIG_COLS)
    assert X.is_bf16(want[big, :X.EMB_BIG_COLS + nb])
    # a lost occurrence of the long run is named by its two counting columns
    q = 5000
    tok = int(((ids == big) & (occ == q)).nonzero())
    drop = want[big] - dout[tok]
    short_cols = (want[big, :X.EMB_BIG_COLS + nb] != drop[:X.EMB_BIG_COLS + nb]).nonzero().view(-1).tolist()
    assert short_cols == [q % X.EMB_BIG_COLS, X.EMB_BIG_COLS + q // X.EMB_BIG_COLS]
    # a lost occurrence of a short run clears its bit
    sid = int(short_ids[lens == X.EMB_CODED_MAX][0])
    tok = int(((ids == sid) & (occ == 3)).nonzero())
    assert int(abs((want[sid, 0] - dout[tok, 0]) - old[sid, 0])) == 255 - 8
    assert len(touched) == len(short_ids) + 1


def test_vector_helper_values_are_exact():
    i = torch.arange(0, 10 ** 8, 9973)
    x16 = (((i * 3) % 255) - 127).double()
    old = ((i % (1 << 20)) - (1 << 19)).double()
    assert X.is_bf16(x16) and torch.equal((old.float() + 0.25 * x16.float()).double(), old + 0.25 * x16)
    b = (((i * 7) % 253) - 126).double() * torch.ldexp(torch.ones(len(i), dtype=torch.float64), -(i % 3))
    assert X.is_bf16(b) and X.is_bf16(x16 * 0.125)
    x32 = (i % (1 << 24)).float() * torch.ldexp(torch.ones(len(i)), -(i % 5).int())
    assert not X.is_bf16(x32.double()), "the cast inputs need rounding"
