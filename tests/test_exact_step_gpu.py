"""Exact-answer tests of the training step's looping kernels at the sizes the benchmark workloads launch them: the fused
cross-entropy (fsb_softmax_xent_fwd_bwd), AdamW over a flat shard (fsb_adamw_flat), the sum of squares (fsb_sumsq), the fp32
accumulate and the cast / add / scale helpers, the column sums (fsb_colsum) and the embedding gather and sorted backward.

Each of these kernels caps its grid and loops over the rest (a grid-stride loop, a strip loop, a run loop), and the older
parity tests run them at sizes where that loop turns once. Here every test restates the kernel's grid from fsb_num_sms() (or
reads the strip count from fsb_colsum_workspace_bytes) and asserts that its size turns the loop at least twice, so a later
grid retune that makes a size single-round fails here instead of quietly dropping coverage.

The inputs come from tests/exact_inputs.py (claims proven in test_exact_inputs_cpu.py) and are functions of the row, element
or token index, built on the device chunk by chunk. Every result is exact in fp32 and compared bit for bit, except the
cross-entropy's row losses and mean, which go through logf and are held to a bound derived from their few fp32 operations.
A failure names the row, element, strip, grid-stride round or occurrence that is wrong.

What notices a wrong term. The library was rebuilt with each of these one-line defects and the older tests of the kernel
(test_kernels_gpu / test_step_ops_gpu / test_layer_ops_gpu) and this file were run against it, on an NVIDIA H100 80GB HBM3:

| defect | older tests | new test that fails, and what it says |
|---|---|---|
| xent: row loop cut to its first round (`t < rows && t < gridDim.x`) | pass (10) | test_xent_exact_rows, all three cases: "gpt2: row_loss of 31712/32768 rows never written; first row 1056 (row-loop round 1 of CTA 0)" |
| xent: label read hoisted out of the row loop (`labels[blockIdx.x + shift]`) | pass (10) | all three: "gpt2: dlogits of 4287 elements in rows 1024..1535 differ; first at row 1056 (row-loop round 1 of CTA 0), column 0: got -3.814697265625e-05, want 0.0 (2^4 live from column 8191 stride 257, label 16383, column live: False)" |
| xent: pass-1 column loop cut to its first 16384 columns | fail (6 of 10) | all three: "gpt2: dlogits of 9837070 elements in rows 0..511 differ; first at row 4 (row-loop round 0 of CTA 4), column 0: got 6.984919309616089e-09, want 0.0 (2^0 live from column 31676 stride 7, label 31676, column live: False)" |
| xent: loss_reduce_kernel reads only its first 1024 rows | pass (10) | all three: "gpt2: loss 2.339430093765259, want 75.28021859305194 +- 0.000197" |
| adamw: grid-stride loop cut to its first round | pass (4) | both sizes: "adamw n=124445184: master of 19619840 elements in 0..33554431 differ; first element 2162688 (vector 540672, grid-stride round 1 of thread 0, slot 0): got -458752.0, want -458753.0; exp_avg holds the gradient of no step: it still holds its initial 5.0, so the element was never updated" |
| adamw: grid stride one vector too long | pass (4) | both sizes: "adamw n=124445184: master of 38 elements in 0..33554431 differ; first element 2162688 (vector 540672, grid-stride round 1 of thread 0, slot 0): got -458752.0, want -458753.0; ..." |
| sumsq: grid-stride loop cut to its first round | pass (2) | both dtypes: "sumsq torch.float32: launch over rounds 0..11: got 2.384185791015625e-07, want 1.3333332538604736; grid-stride rounds (vector slot) lost: [(1, 1), (2, 2), (3, 3), (4, 0), ..., (11, 3)]" |
| accumulate: loop cut to its first round | pass (5) | "accumulate overwrite=False: 97837312/100000000 elements differ; first element 2162688 (vector 540672, grid-stride round 1 of thread 0): got -458752.0, want -458759.0" |
| cast_f32_bf16: loop cut to its first round | pass (5) | "cast: 95674624/100000000 elements differ; first element 4325376 (vector 540672, grid-stride round 1 of thread 0): got nan, want 2162688.0" |
| add: loop cut to its first round | pass (5) | "add: 95674624/100000000 elements differ; first element 4325376 (vector 540672, grid-stride round 1 of thread 0): got nan, want 55.0" |
| scale_inplace: loop cut to its first round | pass (5) | "scale 1/8: 95674624/100000000 elements differ; first element 4325376 (vector 540672, grid-stride round 1 of thread 0): got 71.0, want 8.875" |
| colsum: row loop of a strip cut to its first round | fail (3 of 43) | the four bias-gradient sizes: "colsum gpt2_bias_h pass 0 torch.float32 accumulate=False: 746/768 column sums differ; first column 1: got 1023.0, want 4194303.0; rows lost: strip 0: 12 rows 32..43 (row-loop rounds 1..1, row lanes 0..11)" |
| colsum_finish_kernel sums one strip fewer | fail (41 of 43, most through act_bwd_bias) | all six sizes: "colsum gpt2_bias_h pass 1 torch.float32 accumulate=False: 24/768 column sums differ; first column 702: got 0.0, want 4194303.0; rows lost: strip 42: 22 rows 32256..32277 (row-loop rounds 0..0, row lanes 0..21)" |
| embedding_fwd: loop cut to its first round | pass (6) | both: "embedding gpt2 explicit positions: 20838922 elements differ; first token 5632 column 0 (vector 540672, grid-stride round 1 of thread 0): got -1.8189894035458565e-12, want -1064960.0" |
| embedding_bwd_sorted: run loop stops after its first EMB_R occurrences | fail (4 of 6) | "embedding dW: 1821 rows differ; first id 47 (run of 8 occurrences), column 0: got -241.0, want -1.0; occurrences lost: [4, 5, 6, 7]" |

So the older tests see four of the fifteen (the ones that also shift a small case); the new tests fail on every one and,
except for the mean loss, name the row, element, strip, round or occurrence. The whole file runs in about 7 s of pytest time
with a peak of 9.4 GiB allocated (the 2^29 + 4 AdamW case; every other test stays under 4 GiB).
"""
import math

import pytest
import torch

import exact_inputs as X
from guards import bits, guarded_1d, guarded_2d

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return int(L.load().fsb_num_sms())


def _rounds(work, per_round):
    return -(-work // per_round)


def _ew_threads(work):
    """Threads of an elementwise.cu ew_grid launch (256 per CTA, at most 16 CTAs per SM)."""
    return min(-(-work // 256), 16 * _sms()) * 256


def _first_bad(got, want):
    bad = (bits(got) != bits(want)).nonzero()
    return None if bad.numel() == 0 else (int(bad[0, 0]), len(bad))


# ------------------------------------------------------------------------------------------------------- cross-entropy
XENT_CASES = {
    # name: rows, V, seq, shift, ld pad, grad_scale, ignore
    "gpt2": (32 * 1024, 50264, 1024, 1, 0, 1.0, lambda t: t % 5 == 3),
    "mt5": (32 * 512, 32600, 512, 0, 0, 1.0, lambda t: t % 4 >= 2),
    "bert_strided": (25 * 128, 21128, 128, 1, 16, 3.0, lambda t: t % 9 == 4),
}
XENT_CHUNK = 512


@pytest.mark.parametrize("case", list(XENT_CASES))
def test_xent_exact_rows(case):
    """Rows of 2^j live logits at the row maximum and the rest >= 128 below: the row sum is 2^j, p = 2^-j, so dlogits =
    bf16(fp32((p - onehot) * fp32(grad_scale / n_valid))) bit for bit, and row_loss = M + log(2^j) - logit[label] within
    the bound of its fp32 operations. GPT-2 (shift 1, in place), mT5 (shift 0, n_valid a power of two) and a row-strided
    BERT case with NaN guard columns and a separate dlogits buffer."""
    rows, V, S, shift, pad, gscale, ignore = XENT_CASES[case]
    grid = min(rows, 8 * _sms())
    assert _rounds(rows, grid) >= 2, f"{case}: {rows} rows run the row loop once on a grid of {grid}"
    desc = lambda t: X.xent_rows(t, V, S, shift, ignore=ignore)   # noqa: E731
    t_all = torch.arange(rows, device=DEV)
    d_all = desc(t_all)
    labels = X.xent_labels_array(d_all, S, shift, V)
    n_valid = int(d_all["valid"].sum())
    if case == "mt5":
        assert n_valid & (n_valid - 1) == 0, "the mT5 case is meant to divide by a power of two"
    else:
        assert n_valid & (n_valid - 1) != 0
    in_place = pad == 0
    if in_place:
        logits = torch.empty(rows, V, dtype=BF16, device=DEV)
        view = logits
    else:
        lbuf = guarded_2d(rows, V, BF16, pad_rows=0, pad_cols=pad // 2)
        dbuf = guarded_2d(rows, V, BF16, pad_rows=2, pad_cols=pad // 2)
        assert lbuf.buf.stride(0) == dbuf.buf.stride(0) and lbuf.buf.stride(0) > V
        view = lbuf.view
    for r0 in range(0, rows, XENT_CHUNK):
        view[r0:r0 + XENT_CHUNK] = X.xent_logits(t_all[r0:r0 + XENT_CHUNK], V, desc)[0].to(BF16)
    if not in_place:
        lbuf.before = lbuf.buf.clone()
    row_loss = guarded_1d(rows, F32)
    loss = torch.full((), float("nan"), device=DEV)
    nv = torch.full((), -1, dtype=torch.int32, device=DEV)
    dl = view if in_place else dbuf.view
    L.call("fsb_softmax_xent_fwd_bwd", view.data_ptr(), labels.data_ptr(), dl.data_ptr(), row_loss.view.data_ptr(),
           loss.data_ptr(), nv.data_ptr(), rows, V, view.stride(0), S, shift, -100, gscale, _stream())
    unwritten = torch.isnan(row_loss.view).nonzero()
    if unwritten.numel():
        r = int(unwritten[0])
        raise AssertionError(f"{case}: row_loss of {len(unwritten)}/{rows} rows never written; first row {r} (row-loop round "
                             f"{r // grid} of CTA {r % grid})")
    row_loss.check(f"{case} row_loss")
    assert int(nv) == n_valid, f"{case}: n_valid {int(nv)}, want {n_valid}"
    if not in_place:
        dbuf.check(f"{case} dlogits")
        lbuf.check(f"{case} logits", written=False)
        assert torch.equal(bits(lbuf.buf), bits(lbuf.before)), f"{case}: logits changed although dlogits is separate"
    scale = torch.tensor(X.xent_grad_scale_f32(gscale, n_valid), dtype=F32, device=DEV)
    # dlogits, chunk by chunk
    for r0 in range(0, rows, XENT_CHUNK):
        t = t_all[r0:r0 + XENT_CHUNK]
        _, live, d = X.xent_logits(t, V, desc)
        cols = torch.arange(V, device=DEV)[None, :]
        p = torch.where(live, torch.ldexp(torch.ones_like(d["j"], dtype=F32), -d["j"].int())[:, None], 0.0)
        p = p - (cols == d["label"][:, None]).float()
        p = torch.where(d["valid"][:, None], p, 0.0)
        want = (p * scale).to(BF16)
        got = dl[r0:r0 + XENT_CHUNK]
        if not torch.equal(bits(got), bits(want)):
            bad = (bits(got) != bits(want)).nonzero()
            r, c = int(bad[0, 0]), int(bad[0, 1])
            tr = r0 + r
            raise AssertionError(
                f"{case}: dlogits of {len(bad)} elements in rows {r0}..{r0 + len(t) - 1} differ; first at row {tr} (row-loop "
                f"round {tr // grid} of CTA {tr % grid}), column {c}: got {got[r, c].item()!r}, want {want[r, c].item()!r} "
                f"(2^{int(d['j'][r])} live from column {int(d['base'][r])} stride {int(d['stride'][r])}, label "
                f"{int(d['label'][r])}, column live: {bool(live[r, c])})")
    # row losses and their mean
    lab = d_all["label"]
    dead_lab = torch.where(X.xent_is_live(lab, d_all["base"], d_all["stride"], d_all["n_live"], V), d_all["M"],
                           torch.where(d_all["M"].abs() <= 80, d_all["M"] - X.XENT_GAP - 8 * (lab % 3),
                                       d_all["M"] - X.XENT_GAP * (1 + lab % 3)))
    ref = torch.where(d_all["valid"], X.xent_row_loss_exact(d_all["M"], d_all["j"], dead_lab), 0.0)
    bound = torch.where(d_all["valid"], X.xent_row_loss_bound(d_all["M"], d_all["j"], ref), 0.0)
    got = row_loss.view.double()
    bad = ~((got - ref).abs() <= bound)
    if bad.any():
        r = int(bad.nonzero()[0])
        raise AssertionError(f"{case}: row_loss of {int(bad.sum())}/{rows} rows beyond the bound; first row {r} (round "
                             f"{r // grid} of CTA {r % grid}): got {got[r].item()!r}, want {ref[r].item()!r} +- "
                             f"{bound[r].item():.3g} (M {int(d_all['M'][r])}, 2^{int(d_all['j'][r])} live, label "
                             f"{int(lab[r])})")
    mean_ref = got.sum().item() / n_valid
    mean_tol = X.XENT_MEAN_DEPTH * 2.0 ** -24 * got.abs().sum().item() / n_valid + 2.0 ** -23 * abs(mean_ref)
    assert abs(loss.item() - mean_ref) <= mean_tol, f"{case}: loss {loss.item()!r}, want {mean_ref!r} +- {mean_tol:.3g}"
    exact_mean = ref.sum().item() / n_valid
    assert abs(loss.item() - exact_mean) <= mean_tol + bound.sum().item() / n_valid


# ------------------------------------------------------------------------------------------------------------- AdamW
ADAM_GPT2 = 124_445_184       # gpt2-110m's parameters padded to a multiple of 128: the single-GPU flat shard
ADAM_BIG = 2 ** 29 + 4        # fp32 byte offsets past 2^31
ADAM_CHUNK = 1 << 25
# step: (gradient dtype, device grad_scale, hyper form)
ADAM_STEPS = [(BF16, 2.0 ** -3, False), (F32, None, False), (BF16, 4.0, True), (F32, None, True)]


def _adam_check(n, steps_spec, master, m, v, p16, grid_threads, what):
    steps = len(steps_spec)
    s_last = steps - 1
    gs = steps_spec[-1][1] or 1.0
    for c0 in range(0, n, ADAM_CHUNK):
        i = torch.arange(c0, min(n, c0 + ADAM_CHUNK), device=DEV)
        g = X.adam_grad(i, s_last) * gs
        want = {"master": X.adam_master(i, steps), "exp_avg": g, "exp_avg_sq": g * g}
        for name, got in (("master", master), ("exp_avg", m), ("exp_avg_sq", v)):
            fb = _first_bad(got[c0:c0 + len(i)], want[name])
            if fb is not None:
                k, count = fb
                e = c0 + k
                vec = e // 4
                mv = m[e].item()
                read = "no step: it still holds its initial 5.0, so the element was never updated" if mv == 5.0 else \
                    "?" if mv == 0 or not math.isfinite(mv) else \
                    f"an element = {int(round(math.log2(abs(mv) / gs))) + 60} mod {X.ADAM_EXP_SPAN}"
                raise AssertionError(
                    f"{what}: {name} of {count} elements in {c0}..{c0 + len(i) - 1} differ; first element {e} (vector {vec}, "
                    f"grid-stride round {vec // grid_threads} of thread {vec % grid_threads}, slot {e % 4}): got "
                    f"{got[e].item()!r}, want {want[name][k].item()!r}; exp_avg holds the gradient of {read} (element "
                    f"{e} is {e % X.ADAM_EXP_SPAN} mod {X.ADAM_EXP_SPAN})")
        fb = _first_bad(p16[c0:c0 + len(i)], want["master"].to(BF16))
        assert fb is None, f"{what}: param16 != bf16(master) at element {c0 + fb[0]} ({fb[1]} elements)"


def _adam_run(n, steps_spec, what):
    blocks = -(-(n // 4) // 256)
    grid = min(blocks, 16 * _sms())
    threads = grid * 256
    assert _rounds(n // 4, threads) >= 2, f"{what}: n = {n} runs the grid-stride loop once"
    master = torch.empty(n, device=DEV)
    for c0 in range(0, n, ADAM_CHUNK):
        master[c0:c0 + ADAM_CHUNK] = X.adam_p0(torch.arange(c0, min(n, c0 + ADAM_CHUNK), device=DEV))
    m = torch.full((n,), 5.0, device=DEV)      # finite old moments: with beta = 0 they must drop out
    v = torch.full((n,), 5.0, device=DEV)
    p16 = torch.full((n,), float("nan"), dtype=BF16, device=DEV)
    dtypes = {dt for dt, _, _ in steps_spec}
    grads = {dt: torch.empty(n, dtype=dt, device=DEV) for dt in dtypes}
    for s, (dt, gs, hyper) in enumerate(steps_spec):
        g = grads[dt]
        for c0 in range(0, n, ADAM_CHUNK):
            g[c0:c0 + ADAM_CHUNK] = X.adam_grad(torch.arange(c0, min(n, c0 + ADAM_CHUNK), device=DEV), s).to(dt)
        gsd = None if gs is None else torch.tensor(gs, dtype=F32, device=DEV)
        if hyper:
            h = torch.tensor([X.ADAM_LR, 1.0, 1.0], dtype=F32, device=DEV)
            ops.adamw_flat(master, m, v, g, p16, 1e9, 0.0, 0.0, 0.0, 0.0, 0, grad_scale=gsd, hyper=h)
        else:
            ops.adamw_flat(master, m, v, g, p16, X.ADAM_LR, 0.0, 0.0, 0.0, 0.0, s + 1, grad_scale=gsd)
    del grads
    _adam_check(n, steps_spec, master, m, v, p16, threads, what)


def test_adamw_every_element_every_round_gpt2_shard():
    """beta1 = beta2 = eps = wd = 0, lr 1/4, gradients +-2^e coding the element: m = g, v = g^2 and master = p0 - lr sum sign
    exactly, over four steps (bf16 and fp32 gradients, a power-of-two device grad_scale, the device-hyper form)."""
    _adam_run(ADAM_GPT2, ADAM_STEPS, f"adamw n={ADAM_GPT2}")


def test_adamw_offsets_past_2_31():
    """n = 2^29 + 4: the fp32 arrays' byte offsets pass 2^31. bf16 gradients only (about 8 GB); skipped when the card does
    not have that much free."""
    need = ADAM_BIG * (3 * 4 + 2 + 2) + 4 * ADAM_CHUNK * 8
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"n = 2^29 + 4 needs {need / 2 ** 30:.1f} GiB free; {free / 2 ** 30:.1f} GiB are")
    _adam_run(ADAM_BIG, [st for st in ADAM_STEPS if st[0] == BF16] + [(BF16, None, False)], "adamw n=2^29+4")


# ------------------------------------------------------------------------------------------------------ sum of squares
SUMSQ_N = ADAM_GPT2


@pytest.mark.parametrize("dt", [F32, BF16], ids=["f32", "bf16"])
def test_sumsq_names_every_round(dt):
    """One non-zero element per grid-stride round, 2^(f - 11) in field f of a launch, so the sum of squares carries one bit
    per round (and vector slot r mod 4): a lost round reads as its cleared bit. Then a count of +-1 entries over every slot
    and thread (an integer below 2^24). Accumulating launches add onto 2."""
    threads = 8 * _sms() * 256
    nvec = SUMSQ_N // 4
    n_rounds = _rounds(nvec, threads)
    assert n_rounds >= 2
    x = torch.zeros(SUMSQ_N, dtype=dt, device=DEV)
    out = torch.zeros((), device=DEV)
    for launch, lo in enumerate(range(0, n_rounds, X.SUMSQ_FIELDS)):
        pos = X.sumsq_field_positions(lo, n_rounds, threads, nvec)
        idx = torch.tensor([p for p, _, _ in pos], device=DEV)
        x[idx] = torch.tensor([X.sumsq_field_value(f) * (-1) ** r for _, r, f in pos], dtype=dt, device=DEV)
        acc = launch % 2 == 1
        out.fill_(2.0)
        ops.sumsq(x, out, accumulate=acc)
        want = sum(X.sumsq_field_value(f) ** 2 for _, _, f in pos) + (2.0 if acc else 0.0)
        if out.item() != want:
            got_bits = round((out.item() - (2.0 if acc else 0.0)) * 2 ** 22)
            lost = [(r, p % 4) for p, r, f in pos if not (got_bits >> (2 * f)) & 1]
            raise AssertionError(f"sumsq {dt}: launch over rounds {lo}..{pos[-1][1]}: got {out.item()!r}, want {want!r}; "
                                 f"grid-stride rounds (vector slot) lost: {lost}")
        x[idx] = 0
    for c0 in range(0, SUMSQ_N, ADAM_CHUNK):
        x[c0:c0 + ADAM_CHUNK] = X.sumsq_count_pattern(torch.arange(c0, min(SUMSQ_N, c0 + ADAM_CHUNK), device=DEV)).to(dt)
    out.fill_(3.0)
    ops.sumsq(x, out, accumulate=True)
    want = X.sumsq_count(SUMSQ_N) + 3
    assert out.item() == want, f"sumsq {dt} count: got {out.item()!r}, want {want} ({want - out.item():.0f} entries lost)"


# ------------------------------------------------------------------------------------------------ vector helpers at 1e8
EW_N = 10 ** 8


def _ew_fail(what, got, want, width):
    fb = _first_bad(got, want)
    if fb is None:
        return
    i, count = fb
    vec = i // width
    thr = _ew_threads(EW_N // width)
    raise AssertionError(f"{what}: {count}/{got.numel()} elements differ; first element {i} (vector {vec}, grid-stride "
                         f"round {vec // thr} of thread {vec % thr}): got {got[i].item()!r}, want {want[i].item()!r}")


def test_accumulate_cast_add_scale_at_1e8():
    """ZeRO-2 sized vectors: acc (+)= 2^-2 x with integer x and acc (exact), fp32 -> bf16 casts of values that need
    rounding (against torch's round-to-nearest-even), the bf16 add, scale by 2^-3, and scale by 1, which must leave the
    buffer untouched bit for bit (it holds signalling-NaN patterns that a multiply would quieten)."""
    n = EW_N
    for width in (4, 8):
        assert _rounds(n // width, _ew_threads(n // width)) >= 2
    i = torch.arange(n, device=DEV)
    x16 = (((i * 3) % 255) - 127).to(BF16)
    old = ((i % (1 << 20)) - (1 << 19)).float()
    for overwrite in (False, True):
        acc = guarded_1d(n, F32, fill=0.0, init=old)
        ops.accumulate(acc.view, x16, scale=0.25, overwrite=overwrite)
        acc.check(f"accumulate overwrite={overwrite}", written=False)
        want = (0.0 if overwrite else old) + 0.25 * x16.float()
        _ew_fail(f"accumulate overwrite={overwrite}", acc.view, want, 4)
        del acc, want
    del old
    x32 = (i % (1 << 24)).float() * torch.ldexp(torch.ones(n, device=DEV), -(i % 5).int())
    cast = guarded_1d(n, BF16)
    ops.cast_f32_to_bf16(x32, out=cast.view)
    _ew_fail("cast", cast.view, x32.to(BF16), 8)
    cast.check("cast")
    del x32, cast
    b16 = ((((i * 7) % 253) - 126).float() * torch.ldexp(torch.ones(n, device=DEV), -(i % 3).int())).to(BF16)
    out = guarded_1d(n, BF16)
    ops.add(x16, b16, out=out.view)
    _ew_fail("add", out.view, (x16.float() + b16.float()).to(BF16), 8)
    out.check("add")
    del out, b16
    sc = guarded_1d(n, BF16, fill=0.0, init=x16)
    ops.scale_inplace(sc.view, torch.tensor(0.125, device=DEV))
    sc.check("scale 1/8", written=False)
    _ew_fail("scale 1/8", sc.view, (x16.float() * 0.125).to(BF16), 8)
    snan = x16.clone()
    bits(snan)[i % 1000 == 7] = 0x7F81
    one = guarded_1d(n, BF16, fill=0.0, init=snan)
    ops.scale_inplace(one.view, torch.tensor(1.0, device=DEV))
    one.check("scale 1", written=False)
    _ew_fail("scale by 1 (must not touch memory)", one.view, snan, 8)


# ---------------------------------------------------------------------------------------------------------- column sums
COLSUM_CASES = [
    # name, rows, cols, rows expected to loop (bias-gradient form) or not (learned-position form)
    ("gpt2_bias_h", 32768, 768, True), ("gpt2_bias_ff", 32768, 3072, True),
    ("megatron_bias_h", 16384, 2048, True), ("megatron_bias_ff", 16384, 8192, True),
    ("gpt2_positions", 32, 1024 * 768, False), ("bert_positions", 8, 128 * 768, False),
]


def _colsum_one(x, rows, cols, rr, want_exact, odt, accumulate, old, what, rps):
    init = old.to(odt) if accumulate else None
    out = guarded_1d(cols, odt, fill=0.0 if accumulate else float("nan"), init=init)
    ops.colsum(x, out.view, accumulate=accumulate)
    out.check(what, written=not accumulate)
    want = want_exact + (old.to(odt).double() if accumulate else 0.0)
    wt = want.float() if odt == F32 else want.to(BF16)
    fb = _first_bad(out.view, wt)
    if fb is None:
        return
    c, count = fb
    msg = f"{what}: {count}/{cols} column sums differ; first column {c}: got {out.view[c].item()!r}, want {wt[c].item()!r}"
    if odt == F32:
        got_code = out.view[c].double().item() - (old[c].to(odt).item() if accumulate else 0.0)
        if got_code == int(got_code) and got_code >= 0:
            lost, extra = X.colsum_missing_rows(got_code, want_exact[c].item(), rr[c])
            msg += f"; rows lost: {_name_rows(lost, rps)}" + (f"; bits set that no row owns: {extra}" if extra else "")
    raise AssertionError(msg)


def _name_rows(lost, rps):
    """Lost rows as (strip, row-loop round, row lane), grouped per strip when there are many."""
    if len(lost) <= 4:
        return ", ".join(f"row {r} (strip {r // rps}, row-loop round {(r % rps) // 32}, row lane {r % 32})" for r in lost)
    out = []
    for s in sorted({r // rps for r in lost}):
        rs = [r for r in lost if r // rps == s]
        rounds = sorted({(r % rps) // 32 for r in rs})
        lanes = sorted({r % 32 for r in rs})
        out.append(f"strip {s}: {len(rs)} rows {rs[0]}..{rs[-1]} (row-loop rounds {rounds[0]}..{rounds[-1]}, row lanes "
                   f"{lanes[0]}..{lanes[-1]})")
    return "; ".join(out)


@pytest.mark.parametrize("name,rows,cols,loops", COLSUM_CASES, ids=[c[0] for c in COLSUM_CASES])
def test_colsum_names_lost_rows(name, rows, cols, loops):
    """Column c watches a 22-row window of one strip, row k of the window adding 2^k; passes deal the windows out until
    every row is watched. fp32 and bf16 out, written and accumulated (onto integers); the bias form also through a
    row-strided view with NaN in the padding columns. A wrong fp32 sum is decoded into the rows it lost."""
    ns, rps = X.colsum_plan(rows, cols, _sms())
    assert L.load().fsb_colsum_workspace_bytes(rows, cols) == ns * cols * 4, "colsum_plan restated wrongly"
    if loops:
        assert rps // 32 >= 2 and ns >= 2, f"{name}: {ns} strips of {rps} rows: the row loop turns {rps // 32} times"
    else:
        # one strip and at most one row per row lane: what these sizes cover is the grid of 64-column tiles (and the
        # finishing kernel's 256-column CTAs), many waves of the SMs
        assert ns == 1 and rows <= 32 and (cols + 63) // 64 >= 8 * _sms()
    old = ((torch.arange(cols, device=DEV) % 1000) - 500).float()
    for p in range(X.colsum_passes(rows, cols, rps)):
        rr, strip, win = X.colsum_focus(rows, cols, rps, p)
        rr = rr.to(DEV)
        x, want = X.colsum_matrix(rows, cols, rr, device=DEV)
        views = [("", x)]
        if loops:
            sbuf = torch.full((rows, cols + 64), float("nan"), dtype=BF16, device=DEV)
            sbuf[:, 16:16 + cols] = x
            views.append((" row-strided", sbuf[:, 16:16 + cols]))
        del x
        for vname, xv in views:
            for odt in (F32, BF16):
                for acc in (False, True):
                    _colsum_one(xv, rows, cols, rr, want, odt, acc, old,
                                f"colsum {name} pass {p}{vname} {odt} accumulate={acc}", rps)
        del views


# ------------------------------------------------------------------------------------------------------------ embedding
EMB_FWD_CASES = [("gpt2", 32768, 50264, 768, 1024, 1024, 0), ("megatronbert", 16384, 21128, 2048, 512, 512, 2)]


@pytest.mark.parametrize("name,rows,V,h,S,npos,ntt", EMB_FWD_CASES, ids=[c[0] for c in EMB_FWD_CASES])
def test_embedding_fwd_bit_exact(name, rows, V, h, S, npos, ntt):
    """out = bf16((W[id] + P[pos]) + T[type]) in the kernel's fp32 order, on random bf16 tables of mixed magnitude, with
    explicit positions (offset per sequence) and, for GPT-2, the implicit t % seq_len form as well."""
    vpr = h // 8
    assert _rounds(rows * vpr, _ew_threads(rows * vpr)) >= 2
    g = torch.Generator(device=DEV).manual_seed(rows + h)
    mag = lambda *s: torch.ldexp(torch.randn(*s, device=DEV, generator=g),   # noqa: E731
                                 torch.randint(-20, 21, s, device=DEV, generator=g, dtype=torch.int32)).to(BF16)
    W, P = mag(V, h), mag(npos, h)
    T = mag(ntt, h) if ntt else None
    ids = torch.randint(0, V, (rows,), device=DEV, generator=g)
    ids[:2] = torch.tensor([0, V - 1])
    pos = (torch.arange(rows, device=DEV) + torch.arange(rows, device=DEV) // S * 3) % npos
    tt = torch.randint(0, ntt, (rows,), device=DEV, generator=g) if ntt else None
    want = W[ids].float() + P[pos].float()
    if T is not None:
        want = want + T[tt].float()
    want = want.to(BF16)
    forms = [("explicit positions", pos)]
    if T is None:
        forms.append(("positions t % seq_len", None))
    for fname, pv in forms:
        got = ops.embedding_fwd(ids, W, pos=pv, P=P, token_type=tt, T=T, seq_len=S)
        w = want if pv is not None else (W[ids].float() + P[torch.arange(rows, device=DEV) % S].float()).to(BF16)
        fb = _first_bad(got.view(-1), w.view(-1))
        if fb is not None:
            e, count = fb
            t, c = divmod(e, h)
            vec = t * vpr + c // 8
            thr = _ew_threads(rows * vpr)
            raise AssertionError(f"embedding {name} {fname}: {count} elements differ; first token {t} column {c} (vector "
                                 f"{vec}, grid-stride round {vec // thr} of thread {vec % thr}): got "
                                 f"{got.view(-1)[e].item()!r}, want {w.view(-1)[e].item()!r}")


def test_embedding_bwd_sorted_exact():
    """32768 GPT-2 tokens over V = 50264: one id on half of them, the other half in runs of 1..8 over distinct ids including
    0 and V - 1. Short runs add +-2^q for occurrence q onto -+256 (a lost occurrence is a cleared bit); the long run counts
    occurrences by q mod 384 and q // 384 (a lost one is named by the two columns it leaves short) and sums integers
    elsewhere (exact in fp32, one bf16 rounding). Rows no id hits and the guard rows stay bit-unchanged."""
    T, V, h = 32768, 50264, 768
    big_id = 50256
    ids, short_ids, lens = X.embedding_bwd_ids(T, V, big_id, seed=1)
    occ = X.occurrence_index(ids)
    dout = X.embedding_bwd_dout(ids, occ, h, big_id, seed=2).to(BF16).to(DEV)
    n_big = int((ids == big_id).sum())
    old = X.embedding_bwd_old(V, h, big_id, n_big, short_ids, seed=3)
    assert (n_big // 4) >= 2
    dW = guarded_2d(V, h, BF16, fill=7.0, init=old.to(BF16).to(DEV), pad_cols=0)
    ids_d = ids.to(DEV)
    ops.embedding_bwd(ids_d, dout, dW.view)
    dW.check("embedding dW guard rows", written=False)
    want = old.to(DEV).index_add(0, ids_d, dout.double()).to(BF16)
    got = dW.view
    hit = torch.zeros(V, dtype=torch.bool, device=DEV)
    hit[ids_d] = True
    fb = _first_bad(got[~hit], want[~hit])
    assert fb is None, f"embedding dW: a row no id hits changed ({fb[1]} elements)"
    bad = (bits(got) != bits(want)).any(1).nonzero().view(-1)
    if bad.numel() == 0:
        return
    r = int(bad[0])
    c = int((bits(got[r]) != bits(want[r])).nonzero()[0])
    msg = (f"embedding dW: {len(bad)} rows differ; first id {r} (run of {int((ids == r).sum())} occurrences), column {c}: "
           f"got {got[r, c].item()!r}, want {want[r, c].item()!r}")
    diff = (want[r].double() - got[r].double()).cpu()
    if r == big_id:
        short = [(cc, int(diff[cc])) for cc in range(X.EMB_BIG_COLS + -(-n_big // X.EMB_BIG_COLS)) if diff[cc] != 0]
        mods = [cc for cc, _ in short if cc < X.EMB_BIG_COLS]
        blocks = [cc - X.EMB_BIG_COLS for cc, _ in short if cc >= X.EMB_BIG_COLS]
        lost = sorted(b * X.EMB_BIG_COLS + m for b in blocks for m in mods if b * X.EMB_BIG_COLS + m < n_big)
        msg += (f"; counting columns short: {short[:12]}; occurrences lost (run-loop round q // 4 of row lane q % 4): "
                f"{[(q, q // 4, q % 4) for q in lost[:12]]}{' ...' if len(lost) > 12 else ''}")
    else:
        w = int(abs(want[r, c].double().item() - old[r, c].item()))
        gv = int(abs(got[r, c].double().item() - old[r, c].item()))
        msg += f"; occurrences lost: {[q for q in range(X.EMB_CODED_MAX) if (w >> q) & 1 and not (gv >> q) & 1]}"
    raise AssertionError(msg)
