"""Parity of the per-layer kernels of LLaMA and mT5 that the GEMM / attention / LayerNorm tests do not cover: RMSNorm
forward and backward over every template instance of the norm kernels, rotary embedding on the packed QKV buffer, the
gated and plain activations with the fused bias gradient, the sorted embedding backward and the gradient-clip coefficient.

Each test compares with a plain fp64 torch formula of the same operation on the same bf16 inputs. Outputs the tests pass in
are views of NaN-filled (or, when accumulated into, finite) buffers with guards (tests/guards.py).

Tolerance model:
- A kernel that computes in fp32 and rounds to bf16 once is held to 1 bf16 ulp of the fp64 value (the rounding costs 1/2
  ulp; the fp32 arithmetic before it is ~2^-16 of an ulp) plus an absolute floor for fp32 cancellation:
  - activations: ACT_FLOOR = 2^-18 times the largest factor the activation (or its derivative) is multiplied by: 1 for
    act(x), |dy| for dy * act'(x), |up| / |dout| / |dout * up| for the GLU outputs. It covers fp32 cancellation in
    1 + tanh(u) and 1 - tanh(u)^2 of tanh-GeLU for x in [-5.2, -3], where tanh lies within a few fp32 ulps of -1: there
    act' (~1e-6) is only known to ~2^-23 * |x| * (0.8 + 0.107 x^2) <= 2^-19 (below -5.2 tanh is exactly -1 and the true
    value is under 1e-8); likewise near the zero of SiLU's derivative (x ~ -1.28);
  - rotary embedding: 1e-6 * max|ref| of the tensor (fp32 cancellation in x1 cos - x2 sin);
  - RMSNorm dx: 1e-5 * the row's max|rstd * (g - xhat * mean(g * xhat))|, for the fp32 row sum inside mean(g * xhat).
- Where both sides round the same fp32 value once, the result must be bit-identical (RMSNorm y given the kernel's rstd,
  act_bwd_bias dx against act_bwd, the residual sum).
- Sums of many terms (weight and bias gradients, embedding rows): fp32 accumulation noise, 2e-6 * sum|terms|, plus 1 ulp of
  the result when it is stored in bf16.
"""
import pytest
import torch

from guards import assert_ulp_close, bf16_ulp, bits, guarded_1d, guarded_2d

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"
ACC_REL = 2e-6   # fp32 accumulation noise relative to sum|terms|
ACT_FLOOR = 2.0 ** -18


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return int(L.load().fsb_num_sms())


def _floor(ref, rel=1e-6):
    return rel * ref.double().abs().max().item()


def _sum_close(got, ref, abs_sum, what):
    """got: fp32 or bf16 sums; ref: fp64 sums; abs_sum: fp64 sum of |terms| (including any value accumulated onto)."""
    tol = ACC_REL * abs_sum + 1e-30
    if got.dtype == torch.bfloat16:
        tol = tol + bf16_ulp(ref)
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} sums off; max err {err.max().item():.4g}"


# ----------------------------------------------------------------------------------------------------------- RMSNorm
def _norm_shape(cols, max_vpt):
    """(threads per row, 16-byte vectors per thread) as norm.cu's norm_shape (max_vpt 4) / norm_shape_bwd (3) pick them."""
    nvec, tpr = cols // 8, 32
    while tpr < 256 and -(-nvec // tpr) > max_vpt:
        tpr *= 2
    return tpr, -(-nvec // tpr)


# FSB_NORM_DISPATCH reaches 14 (TPR, VPT) instances per direction; this list runs each of them:
#   cols   fwd       bwd          cols   fwd       bwd
#   8      (32,1)    (32,1)       3080   (128,4)   (256,2)
#   264    (32,2)    (32,2)       4096   (128,4)   (256,2)
#   512    (32,2)    (32,2)       5120   (256,3)   (256,3)
#   520    (32,3)    (32,3)       6152   (256,4)   (256,4)
#   768    (32,3)    (32,3)       8192   (256,4)   (256,4)
#   776    (32,4)    (64,2)       10240  (256,5)   (256,5)
#   1024   (32,4)    (64,2)       12288  (256,6)   (256,6)
#   1032   (64,3)    (64,3)       14336  (256,7)   (256,7)
#   1544   (64,4)    (128,2)      16384  (256,8)   (256,8)
#   2048   (64,4)    (128,2)
#   2056   (128,3)   (128,3)
# 264, 520, 776, 1032, 1544, 2056, 3080 and 6152 leave idle threads in the last vector slot. 512, 768, 1024, 2048 (mT5),
# 4096 and 5120 (LLaMA-7B / 13B) are the model widths.
NORM_WIDTHS = [8, 264, 512, 520, 768, 776, 1024, 1032, 1544, 2048, 2056, 3080, 4096, 5120, 6152, 8192, 10240, 12288,
               14336, 16384]
NORM_INSTANCES = {d: {(32, 1), (32, 2), (32, 3), (64, 3), (128, 3)} | ({(32, 4), (64, 4), (128, 4)} if d == 4 else
                                                                       {(64, 2), (128, 2), (256, 2)})
                  | {(256, v) for v in range(3, 9)} for d in (4, 3)}


def test_norm_widths_cover_every_instance():
    for max_vpt in (4, 3):
        assert {_norm_shape(c, max_vpt) for c in NORM_WIDTHS} == NORM_INSTANCES[max_vpt]


def _norm_rows(cols):
    """1, RPC - 1, a non-multiple of RPC (rows per CTA), and more rows than 2 passes of the 4 * SMs CTA grid cover, so
    every CTA of both kernels runs the grid-stride loop at least twice (the forward's RPC is the larger of the two)."""
    rpc = 256 // _norm_shape(cols, 4)[0]
    big = 9 * _sms() * rpc + 3
    assert big > 2 * 4 * _sms() * rpc
    return sorted({1, max(rpc - 1, 1), 2 * rpc + 1, big})


def _rms_inputs(rows, cols, seed):
    x = _rand(rows, cols, seed=seed)
    r = _rand(rows, cols, seed=seed + 1)
    if rows >= 3:
        x[rows // 2] = 0                          # eps dominates: rstd = eps^-1/2, y = 0
        r[rows // 2] = 0
    x[1::7] *= 100                                # large mean square
    return x, r


@pytest.mark.parametrize("cols", NORM_WIDTHS)
def test_rmsnorm_fwd_bwd_parity(cols):
    """y = scale * bf16(x * rstd) (norms.py: normalise in fp32, cast, then the bf16 product), with and without the fused
    residual; dx = rstd * (g - xhat * mean(g * xhat)) + dres, g = dy * scale; dscale = sum_rows dy * bf16(x * rstd), fp32
    and bf16, written and accumulated. Last case of each width runs the grid-stride loop more than once."""
    eps = 1e-6
    scale = (1 + 0.2 * torch.randn(cols, generator=torch.Generator().manual_seed(cols))).to(torch.bfloat16).to(DEV)
    for k, rows in enumerate(_norm_rows(cols)):
        with_res, with_dres = k % 2 == 0, k in (1, 2)
        wdt, acc = (torch.float32, torch.bfloat16)[k % 2], k >= 2
        what = f"rows={rows} cols={cols} residual={with_res} dres={with_dres} {wdt} accumulate={acc}"
        x, r = _rms_inputs(rows, cols, seed=rows)
        n = rows * cols
        y, st = guarded_1d(n, torch.bfloat16), guarded_1d(rows, torch.float32)
        xs = guarded_1d(n, torch.bfloat16) if with_res else None
        L.call("fsb_rmsnorm_fwd", x.data_ptr(), r.data_ptr() if with_res else None, scale.data_ptr(), y.view.data_ptr(),
               xs.view.data_ptr() if with_res else None, st.view.data_ptr(), rows, cols, eps, _stream())
        y.check(f"rmsnorm y {what}")
        st.check(f"rmsnorm rstd {what}")
        if with_res:
            xs.check(f"rmsnorm sum_out {what}")
            xsum = xs.view.view(rows, cols)
            assert torch.equal(bits(xsum), bits((x.float() + r.float()).to(torch.bfloat16))), \
                f"sum_out is not the bf16 sum x + residual ({what})"
        else:
            xsum = x
        rstd = st.view
        xd = xsum.double()
        rstd_ref = 1.0 / torch.sqrt(xd.pow(2).mean(1) + eps)
        rel = ((rstd.double() - rstd_ref).abs() / rstd_ref).max().item()
        assert rel <= 1e-5, f"rstd off by {rel:.3g} relative ({what})"
        yh = (xsum.float() * rstd[:, None]).to(torch.bfloat16)      # bf16(x * rstd) with the kernel's rstd
        assert torch.equal(bits(y.view.view(rows, cols)), bits(yh * scale)), f"y != scale * bf16(x * rstd) ({what})"
        if rows >= 3:
            assert rstd[rows // 2].item() == pytest.approx(eps ** -0.5, rel=1e-5)

        # backward
        dy = _rand(rows, cols, seed=rows + 7)
        dres = _rand(rows, cols, seed=rows + 8) if with_dres else None
        dx = guarded_1d(n, torch.bfloat16)
        init = torch.full((cols,), 0.5) if acc else None
        dsc = guarded_1d(cols, wdt, fill=0.0 if acc else float("nan"), init=init)
        ws_bytes = int(L.load().fsb_norm_bwd_workspace_bytes(rows, cols, 0))
        ws = ops.workspace(ws_bytes, xsum.device, "norm")

        def bwd(dx_out, dscale_out):
            L.call("fsb_rmsnorm_bwd", dy.data_ptr(), xsum.data_ptr(), scale.data_ptr(), rstd.data_ptr(),
                   dres.data_ptr() if with_dres else None, dx_out.data_ptr(), dscale_out.data_ptr(),
                   L.F32 if wdt == torch.float32 else L.BF16, int(acc), ws.data_ptr(), ws_bytes, rows, cols, _stream())

        bwd(dx.view, dsc.view)
        dx.check(f"rmsnorm dx {what}")
        dsc.check(f"rmsnorm dscale {what}", written=not acc)
        rs = rstd.double()[:, None]
        g = dy.double() * scale.double()
        xhat = xd * rs
        core = rs * (g - xhat * (g * xhat).mean(1, keepdim=True))
        want = core + (dres.double() if with_dres else 0.0)
        floor = 1e-5 * core.abs().amax(1, keepdim=True)
        assert_ulp_close(dx.view.view(rows, cols), want, f"rmsnorm dx {what}", floor=floor)
        terms = dy.double() * yh.double()
        _sum_close(dsc.view, terms.sum(0) + (0.5 if acc else 0.0), terms.abs().sum(0) + (0.5 if acc else 0.0),
                   f"rmsnorm dscale {what}")
        if rows == _norm_rows(cols)[-1]:
            dx2 = torch.empty_like(dx.view)
            dsc2 = torch.full((cols,), 0.5, dtype=wdt, device=DEV) if acc else torch.empty(cols, dtype=wdt, device=DEV)
            bwd(dx2, dsc2)
            assert torch.equal(bits(dx2), bits(dx.view)) and torch.equal(bits(dsc2), bits(dsc.view)), \
                f"two identical backward calls differ ({what})"


@pytest.mark.parametrize("rows,cols", [(3, 8), (1000, 5120), (4096, 1024)])
def test_rmsnorm_bwd_workspace_is_exact(rows, cols):
    """fsb_norm_bwd_workspace_bytes is exactly what the backward uses: that many bytes (a view inside a guarded buffer)
    works and every byte is written, 16 fewer is refused on the host with a message about the workspace."""
    x, dy = _rand(rows, cols, seed=1), _rand(rows, cols, seed=2)
    scale = _rand(cols, seed=3)
    _, rstd, _ = ops.rmsnorm_fwd(x, scale, 1e-6)
    need = int(L.load().fsb_norm_bwd_workspace_bytes(rows, cols, 0))
    assert need > 0 and need % 4 == 0
    ws = guarded_1d(need // 4, torch.float32)
    dx, dsc = torch.empty_like(x), torch.empty(cols, dtype=torch.float32, device=DEV)
    args = (dy.data_ptr(), x.data_ptr(), scale.data_ptr(), rstd.data_ptr(), None, dx.data_ptr(), dsc.data_ptr(), L.F32, 0,
            ws.view.data_ptr())
    L.call("fsb_rmsnorm_bwd", *args, need, rows, cols, _stream())
    ws.check("rmsnorm workspace")
    with pytest.raises(RuntimeError, match="workspace"):
        L.call("fsb_rmsnorm_bwd", *args, need - 16, rows, cols, _stream())


# ----------------------------------------------------------------------------------------------------------- rotary
def _rope_tables(max_pos, hd, base=10000):
    """fp32 cos / sin tables [max_pos, hd/2] built as the LLaMA model builds them (llama.py _ensure_rope)."""
    inv_freq = 1.0 / (base ** (torch.arange(0, hd, 2).float() / hd))
    freqs = torch.einsum("i,j->ij", torch.arange(max_pos, dtype=torch.float32), inv_freq)
    return freqs.cos().contiguous().to(DEV), freqs.sin().contiguous().to(DEV)


def _positions(pattern, T, max_pos, seed):
    g = torch.Generator().manual_seed(seed)
    if pattern == "arange":                        # position_ids = arange(S) over the batch
        B = max(1, T // 2048) if T >= 2048 else (3 if T % 3 == 0 else 1)
        return torch.arange(T // B).repeat(B).to(DEV)
    if pattern == "leftpad":                       # prefill with left padding: cumsum(mask) - 1, pads -> 1
        B = 2 if T % 2 == 0 else 1
        S = T // B
        mask = torch.ones(B, S, dtype=torch.long)
        for b in range(B):
            mask[b, :int(torch.randint(0, S // 2 + 1, (1,), generator=g))] = 0
        pos = mask.cumsum(-1) - 1
        pos.masked_fill_(mask == 0, 1)
        return pos.view(-1).to(DEV)
    pos = torch.randint(0, max_pos, (T,), generator=g)     # decode: one position per row, the table's last row included
    pos[-1] = max_pos - 1
    return pos.to(DEV)


def _rotate_half(v):
    h = v.shape[-1] // 2
    return torch.cat([-v[..., h:], v[..., :h]], -1)


def _rotate_half_t(v):   # transpose of rotate_half
    h = v.shape[-1] // 2
    return torch.cat([v[..., h:], -v[..., :h]], -1)


def _rope_ref(xs, cos, sin, pos, backward):
    """xs [T, nh, hd] bf16 -> fp64 rotate-half rotation on the fp32 tables; backward: the transpose, applied directly."""
    c = torch.cat([cos[pos], cos[pos]], -1).double()[:, None, :]
    s = torch.cat([sin[pos], sin[pos]], -1).double()[:, None, :]
    v = xs.double()
    return v * c + (_rotate_half_t(v) if backward else _rotate_half(v)) * s


def _rope_step(buf, T, nh, hd, cos, sin, pos, slot, backward, what):
    """Rotate slot 0 (q) or 1 (k) of the packed [T, nh, 3, hd] rows of buf[1:T+1] (rows 0 and T+1 are guards); check
    the slot against the reference and every other element for bit equality. Rows with a position outside the table
    must have exactly their head slices of this slot set to NaN."""
    before = buf.clone()
    xs = buf[1:T + 1, :, slot].clone()
    ops.rope_inplace(buf[1:T + 1].view(-1), cos, sin, pos, nh, hd, 3 * nh * hd, 3 * hd, backward=backward,
                     offset=slot * hd)
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[1:T + 1, :, slot] = False
    assert torch.equal(bits(buf)[keep], bits(before)[keep]), f"{what}: elements outside the rotated slot changed"
    bad = (pos < 0) | (pos >= cos.shape[0])
    got = buf[1:T + 1, :, slot]
    if bad.any():
        assert torch.isnan(got[bad].float()).all(), f"{what}: a row with an out-of-range position is not all NaN"
    ok = ~bad
    ref = _rope_ref(xs[ok], cos, sin, pos[ok], backward)
    assert_ulp_close(got[ok], ref, what, floor=_floor(ref))


@pytest.mark.parametrize("hd,nh,T,pattern", [(64, 1, 1, "decode"), (64, 5, 300, "leftpad"), (64, 40, 4096, "arange"),
                                             (128, 1, 1, "decode"), (128, 5, 300, "arange"), (128, 40, 4096, "leftpad"),
                                             (128, 40, 4096, "decode"), (16, 5, 77, "decode"), (96, 40, 300, "leftpad")])
def test_rope_packed_qkv(hd, nh, T, pattern):
    """LLaMA layout: rows of [nh, 3, hd] (q, k, v per head), row_stride 3*nh*hd, head_stride 3*hd. Forward on q, then the
    backward (transposed rotation) on k, each against its own fp64 formula; v and the guard rows stay bit-unchanged."""
    max_pos = 2048
    cos, sin = _rope_tables(max_pos, hd)
    pos = _positions(pattern, T, max_pos, seed=T + nh)
    assert int(pos.min()) >= 0 and int(pos.max()) < max_pos
    if T == 4096:
        assert T * nh * hd // 16 > 16 * _sms() * 256, "the grid-stride loop should run more than once"
    buf = _rand(T + 2, nh, 3, hd, seed=hd + T)
    _rope_step(buf, T, nh, hd, cos, sin, pos, 0, False, f"rope fwd q hd={hd} nh={nh} T={T} {pattern}")
    _rope_step(buf, T, nh, hd, cos, sin, pos, 1, True, f"rope bwd k hd={hd} nh={nh} T={T} {pattern}")


def test_rope_out_of_range_positions_are_nan():
    """A position outside [0, max_pos) never reads the tables: that row's head slices become NaN (the documented
    contract), every other row is rotated normally and nothing else changes."""
    T, nh, hd, max_pos = 64, 5, 128, 256
    cos, sin = _rope_tables(max_pos, hd)
    pos = _positions("decode", T, max_pos, seed=5)
    pos[3], pos[10], pos[T - 1] = -1, max_pos, max_pos
    buf = _rand(T + 2, nh, 3, hd, seed=6)
    _rope_step(buf, T, nh, hd, cos, sin, pos, 0, False, "rope fwd q, out-of-range rows")
    _rope_step(buf, T, nh, hd, cos, sin, pos, 1, True, "rope bwd k, out-of-range rows")


# ----------------------------------------------------------------------------------------------------------- activations
ACTS = {0: lambda x: torch.nn.functional.silu(x),
        1: lambda x: torch.nn.functional.gelu(x, approximate="tanh"),
        2: lambda x: torch.nn.functional.gelu(x),
        3: torch.tanh}


def _act_inputs(n, seed):
    """N(0, 2^2) with every 16th value spread over [-30, 30] (saturated sigmoid / tanh), and values at the zeros of the
    derivatives: SiLU' at x ~ -1.2785, tanh-GeLU' at x ~ -0.7518, and the -3..-7 tail where 1 + tanh cancels."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g) * 2
    i = torch.arange(n)
    for k, fill in ((0, lambda m: torch.rand(m, generator=g) * 60 - 30),
                    (1, lambda m: -1.2785 + 0.01 * torch.randn(m, generator=g)),
                    (2, lambda m: -0.7518 + 0.01 * torch.randn(m, generator=g)),
                    (3, lambda m: -3 - 4 * torch.rand(m, generator=g))):
        sel = i % 16 == k
        x[sel] = fill(int(sel.sum()))
    return x.to(torch.bfloat16).to(DEV)


def _strided(rows, cols, ld, seed, off=8):
    """[rows, cols] bf16 view with row stride ld into a random buffer (the rest of each row is other data)."""
    buf = _rand(rows, ld, seed=seed)
    return buf[:, off:off + cols]


def _glu_ref(act, gate, up, dout):
    gd, ud = gate.double().requires_grad_(True), up.double().requires_grad_(True)
    out = ACTS[act](gd) * ud
    out.backward(dout.double())
    return out.detach(), gd.grad, ud.grad


def _glu_check(act, gate, up, dout, out, dgate, dup, what):
    o_ref, dg_ref, du_ref = _glu_ref(act, gate, up, dout)
    big = lambda t: ACT_FLOOR * t.double().abs().max().item()   # noqa: E731
    assert_ulp_close(out, o_ref, f"glu out {what}", floor=big(up))
    assert_ulp_close(dgate, dg_ref, f"glu dgate {what}", floor=big(dout.double() * up.double()))
    assert_ulp_close(dup, du_ref, f"glu dup {what}", floor=big(dout))


@pytest.mark.parametrize("act,cols", [(0, 13824), (0, 11008), (1, 2816), (1, 1024)])
@pytest.mark.parametrize("rows", [1, 7, 300, 2048])
def test_glu_strided_operands(act, cols, rows):
    """SwiGLU at LLaMA-13B / 7B widths, gated tanh-GeLU at mT5 widths. (a) gate and up in separate buffers with row
    strides ld_gate < ld_up, dout / dgate / dup with three other strides; (b) the model's form: column halves of one
    [rows, 2 ff] buffer, the two gradients into the halves of another."""
    what = f"act={act} rows={rows} cols={cols}"
    x = _act_inputs(rows * cols, seed=rows + cols).view(rows, cols)
    gate = _strided(rows, cols, cols + 8, seed=1)
    gate.copy_(x)
    up = _strided(rows, cols, cols + 56, seed=2)
    dout = _strided(rows, cols, cols + 40, seed=3)
    out = guarded_2d(rows, cols, torch.bfloat16)
    L.call("fsb_glu_fwd", act, gate.data_ptr(), up.data_ptr(), out.view.data_ptr(), rows, cols, gate.stride(0),
           up.stride(0), out.view.stride(0), _stream())
    out.check(f"glu out {what}")
    dg = guarded_2d(rows, cols, torch.bfloat16, pad_cols=8)
    du = guarded_2d(rows, cols, torch.bfloat16, pad_cols=16)
    assert len({gate.stride(0), up.stride(0), dout.stride(0), dg.view.stride(0), du.view.stride(0)}) == 5
    ops.glu_bwd(act, dout, gate, up, dg.view, du.view)
    dg.check(f"glu dgate {what}")
    du.check(f"glu dup {what}")
    _glu_check(act, gate, up, dout, out.view, dg.view, du.view, what)

    gu = torch.cat([x, up], 1)
    dgu = guarded_2d(rows, 2 * cols, torch.bfloat16)
    out2 = ops.glu_fwd(act, gu[:, :cols], gu[:, cols:])
    assert torch.equal(bits(out2), bits(out.view)), f"glu out depends on the operand layout ({what})"
    ops.glu_bwd(act, dout.contiguous(), gu[:, :cols], gu[:, cols:], dgu.view[:, :cols], dgu.view[:, cols:])
    dgu.check(f"glu halves {what}")
    assert torch.equal(bits(dgu.view[:, :cols]), bits(dg.view)) and torch.equal(bits(dgu.view[:, cols:]), bits(du.view)), \
        f"glu gradients into the halves of one buffer differ from separate buffers ({what})"


def _act_n_big():
    """A multiple of 8 with more 8-element vectors than the elementwise grid (16 * SMs CTAs of 256 threads) covers."""
    return (2 * 16 * _sms() * 256 + 37) * 8


@pytest.mark.parametrize("act", [0, 1, 2, 3])
@pytest.mark.parametrize("big", [False, True])
def test_act_fwd_bwd(act, big):
    """y = act(x), dx = dy * act'(x) for SiLU, tanh-GeLU, erf-GeLU and tanh (BERT pooler)."""
    if big:
        n = _act_n_big()
        x = _act_inputs(n, seed=act)
    else:
        n = 8
        x = torch.tensor([-30.0, -5.0, -1.2785, -0.7518, 0.0, 0.5, 3.0, 30.0]).to(torch.bfloat16).to(DEV)
    dy = _rand(n, seed=act + 10)
    y, dx = guarded_1d(n, torch.bfloat16), guarded_1d(n, torch.bfloat16)
    L.call("fsb_act_fwd", act, x.data_ptr(), y.view.data_ptr(), n, _stream())
    L.call("fsb_act_bwd", act, dy.data_ptr(), x.data_ptr(), dx.view.data_ptr(), n, _stream())
    y.check(f"act {act} y")
    dx.check(f"act {act} dx")
    xd = x.double().requires_grad_(True)
    yref = ACTS[act](xd)
    yref.backward(dy.double())
    assert_ulp_close(y.view, yref.detach(), f"act {act} fwd n={n}", floor=ACT_FLOOR)
    assert_ulp_close(dx.view, xd.grad, f"act {act} bwd n={n}", floor=ACT_FLOOR * dy.double().abs().max().item())


@pytest.mark.parametrize("rows", [1, 7, 8, 9, 15, 16, 17, 1000, 8192])
@pytest.mark.parametrize("cols", [8, 264, 3072, 3080])
def test_act_bwd_bias(rows, cols):
    """dx = dy * act'(x) bit-equal to act_bwd, and dbias (+)= the fp32 column sum of the bf16 dx it stored, for every
    strip shape of the two-rows-in-flight loop (rows < 16, not a multiple of 8 or 16, many strips); deterministic."""
    n = rows * cols
    x = _act_inputs(n, seed=rows * cols).view(rows, cols)
    dy = _rand(rows, cols, seed=rows + cols)
    nbytes = int(L.load().fsb_act_bwd_bias_workspace_bytes(rows, cols))
    ws = ops.workspace(nbytes, x.device, "act_bwd_bias")
    for act, wdt, acc in ((1, torch.float32, False), (2, torch.bfloat16, True), (3, torch.bfloat16, False),
                          (1, torch.float32, True)):
        what = f"act={act} rows={rows} cols={cols} {wdt} accumulate={acc}"
        dx = guarded_1d(n, torch.bfloat16)
        init = torch.linspace(-2, 2, cols) if acc else None
        db = guarded_1d(cols, wdt, fill=0.0 if acc else float("nan"), init=init)

        def run(dx_out, db_out):
            L.call("fsb_act_bwd_bias", act, dy.data_ptr(), x.data_ptr(), dx_out.data_ptr(), rows, cols, db_out.data_ptr(),
                   L.F32 if wdt == torch.float32 else L.BF16, int(acc), ws.data_ptr(), nbytes, _stream())

        run(dx.view, db.view)
        dx.check(f"act_bwd_bias dx {what}")
        db.check(f"act_bwd_bias dbias {what}", written=not acc)
        sep = ops.act_bwd(act, dy, x)
        assert torch.equal(bits(dx.view.view(rows, cols)), bits(sep)), f"dx differs from act_bwd ({what})"
        d = sep.double()
        base = init.to(DEV).to(wdt).double() if acc else 0.0
        _sum_close(db.view, d.sum(0) + base, d.abs().sum(0) + (base.abs() if acc else 0.0), f"act_bwd_bias dbias {what}")
        dx2 = torch.empty_like(dx.view)
        db2 = init.to(DEV).to(wdt) if acc else torch.empty(cols, dtype=wdt, device=DEV)
        run(dx2, db2)
        assert torch.equal(bits(dx2), bits(dx.view)) and torch.equal(bits(db2), bits(db.view)), \
            f"two identical act_bwd_bias calls differ ({what})"


def test_act_bwd_bias_rejects_silu():
    x, dy = _rand(16, 64, seed=1), _rand(16, 64, seed=2)
    with pytest.raises(RuntimeError, match="unsupported"):
        ops.act_bwd_bias(0, dy, x, torch.empty(64, dtype=torch.float32, device=DEV))


# ----------------------------------------------------------------------------------------------------------- embedding
@pytest.mark.parametrize("cols", [768, 776, 5120])
def test_embedding_bwd_sorted_wide_rows(cols):
    """dW[id] += sum of the id's dout rows in fp32, one bf16 rounding, at widths of one, two (the second partial) and ten
    64-vector passes; rows no id hits, and the guard rows around dW, stay bit-unchanged."""
    V, T = 32000, 700
    g = torch.Generator().manual_seed(cols)
    hot = torch.tensor([0, 1, 17, 4242, V - 1])
    ids = torch.where(torch.rand(T, generator=g) < 0.6, hot[torch.randint(0, 5, (T,), generator=g)],
                      torch.randint(0, V, (T,), generator=g)).to(DEV)
    dout = _rand(T, cols, seed=cols + 1)
    buf = _rand(V + 2, cols, seed=cols + 2)
    before = buf.clone()
    dW = buf[1:V + 1]
    ops.embedding_bwd(ids, dout, dW)
    hit = torch.zeros(V + 2, dtype=torch.bool, device=DEV)
    hit[ids + 1] = True
    assert torch.equal(bits(buf[~hit]), bits(before[~hit])), "rows no id hits (or the guard rows) changed"
    sums = torch.zeros(V, cols, dtype=torch.float64, device=DEV).index_add_(0, ids, dout.double())
    abss = torch.zeros(V, cols, dtype=torch.float64, device=DEV).index_add_(0, ids, dout.double().abs())
    rows = hit[1:V + 1]
    want = before[1:V + 1][rows].double() + sums[rows]
    assert_ulp_close(dW[rows], want, f"embedding bwd cols={cols}",
                     floor=ACC_REL * (abss[rows] + before[1:V + 1][rows].double().abs()))


# ----------------------------------------------------------------------------------------------------------- clip
@pytest.mark.parametrize("case", ["below", "above", "zero", "disabled"])
def test_clip_coef_matches_clip_grad_norm(case):
    """coef = min(1, max_norm / (||g|| + 1e-6)) as torch.nn.utils.clip_grad_norm_ applies it: exactly 1 below max_norm
    and for an all-zero gradient. max_norm <= 0 means clipping is off (coef 1), where torch would zero the gradients."""
    gen = torch.Generator().manual_seed(3)
    shapes = [(1000,), (64, 68), (4096 + 4,)]
    grads = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    target, max_norm = {"below": (0.5, 1.0), "above": (7.3, 1.0), "zero": (0.0, 1.0), "disabled": (3.0, 0.0)}[case]
    nrm = torch.sqrt(sum(g.double().pow(2).sum() for g in grads)).item()
    grads = [g * (target / nrm) for g in grads]
    flat = torch.cat([g.reshape(-1) for g in grads])
    sumsq = torch.zeros((), dtype=torch.float32, device=DEV)
    ops.sumsq(flat, sumsq)
    coef = torch.full((), float("nan"), device=DEV)
    norm = torch.full((), float("nan"), device=DEV)
    ops.clip_coef(sumsq, max_norm, coef, norm)
    want_norm = torch.sqrt(flat.double().pow(2).sum()).item()
    assert norm.item() == pytest.approx(want_norm, rel=1e-6, abs=1e-30)
    if case == "disabled":
        assert coef.item() == 1.0
        return
    params = [torch.nn.Parameter(torch.zeros_like(g)) for g in grads]
    for p, g in zip(params, grads):
        p.grad = g.clone()
    total = torch.nn.utils.clip_grad_norm_(params, max_norm)
    assert norm.item() == pytest.approx(total.item(), rel=1e-6, abs=1e-30)
    if case == "above":
        want = max_norm / (want_norm + 1e-6)
        assert coef.item() == pytest.approx(want, rel=2e-6)
        for p, g in zip(params, grads):
            assert torch.allclose(g * coef, p.grad, rtol=2e-6, atol=0)
    else:
        assert coef.item() == 1.0, f"coef {coef.item()!r} below max_norm"
        for p, g in zip(params, grads):
            assert torch.equal(p.grad, g)
