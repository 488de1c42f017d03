"""GPU: the split-KV decode-attention kernel (fsb_attn_decode) against a plain fp64 torch formula on the same bf16 inputs.

O is the fp32 result rounded to bf16 once, so it must lie within 1 bf16 ulp of the fp64 value plus a floor of 1e-5 x the row's
max |v| (fp32 sums of the weighted values). Cache slots at and beyond kv_len hold NaN: a single read of one would poison O.
Outputs are written into NaN-guarded views (tests/guards.py)."""
import math

import pytest
import torch

from guards import Guarded, assert_ulp_close, bits
from fsb200 import lib as L
from fsb200 import ops

pytestmark = pytest.mark.gpu

LOG2E = 1.0 / math.log(2.0)


def _cap(n):
    return (n + 200 + 63) // 64 * 64     # well above kv_len, a multiple of 64


def _cache(B, cap, H, D, n, g, packed=False):
    """K and V [B, cap, H, D] bf16, slots >= n set to NaN. packed=True: two strided slices of one [B, cap, 2, H, D] buffer."""
    if packed:
        buf = torch.randn((B, cap, 2, H, D), generator=g, device="cuda").to(torch.bfloat16)
        buf[:, n:] = float("nan")
        return buf[:, :, 0], buf[:, :, 1]
    k = torch.randn((B, cap, H, D), generator=g, device="cuda").to(torch.bfloat16)
    v = torch.randn((B, cap, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k[:, n:] = float("nan")
    v[:, n:] = float("nan")
    return k, v


def _out(B, H, D):
    buf = torch.full((B + 2, H + 1, D + 16), float("nan"), dtype=torch.bfloat16, device="cuda")
    return Guarded(buf, lambda t: t[1:B + 1, :H, 8:8 + D])


def _ref(q, k, v, n, scale, mask=None, rel=None):
    """fp64: (O [B, H, D], lse [B, H] in log2 units, +inf where no key is visible)."""
    cap = k.shape[1]
    qd, kd, vd = q.double(), k[:, :n].double(), v[:, :n].double()
    s = torch.einsum("bhd,bkhd->bhk", qd, kd) * scale
    if rel is not None:
        s = s + rel.double()[:, torch.arange(n, device=q.device) - (n - 1) + cap - 1][None]
    if mask is not None:
        s = s.masked_fill(mask[:, None, :n] == 0, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    o = torch.einsum("bhk,bkhd->bhd", p, vd)
    return o, torch.where(torch.isfinite(lse), lse * LOG2E, torch.full_like(lse, float("inf")))


def _check(q, k, v, n, scale, mask=None, rel=None, what=""):
    B, H, D = q.shape
    g = _out(B, H, D)
    kv_len = torch.tensor([n], dtype=torch.int32, device="cuda")
    _, lse = ops.attn_decode(q, k, v, kv_len, scale, kv_mask=mask, rel_bias=rel, out=g.view)
    torch.cuda.synchronize()
    g.check(what)
    o_ref, lse_ref = _ref(q, k, v, n, scale, mask, rel)
    vmax = v[:, :n].float().nan_to_num(0.0).abs().amax(dim=(1, 3)).double()[:, :, None]   # [B, H, 1]
    assert_ulp_close(g.view, o_ref, what, floor=1e-5 * vmax)
    fin = torch.isfinite(lse_ref)
    assert torch.equal(torch.isfinite(lse), fin), what
    assert torch.allclose(lse.double()[fin], lse_ref[fin], rtol=1e-5, atol=1e-4), what
    return g.view.clone(), lse


# (B, H): 64 x 16 = 1024 rows gives one split on a 132-SM card; 1 x 12 and 4 x 16 give many.
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000, 4096])
@pytest.mark.parametrize("B,H", [(1, 12), (4, 16), (64, 16)])
def test_decode_matches_fp64_and_never_reads_past_kv_len(D, n, B, H):
    if B == 64 and n == 4096:
        pytest.skip("covered at the smaller batches (one split at 4096 keys is the same code path as at 1000)")
    g = torch.Generator(device="cuda").manual_seed(n * 7 + D + B)
    cap = _cap(n)
    q = torch.randn((B, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k, v = _cache(B, cap, H, D, n, g)
    _check(q, k, v, n, 1.0 / math.sqrt(D), what=f"D{D} n{n} B{B} H{H}")


def test_split_counts_cover_one_and_many():
    one = L.load().fsb_attn_decode_workspace_bytes(64, 16, 64, _cap(1000)) // (64 * 16 * 66 * 4)
    many = L.load().fsb_attn_decode_workspace_bytes(1, 12, 64, _cap(1000)) // (12 * 66 * 4)
    assert one == 1 and many > 4, (one, many)


@pytest.mark.parametrize("D", [64, 128])
def test_left_padding_mask_and_fully_masked_row(D):
    B, H, n = 3, 12, 150
    cap = _cap(n)
    g = torch.Generator(device="cuda").manual_seed(11)
    q = torch.randn((B, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k, v = _cache(B, cap, H, D, n, g)
    mask = torch.ones((B, cap), dtype=torch.uint8, device="cuda")
    mask[0, :17] = 0         # left padding
    mask[1, :] = 0           # sees nothing: O = 0, lse = +inf
    mask[2, 40:90] = 0
    o, lse = _check(q, k, v, n, 1.0 / math.sqrt(D), mask=mask, what=f"mask D{D}")
    assert torch.equal(o[1], torch.zeros_like(o[1])) and bool(torch.isinf(lse[1]).all()) and bool((lse[1] > 0).all())


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("n", [1, 37, 256, 320])
def test_rel_bias_at_several_query_positions(D, n):
    from fsb200.models import t5_bias as TB
    B, H, cap = 2, 6, 320
    g = torch.Generator(device="cuda").manual_seed(n)
    table = torch.randn((32, H), generator=g, device="cuda") * 2.0
    rel = TB.rel_bias_vector(table, cap, cap, False)
    q = torch.randn((B, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k, v = _cache(B, cap, H, D, n, g)
    _check(q, k, v, n, 1.0, rel=rel, what=f"rel D{D} n{n}")


@pytest.mark.parametrize("D", [64, 128])
def test_strided_views_of_packed_projection(D):
    B, H, n = 5, 16, 700
    cap = _cap(n)
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = torch.randn((B, 3, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k, v = _cache(B, cap, H, D, n, g, packed=True)
    _check(qkv[:, 0], k, v, n, 0.125, what=f"packed D{D}")


def test_two_calls_identical_bits():
    B, H, D, n = 2, 12, 64, 3000
    cap = _cap(n)
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn((B, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k, v = _cache(B, cap, H, D, n, g)
    kv_len = torch.tensor([n], dtype=torch.int32, device="cuda")
    o1, l1 = ops.attn_decode(q, k, v, kv_len, 0.125)
    o2, l2 = ops.attn_decode(q, k, v, kv_len, 0.125)
    assert torch.equal(bits(o1), bits(o2)) and torch.equal(bits(l1), bits(l2))


def _raw(q, k, v, o, kv_len, ws, ws_bytes):
    B, H, D = q.shape
    return L.load().fsb_attn_decode(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), None, B, H, D, k.shape[1],
                                    kv_len.data_ptr(), q.stride(0), q.stride(1), k.stride(0), k.stride(1), k.stride(2),
                                    v.stride(0), v.stride(1), v.stride(2), o.stride(0), o.stride(1), 0.125, None, None,
                                    ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)


def test_workspace_bytes_exact_and_short_workspace_refused():
    B, H, D, n = 1, 12, 128, 1000
    cap = (n + 63) // 64 * 64                       # kv_len fills every split: every byte of the workspace is written
    g = torch.Generator(device="cuda").manual_seed(9)
    q = torch.randn((B, H, D), generator=g, device="cuda").to(torch.bfloat16)
    k, v = _cache(B, cap, H, D, cap, g)
    kv_len = torch.tensor([cap], dtype=torch.int32, device="cuda")
    nbytes = int(L.load().fsb_attn_decode_workspace_bytes(B, H, D, cap))
    assert nbytes > 0 and nbytes % 4 == 0
    nf = nbytes // 4
    ws = Guarded(torch.full((nf + 64,), float("nan"), dtype=torch.float32, device="cuda"), lambda t: t[32:32 + nf])
    o = _out(B, H, D)
    assert _raw(q, k, v, o.view, kv_len, ws.view, nbytes) == 0
    torch.cuda.synchronize()
    ws.check("workspace")                            # all of it written, nothing beyond it
    o.check("out")
    o2 = _out(B, H, D)
    assert _raw(q, k, v, o2.view, kv_len, ws.view, nbytes - 16) == -1   # FSB_ERR_INVALID
    assert "workspace" in L.last_error()
    torch.cuda.synchronize()
    o2.check("short workspace: no launch", written=False)
    assert bool(torch.isnan(o2.view.float()).all())


def test_head_dim_96_rejected():
    q = torch.zeros((1, 2, 96), dtype=torch.bfloat16, device="cuda")
    k = torch.zeros((1, 64, 2, 96), dtype=torch.bfloat16, device="cuda")
    kv_len = torch.tensor([3], dtype=torch.int32, device="cuda")
    assert L.load().fsb_attn_decode_workspace_bytes(1, 2, 96, 64) == 0
    with pytest.raises(RuntimeError, match="head_dim 96"):
        ops.attn_decode(q, k, k, kv_len, 1.0)


def test_combine_merges_the_splits_in_index_order():
    """q = 0 makes every probability 1/kv_len and every partial's running max 0, so the combine is a plain fp32 sum of the
    partials. Chunks of +X, -X and y (X = 2^24, y = 0.5) sum to 64 y only in split order 0, 1, 2; any other order rounds
    the y chunk away against 64 X. The output pins the order: y / 3, rounded to bf16."""
    B, H, D, cap = 1, 12, 64, 192
    splits = L.load().fsb_attn_decode_workspace_bytes(B, H, D, cap) // (B * H * (D + 2) * 4)
    assert splits == 3
    q = torch.zeros((B, H, D), dtype=torch.bfloat16, device="cuda")
    k = torch.ones((B, cap, H, D), dtype=torch.bfloat16, device="cuda")
    v = torch.empty((B, cap, H, D), dtype=torch.bfloat16, device="cuda")
    v[:, :64], v[:, 64:128], v[:, 128:] = 2.0 ** 24, -(2.0 ** 24), 0.5
    kv_len = torch.tensor([cap], dtype=torch.int32, device="cuda")
    o, lse = ops.attn_decode(q, k, v, kv_len, 1.0)
    want = torch.full_like(o, 0.5 / 3)
    assert torch.equal(bits(o), bits(want)), o.flatten()[:4]
    assert torch.allclose(lse, torch.full_like(lse, math.log2(cap)))
