"""Inputs whose result through the GEMM, weight-only GEMM and attention kernels is known to the bit, and the fp64 reference
of each. Plain torch / numpy; nothing here calls the library. tests/test_exact_inputs_cpu.py proves every claim made below on
the CPU; tests/test_exact_*_gpu.py feed the inputs to the kernels.

Why exact inputs: on random data the honest tolerance of an fp32-accumulating kernel grows with sqrt(K) (or hides one key
among n), and one lost product or one key admitted off by one fits inside it. Here every operand is an exact bf16 value, every
partial sum in any order is an integer below 2^20 (or a dyadic number of as few bits), so fp32 accumulation is exact whatever
the order, the split or the tile walk, and the only rounding is the final store. The comparison needs no tolerance.

Conventions: the GEMM constructors return the logical A [M, K] and B [K, N] in fp64 (tests lay them out for NT / NN / TN);
attention tensors are [B, S, H, D] like the kernels' operands.
"""
import math

import numpy as np
import torch

BUDGET = 2 ** 20          # every partial sum of a GEMM construction stays below this in magnitude


# ------------------------------------------------------------------------------------------------------------ helpers
def is_bf16(t):
    """Every element of the fp64 / fp32 tensor t is exactly a bf16 value."""
    return bool(torch.equal(t.to(torch.bfloat16).to(t.dtype), t))


def bf16_of(exact):
    """Round-to-nearest-even of an exact fp64 value to bf16. The values used here (integers below 2^24, dyadic numbers of
    few bits) are exact in fp32, so going through fp32 rounds once."""
    return exact.to(torch.float32).to(torch.bfloat16)


def _from_patterns(pat):
    """Integer tensor of 16-bit patterns -> bf16 tensor with those bits."""
    return torch.from_numpy(pat.numpy().astype(np.uint16).view(np.int16)).view(torch.bfloat16)


def to_layout(layout, A, B):
    """Logical A [M, K], B [K, N] -> the two matrices as the layout stores them: NT (0) a [M, K] b [N, K]; NN (1) a [M, K]
    b [K, N]; TN (2) a [K, M] b [K, N]."""
    a = A.t() if layout == 2 else A
    b = B.t() if layout == 0 else B
    return a.contiguous(), b.contiguous()


# --------------------------------------------------------------------------------------------------------------- GEMM
def int_amax(K, budget=BUDGET):
    """Largest operand magnitude a with K * a * a < budget (at most 15: four bits per operand)."""
    return max(1, min(15, math.isqrt((budget - 1) // K)))


def int_operands(M, N, K, seed, budget=BUDGET):
    """Integer A [M, K], B [K, N] in [-a, a], a = int_amax(K): zeros and both signs occur, sum_k |A||B| <= K a^2 < budget, so
    every partial sum of A.B in any order and any split is an integer below 2^20 and exact in fp32."""
    g = torch.Generator().manual_seed(seed)
    a = int_amax(K, budget)
    A = torch.randint(-a, a + 1, (M, K), generator=g).double()
    B = torch.randint(-a, a + 1, (K, N), generator=g).double()
    return A, B


def int_vector(n, seed, amax=64):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-amax, amax + 1, (n,), generator=g).double()


POS_FIELDS = 8            # k-blocks coded in one output element: 8 fields of 3 bits = 24 bits, exact in fp32


def position_coded(M, N, K, kb=64):
    """A names one k per k-block, B codes (k-block, k inside it, column), and the product spells the blocks out in base 8.

    A[m, k] = 1 at one k of every k-block: k = kb*blk + (5 m + 3 blk) mod kb (clipped to K in a ragged last block). Column n
    looks at a window of up to 8 consecutive k-blocks starting at block w0(n) = 8 (n mod ceil(nb / 8)): B[k, n] = 8^(blk - w0) c
    with c = 1 + (n + 3 (k mod kb)) mod 7 in 1..7 for the blocks of its window and 0 for all others. So D[m, n] = sum over the
    window of 8^f c_f: field f (3 bits) of the integer D[m, n] is the code of block w0 + f. A block that is dropped reads 0 in
    its field, one that is counted twice reads 2c (a carry into the next field at worst), one read at the wrong k or column
    reads another code. Every B entry is c * 8^f <= 7 * 2^21 (three significant bits) and D < 2^24: exact. With N >= nb / 8
    the columns' windows cover every k-block."""
    nb = (K + kb - 1) // kb
    nwin = (nb + POS_FIELDS - 1) // POS_FIELDS
    A = torch.zeros(M, K, dtype=torch.float64)
    m = torch.arange(M)
    for blk in range(nb):
        A[m, torch.clamp(kb * blk + (5 * m + 3 * blk) % kb, max=K - 1)] = 1.0
    k = torch.arange(K)[:, None]
    n = torch.arange(N)[None, :]
    field = k // kb - POS_FIELDS * (n % nwin)
    c = 1 + (n + 3 * (k % kb)) % 7
    B = torch.where((field >= 0) & (field < POS_FIELDS), 8.0 ** field.clamp(0, POS_FIELDS - 1).double() * c.double(), 0.0)
    return A, B.double()


def position_decode(got, want):
    """First element where the integer matrices differ, as text naming the row, column and the k-block fields that differ."""
    bad = (got != want).nonzero()
    if bad.numel() == 0:
        return None
    m, n = (int(x) for x in bad[0])
    g, w = int(got[m, n]), int(want[m, n])
    fields = [(f, (g >> 3 * f) & 7, (w >> 3 * f) & 7) for f in range(POS_FIELDS) if (g >> 3 * f) & 7 != (w >> 3 * f) & 7]
    return m, n, fields, len(bad)


def position_window_start(n, K, kb=64):
    """First k-block of column n's window."""
    nb = (K + kb - 1) // kb
    return POS_FIELDS * (n % ((nb + POS_FIELDS - 1) // POS_FIELDS))


def normal_bf16_patterns(rows, cols, seed):
    """[rows, cols] bf16 of random *normal* bit patterns over the whole exponent range (biased exponent 1..254, random sign
    and mantissa): no zero, subnormal, inf or NaN."""
    g = torch.Generator().manual_seed(seed)
    exp = torch.randint(1, 255, (rows, cols), generator=g)
    man = torch.randint(0, 128, (rows, cols), generator=g)
    sgn = torch.randint(0, 2, (rows, cols), generator=g)
    return _from_patterns((sgn << 15) | (exp << 7) | man)


def row_selector(M, K, seed):
    """A [M, K] with one 1 per row at column sel[m] (a seeded map onto the K rows of B): A.B copies rows of B."""
    g = torch.Generator().manual_seed(seed)
    sel = torch.randint(0, K, (M,), generator=g)
    A = torch.zeros(M, K, dtype=torch.float64)
    A[torch.arange(M), sel] = 1.0
    return A, sel


def gelu_sweep_values():
    """Every bf16 value x with |x| in {0} or [2^-126, 128] (all normal values up to 128, both signs, and zero), arranged as
    X [64, N]: column n holds 64 consecutive values of one sign in increasing magnitude (the last column of a sign repeats its
    last value; two columns are all zero). Also base [N], the first value of each column: X - base is exactly representable in
    bf16 (at most 63 steps of the column's ulp, the steps doubling at most once) and (X - base) + base == X exactly in fp32."""
    mags = torch.arange(0x0080, 0x4300 + 1, dtype=torch.int32)            # 2^-126 .. 128.0
    cols = []
    for sign in (0, 0x8000):
        pat = mags | sign
        pad = (-len(pat)) % 64
        pat = torch.cat([pat, pat[-1:].expand(pad)])
        cols.append(pat.view(-1, 64))
    cols.append(torch.zeros(2, 64, dtype=torch.int32))      # two zero columns: N = 536, a multiple of 8
    pat = torch.cat(cols).t().contiguous()                                 # [64, N]
    X = _from_patterns(pat).double()
    return X, X[0].clone()


def gelu_tanh(x):
    """0.5 x (1 + tanh u) written as x / (1 + exp(-2 u)): 1 + tanh u cancels to nothing in the negative tail even in fp64."""
    u = math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)
    return x / (1 + torch.exp(-2 * u))


def gelu_erf(x):
    """0.5 x erfc(-x / sqrt 2): erfc keeps the negative tail's digits, which 1 + erf would cancel away."""
    return 0.5 * x * torch.special.erfc(-x / math.sqrt(2))


# --------------------------------------------------------------------------------------------------- weight-only GEMMs
def wq_int_operands(m, n, k, qmax, seed, budget=BUDGET):
    """Integer activations A [m, k], hand-built codes Q [n, k] over the full range [-qmax, qmax] (127 or 7; every code value
    occurs in every row, none comes from the quantiser), with sum_k |A| qmax < budget so that every partial sum of A.Q^T is an
    integer below 2^20. Dense A in [-a, a] where a = budget / (k qmax) is at least 1. For the long k of the Ziya shapes it is
    not; there every 16-wide k-step of every row holds exactly one non-zero (so both sides of every 128-k group boundary do),
    at position (5 row + 3 step) mod 16, of magnitude 1..a with (k / 16) a qmax < budget."""
    g = torch.Generator().manual_seed(seed)
    Q = torch.randint(-qmax, qmax + 1, (n, k), generator=g)
    if k >= 2 * qmax + 1:
        Q[:, :2 * qmax + 1] = torch.arange(-qmax, qmax + 1)[None, :]
    a = min(15, (budget - 1) // (k * qmax))
    if a >= 1:
        A = torch.randint(-a, a + 1, (m, k), generator=g)
    else:
        steps = k // 16
        a = min(15, (budget - 1) // (steps * qmax))
        assert a >= 1 and k % 16 == 0
        val = torch.randint(1, a + 1, (m, steps), generator=g) * (torch.randint(0, 2, (m, steps), generator=g) * 2 - 1)
        pos = (5 * torch.arange(m)[:, None] + 3 * torch.arange(steps)[None, :]) % 16
        A = torch.zeros(m, steps, 16, dtype=torch.int64).scatter_(2, pos[..., None], val[..., None]).view(m, k)
    return A.double(), Q.to(torch.int8)


def w8_scales(n, seed):
    """Per-row power-of-two fp32 scales 2^-9 .. 2^-2."""
    g = torch.Generator().manual_seed(seed)
    return torch.ldexp(torch.ones(n), torch.randint(-9, -1, (n,), generator=g)).float()


def w4_scales(n, groups, seed):
    """Per-row, per-128-k-group power-of-two bf16 scales 2^-4 .. 2^-1, with neighbouring groups of a row never equal: a group
    boundary that slips by one k-step multiplies 16 products by a different power of two. The partial sums are then multiples
    of 2^-4 below 2^19: 23 bits, still exact in fp32."""
    g = torch.Generator().manual_seed(seed)
    e = torch.randint(-4, 0, (n, groups), generator=g)
    for j in range(1, groups):
        same = e[:, j] == e[:, j - 1]
        e[same, j] = -4 + (e[same, j] + 4 + 1) % 4
    return torch.ldexp(torch.ones(n, groups), e).to(torch.bfloat16)


def w8_exact(A, Q, s):
    """fp64 of s[n] * (A . Q^T): an integer below 2^20 times a power of two."""
    return (A @ Q.double().t()) * s.double()[None, :]


def w4_exact(A, Q, s):
    """fp64 of A . W^^T with W^ = q * s[n, k // 128] (exactly a bf16 value: a 3-bit code times a power of two)."""
    W = Q.double() * s.double().repeat_interleave(128, dim=1)
    return A @ W.t()


# ----------------------------------------------------------------------------------------------------------- attention
# The kernels work in base 2: weights are 2^(s * sc - max) with sc = fp32(scale * log2 e) computed on the host in fp32.
# LN2_SCALE is the fp32 softmax scale for which that product is exactly 1, so integer scores stay integers in the
# kernel's domain and ex2 sees integer arguments: 0 for every key tied at the row maximum, <= -GAP for every other key.
LOG2E_F32 = np.float32(1.4426950408889634)
LN2_SCALE = float(np.float32(0.6931471824645996))
GAP = 256                 # least gap between distinct scores: 2^-256 is below fp32's smallest subnormal, so P is exactly 0


def kernel_log2_scale(scale):
    """The factor the kernels multiply scores by: fp32(fp32(scale) * fp32(log2 e))."""
    return float(np.float32(scale) * LOG2E_F32)


def keys_for_scores(score, D):
    """score [B, S, H] integer multiples of GAP with |score| < 2^23 -> (q_vec [D], K [B, S, H, D]) with q_vec . K[b, j, h]
    == score[b, j, h] exactly and every entry a bf16 value. The score is cut into three 7-bit digits of score / 256, each
    stored times its power of two in columns 0..2; columns 3 and 4 hold +p and -p (p = j mod 7 - 3), which cancel in the score
    but make tied keys different vectors (so dQ of a tie is not trivially zero). q_vec = (1, 1, 1, 1, 1, 0, ...)."""
    B, S, H = score.shape
    u = (score // GAP).to(torch.int64)
    assert bool((u * GAP == score).all()) and int(u.abs().max()) < 2 ** 15
    sign = torch.sign(u)
    mag = u.abs()
    K = torch.zeros(B, S, H, D, dtype=torch.float64)
    for c in range(3):
        K[..., c] = (sign * ((mag >> (7 * c)) & 127)).double() * float(GAP * 2 ** (7 * c))
    p = (torch.arange(S) % 7 - 3).double()[None, :, None]
    K[..., 3] = p
    K[..., 4] = -p
    q = torch.zeros(D, dtype=torch.float64)
    q[:5] = 1.0
    return q, K


def queries(B, S, H, D, q_vec):
    """Q [B, S, H, D]: q_vec in every row plus r_i = i mod 5 - 2 in column 5, where every key is 0: it does not move a score
    but makes dK depend on which query rows reached a key."""
    Q = q_vec.expand(B, S, H, D).clone()
    Q[..., 5] = (torch.arange(S) % 5 - 2).double()[None, :, None]
    return Q


def value_codes(B, S, H, D, step=1):
    """V[b, j, h, d] = step * (((j (2 d + 1) + 7 h + 13 b + d) mod 15) - 7): a code of (b, h, j) spread over all D columns,
    integers in [-7 step, 7 step]; two different keys differ in most columns."""
    j = torch.arange(S)[None, :, None, None]
    d = torch.arange(D)[None, None, None, :]
    h = torch.arange(H)[None, None, :, None]
    b = torch.arange(B)[:, None, None, None]
    return (step * (((j * (2 * d + 1) + 7 * h + 13 * b + d) % 15) - 7)).double()


def sparse_pm1(B, S, H, D, seed, nnz=4):
    """dO [B, S, H, D]: `nnz` entries of +-1 per row, the rest 0 (keeps dP = dO . V and with it dS within 8 bits)."""
    g = torch.Generator().manual_seed(seed)
    dO = torch.zeros(B, S, H, D, dtype=torch.float64)
    col = torch.rand(B, S, H, D, generator=g).argsort(-1)[..., :nnz]
    val = (torch.randint(0, 2, (B, S, H, nnz), generator=g) * 2 - 1).double()
    dO.scatter_(-1, col, val)
    return dO


def allowed(B, Sq, Skv, causal, kv_mask):
    """[B, 1, Sq, Skv] bool: key j is permitted for query i."""
    ok = torch.ones(B, 1, Sq, Skv, dtype=torch.bool, device=None if kv_mask is None else kv_mask.device)
    if causal:
        ok &= torch.ones(Sq, Skv, dtype=torch.bool, device=ok.device).tril()
    if kv_mask is not None:
        ok &= kv_mask.bool()[:, None, None, :]
    return ok


def rel_index(Sq, Skv, device=None):
    """[Sq, Skv] index of (query i, key j) into a head's relative-position vector: j - i + Sq - 1."""
    return torch.arange(Skv, device=device)[None, :] - torch.arange(Sq, device=device)[:, None] + Sq - 1


def attention_ref(Q, K, V, scale, causal=False, kv_mask=None, rel=None, dO=None, drel_prior=None):
    """fp64 attention in the kernels' base-2 formulation, on fp64 copies of the operands ([B, S, H, D]; rel [H, Sq + Skv - 1]
    in natural-log units). Scores t = (Q.K) sc + rel log2(e), sc = kernel_log2_scale(scale); weights w = 2^(t - max) over the
    permitted keys, with w below 2^-149 (not representable in fp32) taken as 0; P = w / sum w.
    Returns a dict: O [B, Sq, H, D], lse [B, H, Sq] in natural-log units (+inf for a row with no permitted key, whose O is 0),
    lse2 [B, H, Sq] = max + log2(sum w) in the kernels' base-2 units (meaningful on live rows), P [B, H, Sq, Skv], nwin
    [B, H, Sq] (number of keys at the row maximum), and with dO also dQ, dK, dV (dQ and dK carry the
    fp32 `scale` factor like the kernels' outputs) and drel = drel_prior + the sum of dS along each diagonal."""
    B, Sq, H, D = Q.shape
    Skv = K.shape[1]
    sc = kernel_log2_scale(scale)
    t = torch.einsum("bqhd,bkhd->bhqk", Q, K) * sc
    if rel is not None:
        t = t + (rel.double() * float(np.float64(LOG2E_F32)))[:, rel_index(Sq, Skv, Q.device)][None]
    ok = allowed(B, Sq, Skv, causal, kv_mask).to(Q.device).expand(B, H, Sq, Skv)
    live = ok.any(-1)
    t = torch.where(ok, t, torch.full_like(t, -math.inf))
    mx = torch.where(live, t.amax(-1), torch.zeros_like(t[..., 0]))
    d = t - mx[..., None]
    w = torch.where(d < -149, torch.zeros_like(d), torch.exp2(d))
    l = w.sum(-1)
    P = w / torch.where(live, l, torch.ones_like(l))[..., None]
    out = {"O": torch.einsum("bhqk,bkhd->bqhd", P, V), "P": P, "live": live, "nwin": (d == 0).sum(-1),
           "lse2": mx + torch.log2(torch.where(live, l, torch.ones_like(l))),
           "lse": torch.where(live, (mx + torch.log2(torch.where(live, l, torch.ones_like(l)))) * math.log(2.0),
                              torch.full_like(mx, math.inf))}
    if dO is not None:
        dP = torch.einsum("bqhd,bkhd->bhqk", dO, V)
        delta = (dO * out["O"]).sum(-1).permute(0, 2, 1)                     # [B, H, Sq]
        dS = P * (dP - delta[..., None])
        out["dS"] = dS
        out["dV"] = torch.einsum("bhqk,bqhd->bkhd", P, dO)
        out["dQ"] = torch.einsum("bhqk,bkhd->bqhd", dS, K) * float(np.float32(scale))
        out["dK"] = torch.einsum("bhqk,bqhd->bkhd", dS, Q) * float(np.float32(scale))
        if rel is not None:
            idx = rel_index(Sq, Skv, Q.device).reshape(-1)
            drel = torch.zeros(H, Sq + Skv - 1, dtype=torch.float64, device=Q.device)
            drel.index_add_(1, idx, dS.sum(0).reshape(H, -1))
            out["drel"] = drel + (0 if drel_prior is None else drel_prior.double())
    return out


def ramp_scores(B, S, H, negative=False):
    """score[b, j, h]: a strict ramp in the key index, GAP (h + 1) j, increasing for even b + h and decreasing for odd
    (S - 1 - j in place of j): the winner of a row is the last, respectively the first, key it is permitted to see.
    negative: the whole ramp shifted below zero (<= -GAP), so that a key of score 0 (a zero-filled tail) would beat every
    real key."""
    j = torch.arange(S)[None, :, None]
    h = torch.arange(H)[None, None, :]
    b = torch.arange(B)[:, None, None]
    up = ((b + h) % 2 == 0)
    ramp = torch.where(up, j, S - 1 - j) * (GAP * (h + 1))
    return ramp - GAP * (h + 1) * S if negative else ramp


def peaks_on_ramp(B, S, H, peaks):
    """An increasing ramp GAP j with peaks on top: peaks is a list of (key index, level >= 1); key j gets score
    GAP (S + level S). Keys of one level tie; a higher level beats a lower one whatever the order they arrive in. Rows that see
    no peak (under a causal or padding mask) fall back to the ramp's single winner."""
    score = (torch.arange(S) * GAP)[None, :, None].expand(B, S, H).clone()
    for j, level in peaks:
        score[:, j, :] = GAP * (S + level * S)
    return score


def padding_mask(B, S, edges):
    """uint8 [B, S]; edges[b] = (first, last) permitted key of batch row b (inclusive), so both mask edges are explicit."""
    m = torch.zeros(B, S, dtype=torch.uint8)
    for b, (lo, hi) in enumerate(edges):
        m[b, lo:hi + 1] = 1
    return m


SELECT = 128.0            # bias height of a selected offset: 128 log2(e) = 184.7 base-2 units, so the others weigh exactly 0


def selector_bias(H, Sq, Skv, deltas):
    """rel [H, Sq + Skv - 1] fp32: 0 except SELECT at the offsets deltas[h] (key - query; an int or a tuple) of head h. With
    q = 0 every dot product is 0, so row i selects the keys i + delta that are permitted (several: an exact tie, since
    the same fp32 product SELECT * log2(e) is added to each) and, when none is, the uniform mean over its permitted keys.
    SELECT is a power of two, so SELECT * fp32(log2 e) is exact and so is that plus log2 of a 2- or 4-way tie."""
    rel = torch.zeros(H, Sq + Skv - 1, dtype=torch.float32)
    for h, dl in enumerate(deltas):
        for d in (dl if isinstance(dl, (tuple, list)) else (dl,)):
            rel[h, d + Sq - 1] = SELECT
    return rel


# ================================================================================ the training step's looping kernels
# Constructions for tests/test_exact_step_gpu.py: the fused cross-entropy, AdamW, the sum of squares, the vector helpers,
# the column sums and the embedding gather / sorted backward. Each is a function of the element, row or token index, so the
# GPU tests build multi-GB inputs on the device chunk by chunk and name the index a defect touched.
LN2 = math.log(2.0)
XENT_GAP = 128            # least gap between a dead logit and its row maximum: __expf(-128) = ex2.approx(-184.7) flushes to 0
XENT_MAX_J = 6            # a row has 2^j live logits, j <= 6


def xent_special_columns(V):
    """Columns where a vector, an unrolled load or a loop iteration of the 512-thread row loop begins or ends: 0, V - 1, the
    8-column vector edges around 8, the 4096-column edges of the four loads in flight and the 16384-column iteration edges."""
    cand = [0, V - 1, V - 8, 7, 8, 4095, 4096, 8191, 8192, 16383, 16384, 32767, 32768, 49151, 49152]
    return [c for c in dict.fromkeys(cand) if 0 <= c < V]


def xent_strides(V):
    """Distances between the live columns of a row: neighbours, one lane of consecutive vectors, and wide spreads; every one
    small enough that 64 of them stay distinct modulo V."""
    return [1, 7, 8, 9, 257, V // (2 ** XENT_MAX_J + 1)]


def xent_rows(t, V, S, shift, ignore=None, ignore_index=-100):
    """Per-row description of the exact cross-entropy input, for the int64 row indices t (any device).

    Row t has 2^j live logits equal to its maximum M, at columns base + k stride (mod V), k < 2^j; every other logit is
    M - 128, M - 136 or M - 144 (by column mod 3) for the rows with M in [-80, 80] (even), and M - 128 (1 + column mod 3) for
    the rows with M = 2048 + 128 u in the thousands. The label of row t is a live column (the first or the last), a special
    dead column, or a plain dead column; or ignore_index where ignore(t) holds and on the last `shift` rows of a sequence.
    Returns a dict of tensors shaped like t: j, M, base, stride, n_live, label (ignore_index when ignored), valid."""
    dev = t.device
    sp = torch.tensor(xent_special_columns(V), device=dev)
    st = torch.tensor(xent_strides(V), device=dev)
    j = (t * 5 + t // 3) % (XENT_MAX_J + 1)
    big = t % 11 == 0
    M = torch.where(big, 2048 + 128 * ((t // 11) % 8), 2 * ((t * 37) % 81) - 80)
    base = torch.where(t % 3 == 0, sp[(t // 3) % len(sp)], (t * 7919) % V)
    stride = st[(t // 3) % len(st)]
    n_live = torch.ones_like(j) << j
    kind = (t // 7) % 4
    plain_dead = (base + n_live * stride) % V
    special = sp[(t // 4) % len(sp)]
    special_is_live = xent_is_live(special, base, stride, n_live, V)
    label = torch.where(kind == 0, base, torch.where(kind == 1, (base + (n_live - 1) * stride) % V,
                        torch.where((kind == 2) & ~special_is_live, special, plain_dead)))
    s = t % S
    valid = s + shift < S
    if ignore is not None:
        valid &= ~ignore(t)
    label = torch.where(valid, label, torch.full_like(label, ignore_index))
    return {"j": j, "M": M, "base": base, "stride": stride, "n_live": n_live, "label": label, "valid": valid}


def xent_is_live(c, base, stride, n_live, V):
    """Whether column c is one of the live columns base + k stride (mod V), k < n_live (all broadcast)."""
    d = (c - base) % V
    return (d % stride == 0) & (d // stride < n_live)


def xent_labels_array(rows_desc, S, shift, V):
    """labels[rows] as the kernel reads them (labels[t + shift] for row t): the label of row t stored at t + shift; the first
    `shift` entries of each sequence, which no row reads, hold a plain column."""
    label = rows_desc["label"]
    rows = label.numel()
    arr = torch.full_like(label, V // 2)
    if shift == 0:
        return label.clone()
    s = torch.arange(rows, device=label.device) % S
    keep = s + shift < S
    idx = torch.arange(rows, device=label.device)[keep]
    arr[idx + shift] = label[keep]
    return arr


def xent_logits(t, V, desc_fn):
    """Logits of rows t ([len(t), V] fp32 on t's device, every value a bf16 value)."""
    d = desc_fn(t)
    c = torch.arange(V, device=t.device)[None, :]
    M = d["M"][:, None]
    small = M.abs() <= 80
    dead = torch.where(small, M - XENT_GAP - 8 * (c % 3), M - XENT_GAP * (1 + c % 3))
    live = xent_is_live(c, d["base"][:, None], d["stride"][:, None], d["n_live"][:, None], V)
    return torch.where(live, M, dead).float(), live, d


def xent_grad_scale_f32(grad_scale, n_valid):
    """The kernel's fp32 factor grad_scale / n_valid: one IEEE division of two fp32 values."""
    return float(np.float32(grad_scale) / np.float32(n_valid))


def xent_row_loss_exact(M, j, lab_logit):
    """fp64 M + log(2^j) - logit[label] (the true loss of a row whose row sum is 2^j)."""
    return M.double() + j.double() * LN2 - lab_logit.double()


def xent_row_loss_bound(M, j, ref):
    """What the kernel's lse = M + logf(2^j) then lse - logit[label] may be off by in fp32: logf within 1 ulp of j ln2, and
    one rounding of each of the two additions (ulp(x) <= 2^-23 |x|), doubled."""
    lg = j.double() * LN2
    return 2.0 ** -22 * lg + 2.0 ** -22 * (M.double().abs() + lg) + 2.0 ** -22 * ref.abs()


XENT_MEAN_DEPTH = 42      # longest fp32 addition chain of loss_reduce_kernel: 32 strided terms (rows <= 32768), 5 + 5 tree levels


# ------------------------------------------------------------------------------------------------------------- AdamW
ADAM_LR = 0.25            # a power of two: master moves by exactly +-lr per step
ADAM_EXP_SPAN = 121       # gradient magnitude 2^((i mod 121) - 60): names the element class a thread read


def adam_p0(i):
    """Initial master weight of element i: an integer below 2^19 in magnitude (exact in fp32 with two fraction bits to spare)."""
    return ((i % (1 << 20)) - (1 << 19)).float()


def adam_exponent(i):
    return (i % ADAM_EXP_SPAN) - 60


def adam_sign(i, step):
    """+1 or -1: bit (step + 7) of a multiplicative hash of i, so neighbouring elements and steps differ."""
    return 1 - 2 * (((i * 2654435761) >> (step + 7)) & 1)


def adam_grad(i, step):
    """Gradient of element i at `step`: +-2^e, e in [-60, 60]: exact in bf16 and fp32, and its square (times a grad_scale of
    2^-3 .. 2^2) stays a normal fp32 number."""
    return torch.ldexp(adam_sign(i, step).float(), adam_exponent(i).int())


def adam_master(i, steps):
    """master after `steps` updates with beta1 = beta2 = eps = wd = 0: m = g, v = g^2, denom = |g|, so p -= lr sign(g)."""
    acc = torch.zeros_like(i, dtype=torch.float32)
    for s in range(steps):
        acc += adam_sign(i, s).float()
    return adam_p0(i) - ADAM_LR * acc


# --------------------------------------------------------------------------------------------------------- sum of squares
SUMSQ_FIELDS = 12         # rounds named per launch: value 2^(f - 11), square 2^(2f - 22), f < 12: bits -22 .. 0


def sumsq_field_positions(round_lo, n_rounds, threads, nvec):
    """(flat element index, field f) of the one non-zero element of each grid-stride round round_lo .. round_lo + 11 that
    exists: round r reads vectors r * threads .. (r + 1) * threads - 1; the element sits at a thread that moves with r and
    in vector slot r mod 4. Returns a list of (index, round, field)."""
    out = []
    for f in range(SUMSQ_FIELDS):
        r = round_lo + f
        if r >= n_rounds:
            break
        width = min(threads, nvec - r * threads)
        th = (r * 7919 + 13) % width
        out.append(((r * threads + th) * 4 + r % 4, r, f))
    return out


def sumsq_field_value(f):
    return 2.0 ** (f - 11)


def sumsq_count_pattern(i):
    """+-1 at the elements with i mod 8 == (i // 8) mod 8 (every vector slot and thread over the rounds), 0 elsewhere."""
    on = (i % 8) == ((i // 8) % 8)
    return torch.where(on, 1 - 2 * ((i // 64) % 2), 0).float()


def sumsq_count(n):
    """Number of non-zero elements of sumsq_count_pattern over [0, n)."""
    full, rem = divmod(n, 64)
    return full * 8 + sum(1 for k in range(rem) if k % 8 == k // 8)


# ---------------------------------------------------------------------------------------------------------- column sums
COLSUM_BITS = 22          # rows coded per column: row j of a window adds 2^j, so a column sum has at most 22 bits


def colsum_plan(rows, cols, sms):
    """(strips, rows per strip) as elementwise.cu's colsum_plan picks them."""
    col_tiles = (cols + 63) // 64
    want = (4 * sms + col_tiles - 1) // col_tiles
    want = max(1, min(want, (rows + 31) // 32, 1024))
    rps = ((rows + want - 1) // want + 31) // 32 * 32
    return (rows + rps - 1) // rps, rps


def colsum_focus(rows, cols, rps, pass_idx=0):
    """Column c watches one window of COLSUM_BITS consecutive rows of one strip: rows strip * rps + 22 w .. + 21 (clipped to
    the strip and the matrix), row k of the window holding 2^k in that column and every other row 0. The (strip, window)
    pairs are dealt out to the columns cyclically, shifted by pass_idx * cols, so that n_passes(...) passes cover every row.
    Returns (row index [cols, 22] int64 with -1 where the window is short, strip [cols], window [cols])."""
    ns = (rows + rps - 1) // rps
    nw = (rps + COLSUM_BITS - 1) // COLSUM_BITS
    tup = (torch.arange(cols) + pass_idx * cols) % (ns * nw)
    strip, win = tup // nw, tup % nw
    k = torch.arange(COLSUM_BITS)
    r = strip[:, None] * rps + win[:, None] * COLSUM_BITS + k[None, :]
    ok = (win[:, None] * COLSUM_BITS + k[None, :] < rps) & (r < rows)
    return torch.where(ok, r, torch.full_like(r, -1)), strip, win


def colsum_passes(rows, cols, rps):
    ns = (rows + rps - 1) // rps
    return -(-(ns * ((rps + COLSUM_BITS - 1) // COLSUM_BITS)) // cols)


def colsum_matrix(rows, cols, rr, device=None):
    """The bf16 [rows, cols] matrix of colsum_focus rows rr, and its exact column sums (fp64)."""
    x = torch.zeros(rows, cols, dtype=torch.float32, device=device)
    k = torch.arange(COLSUM_BITS, device=device).expand_as(rr)
    c = torch.arange(cols, device=device)[:, None].expand_as(rr)
    ok = rr >= 0
    x[rr[ok], c[ok]] = torch.ldexp(torch.ones(int(ok.sum()), device=device), k[ok].int())
    want = torch.where(ok, torch.ldexp(torch.ones_like(rr, dtype=torch.float64), k), 0.0).sum(1)
    return x.to(torch.bfloat16), want


def colsum_missing_rows(got, want, rr_col):
    """The rows of one column whose bit is set in want but not in got (both integers), and those set only in got."""
    g, w = int(got), int(want)
    lost = [int(rr_col[k]) for k in range(COLSUM_BITS) if (w >> k) & 1 and not (g >> k) & 1]
    extra = [k for k in range(COLSUM_BITS + 2) if (g >> k) & 1 and not (w >> k) & 1]
    return lost, extra


# ------------------------------------------------------------------------------------------------ sorted embedding backward
EMB_CODED_MAX = 8         # a short run has 1..8 occurrences; occurrence q adds +-2^q: a run sum fits bf16's 8 bits
EMB_BIG_COLS = 384        # the long run: columns c < 384 count occurrences q = c mod 384; 384 + b counts block q // 384


def embedding_bwd_ids(tokens, V, big_id, seed):
    """ids [tokens] int64: half the tokens carry big_id (one long run), the other half runs of 1..8 occurrences over distinct
    ids that include 0 (the run at sorted position 0) and V - 1 (the run that ends at the last sorted position), token order
    shuffled. Returns (ids, short_ids, short_lengths)."""
    g = torch.Generator().manual_seed(seed)
    half = tokens // 2
    lengths = []
    total = 0
    while total < tokens - half:
        ln = 1 + len(lengths) % EMB_CODED_MAX
        ln = min(ln, tokens - half - total)
        lengths.append(ln)
        total += ln
    nrun = len(lengths)
    pool = torch.randperm(V - 2, generator=g)[:nrun + 1] + 1
    pool = pool[pool != big_id][:nrun - 2]
    short_ids = torch.cat([torch.tensor([0]), pool, torch.tensor([V - 1])])
    lens = torch.tensor(lengths)
    ids = torch.cat([torch.full((half,), big_id), short_ids.repeat_interleave(lens)])
    perm = torch.randperm(tokens, generator=g)
    return ids[perm].contiguous(), short_ids, lens


def occurrence_index(ids):
    """For each token, how many earlier tokens (in token order) carry the same id: its place in a stable sort's run."""
    order = torch.sort(ids, stable=True).indices
    sorted_ids = ids[order]
    start = torch.ones_like(sorted_ids, dtype=torch.bool)
    start[1:] = sorted_ids[1:] != sorted_ids[:-1]
    pos = torch.arange(len(ids))
    run_start = torch.cummax(torch.where(start, pos, torch.zeros_like(pos)), 0).values
    occ = torch.empty_like(ids)
    occ[order] = pos - run_start
    return occ


def embedding_bwd_dout(ids, occ, cols, big_id, seed):
    """dout [tokens, cols] fp32 (bf16 values) and the old dW rows of the touched ids:
    - short runs: occurrence q adds s 2^q in column c, s = +1 on even 8-column vectors and -1 on odd ones; the old value is
      -256 s, so old + run sum is in [-256, 256] in magnitude: a bf16 integer, and a lost or doubled occurrence flips its bit;
    - the long run: columns c < 384 hold 1 where q mod 384 == c, columns 384 + b hold 1 where q // 384 == b (old -256), so one
      lost occurrence q is named by the pair of columns it leaves short; the remaining columns hold integers in [-3, 3] (old
      a small integer), summed exactly in fp32 and rounded once to bf16."""
    g = torch.Generator().manual_seed(seed)
    T = len(ids)
    c = torch.arange(cols)[None, :]
    sgn = 1.0 - 2.0 * ((c // 8) % 2).double()
    short = (ids != big_id)[:, None]
    q = occ[:, None]
    d_short = sgn * torch.ldexp(torch.ones(T, 1, dtype=torch.float64), q.clamp(max=30))
    nb = -(-int((ids == big_id).sum()) // EMB_BIG_COLS)
    d_big = torch.where(c < EMB_BIG_COLS, (q % EMB_BIG_COLS == c).double(),
                        torch.where(c < EMB_BIG_COLS + nb, (q // EMB_BIG_COLS == c - EMB_BIG_COLS).double(),
                                    torch.randint(-3, 4, (T, cols), generator=g).double()))
    dout = torch.where(short, d_short, d_big)
    return dout


def embedding_bwd_old(V, cols, big_id, n_big, short_ids, seed):
    """Initial dW [V, cols] fp64: random integers in [-50, 50] on the rows no id hits, -256 s on the short runs' rows, -256 on
    the long run's counting columns and a small integer elsewhere on its row."""
    g = torch.Generator().manual_seed(seed)
    old = torch.randint(-50, 51, (V, cols), generator=g).double()
    c = torch.arange(cols)
    sgn = 1.0 - 2.0 * ((c // 8) % 2).double()
    old[short_ids] = -256.0 * sgn
    old[big_id, c < EMB_BIG_COLS + -(-n_big // EMB_BIG_COLS)] = -256.0
    return old
