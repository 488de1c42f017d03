"""The write contract of every public `fsb200.ops` function, and the check that a call keeps to it.

`WRITES[op](arguments)` lists what a call may write among its ARGUMENTS (the bound arguments, defaults applied), each a
`Write(arg, view, kind, rows)`: `view` a tensor view of argument `arg`, `rows` an optional index of the view's first
dimension (only those rows are written), and `kind`
  - OVERWRITE: every element of the view is written, so the call's result does not depend on what was there;
  - UPDATE: the elements may change and their old values may be read (accumulation, in-place ops).
The entries follow include/fsb200.h and the ops docstrings, and every declared view is a view of the argument itself or a
subset of it: where a C entry addresses memory from a pointer and sizes (flat spans, a shared row stride), the ops wrapper
refuses an argument whose extent differs, so no declared write can reach past the tensor it names. The flags of the call choose the kind (`gemm`'s out is UPDATE
under accumulate=True and OVERWRITE otherwise). An OVERWRITE view whose bytes overlap a read-only tensor argument (an
out= that aliases an input, which fsb_add and fsb_dropout allow) is treated as UPDATE.

Tensors an op allocates itself (`torch.empty` / `torch.empty_like` in fsb200/ops.py; ops.py calls no `new_empty`) need no
entry: they are all checked as OVERWRITE. One that is legitimately left partly unwritten would be listed in
`FRESH_PARTIAL[op]` with the reason; no op has one.

`check_footprint(op, fn, args, kwargs)` runs `fn(*args, **kwargs)` (the op, or the Recorder's `real` call of it) and checks:
  - every byte of every storage an argument refers to is unchanged outside the declared write views (the storage is
    snapshotted before the call and compared byte for byte through uint8 views, so views of different dtypes over one
    storage are handled);
  - no poison is left inside an OVERWRITE view or a fresh allocation (NaN for floating types, a byte pattern no kernel
    output takes for integer and FP8 codes: int8 -128, uint8 0 (int4 codes are 1 .. 15 per nibble, the mask bytes that
    kv_append sets are 1), 0xA5 bytes for int32 / int64, 0x7f for FP8, a NaN encoding in both formats);
  - every workspace the op asks `ops.workspace` for is a fresh view of exactly the requested bytes, 4 KiB (a 256-byte
    aligned offset) into a buffer of 0xA5 bytes with at least 4 KiB after it, and both guards are bit-identical afterwards.
A failure names the op, the argument and the storage byte offset and count of what changed.

Blind spot: a write into an allocation that no argument of the call refers to (another tensor that happens to lie
elsewhere in device memory) is not visible to this check.
"""
import inspect
from typing import NamedTuple, Optional

import torch

from fsb200 import ops

OVERWRITE, UPDATE = "overwrite", "update"
WS_GUARD = 4096          # guard bytes before every workspace view (a multiple of 256: the view keeps 256-byte alignment)
WS_SENTINEL = 0xA5
CMP_CHUNK = 1 << 28      # bytes compared per step (bounds the temporaries of a compare over a multi-GB storage)
_INT_POISON = {torch.int8: 0x80, torch.uint8: 0x00, torch.int16: 0xA5, torch.int32: 0xA5, torch.int64: 0xA5}
_FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)


class Write(NamedTuple):
    arg: str
    view: torch.Tensor
    kind: str
    rows: Optional[torch.Tensor] = None


# ------------------------------------------------------------------------------------------------------ byte views
def storage_bytes(t):
    """The whole storage of t as a contiguous uint8 tensor sharing its memory."""
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage())


def byte_view(t, sb=None):
    """t's bytes as a uint8 [*t.shape, element_size] view of `sb` (default: t's own storage)."""
    es = t.element_size()
    sb = storage_bytes(t) if sb is None else sb
    return sb.as_strided((*t.shape, es), (*(s * es for s in t.stride()), 1), t.storage_offset() * es)


def extent(t):
    """[first, last + 1) storage bytes t's view touches."""
    es = t.element_size()
    lo = t.storage_offset() * es
    if t.numel() == 0:
        return lo, lo
    return lo, lo + (sum((n - 1) * s for n, s in zip(t.shape, t.stride())) + 1) * es


def _key(t):
    return (t.device, t.untyped_storage().data_ptr())


def _overlap(x, y):
    """Do the byte sets of two views of one storage intersect?"""
    (lx, hx), (ly, hy) = extent(x), extent(y)
    if max(lx, ly) >= min(hx, hy):
        return False
    lo, hi = min(lx, ly), max(hx, hy)
    m = torch.zeros(hi - lo, dtype=torch.uint8, device=x.device)
    bx, by = byte_view(x), byte_view(y)
    m.as_strided(bx.shape, bx.stride(), lx - lo).fill_(1)
    return bool(m.as_strided(by.shape, by.stride(), ly - lo).any())


# ------------------------------------------------------------------------------------------------------ poison
def poison(t):
    if t.numel() == 0:
        return
    if t.dtype in _FP8:
        byte_view(t).fill_(0x7F)
    elif t.dtype.is_floating_point:
        t.fill_(float("nan"))
    else:
        byte_view(t).fill_(_INT_POISON[t.dtype])


def poisoned(t, rows=None):
    """Bool mask of t's elements (of the rows `rows`) that still hold the poison."""
    if t.dtype in _FP8:
        m = (byte_view(t) == 0x7F).all(-1)
    elif t.dtype.is_floating_point:
        m = torch.isnan(t)
    else:
        m = (byte_view(t) == _INT_POISON[t.dtype]).all(-1)
    return m if rows is None else m[rows]


# ------------------------------------------------------------------------------------------------------ the table
def _acc(a, flag="accumulate"):
    return UPDATE if a[flag] else OVERWRITE


def _given(a, name, view_of, kind):
    t = a.get(name)
    return [] if t is None else [Write(name, view_of(t), kind)]


def _gemm(a):
    """out (when given) and aux, the pre-activation copy acc + bias (ops.gemm refuses either unless it is [M, N])."""
    return _given(a, "out", lambda t: t, _acc(a)) + _given(a, "aux", lambda t: t, OVERWRITE)


def _norm_bwd(*wgrads):
    def entry(a):
        return [Write(n, a[n], _acc(a)) for n in wgrads]
    return entry


def _glu_bwd(a):
    return [Write(n, a[n], OVERWRITE) for n in ("dgate", "dup")]


def _embedding_bwd(a):
    dW, rows = a["dW"], a["dout"].shape[0]
    if a["ids"] is None:                         # row t % idx_mod
        hit = torch.arange(min(rows, a["idx_mod"]), device=dW.device)
    else:
        hit = torch.unique(a["ids"].reshape(-1))
    return [Write("dW", dW, UPDATE, hit)]


def _softmax_xent(a):
    lg, dl = a["logits"], a["dlogits"]
    if dl is None or isinstance(dl, str):        # "inplace": the gradient replaces the logits it was computed from
        return [Write("logits", lg, UPDATE)] if dl == "inplace" else []
    return [Write("dlogits", dl, OVERWRITE)]


def _adamw(a):
    return [Write(k, a[k], UPDATE) for k in ("master", "m", "v")] + _given(a, "param16", lambda t: t, OVERWRITE)


def _kv_append(a):
    """Slot kv_len - 1 of every row (and that mask byte); nothing when the slot lies outside [0, cap)."""
    s = int(a["kv_len"].reshape(-1)[0].item()) - 1
    if not 0 <= s < a["k_cache"].shape[1]:
        return []
    w = [Write(n, a[n][:, s], OVERWRITE) for n in ("k_cache", "v_cache")]
    return w + _given(a, "kv_mask", lambda t: t[:, s], OVERWRITE)


def _kv_reorder(a):
    """The live slots [0, kv_len) of every dst row whose index is in range; nothing else."""
    dst, index = a["dst"], a["index"]
    rows, cap = dst.shape[1], dst.shape[2]
    live = min(max(int(a["kv_len"].reshape(-1)[0].item()), 0), cap)
    ok = [r for r, i in enumerate(index.tolist()) if 0 <= i < rows]
    return [Write("dst", dst[:, r, :live], OVERWRITE) for r in ok]


def _sdpa_bwd(a):
    return [Write(n, a[n], OVERWRITE) for n in ("dq", "dk", "dv")] + _given(a, "drel_bias", lambda t: t, UPDATE)


def _rope(a):
    x = a["x"]
    v = torch.as_strided(x, (a["positions"].numel(), a["nheads"], a["head_dim"]), (a["row_stride"], a["head_stride"], 1),
                         x.storage_offset() + a["offset"])
    return [Write("x", v, UPDATE)]


def _whole(name, kind):
    """The whole argument `name` (when given)."""
    return lambda a: _given(a, name, lambda t: t, kind)


NOTHING = lambda a: []   # noqa: E731  (every output is a fresh allocation, or there is no kernel)

WRITES = {
    "gemm": _gemm,
    "quantize_w8": lambda a: _given(a, "q", lambda t: t, OVERWRITE) + _given(a, "s", lambda t: t, OVERWRITE),
    "gemm_w8a16": lambda a: _given(a, "out", lambda t: t, OVERWRITE),
    "quantize_w4": lambda a: _given(a, "q", lambda t: t, OVERWRITE) + _given(a, "s", lambda t: t, OVERWRITE),
    "gemm_w4a16": lambda a: _given(a, "out", lambda t: t, OVERWRITE),
    "fp8_quantize": NOTHING,                                   # y, yt and [scale_inv, amax] are fresh
    "gemm_fp8": lambda a: _given(a, "out", lambda t: t, _acc(a)),
    "rmsnorm_fwd": NOTHING, "layernorm_fwd": NOTHING,          # y, the statistics and x_sum are fresh
    "rmsnorm_bwd": _norm_bwd("dscale_out"), "rmsnorm_bwd_dropout": _norm_bwd("dscale_out"),
    "layernorm_bwd": _norm_bwd("dgamma_out", "dbeta_out"),
    "layernorm_bwd_dropout": _norm_bwd("dgamma_out", "dbeta_out"),
    "dropout_advance": _whole("counter", UPDATE),
    "dropout": _whole("out", OVERWRITE),
    "rope_inplace": _rope,
    "glu_fwd": NOTHING, "glu_bwd": _glu_bwd,
    "act_fwd": NOTHING, "act_bwd": NOTHING,
    "act_bwd_bias": lambda a: [Write("dbias", a["dbias"], _acc(a))],
    "add": _whole("out", OVERWRITE),
    "accumulate": lambda a: [Write("acc32", a["acc32"], OVERWRITE if a["overwrite"] else UPDATE)],
    "scale_inplace": _whole("x16", UPDATE),
    "colsum": lambda a: [Write("out", a["out"], _acc(a))],
    "embedding_fwd": NOTHING,
    "embedding_bwd": _embedding_bwd,
    "cast_f32_to_bf16": _whole("out", OVERWRITE),
    "softmax_xent": _softmax_xent,
    "adamw_flat": _adamw,
    "sumsq": _whole("out", UPDATE),
    "clip_coef": lambda a: _whole("coef_out", UPDATE)(a) + _whole("norm_out", UPDATE)(a),
    "sdpa_fwd": lambda a: _given(a, "out", lambda t: t, OVERWRITE),
    "attn_decode": lambda a: _given(a, "out", lambda t: t, OVERWRITE),
    "kv_append": _kv_append,
    "kv_reorder": _kv_reorder,
    "sdpa_bwd": _sdpa_bwd,
    "segment_bounds": NOTHING,                                 # torch ops only, fresh bounds
    "sdpa_segments_fwd": lambda a: _given(a, "out", lambda t: t, OVERWRITE),
    "sdpa_segments_bwd": lambda a: [Write(n, a[n], OVERWRITE) for n in ("dq", "dk", "dv")],
}

# op -> {index of the allocation in call order: why it may be left partly unwritten}
FRESH_PARTIAL = {}


# ------------------------------------------------------------------------------------------------------ the check
class Stats:
    """Per op: footprint-checked calls and the bytes verified unchanged (storage bytes outside the writes + guards)."""

    def __init__(self):
        self.checked, self.guard_bytes = {}, {}

    def add(self, op, nbytes):
        self.checked[op] = self.checked.get(op, 0) + 1
        self.guard_bytes[op] = self.guard_bytes.get(op, 0) + nbytes


STATS = Stats()


class _Fresh:
    """Stands in for `torch` inside fsb200.ops during a check: empty / empty_like return poisoned tensors and are kept."""

    def __init__(self):
        self.allocs = []

    def __getattr__(self, name):
        return getattr(torch, name)

    def _keep(self, t):
        poison(t)
        self.allocs.append(t)
        return t

    def empty(self, *a, **k):
        return self._keep(torch.empty(*a, **k))

    def empty_like(self, *a, **k):
        return self._keep(torch.empty_like(*a, **k))


class _Workspaces:
    """Stands in for ops.workspace during a check: a fresh exact-size view between sentinel guards per request."""

    def __init__(self):
        self.bufs = []

    def __call__(self, nbytes, device, tag="default"):
        n = int(nbytes)
        buf = torch.full((WS_GUARD + n + WS_GUARD + (-n) % 256,), WS_SENTINEL, dtype=torch.uint8, device=device)
        self.bufs.append((tag, buf, n))
        return buf[WS_GUARD:WS_GUARD + n]

    def problems(self, op):
        bad, nbytes = [], 0
        for tag, buf, n in self.bufs:
            for side, g, base in (("before", buf[:WS_GUARD], -WS_GUARD), ("after", buf[WS_GUARD + n:], n)):
                nbytes += g.numel()
                diff = (g != WS_SENTINEL).nonzero()
                if diff.numel():
                    first = int(diff[0]) + base
                    bad.append(f"ops.{op}: workspace '{tag}' ({n} bytes): {diff.numel()} guard bytes {side} it changed, "
                               f"first at byte {first} relative to the workspace start")
        return bad, nbytes


def _tensor_args(a):
    out = []
    for name, v in a.items():
        if isinstance(v, torch.Tensor):
            out.append((name, v))
        elif isinstance(v, ops.Dropout):
            out.append((f"{name}.base", v.base))
    return out


def _changed(cur, snap):
    """(count, first index) of the bytes where two equal-length uint8 tensors differ, compared in chunks."""
    n, first = 0, None
    for i in range(0, cur.numel(), CMP_CHUNK):
        d = cur[i:i + CMP_CHUNK] != snap[i:i + CMP_CHUNK]
        if d.any():
            c = int(d.sum())
            n += c
            if first is None:
                first = i + int(d.nonzero()[0])
    return n, first


def bound_arguments(op, args, kwargs):
    sig = inspect.signature(getattr(ops, op))
    b = sig.bind(*args, **kwargs)
    b.apply_defaults()
    return dict(b.arguments)


def check_footprint(op, fn, args, kwargs, stats=STATS):
    """Run fn(*args, **kwargs) as a call of ops.<op> and check its write footprint (module docstring). Returns fn's result."""
    entry = WRITES.get(op)
    if entry is None:
        raise AssertionError(f"ops.{op} has no write-footprint entry (WRITES in tests/footprint.py)")
    a = bound_arguments(op, args, kwargs)
    tensors = _tensor_args(a)
    writes = entry(a)
    write_args = {w.arg for w in writes}
    reads = [(n, t) for n, t in tensors if n not in write_args]
    storages = {}
    for n, t in tensors:
        k = _key(t)
        if k not in storages:
            storages[k] = (storage_bytes(t).clone(), [n])
        elif n not in storages[k][1]:
            storages[k][1].append(n)
    poisoned_writes = []
    for w in writes:
        if w.kind != OVERWRITE or any(_key(t) == _key(w.view) and _overlap(w.view, t) for _, t in reads):
            continue
        v = w.view if w.rows is None else w.view[w.rows]
        if w.rows is None:
            poison(w.view)
        else:
            pv = v.clone(); poison(pv); w.view[w.rows] = pv
        poisoned_writes.append(w)

    fresh, wss = _Fresh(), _Workspaces()
    saved = ops.torch, ops.workspace
    ops.torch, ops.workspace = fresh, wss
    try:
        ret = fn(*args, **kwargs)
    finally:
        ops.torch, ops.workspace = saved

    bad = []
    for w in poisoned_writes:
        left = poisoned(w.view, w.rows)
        if left.any():
            bad.append(f"ops.{op}: {int(left.sum())}/{left.numel()} elements of the overwrite argument '{w.arg}' were never "
                       f"written (poison left)")
    for i, t in enumerate(fresh.allocs):
        if i in FRESH_PARTIAL.get(op, {}):
            continue
        left = poisoned(t)
        if left.any():
            bad.append(f"ops.{op}: {int(left.sum())}/{left.numel()} elements of the tensor it allocated (#{i}, "
                       f"{tuple(t.shape)} {t.dtype}) were never written (poison left)")
    nbytes = 0
    for k, (snap, names) in storages.items():
        cur = None
        for w in writes:
            if _key(w.view) != k:
                continue
            cur = storage_bytes(w.view) if cur is None else cur
            sv, cv = byte_view(w.view, snap), byte_view(w.view, cur)
            if w.rows is None:
                sv.copy_(cv)
            else:
                sv[w.rows] = cv[w.rows]
        cur = storage_bytes(dict(tensors)[names[0]]) if cur is None else cur
        nbytes += cur.numel()
        n, first = _changed(cur, snap)
        if n:
            owner = [nm for nm, t in tensors if _key(t) == k and extent(t)[0] <= first < extent(t)[1]]
            where = f"argument '{owner[0]}'" if owner else f"the storage of argument(s) {names}, outside every argument view"
            bad.append(f"ops.{op}: {n} bytes changed outside the declared writes in {where}; first at storage byte "
                       f"offset {first}")
    ws_bad, ws_bytes = wss.problems(op)
    bad += ws_bad
    if bad:
        raise AssertionError("; ".join(bad))
    stats.add(op, nbytes + ws_bytes)
    return ret


def footprint_checkers(stats=STATS):
    """launch_census.Recorder checkers: check_footprint for every op the census may meet (an op without a WRITES entry
    fails by name when it is first called)."""
    import launch_census
    return {name: (lambda name: lambda real, bound, *a, **k: check_footprint(name, real, a, k, stats))(name)
            for name in launch_census.ops_functions()}


def missing_entries():
    """Public ops functions (launch_census.ops_functions) without a WRITES entry, in definition order."""
    import launch_census
    return [n for n in launch_census.ops_functions() if n not in WRITES]
