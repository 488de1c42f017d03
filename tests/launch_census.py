"""The launch census recorder shared by tests/test_workload_launches_gpu.py and tests/test_path_launches_gpu.py.

`Recorder` wraps every public `fsb200.ops` function. The outermost call (a reentrancy guard skips calls an op makes through
another) is keyed by its signature: the op, each tensor's shape, strides, dtype and 16-byte alignment class, the scalar
flags, which optional operands are present, and whatever `extra_key(op, arguments)` adds (the dropout site, so that every
site is value-checked once). The first call of every signature goes through its tests/launch_refs.py checker, and so does
every call of the ops named in `check_all` (the decode ops, whose result depends on the device-held kv_len); the rest are
counted. `observe(op, arguments, result)` sees every outermost call after it ran (the dropout stream log).
"""
import functools
import inspect

import torch

import launch_refs as R
from fsb200 import lib as L, ops

# public ops functions that launch no kernel of their own: they are not recorded
NOT_LAUNCHES = {"workspace", "set_profiler", "set_reserved_sms"}


def ops_functions():
    return {n: f for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__
            and not n.startswith("_") and n not in NOT_LAUNCHES}


def _key_of(v):
    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype), v.data_ptr() % 16)
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    return type(v).__name__


class Recorder:
    """Wraps the public ops functions; see the module docstring."""

    def __init__(self, checkers, check_all=(), extra_key=None, observe=None):
        self.checkers = checkers
        self.check_all = set(check_all)
        self.extra_key = extra_key
        self.observe = observe
        self.depth = 0
        self.calls = {}          # (op, signature) -> count
        self.checked = {}        # (op, signature) -> checked calls
        self.worst = {}          # (op, signature) -> largest err / bound of its checked calls
        self.wrapped_launches = 0
        self.extra_launches = 0  # launches the checkers issue themselves (the aux re-run of a GeLU GEMM)
        self.check_mem = {}      # (op, signature) -> device memory its checked call needed above what was allocated before
        self.peak = 0            # peak allocated over the run (torch's peak counter is reset around each check)

    def install(self, monkeypatch):
        for name, fn in ops_functions().items():
            monkeypatch.setattr(ops, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)

        @functools.wraps(fn)
        def wrapper(*args, **kwargs):
            if self.depth:
                return fn(*args, **kwargs)
            arguments = sig.bind(*args, **kwargs).arguments
            key = tuple((k, _key_of(v)) for k, v in arguments.items())
            if self.extra_key is not None:
                key = key + (("extra", self.extra_key(name, arguments)),)
            key = (name, key)
            first = key not in self.calls
            self.calls[key] = self.calls.get(key, 0) + 1
            self.depth += 1
            try:
                if not (first or name in self.check_all):
                    c0 = L.launch_count
                    ret = fn(*args, **kwargs)
                    self.wrapped_launches += L.launch_count - c0
                else:
                    ret = self._checked(name, key, fn, args, kwargs)
                if self.observe is not None:
                    self.observe(name, arguments, ret)
                return ret
            finally:
                self.depth -= 1
        return wrapper

    def _checked(self, name, key, fn, args, kwargs):
        chk = self.checkers.get(name)
        if chk is None:
            raise AssertionError(f"ops.{name} has no launch reference in tests/launch_refs.py")
        deltas = []       # launches of each invocation of `real`: the first is the step's own call

        def real(*a, **kw):
            c0 = L.launch_count
            r = fn(*a, **kw)
            deltas.append(L.launch_count - c0)
            return r
        b = R.Bound(f"{name} {key[1]}")
        self.peak = max(self.peak, torch.cuda.max_memory_allocated())
        torch.cuda.reset_peak_memory_stats()
        m0 = torch.cuda.memory_allocated()
        ret = chk(real, b, *args, **kwargs)
        m1 = torch.cuda.max_memory_allocated()
        self.peak = max(self.peak, m1)
        self.check_mem[key] = max(self.check_mem.get(key, 0), m1 - m0)
        self.wrapped_launches += deltas[0]
        self.extra_launches += sum(deltas[1:])   # re-runs inside the checker (the plain GEMM an aux is compared with)
        self.worst[key] = max(self.worst.get(key, 0.0), b.worst)
        self.checked[key] = self.checked.get(key, 0) + 1
        return ret


def free_gib():
    free, _ = torch.cuda.mem_get_info()
    return free / 2 ** 30


def print_table(name, rec, secs, peak):
    rows = {}
    for (op, sig), n in rec.calls.items():
        r = rows.setdefault(op, [0, 0, 0, 0.0, 0])
        r[0] += 1; r[1] += n; r[2] += rec.checked.get((op, sig), 0)
        r[3] = max(r[3], rec.worst.get((op, sig), 0.0))
        r[4] = max(r[4], rec.check_mem.get((op, sig), 0))
    print(f"\n[census] {name}: {sum(r[0] for r in rows.values())} signatures, {sum(r[1] for r in rows.values())} calls, "
          f"{sum(r[2] for r in rows.values())} checked, {secs:.1f} s wall, peak {peak / 2 ** 30:.1f} GiB")
    print(f"[census] {'op':<22} {'signatures':>10} {'calls':>6} {'checked':>7} {'worst err/bound':>16} {'check GiB':>10}")
    for op in sorted(rows):
        s, n, c, wr, mem = rows[op]
        print(f"[census] {op:<22} {s:>10} {n:>6} {c:>7} {wr:>16.3g} {mem / 2 ** 30:>10.2f}")


# ------------------------------------------------------------------------------------------------ dropout stream log
# The ops that draw a dropout mask, by the layout kind their mask has; forward and backward of one site must agree on it.
DROP_KIND = {"sdpa_fwd": "attention", "sdpa_bwd": "attention", "layernorm_fwd": "layernorm",
             "layernorm_bwd_dropout": "layernorm", "rmsnorm_fwd": "rmsnorm", "rmsnorm_bwd_dropout": "rmsnorm",
             "glu_fwd": "glu", "glu_bwd": "glu", "dropout": "dropout"}
DROP_BACKWARD = {"sdpa_bwd", "layernorm_bwd_dropout", "rmsnorm_bwd_dropout", "glu_bwd"}


def _mask_shape(op, a):
    if op in ("sdpa_fwd", "sdpa_bwd"):
        B, Sq, H, _ = a["q"].shape
        return (B, H, Sq, a["k"].shape[1])
    t = a.get("x", a.get("gate"))
    return tuple(t.shape)


class DropoutLog:
    """The dropout streams a run draws: every dropout_advance (old base, n) and every masked call (op, base, site, p, seed,
    mask shape). Pass `observe` to a Recorder."""

    def __init__(self):
        self.advances, self.uses = [], []

    def observe(self, op, a, ret):
        if op == "dropout_advance":
            self.advances.append((int(ret.item()), int(a["n"])))
        elif op in DROP_KIND and a.get("drop") is not None:
            d = a["drop"]
            self.uses.append((op, int(d.base.item()), d.site, d.p, d.seed, _mask_shape(op, a)))


def site_of(op, a):
    """Recorder extra_key: the dropout site of a masked call (None for every other call)."""
    d = a.get("drop") if op in DROP_KIND else None
    return None if d is None else d.site


def dropout_stream_problems(advances, uses):
    """The whole-step invariants of the dropout streams, as messages (empty when they hold):
    (1) the sites used under each base are exactly range(n) of the dropout_advance(n) that returned it (a smaller n would
    let the next forward's streams overlap this one's); (2) each advance starts where the previous one ended; (3) every
    (base, site) is drawn by exactly one forward and one backward call of one mask kind (two ops.dropout calls for the
    standalone kind), with the same p, seed and mask shape."""
    bad = []
    for (b0, n0), (b1, _) in zip(advances, advances[1:]):
        if b1 != b0 + n0:
            bad.append(f"dropout_advance returned base {b1} after base {b0} + n {n0}: the counter did not advance by n")
    by_base = {}
    for u in uses:
        by_base.setdefault(u[1], []).append(u)
    ns = dict(advances)
    for base, us in sorted(by_base.items()):
        if base not in ns:
            bad.append(f"base {base} was not returned by any dropout_advance")
            continue
        sites = {u[2] for u in us}
        if sites != set(range(ns[base])):
            extra, missing = sorted(sites - set(range(ns[base]))), sorted(set(range(ns[base])) - sites)
            bad.append(f"base {base}: sites used are not range({ns[base]}): outside {extra[:8]}, unused {missing[:8]}")
    pairs = {}
    for u in uses:
        pairs.setdefault((u[1], u[2]), []).append(u)
    for (base, site), us in sorted(pairs.items()):
        kinds = {DROP_KIND[u[0]] for u in us}
        nb = sum(u[0] in DROP_BACKWARD for u in us)
        if len(us) != 2 or len(kinds) != 1 or (kinds != {"dropout"} and nb != 1):
            bad.append(f"stream (base {base}, site {site}) is drawn by {[u[0] for u in us]}: want one forward and one "
                       f"backward of one kind")
        elif len({(u[3], u[4], u[5]) for u in us}) != 1:
            bad.append(f"stream (base {base}, site {site}): forward and backward differ in (p, seed, mask shape): "
                       f"{[(u[3], u[4], u[5]) for u in us]}")
    return bad
