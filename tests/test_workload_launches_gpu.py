"""Census of the benchmark's training step: every launch of each bench.WORKLOADS entry, checked against fp64.

Each workload is built at full width with 2 layers (T5: 2 encoder and 2 decoder layers; the middle layers repeat the first
and last layer's launches) at the benchmark's micro-batch, sequence lengths and ZeRO stage, with ga = min(bench ga, 2), and
runs one eager optimizer step. Every public `fsb200.ops` function is wrapped by a recorder: the outermost call (a
reentrancy guard skips calls an op makes through another) is keyed by its signature — the op, each tensor's shape, strides,
dtype and 16-byte alignment class, the scalar flags, which optional operands are present. The first call of every signature
goes through its tests/launch_refs.py checker; the rest are counted. The engine reaches AdamW, the gradient norm and the
fp32 accumulation through the `ops` module (ZeroEngine's default `kernels`), so the patch reaches the optimizer too.

Asserted: (a) every op the step called has a checker, (b) lib.launch_count grew by exactly the launches of the wrapped calls
(no kernel bypassed `ops`), (c) every checked signature is within its bound, (d) the loss is finite. `-s` prints the census.
"""
import functools
import gc
import inspect
import math
import os
import sys
import time

import pytest
import torch

import launch_refs as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (read only: WORKLOADS, build_model, make_host_batches)

from fsb200 import lib as L, ops  # noqa: E402

# public ops functions that launch no kernel of their own: they are not recorded
NOT_LAUNCHES = {"workspace", "set_profiler", "set_reserved_sms"}
# device memory (GiB) each census run needs, its fp64 checks included: the peak allocated on one H100 80GB HBM3 (GPT-2 9.6,
# BERT-base 1.8, MegatronBERT 8.9, T5 7.2, LLaMA 25.2; no check needs more than 6 GiB above the step's own memory) plus
# 2 GiB for the allocator's rounding
NEED_GIB = {"gpt2-110m": 12, "bert-base": 4, "megatronbert-1.3b": 11, "randeng-t5-784m": 10, "ziya-llama-13b": 28}


def _ops_functions():
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

    def __init__(self, checkers):
        self.checkers = checkers
        self.depth = 0
        self.calls = {}          # (op, signature) -> count
        self.worst = {}          # (op, signature) -> err / bound of its checked call
        self.wrapped_launches = 0
        self.extra_launches = 0  # launches the checkers issue themselves (the aux re-run of a GeLU GEMM)
        self.check_mem = {}      # (op, signature) -> device memory its checked call needed above what was allocated before
        self.peak = 0            # peak allocated over the step (torch's peak counter is reset around each check)

    def install(self, monkeypatch):
        for name, fn in _ops_functions().items():
            monkeypatch.setattr(ops, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)

        @functools.wraps(fn)
        def wrapper(*args, **kwargs):
            if self.depth:
                return fn(*args, **kwargs)
            bound_args = sig.bind(*args, **kwargs)
            key = (name, tuple((k, _key_of(v)) for k, v in bound_args.arguments.items()))
            first = key not in self.calls
            self.calls[key] = self.calls.get(key, 0) + 1
            self.depth += 1
            try:
                if not first:
                    c0 = L.launch_count
                    ret = fn(*args, **kwargs)
                    self.wrapped_launches += L.launch_count - c0
                    return ret
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
                self.check_mem[key] = m1 - m0
                self.wrapped_launches += deltas[0]
                self.extra_launches += sum(deltas[1:])   # re-runs inside the checker (the plain GEMM an aux is compared with)
                self.worst[key] = b.worst
                return ret
            finally:
                self.depth -= 1
        return wrapper


def _free_gib():
    free, _ = torch.cuda.mem_get_info()
    return free / 2 ** 30


def _layers(w):
    w = dict(w)
    for k in ("n_layer", "num_hidden_layers", "num_layers"):
        if k in w:
            w[k] = 2
    return w


def _run_census(name, monkeypatch, checkers=None):
    torch.manual_seed(0)
    w = _layers(bench.workload(name))
    w["micro"] = min(w["micro"], w["per_gpu"])
    ga = min(w["per_gpu"] // w["micro"], 2)
    from fsb200.schedules import polynomial_lr
    from fsb200.trainer import PretrainStep
    dev = torch.device("cuda", torch.cuda.current_device())
    model = bench.build_model(w, dev, 1)
    stepper = PretrainStep(model, lambda s_: polynomial_lr(s_, w["lr"], 10, 1000, 1e-7), lr=w["lr"], betas=w["betas"],
                           weight_decay=w["wd"], grad_clip=w["clip"], ga_steps=ga, stage=w.get("stage", 2),
                           cuda_graph=False)
    batches = [{k: v.to(dev) for k, v in b.items()} for b in bench.make_host_batches(w, ga, 0)]
    rec = Recorder(R.CHECKERS if checkers is None else checkers)
    rec.install(monkeypatch)
    torch.cuda.synchronize()
    c0 = L.launch_count
    try:
        loss = stepper.step_device(batches)
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    growth = L.launch_count - c0
    return rec, growth, loss


def _census(name, monkeypatch, checkers=None):
    """_run_census with the model freed on failure too: the failure is re-raised without the traceback that holds it, so
    the next workload finds the device memory free."""
    msg = None
    try:
        return _run_census(name, monkeypatch, checkers)
    except AssertionError as e:
        msg = str(e)
    gc.collect(); torch.cuda.empty_cache()
    raise AssertionError(msg)


def _table(name, rec, secs, peak):
    rows = {}
    for (op, sig), n in rec.calls.items():
        r = rows.setdefault(op, [0, 0, 0.0, 0])
        r[0] += 1; r[1] += n
        r[2] = max(r[2], rec.worst.get((op, sig), 0.0))
        r[3] = max(r[3], rec.check_mem.get((op, sig), 0))
    print(f"\n[census] {name}: {sum(r[0] for r in rows.values())} signatures, {sum(r[1] for r in rows.values())} calls, "
          f"{secs:.1f} s wall, peak {peak / 2 ** 30:.1f} GiB")
    print(f"[census] {'op':<18} {'signatures':>10} {'calls':>6} {'worst err/bound':>16} {'check GiB':>10}")
    for op in sorted(rows):
        s, n, wr, mem = rows[op]
        print(f"[census] {op:<18} {s:>10} {n:>6} {wr:>16.3g} {mem / 2 ** 30:>10.2f}")


@pytest.mark.parametrize("name", list(bench.WORKLOADS))
def test_every_launch_of_the_step_against_fp64(name, monkeypatch):
    need = NEED_GIB[name]
    gc.collect(); torch.cuda.empty_cache()     # what earlier tests left in torch's cache counts as free here
    if _free_gib() < need:
        pytest.skip(f"{name} at full width with 2 layers, its ZeRO state and the fp64 checks need about {need} GiB free; "
                    f"{_free_gib():.1f} GiB are")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    rec, growth, loss = _census(name, monkeypatch)
    secs = time.time() - t0
    _table(name, rec, secs, max(rec.peak, torch.cuda.max_memory_allocated()))
    assert growth - rec.extra_launches == rec.wrapped_launches, \
        (f"lib.launch_count grew by {growth - rec.extra_launches} over the step (checker re-runs excluded) but the wrapped "
         f"ops calls launched {rec.wrapped_launches}: a kernel was reached without going through fsb200.ops")
    assert math.isfinite(float(loss.item())), f"{name}: loss {loss.item()}"
    gc.collect(); torch.cuda.empty_cache()


def test_census_names_an_op_without_checker(monkeypatch):
    """Deleting a checker makes the census fail and name the op it lost."""
    checkers = dict(R.CHECKERS)
    del checkers["layernorm_bwd"]
    with pytest.raises(AssertionError, match="ops.layernorm_bwd has no launch reference"):
        _census("bert-base", monkeypatch, checkers)
    gc.collect(); torch.cuda.empty_cache()


def test_census_catches_a_launch_that_bypasses_ops(monkeypatch):
    """An fsb_add issued through lib.call outside any ops wrapper makes assertion (b) fail; without it (b) holds."""
    a = torch.ones(64, dtype=torch.bfloat16, device="cuda")
    rec = Recorder(R.CHECKERS)
    rec.install(monkeypatch)
    c0 = L.launch_count
    ops.add(a, a)
    assert L.launch_count - c0 - rec.extra_launches == rec.wrapped_launches == 1
    out = torch.empty_like(a)
    L.call("fsb_add", a.data_ptr(), a.data_ptr(), out.data_ptr(), a.numel(), torch.cuda.current_stream().cuda_stream)
    assert L.launch_count - c0 - rec.extra_launches != rec.wrapped_launches
    monkeypatch.undo()
