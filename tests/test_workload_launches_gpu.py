"""Census of the benchmark's training step: every launch of each bench.WORKLOADS entry, checked against fp64.

Each workload is built at full width with 2 layers (T5: 2 encoder and 2 decoder layers; the middle layers repeat the first
and last layer's launches) at the benchmark's micro-batch, sequence lengths and ZeRO stage, with ga = min(bench ga, 2), and
runs one eager optimizer step. Every public `fsb200.ops` function is wrapped by the recorder of tests/launch_census.py: the
outermost call (a reentrancy guard skips calls an op makes through another) is keyed by its signature — the op, each
tensor's shape, strides, dtype and 16-byte alignment class, the scalar flags, which optional operands are present. The first
call of every signature goes through its tests/launch_refs.py checker; the rest are counted. The engine reaches AdamW, the
gradient norm and the fp32 accumulation through the `ops` module (ZeroEngine's default `kernels`), so the patch reaches the
optimizer too.

Asserted: (a) every op the step called has a checker, (b) lib.launch_count grew by exactly the launches of the wrapped calls
(no kernel bypassed `ops`), (c) every checked signature is within its bound, (d) the loss is finite. `-s` prints the census.
"""
import gc
import math
import os
import sys
import time

import pytest
import torch

import launch_refs as R
from launch_census import Recorder, free_gib as _free_gib, print_table as _table

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (read only: WORKLOADS, build_model, make_host_batches)

from fsb200 import lib as L, ops  # noqa: E402

# device memory (GiB) each census run needs, its fp64 checks included: the peak allocated on one H100 80GB HBM3 (GPT-2 9.6,
# BERT-base 1.8, MegatronBERT 8.9, T5 7.2, LLaMA 25.2; no check needs more than 6 GiB above the step's own memory) plus
# 2 GiB for the allocator's rounding
NEED_GIB = {"gpt2-110m": 12, "bert-base": 4, "megatronbert-1.3b": 11, "randeng-t5-784m": 10, "ziya-llama-13b": 28}


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
