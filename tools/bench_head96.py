"""GPT-2 at head width 96 (the 3.5B Wenzhong / Yuyuan shape: 30 layers, 32 heads x 96, hidden 3072, seq 1024) on one GPU.

1. Attention (`attn`): causal forward and backward at batch 8, seq 1024, dropout 0 and 0.1, for 32 x 96 against 24 x 128
   and 48 x 64. All three have heads x head_dim = 3072, so they do the same useful FLOPs per token; TFLOP/s is credited with
   the useful causal FLOPs (forward 2 matmuls, backward 5, half of each S x S product). Each shape's forward and backward
   are timed between CUDA events over `--iters` calls; the shapes alternate for `--reps` rounds; the median and the range
   over the rounds are reported.
2. Training step (`step`): full width (3072, 32 heads, V 50304) at `--layers` layers, seq 1024 x micro-batch 1/2/4, one
   ZeroEngine optimizer step (ZeRO-2, one GPU) per micro-batch: tokens/s, model TFLOP/s (bench.flops_per_token, which
   credits 6 N_mm + 3 F_attn per token) and peak allocated memory, median and range over `--reps` timed windows of
   `--steps` steps. `--full-depth` also tries all 30 layers at micro-batch 1 and reports whether they fit.
3. Generation (`generate`): all 30 layers (random weights, bf16), the Wenzhong README's sampling call (max_length 150,
   top_p 0.9, 5 return sequences), graph decode against eager decode (FSB_GENERATE_GRAPH), alternated `--reps` times:
   generated tokens/s and peak allocated memory.

  python tools/bench_head96.py [--sections attn step generate] [--layers 4 8] [--full-depth] [--out DIR]

Prints one JSON line per record, the card's name, power limit and max SM clock first; --out also writes them to
DIR/bench_head96.jsonl."""
import argparse
import gc
import json
import math
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
import bench  # noqa: E402  (read only: workload, build_model, flops_per_token)
from bench_int8 import card  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.engine import ZeroEngine  # noqa: E402

GIB = 2 ** 30
WIDTH = dict(n_embd=3072, n_head=32, vocab_size=50304, n_positions=1024)


def spread(xs):
    return dict(median=round(statistics.median(xs), 4), min=round(min(xs), 4), max=round(max(xs), 4), n=len(xs))


# ------------------------------------------------------------------------------------------------ 1. attention
def attn_case(H, D, B, S, p):
    g = torch.Generator(device="cuda").manual_seed(H)
    qkv = torch.randn(B, S, 3, H, D, device="cuda", generator=g).to(torch.bfloat16)
    dout = torch.randn(B, S, H, D, device="cuda", generator=g).to(torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    scale = 1.0 / math.sqrt(D)
    base = torch.zeros(1, dtype=torch.int64, device="cuda")
    drop = ops.Dropout(p, 1234, base, 1) if p > 0 else None
    out, lse = ops.sdpa_fwd(q, k, v, scale, True, drop=drop)

    def fwd():
        ops.sdpa_fwd(q, k, v, scale, True, drop=drop)

    def bwd():
        ops.sdpa_bwd(q, k, v, out, dout, lse, scale, True, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], drop=drop)
    return fwd, bwd


def event_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def section_attn(emit, iters, reps):
    B, S = 8, 1024
    shapes = [(32, 96), (24, 128), (48, 64)]
    useful = B * S * S * 3072 / 2 * 2    # one causal S x S x (H D) matmul: 2 flops per MAC, half the square
    for p in (0.0, 0.1):
        cases = {hd: attn_case(*hd, B, S, p) for hd in shapes}
        for fwd, bwd in cases.values():      # warm-up: module load, tensor maps
            for _ in range(3):
                fwd(); bwd()
        torch.cuda.synchronize()
        t = {hd: ([], []) for hd in shapes}
        for r in range(reps):
            order = shapes if r % 2 == 0 else shapes[::-1]
            for hd in order:
                fwd, bwd = cases[hd]
                t[hd][0].append(event_ms(fwd, iters))
                t[hd][1].append(event_ms(bwd, iters))
        for (H, D) in shapes:
            f, b = t[(H, D)]
            emit(dict(kind="attn", heads=H, head_dim=D, batch=B, seq=S, p=p, fwd_ms=spread(f), bwd_ms=spread(b),
                      fwd_tflops=round(2 * useful / (statistics.median(f) * 1e-3) / 1e12, 1),
                      bwd_tflops=round(5 * useful / (statistics.median(b) * 1e-3) / 1e12, 1)))
        del cases
        gc.collect(); torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 2. training step
def workload(L):
    return dict(bench.workload("gpt2-110m"), n_layer=L, **WIDTH)


def section_step(emit, layers, micros, steps, reps, full_depth):
    dev = torch.device("cuda", torch.cuda.current_device())
    configs = [(L, B) for L in layers for B in micros] + ([(30, 1)] if full_depth else [])
    for L in sorted({c[0] for c in configs}):
        w = workload(L)
        model = eng = None
        try:
            model = bench.build_model(w, dev, 1)
            eng = ZeroEngine(model, lr=1e-4, betas=w["betas"], weight_decay=w["wd"], grad_clip=w["clip"], stage=2)
            for B in [b for (l, b) in configs if l == L]:
                S = 1024
                g = torch.Generator(device="cuda").manual_seed(1)
                ids = torch.randint(0, w["vocab_size"], (B, S), device="cuda", generator=g)

                def one():
                    out = model(input_ids=ids, labels=ids)
                    out.loss.backward()
                    eng.backward_done()
                    eng.step()
                for _ in range(2):
                    one()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                times = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    for _ in range(steps):
                        one()
                    torch.cuda.synchronize()
                    times.append((time.perf_counter() - t0) / steps)
                dt = statistics.median(times)
                tok = [B * S / x for x in times]
                emit(dict(kind="step", layers=L, seq=S, micro=B, zero_stage=2, step_ms=spread([1e3 * x for x in times]),
                          tokens_per_s=spread(tok),
                          model_tflops=round(B * S / dt * bench.flops_per_token(dict(w, seq=S)) / 1e12, 1),
                          peak_alloc_gib=round(torch.cuda.max_memory_allocated() / GIB, 2)))
        except torch.cuda.OutOfMemoryError as e:
            emit(dict(kind="step", layers=L, fits=False, reason=f"out of memory on one card: {str(e).splitlines()[0]}"))
        finally:
            del model, eng
            gc.collect(); torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 3. generate
def section_generate(emit, reps):
    dev = torch.device("cuda", torch.cuda.current_device())
    w = workload(30)
    model = bench.build_model(w, dev, 1)
    model.eval()
    prompt = torch.randint(4, w["vocab_size"], (1, 32), generator=torch.Generator().manual_seed(0)).cuda()
    kw = dict(max_length=150, do_sample=True, top_p=0.9, num_return_sequences=5, return_dict_in_generate=True,
              output_scores=True, eos_token_id=w["vocab_size"] - 1, pad_token_id=0)
    res = {"0": [], "1": []}
    peak = {}
    for flag in ("0", "1"):       # warm-up (graph capture included in the first graphed call)
        os.environ["FSB_GENERATE_GRAPH"] = flag
        torch.manual_seed(0)
        model.generate(input_ids=prompt, **kw)
    for r in range(reps):
        for flag in (("0", "1") if r % 2 == 0 else ("1", "0")):
            os.environ["FSB_GENERATE_GRAPH"] = flag
            torch.manual_seed(0)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            out = model.generate(input_ids=prompt, **kw)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            new = (out.sequences.shape[1] - prompt.shape[1]) * out.sequences.shape[0]
            res[flag].append(new / dt)
            peak[flag] = max(peak.get(flag, 0), torch.cuda.max_memory_allocated())
    for flag, name in (("0", "eager"), ("1", "graph")):
        emit(dict(kind="generate", decode=name, layers=30, prompt=32, max_length=150, top_p=0.9, num_return_sequences=5,
                  tokens_per_s=spread(res[flag]), peak_alloc_gib=round(peak[flag] / GIB, 2)))
    del model
    gc.collect(); torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", nargs="+", default=["attn", "step", "generate"])
    ap.add_argument("--layers", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--micro", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--full-depth", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_head96: needs a CUDA device")
    sink = []

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        sink.append(line)

    emit(dict(kind="card", **card()))
    if "attn" in a.sections:
        section_attn(emit, a.iters, a.reps)
    if "step" in a.sections:
        section_step(emit, a.layers, a.micro, a.steps, a.reps, a.full_depth)
    if "generate" in a.sections:
        section_generate(emit, a.reps)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_head96.jsonl"), "w") as f:
            f.write("\n".join(sink) + "\n")


if __name__ == "__main__":
    main()
