"""Decode-attention kernel A/B and end-to-end KV-cache generation throughput on one GPU.

1. Kernel: fsb_attn_decode (split-KV) against fsb_sdpa_fwd with one query row over the same masked cache (how LLaMA's decode
   step attends). Device time per call: 50 calls captured in one CUDA graph, the graph replayed under CUDA events, so host
   launch overhead is out of the figure (an eager loop of these ~30 us calls measures the Python / ctypes path instead; it is
   reported as *_eager_us). Shapes: GPT-2 (12 x 64) and mT5-784M (16 x 64) heads, rows 1 / 8 / 32,
   kv_len 128 / 512 / 1024 with kv_cap the next multiple of 64 above kv_len. Bytes = the K/V a row must read,
   2 * kv_len * heads * head_dim * 2 B per row; the share is against the 3.35 TB/s HBM3 data-sheet figure.
2. End to end: tokens/s of `generate` (greedy; beam 2 for T5), host wall time per new token, and the device (kernel) time per
   token from torch.profiler in a separate run. The gap between the two is host launch overhead.
   C5 Randeng-T5-784M: encoder 512, 64 new tokens, batch 8. C2 GPT-2 110M: prompt 512, 128 new tokens, batch 8.
   Random weights; eos is set to an id outside the vocabulary, which no step can produce, so every run generates exactly
   the stated number of tokens.

  python tools/bench_generate.py [--iters 200] [--out DIR]

Prints one JSON line per measurement with the card's name and power limit; --out also writes them to DIR/bench_generate.jsonl."""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402  (workload table, model builder)
from bench_validation import card  # noqa: E402
from fsb200 import ops  # noqa: E402

HBM = 3.35e12


def time_us(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / iters


def graph_us(fn, calls=50, reps=20):
    """Device time of one call: `calls` calls captured in a CUDA graph, replayed `reps` times between CUDA events."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / (reps * calls)


def kernel_ab(iters, emit):
    g = torch.Generator(device="cuda").manual_seed(0)
    for model, H in (("gpt2", 12), ("mt5-784m", 16)):
        D = 64
        for rows in (1, 8, 32):
            for n in (128, 512, 1024):
                cap = (n // 64 + 1) * 64
                q = torch.randn((rows, 1, H, D), generator=g, device="cuda").to(torch.bfloat16)
                k = torch.randn((rows, cap, H, D), generator=g, device="cuda").to(torch.bfloat16)
                v = torch.randn((rows, cap, H, D), generator=g, device="cuda").to(torch.bfloat16)
                mask = torch.zeros((rows, cap), dtype=torch.uint8, device="cuda")
                mask[:, :n] = 1
                kv_len = torch.tensor([n], dtype=torch.int32, device="cuda")
                scale = 1.0 / math.sqrt(D)
                o_ref, _ = ops.sdpa_fwd(q, k, v, scale, False, kv_mask=mask)
                o_new, _ = ops.attn_decode(q[:, 0], k, v, kv_len, scale, kv_mask=mask)
                diff = (o_ref[:, 0].float() - o_new.float()).abs().max().item()
                old = lambda: ops.sdpa_fwd(q, k, v, scale, False, kv_mask=mask)              # noqa: E731
                new = lambda: ops.attn_decode(q[:, 0], k, v, kv_len, scale, kv_mask=mask)    # noqa: E731
                e_old, e_new = time_us(old, iters), time_us(new, iters)
                t_old, t_new = graph_us(old), graph_us(new)
                nbytes = 2 * n * H * D * 2 * rows
                emit(dict(bench="attn_decode_ab", model=model, heads=H, head_dim=D, rows=rows, kv_len=n, kv_cap=cap,
                          sdpa_fwd_us=round(t_old, 2), attn_decode_us=round(t_new, 2), speedup=round(t_old / t_new, 2),
                          sdpa_fwd_eager_us=round(e_old, 2), attn_decode_eager_us=round(e_new, 2),
                          sdpa_fwd_GBps=round(nbytes / t_old / 1e3, 1), attn_decode_GBps=round(nbytes / t_new / 1e3, 1),
                          attn_decode_share_of_hbm=round(nbytes / t_new / 1e-6 / HBM, 3), max_abs_diff=diff))


def end_to_end(emit):
    cases = (("C5", "randeng-t5-784m", 512, 64, 8, dict()), ("C5", "randeng-t5-784m", 512, 64, 8, dict(num_beams=2)),
             ("C2", "gpt2-110m", 512, 128, 8, dict()))
    for tag, name, S, new, B, kw in cases:
        w = bench.workload(name)
        model = bench.build_model(w, "cuda", 1)
        ids = torch.randint(2, w["vocab_size"] - 8, (B, S), generator=torch.Generator().manual_seed(1)).cuda()
        args = dict(input_ids=ids, max_new_tokens=new, eos_token_id=w["vocab_size"], **kw)
        out = model.generate(**args)                     # warm-up: module load, workspaces, allocator
        torch.cuda.synchronize()
        reps = 3
        t0 = time.perf_counter()
        for _ in range(reps):
            out = model.generate(**args)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) / reps
        steps = out.shape[1] - (S if w["family"] == "gpt2" else 1)
        assert steps == new, (steps, new)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model.generate(**args)
            torch.cuda.synchronize()
        dev_us = sum(e.self_device_time_total for e in prof.key_averages())
        emit(dict(bench="generate", config=tag, model=name, batch=B, prompt=S, new_tokens=steps,
                  num_beams=kw.get("num_beams", 1), tokens_per_s=round(B * steps / wall, 1),
                  wall_ms_per_step=round(1e3 * wall / steps, 3), device_ms_per_step=round(dev_us / 1e3 / steps, 3)))
        del model
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_generate: no CUDA device")
    name, power = card()
    lines = []

    def emit(d):
        d.update(gpu=name, power_limit=power)
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    kernel_ab(a.iters, emit)
    if not a.skip_e2e:
        end_to_end(emit)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_generate.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
