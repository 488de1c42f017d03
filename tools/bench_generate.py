"""Decode-attention kernel A/B and end-to-end KV-cache generation throughput on one GPU.

1. Kernel: fsb_attn_decode (split-KV) against fsb_sdpa_fwd with one query row over the same masked cache (how LLaMA's decode
   step attends). Device time per call: 50 calls captured in one CUDA graph, the graph replayed under CUDA events, so host
   launch overhead is out of the figure (an eager loop of these ~30 us calls measures the Python / ctypes path instead; it is
   reported as *_eager_us). Shapes: GPT-2 (12 x 64) and mT5-784M (16 x 64) heads, rows 1 / 8 / 32,
   kv_len 128 / 512 / 1024 with kv_cap the next multiple of 64 above kv_len. Bytes = the K/V a row must read,
   2 * kv_len * heads * head_dim * 2 B per row; the share is against the 3.35 TB/s HBM3 data-sheet figure.
2. Beam reorder: fsb_kv_reorder (every layer in one launch, live slots only) against the per-layer full-capacity index_select
   it replaced, at the C5 beam shape, timed the same way.
3. End to end: the CUDA-graph decode step against the same step body run eagerly (FSB_GENERATE_GRAPH=0), the two alternated
   `--reps` times in one process (medians reported): tokens/s and host wall time per new token, device (kernel) time per
   token from torch.profiler in a separate run, host `fsb_*` calls per token, the host time spent capturing, and the peak
   memory `generate` allocates above the model (the beam twin included). The two modes must produce the same tokens.
   C5 Randeng-T5-784M: encoder 512, 64 new tokens, batch 8, greedy and 2 beams. C2 GPT-2 110M: prompt 512, 128 new tokens,
   batch 8; and 3 new tokens, the shortest run with a capture, where the capture is not amortised. Ziya-LLaMA-13B width
   (hidden 5120, 40 heads) at 8 of its 40 layers: prompt 512, 128 new tokens, batch 8.
   Random weights; eos is set to an id outside the vocabulary (LLaMA: none), so every run generates exactly the stated
   number of tokens.

  python tools/bench_generate.py [--iters 200] [--reps 3] [--skip-e2e] [--out DIR]

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
from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.decode_graph import DecodeGraphs  # noqa: E402

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


def _count_calls():
    """Wrap lib.call with a counter of host `fsb_*` calls; returns the counter (a one-element list)."""
    n = [0]
    real = L.call

    def counted(name, *args, **kw):
        n[0] += 1
        return real(name, *args, **kw)
    L.call = counted
    return n


def _time_captures():
    """Wrap DecodeGraphs._capture with a host clock; returns the running total in seconds (a one-element list)."""
    total = [0.0]
    real = DecodeGraphs._capture

    def timed(self, key):
        torch.cuda.synchronize()         # the work queued before the capture is not part of it
        t0 = time.perf_counter()
        real(self, key)
        torch.cuda.synchronize()
        total[0] += time.perf_counter() - t0
    DecodeGraphs._capture = timed
    return total


LLAMA_LAYERS = 8   # Ziya-LLaMA-13B width (hidden 5120, 40 heads, vocabulary 39424) at 8 of its 40 layers on one GPU


def end_to_end(emit, reps):
    """Graphed decode step against the same step run eagerly (FSB_GENERATE_GRAPH=0), alternated in one process."""
    calls, capture_s = _count_calls(), _time_captures()
    cases = (("C5", "randeng-t5-784m", 512, 64, 8, dict()), ("C5", "randeng-t5-784m", 512, 64, 8, dict(num_beams=2)),
             ("C2", "gpt2-110m", 512, 128, 8, dict()), ("C4-width", f"ziya-llama-13b-L{LLAMA_LAYERS}", 512, 128, 8, dict()),
             ("C2", "gpt2-110m", 512, 3, 8, dict()))
    for tag, name, S, new, B, kw in cases:
        w = bench.workload(name)
        model = bench.build_model(w, "cuda", 1)
        ids = torch.randint(2, w["vocab_size"] - 8, (B, S), generator=torch.Generator().manual_seed(1)).cuda()
        if w["family"] == "llama":
            gen = lambda: model.generate(ids, max_length=S + new)                                   # noqa: E731
        else:
            gen = lambda: model.generate(input_ids=ids, max_new_tokens=new, eos_token_id=w["vocab_size"], **kw)  # noqa: E731
        modes = ("eager", "graph")
        res = {m: dict(wall=[], calls=0, capture=0.0, peak=0, out=None) for m in modes}
        base = torch.cuda.memory_allocated()
        for m in modes:                                  # warm-up: module load, workspaces, allocator
            os.environ["FSB_GENERATE_GRAPH"] = "0" if m == "eager" else "1"
            gen()
        for _ in range(reps):
            for m in modes:
                os.environ["FSB_GENERATE_GRAPH"] = "0" if m == "eager" else "1"
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                calls[0], capture_s[0] = 0, 0.0
                t0 = time.perf_counter()
                out = gen()
                torch.cuda.synchronize()
                r = res[m]
                r["wall"].append(time.perf_counter() - t0)
                r["calls"], r["capture"] = calls[0], capture_s[0]
                r["peak"] = max(r["peak"], torch.cuda.max_memory_allocated() - base)
                r["out"] = out
        assert torch.equal(res["eager"]["out"], res["graph"]["out"]), "graphed decode differs from the eager decode"
        steps = res["graph"]["out"].shape[1] - (S if w["family"] != "t5" else 1)
        assert steps == new, (steps, new)
        from torch.profiler import ProfilerActivity, profile
        for m in modes:
            os.environ["FSB_GENERATE_GRAPH"] = "0" if m == "eager" else "1"
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                gen()
                torch.cuda.synchronize()
            res[m]["dev_us"] = sum(e.self_device_time_total for e in prof.key_averages())
        line = dict(bench="generate_graph_ab", config=tag, model=name, batch=B, prompt=S, new_tokens=steps,
                    num_beams=kw.get("num_beams", 1), reps=reps)
        for m in modes:
            r = res[m]
            wall = sorted(r["wall"])[len(r["wall"]) // 2]
            line.update({f"{m}_tokens_per_s": round(B * steps / wall, 1), f"{m}_wall_ms_per_token": round(1e3 * wall / steps, 3),
                         f"{m}_device_ms_per_token": round(r["dev_us"] / 1e3 / steps, 3),
                         f"{m}_host_calls_per_token": round(r["calls"] / steps, 1),
                         f"{m}_peak_mem_MiB": round(r["peak"] / 2 ** 20, 1)})
        line["graph_capture_ms"] = round(1e3 * res["graph"]["capture"], 2)
        line["graph_speedup"] = round(line["graph_tokens_per_s"] / line["eager_tokens_per_s"], 3)
        emit(line)
        del model, gen, res
        torch.cuda.empty_cache()
    os.environ.pop("FSB_GENERATE_GRAPH", None)


def reorder_ab(emit):
    """fsb_kv_reorder (all layers, live slots only, one launch) against the per-layer full-capacity index_select it replaces,
    at the C5 beam shape: 24 decoder layers, 8 items x 2 beams, 16 heads x 64, capacity 128 (64 new tokens)."""
    w = bench.workload("randeng-t5-784m")
    Ly, R, cap, H, D = w["num_layers"], 16, 128, w["num_heads"], w["d_kv"]
    g = torch.Generator(device="cuda").manual_seed(0)
    src = torch.randn((Ly, R, cap, 2, H, D), generator=g, device="cuda").to(torch.bfloat16)
    dst = torch.empty_like(src)
    idx = (torch.arange(R, device="cuda") // 2) * 2 + torch.randint(0, 2, (R,), generator=g, device="cuda")
    layers = list(src.unbind(0))
    for n in (1, 32, 64):
        kv_len = torch.tensor([n], dtype=torch.int32, device="cuda")
        ops.kv_reorder(src, dst, idx, kv_len)
        assert torch.equal(dst[:, :, :n], src.index_select(1, idx)[:, :, :n])
        t_new = graph_us(lambda: ops.kv_reorder(src, dst, idx, kv_len))                      # noqa: B023
        t_old = graph_us(lambda: [kv.index_select(0, idx) for kv in layers])                   # noqa: B023
        nbytes = 2 * Ly * R * n * 2 * H * D * 2
        emit(dict(bench="kv_reorder_ab", layers=Ly, rows=R, kv_cap=cap, heads=H, head_dim=D, kv_len=n,
                  kv_reorder_us=round(t_new, 2), index_select_us=round(t_old, 2), speedup=round(t_old / t_new, 2),
                  kv_reorder_GBps=round(nbytes / t_new / 1e3, 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
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
    reorder_ab(emit)
    if not a.skip_e2e:
        end_to_end(emit, a.reps)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_generate.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
