"""FP8 (fp8=True) against bf16 LLaMA training on one GPU.

1. Kernels at Ziya-LLaMA-13B width (hidden 5120, ff 13824) with 8192 token rows, for each projection (query_key_value,
   dense, w1|w3, w2) in its three roles: forward (m = 8192, n = out, k = in), data gradient (m = 8192, n = in, k = out) and
   weight gradient (m = out, n = in, k = 8192). fsb_gemm_fp8 against fsb_gemm_bf16 (NT / NN / TN) on the same shape, device
   time per call from `calls` calls captured in one CUDA graph and replayed under CUDA events, the two alternated `--reps`
   times (medians and the spread). TFLOP/s = 2mnk / time, beside the 1,979 (FP8) / 989 (bf16) dense data-sheet figures.
   fsb_fp8_quantize of the GEMM's A operand (both layouts): GB/s of 2 reads of the bf16 tensor (amax, cast) plus the two
   code writes, beside 3.35 TB/s.
2. The Ziya-width 4-layer training step (vocabulary 39424, 40 heads, seq 2048, micro-batch 4), ZeRO engine on one GPU: tokens/s
   over `--steps` steps after `--warmup`, and peak torch.cuda.max_memory_allocated over the timed steps, fp8 and bf16
   alternated `--reps` times, which one goes first swapped every repetition. One model is alive at a time: the model and
   its engine reference each other (the engine's gradient hook), so each run ends with gc.collect() before empty_cache(),
   and every run checks that the allocated memory is back within 64 MiB of the level it started from, apart from the
   library's grow-only scratch buffers (fsb200.ops.workspace).

  python tools/bench_fp8.py [--reps 3] [--steps 6] [--warmup 2] [--skip-kernels] [--skip-step] [--out DIR]

Prints one JSON line per measurement, the card's name, power limit and max SM clock first; --out also writes them to
DIR/bench_fp8.jsonl."""
import argparse
import gc
import json
import os
import statistics
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
from bench_int8 import card, graph_us  # noqa: E402
from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.engine import ZeroEngine  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402

H, FF, T = 5120, 13824, 8192
PROJ = (("qkv", 3 * H, H), ("dense", H, H), ("w1w3", 2 * FF, H), ("w2", H, FF))
HBM, PEAK_FP8, PEAK_BF16 = 3.35e12, 1979e12, 989e12


def emit(rec, sink):
    line = json.dumps(rec)
    print(line, flush=True)
    sink.append(line)


def kernels(reps, sink):
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n_out, k_in in PROJ:
        for role, (m, n, k) in (("fwd", (T, n_out, k_in)), ("dgrad", (T, k_in, n_out)), ("wgrad", (n_out, k_in, T))):
            a_fmt = "e4m3" if role == "fwd" else "e5m2"
            a16 = torch.randn((m, k), device="cuda", generator=g).to(torch.bfloat16)
            b16 = (torch.randn((n, k), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
            aq, _, sa = ops.fp8_quantize(a16, a_fmt)
            bq, _, sb = ops.fp8_quantize(b16, "e4m3")
            d = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
            # the bf16 GEMM in the layout the bf16 model runs for this role, on operands of the same extents
            if role == "fwd":
                bf = lambda: ops.gemm(L.GEMM_NT, a16, b16, out=d)
            elif role == "dgrad":
                bt = b16.t().contiguous()          # [k, n]
                bf = lambda: ops.gemm(L.GEMM_NN, a16, bt, out=d)
            else:
                at, btt = a16.t().contiguous(), b16.t().contiguous()   # [k, m], [k, n]
                bf = lambda: ops.gemm(L.GEMM_TN, at, btt, out=d)
            f8 = lambda: ops.gemm_fp8(aq, sa, bq, sb, out=d)
            q8 = lambda: ops.fp8_quantize(a16, a_fmt, rowwise=True, colwise=True)
            t8, t16, tq = [], [], []
            for _ in range(reps):
                t8.append(graph_us(f8)); t16.append(graph_us(bf)); tq.append(graph_us(q8, calls=20))
            flops = 2.0 * m * n * k
            qbytes = 2 * (2 * m * k) + 2 * m * k
            u8, u16, uq = statistics.median(t8), statistics.median(t16), statistics.median(tq)
            emit(dict(kind="gemm", proj=name, role=role, m=m, n=n, k=k,
                      fp8_us=round(u8, 1), fp8_us_all=[round(x, 1) for x in t8],
                      bf16_us=round(u16, 1), bf16_us_all=[round(x, 1) for x in t16],
                      fp8_tflops=round(flops / u8 / 1e6, 1), bf16_tflops=round(flops / u16 / 1e6, 1),
                      fp8_of_1979=round(flops / u8 / 1e6 / (PEAK_FP8 / 1e12), 3),
                      bf16_of_989=round(flops / u16 / 1e6 / (PEAK_BF16 / 1e12), 3),
                      speedup=round(u16 / u8, 3),
                      quantize_us=round(uq, 1), quantize_gbs=round(qbytes / uq / 1e3, 1),
                      quantize_of_3350=round(qbytes / uq / 1e3 / 3350, 3)), sink)
            del a16, b16, aq, bq, d
            torch.cuda.empty_cache()


def _scratch_bytes():
    return sum(b.numel() * b.element_size() for b in ops._ws_cache.values())


def step(fp8, steps, warmup, sink):
    gc.collect()
    torch.cuda.empty_cache()
    base, ws0 = torch.cuda.memory_allocated(), _scratch_bytes()
    cfg = SimpleNamespace(vocab_size=39424, hidden_size=H, num_hidden_layers=4, num_attention_heads=40,
                          rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                          llama_mlp_multiple_of=256)
    B, S = 4, 2048
    model = LlamaForCausalLM(cfg, device="cuda", fp8=fp8)
    eng = ZeroEngine(model, lr=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=g)
    losses = []

    def one():
        out = model(input_ids=ids, labels=ids)
        out.loss.backward()
        eng.backward_done()
        eng.step()
        return out.loss

    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for _ in range(steps):
        losses.append(one().detach())
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rec = dict(kind="step", fp8=fp8, layers=4, batch=B, seq=S, steps=steps, tokens_per_s=round(B * S * steps / dt),
               step_ms=round(1e3 * dt / steps, 1), peak_alloc_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
               alloc_before_gib=round(base / 2 ** 30, 3), loss_last=round(float(losses[-1]), 4))
    del model, eng, losses, one
    gc.collect()          # the model <-> engine reference cycle: without it the model's memory outlives the run
    torch.cuda.empty_cache()
    left, grown = torch.cuda.memory_allocated(), _scratch_bytes() - ws0
    rec["alloc_after_gib"] = round(left / 2 ** 30, 3)
    rec["scratch_grown_mib"] = round(grown / 2 ** 20, 1)
    rec["other_left_bytes"] = left - base - grown
    emit(rec, sink)
    # Beyond the library's grow-only scratch (ops.workspace), small process-wide caches may stay (tens of KB); a model that
    # outlived its run would leave GiBs and inflate the next run's peak.
    if left - base - grown > 64 << 20:
        raise SystemExit(f"bench_fp8: {left - base - grown} bytes still allocated after the {'fp8' if fp8 else 'bf16'} run")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8: needs a CUDA device")
    sink = []
    emit(dict(kind="card", **card()), sink)
    if not a.skip_kernels:
        kernels(a.reps, sink)
    if not a.skip_step:
        for r in range(a.reps):
            for fp8 in ((True, False) if r % 2 == 0 else (False, True)):
                step(fp8, a.steps, a.warmup, sink)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fp8.jsonl"), "w") as f:
            f.write("\n".join(sink) + "\n")


if __name__ == "__main__":
    main()
