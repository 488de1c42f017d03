"""Int8 (W8A16) and int4 (W4A16) weight-only LLaMA inference on one GPU.

1. Kernel A/B/C: fsb_gemm_w8a16 and fsb_gemm_w4a16 against fsb_gemm_bf16 (NT) on the Ziya-LLaMA-13B projection shapes
   (n, k) = (15360, 5120) query_key_value, (5120, 5120) dense, (27648, 5120) w1|w3, (5120, 13824) w2, at m = 1, 8, 32 token
   rows (decode) and 4096 (prefill). Device time per call: 50 calls captured in one CUDA graph, the graph replayed under
   CUDA events; the three kernels alternated `--reps` times, medians reported. Bytes per call: int8 n*k + 4n (weights and
   scales) + 2mk + 2mn, int4 n*k/2 + 2n*k/128 + 2mk + 2mn, bf16 2nk + 2mk + 2mn; GB/s and the share of the 3.35 TB/s HBM3
   data-sheet figure for m <= 32, TFLOP/s (2mnk) at 4096.
2. End to end: `generate` at Ziya width (hidden 5120, 40 heads, ff 13824, vocabulary 39424), prompt 512, 128 new tokens,
   batch 1 and 8, greedy, random weights: bf16, int8 and int4 at 8 of the 40 layers, int8 and int4 at all 40. Tokens/s (host wall clock,
   median of `--reps`), device time per new token (torch.profiler, prefill included, separate run), host `fsb_*` calls per
   new token, and the peak of torch.cuda.max_memory_allocated over building the model and generating, above what was
   allocated before.

With --model gpt2, int8 / int4 GPT-2 at the 3.5B Wenzhong / Yuyuan width (hidden 3072, 32 heads x 96, inner 12288,
vocabulary 50304, 30 layers):
1. Kernel A/B/C: fsb_gemm_w8a16_bias and fsb_gemm_w4a16_bias against fsb_gemm_bf16 (NN, the Conv1D layout) with the same
   bias / GELU epilogue, at (n, k) = (9216, 3072) c_attn, (3072, 3072) attn.c_proj, (12288, 3072) mlp.c_fc (bias + gelu_new),
   (3072, 12288) mlp.c_proj; m = 1, 5, 8, 32 (GB/s, bytes as above plus 2n of bias) and 1024 (TFLOP/s).
2. End to end: `generate` with random weights at all 30 layers in bf16, int8 and int4, CUDA-graph decode: the Wenzhong README
   sampling call (32-token prompt, max_length 150, top_p 0.9, 5 return sequences) and greedy at batch 1 and 8 (32-token
   prompt, 118 new tokens). Tokens/s (host wall clock, median of `--reps`), peak memory and get_memory_footprint.

  python tools/bench_int8.py [--model llama|gpt2] [--reps 3] [--skip-e2e] [--skip-40] [--out DIR]

Prints one JSON line per measurement, the card's name, power limit and max SM clock first; --out also writes them to
DIR/bench_int8.jsonl."""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.models.gpt2 import GPT2LMHeadModel  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402

HBM = 3.35e12
ZIYA = dict(vocab_size=39424, hidden_size=5120, num_attention_heads=40)
SHAPES = (("qkv", 15360, 5120), ("dense", 5120, 5120), ("w1w3", 27648, 5120), ("w2", 5120, 13824))
WENZHONG = dict(vocab_size=50304, n_positions=1024, n_embd=3072, n_head=32, n_layer=30)
GPT2_SHAPES = (("c_attn", 9216, 3072, L.EPI_NONE), ("attn.c_proj", 3072, 3072, L.EPI_NONE),
               ("mlp.c_fc", 12288, 3072, L.EPI_GELU_TANH), ("mlp.c_proj", 3072, 12288, L.EPI_NONE))


def card():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", bus],
                       capture_output=True, text=True, check=True)
    name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


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


def kernel_ab(reps, emit):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, n, k in SHAPES:
        w = (torch.randn((n, k), generator=gen, device="cuda") * 0.02).to(torch.bfloat16)
        q, s = ops.quantize_w8(w)
        q4, s4 = ops.quantize_w4(w)
        w4 = dequantize_w4(q4, s4)
        for m in (1, 8, 32, 4096):
            a = torch.randn((m, k), generator=gen, device="cuda").to(torch.bfloat16)
            d8 = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
            d4 = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
            d16 = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
            f16 = lambda: ops.gemm(L.GEMM_NT, a, w, out=d16)            # noqa: E731  (the decode step's bf16 call)
            f8 = lambda: ops.gemm_w8a16(a, q, s, out=d8)                # noqa: E731
            f4 = lambda: ops.gemm_w4a16(a, q4, s4, out=d4)              # noqa: E731
            t16, t8, t4 = [], [], []
            for _ in range(reps):
                t16.append(graph_us(f16))
                t8.append(graph_us(f8))
                t4.append(graph_us(f4))
            t16, t8, t4 = sorted(t16)[reps // 2], sorted(t8)[reps // 2], sorted(t4)[reps // 2]
            # each result against the bf16 GEMM of its dequantised weight (a sanity figure, not a test)
            ref = ops.gemm(L.GEMM_NT, a, (q.float() * s[:, None]).to(torch.bfloat16)).float()
            rel = float((d8.float() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
            ref4 = ops.gemm(L.GEMM_NT, a, w4).float()
            rel4 = float((d4.float() - ref4).abs().max() / ref4.abs().max().clamp_min(1e-30))
            b8 = n * k + 4 * n + 2 * m * k + 2 * m * n
            b4 = n * k // 2 + 2 * n * (k // 128) + 2 * m * k + 2 * m * n
            b16 = 2 * n * k + 2 * m * k + 2 * m * n
            line = dict(bench="gemm_weight_only_ab", shape=name, m=m, n=n, k=k, bf16_us=round(t16, 2), int8_us=round(t8, 2),
                        int4_us=round(t4, 2), speedup=round(t16 / t8, 3), int4_speedup=round(t16 / t4, 3),
                        int4_over_int8=round(t8 / t4, 3),
                        splitk_workspace_bytes=int(L.load().fsb_gemm_w8a16_workspace_bytes(m, n, k)),
                        max_rel_diff_vs_dequantised_bf16=rel, int4_max_rel_diff_vs_dequantised_bf16=rel4, reps=reps)
            if m <= 32:
                line.update(int8_GBps=round(b8 / t8 / 1e3, 1), int4_GBps=round(b4 / t4 / 1e3, 1), bf16_GBps=round(b16 / t16 / 1e3, 1),
                            int8_share_of_hbm=round(b8 / (t8 * 1e-6) / HBM, 3), int4_share_of_hbm=round(b4 / (t4 * 1e-6) / HBM, 3),
                            bf16_share_of_hbm=round(b16 / (t16 * 1e-6) / HBM, 3))
            else:
                line.update(int8_TFLOPs=round(2 * m * n * k / t8 / 1e6, 1), int4_TFLOPs=round(2 * m * n * k / t4 / 1e6, 1),
                            bf16_TFLOPs=round(2 * m * n * k / t16 / 1e6, 1))
            emit(line)
            del a, d8, d4, d16, ref, ref4
        del w, q, s, q4, s4, w4
        torch.cuda.empty_cache()


def kernel_ab_gpt2(reps, emit):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, n, k, epi in GPT2_SHAPES:
        w = (torch.randn((n, k), generator=gen, device="cuda") * 0.02).to(torch.bfloat16)
        wt = w.t().contiguous()                                          # the Conv1D weight [in, out]
        bias = (torch.randn((n,), generator=gen, device="cuda") * 0.02).to(torch.bfloat16)
        q, s = ops.quantize_w8(w)
        q4, s4 = ops.quantize_w4(w)
        w8t = (q.float() * s[:, None]).to(torch.bfloat16).t().contiguous()
        w4t = dequantize_w4(q4, s4).t().contiguous()
        for m in (1, 5, 8, 32, 1024):
            a = torch.randn((m, k), generator=gen, device="cuda").to(torch.bfloat16)
            d8, d4, d16 = (torch.empty((m, n), dtype=torch.bfloat16, device="cuda") for _ in range(3))
            f16 = lambda: ops.gemm(L.GEMM_NN, a, wt, out=d16, bias=bias, epilogue=epi)          # noqa: E731
            f8 = lambda: ops.gemm_w8a16(a, q, s, out=d8, bias=bias, epilogue=epi)              # noqa: E731
            f4 = lambda: ops.gemm_w4a16(a, q4, s4, out=d4, bias=bias, epilogue=epi)            # noqa: E731
            t16, t8, t4 = [], [], []
            for _ in range(reps):
                t16.append(graph_us(f16))
                t8.append(graph_us(f8))
                t4.append(graph_us(f4))
            t16, t8, t4 = sorted(t16)[reps // 2], sorted(t8)[reps // 2], sorted(t4)[reps // 2]
            ref = ops.gemm(L.GEMM_NN, a, w8t, bias=bias, epilogue=epi).float()
            rel = float((d8.float() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
            ref4 = ops.gemm(L.GEMM_NN, a, w4t, bias=bias, epilogue=epi).float()
            rel4 = float((d4.float() - ref4).abs().max() / ref4.abs().max().clamp_min(1e-30))
            b8 = n * k + 4 * n + 2 * n + 2 * m * k + 2 * m * n
            b4 = n * k // 2 + 2 * n * (k // 128) + 2 * n + 2 * m * k + 2 * m * n
            b16 = 2 * n * k + 2 * n + 2 * m * k + 2 * m * n
            line = dict(bench="gemm_weight_only_bias_ab", shape=name, epilogue="bias+gelu_new" if epi else "bias", m=m, n=n,
                        k=k, bf16_us=round(t16, 2), int8_us=round(t8, 2), int4_us=round(t4, 2),
                        speedup=round(t16 / t8, 3), int4_speedup=round(t16 / t4, 3),
                        splitk_workspace_bytes=int(L.load().fsb_gemm_w8a16_workspace_bytes(m, n, k)),
                        max_rel_diff_vs_dequantised_bf16=rel, int4_max_rel_diff_vs_dequantised_bf16=rel4, reps=reps)
            if m <= 32:
                line.update(int8_GBps=round(b8 / t8 / 1e3, 1), int4_GBps=round(b4 / t4 / 1e3, 1),
                            bf16_GBps=round(b16 / t16 / 1e3, 1))
            else:
                line.update(int8_TFLOPs=round(2 * m * n * k / t8 / 1e6, 1), int4_TFLOPs=round(2 * m * n * k / t4 / 1e6, 1),
                            bf16_TFLOPs=round(2 * m * n * k / t16 / 1e6, 1))
            emit(line)
            del a, d8, d4, d16, ref, ref4
        del w, wt, q, s, q4, s4, w8t, w4t
        torch.cuda.empty_cache()


def end_to_end_gpt2(reps, emit, layers=30):
    import transformers
    calls = _count_calls()
    S = 32
    runs = (("sample_5x", 1, dict(max_length=150, do_sample=True, top_p=0.9, num_return_sequences=5)),
            ("greedy", 1, dict(max_length=150)), ("greedy", 8, dict(max_length=150)))
    for fmt in ("bf16", "int8", "int4"):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        cfg = transformers.GPT2Config(**dict(WENZHONG, n_layer=layers), bos_token_id=50256, eos_token_id=50256,
                                      resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0, activation_function="gelu_new")
        t0 = time.perf_counter()
        model = GPT2LMHeadModel(cfg, device="cuda", world_size=1, load_in_8bit=fmt == "int8", load_in_4bit=fmt == "int4")
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        for mode, B, kw in runs:
            # ids below the eos id: random weights would otherwise end rows early at different steps per format
            ids = torch.randint(0, 50000, (B, S), generator=torch.Generator().manual_seed(1)).cuda()
            gen = lambda: model.generate(input_ids=ids, pad_token_id=0, **kw)   # noqa: E731
            out = gen()                                                         # warm-up: workspaces, graph capture
            rows = B * kw.get("num_return_sequences", 1)
            wall, toks = [], 0
            for _ in range(reps):
                torch.manual_seed(0)
                torch.cuda.synchronize()
                calls[0] = 0
                t0 = time.perf_counter()
                out = gen()
                torch.cuda.synchronize()
                wall.append(time.perf_counter() - t0)
            new = out.shape[1] - S
            w = sorted(wall)[len(wall) // 2]
            emit(dict(bench="generate_weight_only", model=f"wenzhong-3.5b-L{layers}", weights=fmt, mode=mode, batch=B,
                      rows=rows, prompt=S, new_tokens=new, reps=reps, tokens_per_s=round(rows * new / w, 1),
                      ms_per_step=round(1e3 * w / new, 3), host_calls_per_step=round(calls[0] / new, 2),
                      peak_mem_GiB=round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3),
                      model_footprint_GiB=round(model.get_memory_footprint() / 2 ** 30, 3), build_s=round(build_s, 1)))
            del ids, gen, out
        del model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def dequantize_w4(q, s):
    """W^ = bf16(q * s) of an int4 weight, unpacked on the device by the layout of include/fsb200.h (bench sanity check)."""
    n2, k = q.shape
    b = q.view(n2, k // 16, 4, 2, 2).to(torch.int16)                          # [p, block, t, b, h]
    u = torch.stack([b & 0xF, b >> 4], dim=-1) - 8                           # [p, block, t, b, h, row]
    qi = u.permute(0, 5, 1, 4, 2, 3).reshape(2 * n2, k).float()
    return (qi.view(2 * n2, k // 128, 128) * s.float()[:, :, None]).view(2 * n2, k).to(torch.bfloat16)


def _count_calls():
    n = [0]
    real = L.call

    def counted(name, *args, **kw):
        n[0] += 1
        return real(name, *args, **kw)
    L.call = counted
    return n


def end_to_end(reps, emit, S=512, new=128, full=True):
    calls = _count_calls()
    runs = [(8, "bf16"), (8, "int8"), (8, "int4")] + ([(40, "int8"), (40, "int4")] if full else [])
    for layers, fmt in runs:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        cfg = SimpleNamespace(num_hidden_layers=layers, rms_norm_epsilon=1e-6, max_position_embeddings=2048,
                              rotary_emb_base=10000, llama_mlp_multiple_of=256, **ZIYA)
        t0 = time.perf_counter()
        model = LlamaForCausalLM(cfg, device="cuda", world_size=1, load_in_8bit=fmt == "int8", load_in_4bit=fmt == "int4")
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        for B in (1, 8):
            ids = torch.randint(2, ZIYA["vocab_size"] - 8, (B, S), generator=torch.Generator().manual_seed(1)).cuda()
            gen = lambda: model.generate(ids, max_length=S + new)     # noqa: E731
            out = gen()                                                # warm-up: workspaces, graph capture paths
            assert out.shape == (B, S + new), out.shape
            wall = []
            for _ in range(reps):
                torch.cuda.synchronize()
                calls[0] = 0
                t0 = time.perf_counter()
                gen()
                torch.cuda.synchronize()
                wall.append(time.perf_counter() - t0)
            ncalls = calls[0]
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                gen()
                torch.cuda.synchronize()
            dev_us = sum(e.self_device_time_total for e in prof.key_averages())
            w = sorted(wall)[len(wall) // 2]
            emit(dict(bench="generate_weight_only", model=f"ziya-llama-13b-L{layers}", weights=fmt, batch=B,
                      prompt=S, new_tokens=new, reps=reps, tokens_per_s=round(B * new / w, 1),
                      wall_ms_per_token=round(1e3 * w / new, 3), device_ms_per_token=round(dev_us / 1e3 / new, 3),
                      host_calls_per_token=round(ncalls / new, 2),
                      peak_mem_GiB=round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3),
                      model_footprint_GiB=round(model.get_memory_footprint() / 2 ** 30, 3), build_s=round(build_s, 1)))
            del ids, gen, out
        del model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=("llama", "gpt2"), default="llama")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--layers", type=int, default=30, help="--model gpt2: layers of the end-to-end model")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--skip-40", action="store_true", help="end to end at 8 layers only")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_int8: needs a CUDA GPU")
    info = card()
    lines = []

    def emit(d):
        d.update(info)
        lines.append(d)
        print(json.dumps(d), flush=True)
    emit(dict(bench="card"))
    if args.model == "gpt2":
        kernel_ab_gpt2(args.reps, emit)
        if not args.skip_e2e:
            end_to_end_gpt2(args.reps, emit, layers=args.layers)
    else:
        kernel_ab(args.reps, emit)
        if not args.skip_e2e:
            end_to_end(args.reps, emit, full=not args.skip_40)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_int8.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
