"""Activation recompute (gradient_checkpointing) against keeping every layer's activations, LLaMA training on one GPU.

At Ziya-LLaMA-13B width (hidden 5120, 40 heads of 128, ff 13824, vocabulary 39424) with `--layers` layers (default 4 and 8,
depths one card holds with their ZeRO optimizer state), for every sequence length in `--seqs` and micro-batch in `--micro`:
one optimizer step per micro-batch (ZeroEngine on one GPU, ZeRO-2, clip 1.0 as bench.py's C4), recompute off and on
alternated on the same model and engine, which one goes first swapped from one configuration to the next. Per run: step
time over `--steps` steps after `--warmup` (host clock around work that ends in a device synchronise), tokens/s, model
TFLOP/s and the peak of torch.cuda.max_memory_allocated over the timed steps, with the allocation before them (parameters,
gradients, optimizer state) beside it.

Model FLOPs are bench.flops_per_token, 6 N_mm + 3 F_attn per token: the work of one forward and one backward. The forward
the recompute runs a second time inside the backward is NOT credited, so a recomputed step shows a lower model TFLOP/s for
the same kernels.

A configuration whose predicted need (its activations and head from the tensor shapes, with a margin) exceeds the free
device memory is skipped with a message instead of run.

The `headline` record of each depth compares tokens/s at seq 2048, micro-batch 4 with recompute against seq 1024,
micro-batch 1 without (what bench.py's C4 runs), and `per_layer` records give the growth of the activation peak per layer
between the two depths, the input of the 40-layer arithmetic in DESIGN §2.

  python tools/bench_recompute.py [--layers 4 8] [--seqs 1024 2048] [--micro 1 2 4] [--steps 4] [--warmup 2] [--out DIR]

Prints one JSON line per record, the card's name, power limit and max SM clock first; --out also writes them to
DIR/bench_recompute.jsonl."""
import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
import bench  # noqa: E402  (read only: workload, build_model, flops_per_token)
from bench_int8 import card  # noqa: E402
from fsb200.engine import ZeroEngine  # noqa: E402

GIB = 2 ** 30


def layer_saved_bytes(w, T):
    """Bytes of what one layer's backward reads at T tokens (LlamaForCausalLM._layer's saved tuple): x, h1, o, x1, h2
    [T, h] and q|k|v [T, 3h] in bf16, w1|w3 [T, 2ff] and act [T, ff] in bf16, the two rstd [T] and lse [T, heads] in fp32."""
    h, nh = w["hidden_size"], w["num_attention_heads"]
    ff = 256 * ((int(2 * h * 4 / 3) + 255) // 256)
    return T * (8 * h * 2 + 3 * ff * 2 + 2 * 4 + nh * 4)


def predicted_need(w, T, recompute):
    """Activation and head bytes of one micro-batch of T tokens, from the shapes, with a margin: the layers' saved sets (or
    their inputs and one recomputed set), one more set for a layer's transients, the logits and their fp32 loss temporaries."""
    h, L, V = w["hidden_size"], w["num_hidden_layers"], w["vocab_size"]
    one = layer_saved_bytes(w, T)
    layers = L * T * h * 2 + one if recompute else L * one
    return int(1.25 * (layers + one + T * V * (2 + 2 + 4))) + GIB


def run(model, eng, w, B, S, recompute, steps, warmup):
    """Time `steps` optimizer steps of one [B, S] micro-batch with recompute on or off; -> record, or None when skipped."""
    T = B * S
    if recompute:
        model.gradient_checkpointing_enable()
    else:
        model.gradient_checkpointing_disable()
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    need = predicted_need(w, T, recompute)
    tag = dict(layers=w["num_hidden_layers"], seq=S, micro=B, recompute=recompute)
    if need > free:
        return dict(kind="skipped", **tag, predicted_gib=round(need / GIB, 2), free_gib=round(free / GIB, 2),
                    reason="predicted need exceeds free device memory")
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, w["vocab_size"], (B, S), device="cuda", generator=g)
    losses = []

    def one():
        out = model(input_ids=ids, labels=ids)
        out.loss.backward()
        eng.backward_done()
        eng.step()
        return out.loss.detach()

    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for _ in range(steps):
        losses.append(one())
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    peak = torch.cuda.max_memory_allocated()
    wf = dict(w, seq=S)
    tok_s = T / dt
    rec = dict(kind="step", **tag, steps=steps, step_ms=round(1e3 * dt, 1), tokens_per_s=round(tok_s),
               model_tflops=round(tok_s * bench.flops_per_token(wf) / 1e12, 1),
               peak_alloc_gib=round(peak / GIB, 3), alloc_before_gib=round(before / GIB, 3),
               activation_peak_gib=round((peak - before) / GIB, 3), predicted_gib=round(need / GIB, 2),
               loss_last=round(float(losses[-1]), 4))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--seqs", type=int, nargs="+", default=[1024, 2048])
    ap.add_argument("--micro", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_recompute: needs a CUDA device")
    sink = []

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        sink.append(line)

    emit(dict(kind="card", **card(), note="model_tflops credits 6 N_mm + 3 F_attn per token (bench.flops_per_token); the "
              "forward recomputed in the backward is not credited"))
    act = {}     # (layers, seq, micro, recompute) -> activation peak bytes
    flip = False
    for L in a.layers:
        w = bench.workload(f"ziya-llama-13b-L{L}")
        model = bench.build_model(w, torch.device("cuda", torch.cuda.current_device()), 1)
        eng = ZeroEngine(model, lr=1e-4, betas=w["betas"], weight_decay=w["wd"], grad_clip=w["clip"], stage=2)
        res = {}
        for S in a.seqs:
            for B in a.micro:
                for rc in ((True, False) if flip else (False, True)):
                    rec = run(model, eng, w, B, S, rc, a.steps, a.warmup)
                    emit(rec)
                    if rec["kind"] == "step":
                        res[(S, B, rc)] = rec
                        act[(L, S, B, rc)] = rec["activation_peak_gib"]
                flip = not flip
        on, off = res.get((2048, 4, True)), res.get((1024, 1, False))
        if on and off:
            emit(dict(kind="headline", layers=L, recomputed_seq2048_micro4_tokens_per_s=on["tokens_per_s"],
                      kept_seq1024_micro1_tokens_per_s=off["tokens_per_s"],
                      ratio=round(on["tokens_per_s"] / off["tokens_per_s"], 3)))
        del model, eng, res
        gc.collect()          # the model <-> engine reference cycle: without it the model's memory outlives the depth
        torch.cuda.empty_cache()
    if len(a.layers) >= 2:
        l0, l1 = min(a.layers), max(a.layers)
        for (L, S, B, rc), v in sorted(act.items()):
            if L == l0 and (l1, S, B, rc) in act:
                emit(dict(kind="per_layer", seq=S, micro=B, recompute=rc, depths=[l0, l1],
                          activation_peak_gib_per_layer=round((act[(l1, S, B, rc)] - v) / (l1 - l0), 4)))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_recompute.jsonl"), "w") as f:
            f.write("\n".join(sink) + "\n")


if __name__ == "__main__":
    main()
