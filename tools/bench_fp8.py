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

--model megatronbert measures Erlangshen-MegatronBERT-1.3B (C3) instead:
1. Kernels at C3 width (hidden 2048, MLP 8192) with 32 x 512 = 16384 token rows, for each projection (query|key|value,
   attention output, intermediate, output) in the same three roles. The forward runs each projection's epilogue in both
   GEMMs: its bias, and on the intermediate the GELU (erf) with the pre-activation copy (aux). The quantiser rows are the
   passes each role needs: the forward's input in both layouts (e4m3), the gradient's in both layouts (e5m2).
2. The C3-width step (24 layers, 32 heads, vocabulary 21248, seq 512, micro-batch 32, MLM + sentence order) at dropout 0
   and 0.1, fp8 and bf16 alternated as above.

  python tools/bench_fp8.py [--model llama|megatronbert] [--reps 3] [--steps 6] [--warmup 2] [--skip-kernels]
                            [--skip-step] [--out DIR]

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
from fsb200.models.bert import MegatronBertForPreTraining  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402

H, FF, T = 5120, 13824, 8192
PROJ = (("qkv", 3 * H, H), ("dense", H, H), ("w1w3", 2 * FF, H), ("w2", H, FF))
C3_H, C3_FF, C3_T = 2048, 8192, 32 * 512
# (name, out, in, forward epilogue, forward writes aux): every C3 projection has a bias
C3_PROJ = (("qkv", 3 * C3_H, C3_H, L.EPI_NONE, False), ("attn_out", C3_H, C3_H, L.EPI_NONE, False),
           ("inter", C3_FF, C3_H, L.EPI_GELU_ERF, True), ("out", C3_H, C3_FF, L.EPI_NONE, False))
HBM, PEAK_FP8, PEAK_BF16 = 3.35e12, 1979e12, 989e12


def emit(rec, sink):
    line = json.dumps(rec)
    print(line, flush=True)
    sink.append(line)


def kernels(reps, sink, proj=tuple(p + (L.EPI_NONE, False) for p in PROJ), T=T, bias=False):
    """bias: the forward adds a bias (and runs each projection's epilogue) in both GEMMs."""
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n_out, k_in, epi, with_aux in proj:
        for role, (m, n, k) in (("fwd", (T, n_out, k_in)), ("dgrad", (T, k_in, n_out)), ("wgrad", (n_out, k_in, T))):
            a_fmt = "e4m3" if role == "fwd" else "e5m2"
            a16 = torch.randn((m, k), device="cuda", generator=g).to(torch.bfloat16)
            b16 = (torch.randn((n, k), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
            aq, _, sa = ops.fp8_quantize(a16, a_fmt)
            bq, _, sb = ops.fp8_quantize(b16, "e4m3")
            d = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
            fwd = role == "fwd"
            bv = (torch.randn(n, device="cuda", generator=g) * 0.1).to(torch.bfloat16) if bias and fwd else None
            ep = epi if fwd else L.EPI_NONE
            aux = torch.empty((m, n), dtype=torch.bfloat16, device="cuda") if with_aux and fwd else None
            # the bf16 GEMM in the layout the bf16 model runs for this role, on operands of the same extents
            if role == "fwd":
                bf = lambda: ops.gemm(L.GEMM_NT, a16, b16, out=d, bias=bv, epilogue=ep, aux=aux)
            elif role == "dgrad":
                bt = b16.t().contiguous()          # [k, n]
                bf = lambda: ops.gemm(L.GEMM_NN, a16, bt, out=d)
            else:
                at, btt = a16.t().contiguous(), b16.t().contiguous()   # [k, m], [k, n]
                bf = lambda: ops.gemm(L.GEMM_TN, at, btt, out=d)
            f8 = lambda: ops.gemm_fp8(aq, sa, bq, sb, out=d, bias=bv, epilogue=ep, aux=aux)
            q8 = lambda: ops.fp8_quantize(a16, a_fmt, rowwise=True, colwise=True)
            t8, t16, tq = [], [], []
            for _ in range(reps):
                t8.append(graph_us(f8)); t16.append(graph_us(bf)); tq.append(graph_us(q8, calls=20))
            flops = 2.0 * m * n * k
            qbytes = 2 * (2 * m * k) + 2 * m * k
            u8, u16, uq = statistics.median(t8), statistics.median(t16), statistics.median(tq)
            epi_keys = dict(bias=bv is not None, epilogue=ep, aux=aux is not None) if bias else {}
            emit(dict(kind="gemm", proj=name, role=role, m=m, n=n, k=k, **epi_keys,
                      fp8_us=round(u8, 1), fp8_us_all=[round(x, 1) for x in t8],
                      bf16_us=round(u16, 1), bf16_us_all=[round(x, 1) for x in t16],
                      fp8_tflops=round(flops / u8 / 1e6, 1), bf16_tflops=round(flops / u16 / 1e6, 1),
                      fp8_of_1979=round(flops / u8 / 1e6 / (PEAK_FP8 / 1e12), 3),
                      bf16_of_989=round(flops / u16 / 1e6 / (PEAK_BF16 / 1e12), 3),
                      speedup=round(u16 / u8, 3),
                      quantize_us=round(uq, 1), quantize_gbs=round(qbytes / uq / 1e3, 1),
                      quantize_of_3350=round(qbytes / uq / 1e3 / 3350, 3)), sink)
            del a16, b16, aq, bq, d, bv, aux
            torch.cuda.empty_cache()


def _scratch_bytes():
    return sum(b.numel() * b.element_size() for b in ops._ws_cache.values())


def _llama(fp8, _dropout):
    cfg = SimpleNamespace(vocab_size=39424, hidden_size=H, num_hidden_layers=4, num_attention_heads=40,
                          rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                          llama_mlp_multiple_of=256)
    B, S = 4, 2048
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=g)
    return LlamaForCausalLM(cfg, device="cuda", fp8=fp8), dict(input_ids=ids, labels=ids), dict(layers=4, batch=B, seq=S)


def _megatronbert(fp8, dropout):
    """C3 width: Erlangshen-MegatronBERT-1.3B's config (24 layers) at seq 512, micro-batch 32; MLM labels on 15 % of the
    tokens, sentence-order labels."""
    nl, V, B, S = 24, 21248, 32, 512
    cfg = SimpleNamespace(vocab_size=V, hidden_size=C3_H, num_hidden_layers=nl, num_attention_heads=32,
                          intermediate_size=C3_FF, max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu",
                          layer_norm_eps=1e-12, hidden_dropout_prob=dropout, attention_probs_dropout_prob=dropout)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(1, V, (B, S), device="cuda", generator=g)
    sel = torch.rand((B, S), device="cuda", generator=g) < 0.15
    tt = torch.zeros_like(ids)
    tt[:, S // 2:] = 1
    batch = dict(input_ids=ids, token_type_ids=tt, attention_mask=torch.ones_like(ids),
                 labels=torch.where(sel, ids, torch.full_like(ids, -100)),
                 next_sentence_label=torch.randint(0, 2, (B,), device="cuda", generator=g))
    return MegatronBertForPreTraining(cfg, device="cuda", fp8=fp8), batch, dict(layers=nl, batch=B, seq=S)


def step(fp8, steps, warmup, sink, build=_llama, dropout=0.0):
    gc.collect()
    torch.cuda.empty_cache()
    base, ws0 = torch.cuda.memory_allocated(), _scratch_bytes()
    model, batch, shape = build(fp8, dropout)
    B, S = shape["batch"], shape["seq"]
    eng = ZeroEngine(model, lr=1e-4)
    losses = []

    def one():
        out = model(**batch)
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
    extra = dict(model="megatronbert", dropout=dropout) if build is _megatronbert else {}
    rec = dict(kind="step", **extra, fp8=fp8, **shape, steps=steps,
               tokens_per_s=round(B * S * steps / dt),
               step_ms=round(1e3 * dt / steps, 1), peak_alloc_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
               alloc_before_gib=round(base / 2 ** 30, 3), loss_last=round(float(losses[-1]), 4))
    del model, eng, losses, one, batch
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
    ap.add_argument("--model", choices=("llama", "megatronbert"), default="llama")
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
    bert = a.model == "megatronbert"
    if not a.skip_kernels:
        if bert:
            kernels(a.reps, sink, C3_PROJ, C3_T, bias=True)
        else:
            kernels(a.reps, sink)
    if not a.skip_step:
        for dropout in ((0.0, 0.1) if bert else (0.0,)):
            for r in range(a.reps):
                for fp8 in ((True, False) if r % 2 == 0 else (False, True)):
                    step(fp8, a.steps, a.warmup, sink, _megatronbert if bert else _llama, dropout)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fp8.jsonl"), "w") as f:
            f.write("\n".join(sink) + "\n")


if __name__ == "__main__":
    main()
