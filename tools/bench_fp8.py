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

--model t5 measures Randeng-T5-784M (C5) width instead:
1. Kernels at C5 width (d_model 1024, d_ff 2816, 16 heads of 64) with 32 x 512 = 16384 token rows on either side, for each
   distinct projection shape (self q|k|v, the attention output projections, cross q, cross k|v, wi_0|wi_1, wo) in the same
   three roles. mT5's projections have no bias and no epilogue. The quantiser rows as above.
2. A C5-width step at reduced depth (12 encoder and 12 decoder layers, vocabulary 32600, encoder and decoder length 512,
   micro-batch 32, span-corruption-shaped labels) at dropout 0 and 0.1, fp8 and bf16 alternated as above.

--model gpt2 measures GPT-2 / Wenzhong, whose Conv1D weights are [in, out]:
1. Kernels at C2 width (hidden 768, 32 x 1024 token rows) and at the 3.5B Wenzhong / Yuyuan width (hidden 3072, 4 x 1024
   rows), for each projection (c_attn, attn.c_proj, c_fc with bias + gelu_new + pre-activation aux, mlp.c_proj) in the
   three roles, each against the bf16 GEMM in the layout the bf16 model runs (forward NN, dgrad NT, wgrad TN). The forward
   carries the bias on every projection. The weight gradient runs fsb_gemm_fp8_t (the transposed store into [in, out]); a
   second row times plain fsb_gemm_fp8 on the same operands (its [out, in] result), so the transposed epilogue's cost
   stands alone.
2. Steps, ZeRO-2 on one GPU, fp8 and bf16 alternated as above: C2 width at 12 layers, 32 x 1024, dropout 0 and 0.1; the
   3.5B width at 8 layers, seq 1024 x micro-batch 1, 2, 4; all 30 layers at micro-batch 1. Model TFLOP/s from
   bench.flops_per_token. Then, per precision, the largest micro-batch at which 30 layers train, tried in increasing
   order from 1 and stopped at the first out-of-memory error.

  python tools/bench_fp8.py [--model llama|megatronbert|t5|gpt2] [--reps 3] [--steps 6] [--warmup 2] [--skip-kernels]
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
import bench  # noqa: E402  (read only: workload, flops_per_token)
from bench_int8 import card, graph_us  # noqa: E402
from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.engine import ZeroEngine  # noqa: E402
from fsb200.models.bert import MegatronBertForPreTraining  # noqa: E402
from fsb200.models.gpt2 import GPT2LMHeadModel  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402
from fsb200.models.t5 import MT5ForConditionalGeneration  # noqa: E402

H, FF, T = 5120, 13824, 8192
PROJ = (("qkv", 3 * H, H), ("dense", H, H), ("w1w3", 2 * FF, H), ("w2", H, FF))
C3_H, C3_FF, C3_T = 2048, 8192, 32 * 512
# (name, out, in, forward epilogue, forward writes aux): every C3 projection has a bias
C3_PROJ = (("qkv", 3 * C3_H, C3_H, L.EPI_NONE, False), ("attn_out", C3_H, C3_H, L.EPI_NONE, False),
           ("inter", C3_FF, C3_H, L.EPI_GELU_ERF, True), ("out", C3_H, C3_FF, L.EPI_NONE, False))
C5_D, C5_FF, C5_INNER, C5_T = 1024, 2816, 16 * 64, 32 * 512
# (name, out, in, forward epilogue, forward writes aux): the distinct C5 projection shapes; o stands for the encoder's and the
# decoder's self- and cross-attention output projections, cq for the cross-attention query
C5_PROJ = (("qkv", 3 * C5_INNER, C5_D, L.EPI_NONE, False), ("o", C5_D, C5_INNER, L.EPI_NONE, False),
           ("cq", C5_INNER, C5_D, L.EPI_NONE, False), ("ckv", 2 * C5_INNER, C5_D, L.EPI_NONE, False),
           ("wi", 2 * C5_FF, C5_D, L.EPI_NONE, False), ("wo", C5_D, C5_FF, L.EPI_NONE, False))
HBM, PEAK_FP8, PEAK_BF16 = 3.35e12, 1979e12, 989e12
# GPT-2 (name, out, in, forward epilogue, forward writes aux) at hidden h; every projection has a bias
GPT2_PROJ = lambda h: (("c_attn", 3 * h, h, L.EPI_NONE, False), ("attn_proj", h, h, L.EPI_NONE, False),
                       ("c_fc", 4 * h, h, L.EPI_GELU_TANH, True), ("mlp_proj", h, 4 * h, L.EPI_NONE, False))
GPT2_WIDTHS = (("c2", 768, 32 * 1024), ("3.5b", 3072, 4 * 1024))


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


def gpt2_kernels(reps, sink):
    """GPT-2's Conv1D roles: the bf16 GEMM in the bf16 model's layouts (weight [in, out]) against the FP8 GEMMs on the codes
    Fp8Conv1D passes. wgrad: fsb_gemm_fp8_t into [in, out]; wgrad_plain: fsb_gemm_fp8 on the same operands into [out, in]."""
    g = torch.Generator(device="cuda").manual_seed(0)
    for width, h, T in GPT2_WIDTHS:
        for name, n_out, k_in, epi, with_aux in GPT2_PROJ(h):
            x = torch.randn((T, k_in), device="cuda", generator=g).to(torch.bfloat16)
            w = (torch.randn((k_in, n_out), device="cuda", generator=g) * 0.02).to(torch.bfloat16)   # Conv1D [in, out]
            dy = (torch.randn((T, n_out), device="cuda", generator=g) * 1e-3).to(torch.bfloat16)
            bv = (torch.randn(n_out, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
            aux = torch.empty((T, n_out), dtype=torch.bfloat16, device="cuda") if with_aux else None
            xq, xt, sx = ops.fp8_quantize(x, "e4m3", rowwise=True, colwise=True)
            wq, wt, sw = ops.fp8_quantize(w, "e4m3", rowwise=True, colwise=True)
            dyq, dyt, sdy = ops.fp8_quantize(dy, "e5m2", rowwise=True, colwise=True)
            y = torch.empty((T, n_out), dtype=torch.bfloat16, device="cuda")
            dx = torch.empty((T, k_in), dtype=torch.bfloat16, device="cuda")
            dw = torch.empty((k_in, n_out), dtype=torch.bfloat16, device="cuda")
            dwt = torch.empty((n_out, k_in), dtype=torch.bfloat16, device="cuda")
            roles = (
                ("fwd", (T, n_out, k_in), lambda: ops.gemm(L.GEMM_NN, x, w, out=y, bias=bv, epilogue=epi, aux=aux),
                 lambda: ops.gemm_fp8(xq, sx, wt, sw, out=y, bias=bv, epilogue=epi, aux=aux),
                 lambda: ops.fp8_quantize(x, "e4m3", rowwise=True, colwise=True)),
                ("dgrad", (T, k_in, n_out), lambda: ops.gemm(L.GEMM_NT, dy, w, out=dx),
                 lambda: ops.gemm_fp8(dyq, sdy, wq, sw, out=dx),
                 lambda: ops.fp8_quantize(dy, "e5m2", rowwise=True, colwise=True)),
                ("wgrad", (n_out, k_in, T), lambda: ops.gemm(L.GEMM_TN, x, dy, out=dw),
                 lambda: ops.gemm_fp8(dyt, sdy, xt, sx, out=dw, store_transposed=True), None),
                ("wgrad_plain", (n_out, k_in, T), lambda: ops.gemm(L.GEMM_TN, x, dy, out=dw),
                 lambda: ops.gemm_fp8(dyt, sdy, xt, sx, out=dwt), None))
            for role, (m, n, k), bf, f8, q8 in roles:
                t8, t16, tq = [], [], []
                for _ in range(reps):
                    t8.append(graph_us(f8)); t16.append(graph_us(bf))
                    if q8 is not None:
                        tq.append(graph_us(q8, calls=20))
                flops = 2.0 * m * n * k
                u8, u16 = statistics.median(t8), statistics.median(t16)
                rec = dict(kind="gemm", model="gpt2", width=width, proj=name, role=role, m=m, n=n, k=k,
                           epilogue=epi if role == "fwd" else L.EPI_NONE, aux=role == "fwd" and with_aux,
                           fp8_us=round(u8, 1), fp8_us_all=[round(v, 1) for v in t8],
                           bf16_us=round(u16, 1), bf16_us_all=[round(v, 1) for v in t16],
                           fp8_tflops=round(flops / u8 / 1e6, 1), bf16_tflops=round(flops / u16 / 1e6, 1),
                           speedup=round(u16 / u8, 3))
                if tq:
                    rows, cols = (T, k_in) if role == "fwd" else (T, n_out)
                    qbytes = 2 * (2 * rows * cols) + 2 * rows * cols
                    uq = statistics.median(tq)
                    rec.update(quantize_us=round(uq, 1), quantize_gbs=round(qbytes / uq / 1e3, 1))
                emit(rec, sink)
            del x, w, dy, bv, aux, xq, xt, wq, wt, dyq, dyt, y, dx, dw, dwt
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


def _t5(fp8, dropout):
    """C5 width: Randeng-T5-784M's config at 12 + 12 layers (of its 24 + 24), encoder and decoder length 512, micro-batch
    32; the last 3 decoder positions of every row unlabelled, as hf_oracle.make_t5_batch does."""
    nl, V, B, S = 12, 32600, 32, 512
    cfg = SimpleNamespace(vocab_size=V, d_model=C5_D, d_kv=64, d_ff=C5_FF, num_layers=nl, num_decoder_layers=nl,
                          num_heads=16, relative_attention_num_buckets=32, relative_attention_max_distance=128,
                          dropout_rate=dropout, feed_forward_proj="gated-gelu", tie_word_embeddings=True,
                          layer_norm_epsilon=1e-6, pad_token_id=0, decoder_start_token_id=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(2, V, (B, S), device="cuda", generator=g)
    labels = torch.randint(2, V, (B, S), device="cuda", generator=g)
    labels[:, -3:] = -100
    return MT5ForConditionalGeneration(cfg, device="cuda", fp8=fp8), dict(input_ids=ids, labels=labels), \
        dict(layers=nl, batch=B, seq=S)


def _gpt2_shape(layers, h, heads, B, S=1024):
    """A GPT-2 step builder: Wenzhong's vocabulary (50257 padded to 50304), `layers` blocks at hidden h, seq S, micro-batch
    B, random ids."""
    def build(fp8, dropout):
        w = dict(bench.workload("gpt2-110m"), n_layer=layers, n_embd=h, n_head=heads, vocab_size=50304, n_positions=1024)
        cfg = SimpleNamespace(vocab_size=w["vocab_size"], n_positions=w["n_positions"], n_embd=h, n_layer=layers,
                              n_head=heads, layer_norm_epsilon=1e-5, initializer_range=0.02, resid_pdrop=dropout,
                              embd_pdrop=dropout, attn_pdrop=dropout, activation_function="gelu_new")
        g = torch.Generator(device="cuda").manual_seed(1)
        ids = torch.randint(0, w["vocab_size"], (B, S), device="cuda", generator=g)
        return GPT2LMHeadModel(cfg, device="cuda", fp8=fp8), dict(input_ids=ids, labels=ids), \
            dict(layers=layers, batch=B, seq=S, model_tflops_per_token=bench.flops_per_token(dict(w, seq=S)))
    build.gpt2 = dict(model="gpt2", width=h)
    return build


def gpt2_largest_micro_batch(fp8, sink, layers=30, limit=64):
    """The largest micro-batch at which `layers` 3.5B-width blocks run a step (ZeRO-2, one GPU), trying 1, 2, ... and
    stopping at the first out-of-memory error."""
    best, reason = 0, None
    gc.collect()
    torch.cuda.empty_cache()
    base, ws0 = torch.cuda.memory_allocated(), _scratch_bytes()
    for B in range(1, limit + 1):
        model = eng = batch = loss = None
        try:
            model, batch, _ = _gpt2_shape(layers, 3072, 32, B)(fp8, 0.0)
            eng = ZeroEngine(model, lr=1e-4, stage=2)
            loss = model(**batch).loss
            loss.backward()
            eng.backward_done()
            eng.step()
            torch.cuda.synchronize()
            best = B
        except torch.cuda.OutOfMemoryError as e:
            reason = str(e).splitlines()[0]
            break
        finally:
            # the loss's autograd graph holds the model: drop it too, or the next try starts beside this one
            del model, eng, batch, loss
            gc.collect()
            torch.cuda.empty_cache()
    left = torch.cuda.memory_allocated() - base - (_scratch_bytes() - ws0)
    if left > 64 << 20:
        raise SystemExit(f"bench_fp8: {left} bytes still allocated after the micro-batch search")
    emit(dict(kind="largest_micro_batch", model="gpt2", width=3072, layers=layers, seq=1024, fp8=fp8, micro_batch=best,
              stopped_by=reason), sink)


def step(fp8, steps, warmup, sink, build=_llama, dropout=0.0):
    gc.collect()
    torch.cuda.empty_cache()
    base, ws0 = torch.cuda.memory_allocated(), _scratch_bytes()
    model, batch, shape = build(fp8, dropout)
    B, S = shape["batch"], shape["seq"]
    eng = ZeroEngine(model, lr=1e-4)
    per_token = shape.pop("model_tflops_per_token", None)
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
    extra = {_megatronbert: dict(model="megatronbert", dropout=dropout), _t5: dict(model="t5", dropout=dropout)}.get(build, {})
    if hasattr(build, "gpt2"):
        extra = dict(build.gpt2, dropout=dropout, zero_stage=2,
                     model_tflops=round(B * S * steps / dt * per_token / 1e12, 1))
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
    ap.add_argument("--model", choices=("llama", "megatronbert", "t5", "gpt2"), default="llama")
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
    bert, t5, gpt2 = a.model == "megatronbert", a.model == "t5", a.model == "gpt2"
    if not a.skip_kernels:
        if gpt2:
            gpt2_kernels(a.reps, sink)
        elif bert:
            kernels(a.reps, sink, C3_PROJ, C3_T, bias=True)
        elif t5:
            kernels(a.reps, sink, C5_PROJ, C5_T)
        else:
            kernels(a.reps, sink)
    if not a.skip_step and gpt2:
        runs = [(_gpt2_shape(12, 768, 12, 32), p) for p in (0.0, 0.1)] + \
               [(_gpt2_shape(8, 3072, 32, B), 0.0) for B in (1, 2, 4)] + [(_gpt2_shape(30, 3072, 32, 1), 0.0)]
        for build, dropout in runs:
            for r in range(a.reps):
                for fp8 in ((True, False) if r % 2 == 0 else (False, True)):
                    step(fp8, a.steps, a.warmup, sink, build, dropout)
        for fp8 in (False, True):
            gpt2_largest_micro_batch(fp8, sink)
    elif not a.skip_step:
        build = _megatronbert if bert else _t5 if t5 else _llama
        for dropout in ((0.0, 0.1) if bert or t5 else (0.0,)):
            for r in range(a.reps):
                for fp8 in ((True, False) if r % 2 == 0 else (False, True)):
                    step(fp8, a.steps, a.warmup, sink, build, dropout)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fp8.jsonl"), "w") as f:
            f.write("\n".join(sink) + "\n")


if __name__ == "__main__":
    main()
