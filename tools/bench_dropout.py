"""Cost of dropout on an H100: attention forward / backward device time with p = 0 and p = 0.1, and BERT / MegatronBERT / mT5
training-step throughput with dropout-0 and dropout-0.1 configs, alternated in one process (median of 3 windows each). Attention,
RMSNorm and gated-activation times are kernel times from torch.profiler; step throughput is wall time over device-synchronised
windows.

    python tools/bench_dropout.py [--steps 20] [--out result.json]

Shapes: C3 attention = micro-batch 32 x 512, 32 heads, head dim 64; C1 attention = 8 x 128, 12 heads. Steps: C1 = BERT-base
(12 layers, hidden 768) at 8 x 128; C3 = the Erlangshen MegatronBERT width (hidden 2048, 32 heads) at 32 x 512 with 4 layers
(the full 24-layer model's optimizer state and activations are not needed to price the per-layer dropout work). C5 =
Randeng-T5-784M width (d 1024, 16 heads x 64, d_ff 2816) at 32 x (enc 512 + dec 512): attention of the encoder (relative bias +
padding mask), of the decoder (the causal flag with the bias) and cross-attention; RMSNorm with a residual and the gated GeLU
over the 16384 tokens; a 4 + 4-layer step with its peak memory. C2 = Wenzhong-GPT2-110M (12 layers, hidden 768, 12 heads x 64) at 32 x 1024: causal attention at p = 0 and p = 0.1
(the causal flag, which is what the model runs), the same attention at p = 0.1 with the causal mask folded into a bias vector
instead (for reference: no tile is skipped; no bias gradient), and the 12-layer step with all three probabilities 0 against 0.1.
Prints one JSON line; card name and power limit come from nvidia-smi in the same process."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))

import torch  # noqa: E402

from fsb200 import ops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def kernel_ms(fn, iters, match=("attn_",)):
    """Device time per call of the kernels fn launches whose names contain one of `match` (default: the attention kernels
    attn_fwd / attn_delta / attn_bwd_dq / attn_bwd_dkv / attn_dbias), from torch.profiler's CUDA activity records: kernel
    execution only, not the host time of the call."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for evt in prof.key_averages():
        if any(m in evt.key for m in match):
            us += getattr(evt, "self_device_time_total", None) or evt.self_cuda_time_total
    if us == 0.0:
        raise RuntimeError(f"bench_dropout: the profiler recorded no kernel matching {match}")
    return us / 1e3 / iters


def attention(B, S, H, D, iters=50):
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).cuda()
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).cuda()
    mask = torch.ones(B, S, dtype=torch.uint8, device="cuda")
    mask[:, S - S // 8:] = 0
    dq = torch.empty_like(qkv)
    base = torch.zeros(1, dtype=torch.int64, device="cuda")
    scale = 1.0 / math.sqrt(D)
    res = {}
    for _ in range(3):   # alternate p = 0 / 0.1 windows
        for p in (0.0, 0.1):
            drop = None if p == 0 else ops.Dropout(p, 1, base, 0)
            o, lse = ops.sdpa_fwd(q, k, v, scale, False, kv_mask=mask, drop=drop)
            f = kernel_ms(lambda: ops.sdpa_fwd(q, k, v, scale, False, kv_mask=mask, drop=drop), iters)
            b = kernel_ms(lambda: ops.sdpa_bwd(q, k, v, o, dout, lse, scale, False, dq[:, :, 0], dq[:, :, 1], dq[:, :, 2],
                                             kv_mask=mask, drop=drop), iters)
            res.setdefault(p, []).append((f, b))
    return {f"p={p}": {"fwd_ms": statistics.median(x[0] for x in v), "bwd_ms": statistics.median(x[1] for x in v)}
            for p, v in res.items()}


def attention_t5(B, S, H, D, iters=50):
    """The three attention forms of the C5 layer stack, p = 0 against p = 0.1 as the model runs them."""
    import fsb200.models.t5_bias as TB
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).cuda()
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).cuda()
    mask = torch.ones(B, S, dtype=torch.uint8, device="cuda")
    mask[:, S - S // 8:] = 0
    table = 0.1 * torch.randn(32, H, generator=g).cuda()
    rel_e = TB.rel_bias_vector(table, S, S, True, 32, 128)
    rel_d = TB.rel_bias_vector(table, S, S, False, 32, 128)
    dq = torch.empty_like(qkv)
    base = torch.zeros(1, dtype=torch.int64, device="cuda")
    forms = {   # name -> {p: (causal, kv_mask, rel_bias)}
        "encoder_self": {0.0: (False, mask, rel_e), 0.1: (False, mask, rel_e)},
        "decoder_self": {0.0: (True, None, rel_d), 0.1: (True, None, rel_d)},
        "cross": {0.0: (False, mask, None), 0.1: (False, mask, None)},
    }
    out = {}
    for name, by_p in forms.items():
        res = {}
        for _ in range(3):   # alternate p = 0 / 0.1 windows
            for p, (causal, km, rel) in by_p.items():
                drop = None if p == 0 else ops.Dropout(p, 1, base, 0)
                drel = None if rel is None else torch.zeros_like(rel)
                o, lse = ops.sdpa_fwd(q, k, v, 1.0, causal, kv_mask=km, rel_bias=rel, drop=drop)
                f = kernel_ms(lambda: ops.sdpa_fwd(q, k, v, 1.0, causal, kv_mask=km, rel_bias=rel, drop=drop), iters)
                b = kernel_ms(lambda: ops.sdpa_bwd(q, k, v, o, dout, lse, 1.0, causal, dq[:, :, 0], dq[:, :, 1], dq[:, :, 2],
                                                 kv_mask=km, rel_bias=rel, drel_bias=drel, drop=drop), iters)
                res.setdefault(p, []).append((f, b))
        out[name] = {f"p={p}": {"fwd_ms": statistics.median(x[0] for x in v), "bwd_ms": statistics.median(x[1] for x in v)}
                     for p, v in res.items()}
    return out


def attention_gpt2(B, S, H, D, iters=50):
    """C2 causal self-attention: the causal flag at p = 0 and p = 0.1, and the causal mask folded into a bias at p = 0.1."""
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).cuda()
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).cuda()
    folded = torch.zeros(H, 2 * S - 1, device="cuda")
    folded[:, S:] = float("-inf")          # offsets k - q > 0
    dq = torch.empty_like(qkv)
    base = torch.zeros(1, dtype=torch.int64, device="cuda")
    scale = 1.0 / math.sqrt(D)
    forms = {"causal p=0.0": (0.0, True, None), "causal p=0.1": (0.1, True, None), "folded_bias p=0.1": (0.1, False, folded)}
    res = {}
    for _ in range(3):   # alternate the forms' windows
        for name, (p, causal, rel) in forms.items():
            drop = None if p == 0 else ops.Dropout(p, 1, base, 0)
            fwd = lambda: ops.sdpa_fwd(q, k, v, scale, causal, rel_bias=rel, drop=drop)
            bwd = lambda: ops.sdpa_bwd(q, k, v, o, dout, lse, scale, causal, dq[:, :, 0], dq[:, :, 1], dq[:, :, 2],
                                       rel_bias=rel, drop=drop)
            o, lse = fwd()
            f = kernel_ms(fwd, iters)
            b = kernel_ms(bwd, iters)
            res.setdefault(name, []).append((f, b))
    return {name: {"fwd_ms": statistics.median(x[0] for x in v), "bwd_ms": statistics.median(x[1] for x in v)}
            for name, v in res.items()}


def step_gpt2(B, S, steps):
    """The 12-layer C2 step (Wenzhong-GPT2-110M) on one micro-batch of B x S: tokens per second with embd_pdrop, attn_pdrop
    and resid_pdrop all 0 against all 0.1."""
    from fsb200.models.gpt2 import GPT2LMHeadModel
    from fsb200.trainer import PretrainStep
    cfg = dict(vocab_size=50264, n_positions=1024, n_embd=768, n_layer=12, n_head=12, layer_norm_epsilon=1e-5,
               initializer_range=0.02, activation_function="gelu_new")
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, cfg["vocab_size"] - 8, (B, S), generator=g).cuda()
    batch = {"input_ids": ids, "labels": ids.clone()}
    runs = {}
    for p in (0.0, 0.1):
        torch.manual_seed(0)
        model = GPT2LMHeadModel(SimpleNamespace(embd_pdrop=p, attn_pdrop=p, resid_pdrop=p, **cfg), device="cuda")
        runs[p] = PretrainStep(model, lambda s_: 1e-4, lr=1e-4, weight_decay=0.1, grad_clip=0.0)
        for _ in range(3):
            runs[p].step_device([batch])
    torch.cuda.synchronize()
    res = {}
    for _ in range(3):
        for p in (0.0, 0.1):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(steps):
                runs[p].step_device([batch])
            ev1.record()
            torch.cuda.synchronize()
            res.setdefault(p, []).append(B * S * steps / (ev0.elapsed_time(ev1) / 1e3))
    del runs
    torch.cuda.empty_cache()
    return {f"p={p}": {"tokens_per_s": statistics.median(v)} for p, v in res.items()}


def pointwise_t5(T, d, ff, iters=50):
    """RMSNorm (with the residual add) forward / backward and the gated GeLU forward / backward of a C5 layer over T tokens."""
    from fsb200 import lib as L
    g = torch.Generator().manual_seed(0)
    x, r, dy = (torch.randn(T, d, generator=g).to(torch.bfloat16).cuda() for _ in range(3))
    w = torch.ones(d, dtype=torch.bfloat16, device="cuda")
    gw = torch.zeros(d, dtype=torch.float32, device="cuda")
    gu = torch.randn(T, 2 * ff, generator=g).to(torch.bfloat16).cuda()
    da = torch.randn(T, ff, generator=g).to(torch.bfloat16).cuda()
    dgu = torch.empty_like(gu)
    base = torch.zeros(1, dtype=torch.int64, device="cuda")
    res = {}
    for _ in range(3):
        for p in (0.0, 0.1):
            drop = None if p == 0 else ops.Dropout(p, 1, base, 0)
            _, rstd, xs = ops.rmsnorm_fwd(x, w, 1e-6, residual=r, drop=drop)
            if drop is None:
                nb = lambda: ops.rmsnorm_bwd(dy, xs, w, rstd, gw, dres=r)
            else:
                nb = lambda: ops.rmsnorm_bwd_dropout(dy, xs, w, rstd, gw, drop, dres=r)
            t = (kernel_ms(lambda: ops.rmsnorm_fwd(x, w, 1e-6, residual=r, drop=drop), iters, ("norm_fwd",)),
                 kernel_ms(nb, iters, ("norm_bwd", "colsum")),
                 kernel_ms(lambda: ops.glu_fwd(L.ACT_GELU_TANH, gu[:, :ff], gu[:, ff:], drop=drop), iters, ("glu_fwd",)),
                 kernel_ms(lambda: ops.glu_bwd(L.ACT_GELU_TANH, da, gu[:, :ff], gu[:, ff:], dgu[:, :ff], dgu[:, ff:], drop=drop),
                           iters, ("glu_bwd",)))
            res.setdefault(p, []).append(t)
    keys = ("rmsnorm_fwd_ms", "rmsnorm_bwd_ms", "glu_fwd_ms", "glu_bwd_ms")
    return {f"p={p}": {k: statistics.median(x[i] for x in v) for i, k in enumerate(keys)} for p, v in res.items()}


def step_t5(B, S, steps):
    """Randeng-T5-784M width with 4 + 4 layers, one micro-batch of B x (enc S + dec S): tokens (enc + dec) per second and
    the peak of allocated device memory, dropout_rate 0 against 0.1."""
    from fsb200.models.t5 import MT5ForConditionalGeneration
    from fsb200.trainer import PretrainStep
    cfg = dict(vocab_size=32600, d_model=1024, d_kv=64, d_ff=2816, num_layers=4, num_decoder_layers=4, num_heads=16,
               relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
               feed_forward_proj="gated-gelu", tie_word_embeddings=False, pad_token_id=0, decoder_start_token_id=0)
    g = torch.Generator().manual_seed(1)
    batch = {"input_ids": torch.randint(2, cfg["vocab_size"], (B, S), generator=g).cuda(),
             "labels": torch.randint(2, cfg["vocab_size"], (B, S), generator=g).cuda()}
    runs, peak = {}, {}
    for p in (0.0, 0.1):
        torch.manual_seed(0)
        model = MT5ForConditionalGeneration(SimpleNamespace(dropout_rate=p, **cfg), device="cuda")
        runs[p] = PretrainStep(model, lambda s_: 1e-4, lr=1e-4, weight_decay=0.01, grad_clip=1.0)
        torch.cuda.synchronize()
        base_mem = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        for _ in range(3):
            runs[p].step_device([batch])
        torch.cuda.synchronize()
        peak[p] = (torch.cuda.max_memory_allocated() - base_mem) / 2 ** 30
    res = {}
    for _ in range(3):
        for p in (0.0, 0.1):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(steps):
                runs[p].step_device([batch])
            ev1.record()
            torch.cuda.synchronize()
            res.setdefault(p, []).append(2 * B * S * steps / (ev0.elapsed_time(ev1) / 1e3))
    del runs
    torch.cuda.empty_cache()
    return {f"p={p}": {"tokens_per_s": statistics.median(v), "step_peak_gib_above_model": peak[p]} for p, v in res.items()}


def step_throughput(kind, B, S, steps):
    from fsb200.models.bert import BertForMaskedLM, MegatronBertForPreTraining
    from fsb200.trainer import PretrainStep
    if kind == "C1":
        cfg = dict(vocab_size=21128, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                   max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", layer_norm_eps=1e-12)
        cls = BertForMaskedLM
    else:
        cfg = dict(vocab_size=21248, hidden_size=2048, num_hidden_layers=4, num_attention_heads=32, intermediate_size=8192,
                   max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu_new", layer_norm_eps=1e-12)
        cls = MegatronBertForPreTraining
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, cfg["vocab_size"], (B, S), generator=g)
    labels = torch.where(torch.rand(B, S, generator=g) < 0.15, ids, torch.full_like(ids, -100))
    batch = {"input_ids": ids.cuda(), "token_type_ids": torch.zeros_like(ids).cuda(), "labels": labels.cuda()}
    if kind == "C3":
        batch["next_sentence_label"] = torch.randint(0, 2, (B,), generator=g).cuda()
    runs = {}
    for p in (0.0, 0.1):
        torch.manual_seed(0)
        model = cls(SimpleNamespace(hidden_dropout_prob=p, attention_probs_dropout_prob=p, **cfg), device="cuda")
        runs[p] = PretrainStep(model, lambda s_: 1e-4, lr=1e-4, weight_decay=0.01, grad_clip=1.0)
        for _ in range(3):
            runs[p].step_device([batch])
    torch.cuda.synchronize()
    res = {}
    for _ in range(3):
        for p in (0.0, 0.1):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(steps):
                runs[p].step_device([batch])
            ev1.record()
            torch.cuda.synchronize()
            res.setdefault(p, []).append(B * S * steps / (ev0.elapsed_time(ev1) / 1e3))
    del runs
    torch.cuda.empty_cache()
    return {f"p={p}": {"tokens_per_s": statistics.median(v)} for p, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropout: needs a GPU (no CPU timing is meaningful)")
    out = {"card": card(),
           "attention_C3_32x512_h32_d64": attention(32, 512, 32, 64),
           "attention_C1_8x128_h12_d64": attention(8, 128, 12, 64),
           "step_C1_bert_base_8x128": step_throughput("C1", 8, 128, a.steps),
           "step_C3_width_4_layers_32x512": step_throughput("C3", 32, 512, max(3, a.steps // 4)),
           "attention_C5_32x512_h16_d64": attention_t5(32, 512, 16, 64),
           "pointwise_C5_16384_tokens_d1024_ff2816": pointwise_t5(32 * 512, 1024, 2816),
           "step_C5_width_4_4_layers_32x512": step_t5(32, 512, max(3, a.steps // 4)),
           "attention_C2_32x1024_h12_d64": attention_gpt2(32, 1024, 12, 64),
           "step_C2_gpt2_110m_32x1024": step_gpt2(32, 1024, max(3, a.steps // 2))}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
