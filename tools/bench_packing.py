"""Packed against padded batches on one GPU: Ziya-LLaMA SFT (--model llama, the default), Wenzhong-GPT2 QA (--model gpt2),
Erlangshen-MegatronBERT MLM + sentence-order pretraining (--model megatronbert) or Randeng-T5 / mT5 LCSTS summarisation
(--model mt5).

No corpus is read: the length mix is a seeded log-normal chosen here, and the gain depends on it.
  llama: SFT-like sample lengths, median 320 tokens, sigma 0.9, seed 20231018, capped at max_seq_length = 2048; 40 % of
         each sample is prompt (label -100), the rest labelled output.
  gpt2 : question + answer lengths, median 160 tokens, sigma 0.7, seed 20231018, capped at max_seq_length = 1024; every
         token labelled, as GPT2QADataset.encode labels everything but the pads.
  megatronbert: document lengths, median 200 tokens, sigma 0.6, seed 20231018, capped at max_seq_length = 512; [CLS]
         first, ~15 % of the other tokens MLM-labelled, one sentence-order label per document, padded to 512 as
         ErLangShenCollator pads.
  mt5  : LCSTS-like source lengths, median 75 tokens (the reference's own statistic of LCSTS: mean 74.7, max 132),
         sigma 0.4, seed 20231018, capped at max_enc_length = 128. Targets are max_dec_length = 64 tokens, ALL labelled:
         LCSTSDataset.encode leaves its pad ids labelled (its `labels[target == pad_token_id] = -100` compares a list with
         an int), so a target keeps its full padded length and the decoder does the padded batch's work; packing removes
         the source pads only. Packed rows: 4 x 128 = 512 encoder tokens and 4 x 64 = 256 decoder tokens.

1. Attention at the model's head shape (llama: 40 heads x 128, S 2048; gpt2: 12 heads x 64, S 1024, attention dropout
   p = 0.1): the samples packed first fit into `--rows` rows. The segment kernels (the causal segment form of
   fsb_sdpa_{fwd,bwd}, with or without dropout) against what the padded batch runs today: llama fsb_sdpa_fwd / _bwd with
   causal = 1 on the same [rows, S] tensors; gpt2 the causal + key-mask + dropout kernels (fsb_sdpa_{fwd,bwd} with p > 0) on
   the padded [samples, S] tensors, one sample per row; megatronbert (32 heads x 64, S 512, p = 0.1) the bidirectional
   segment kernels (the bidirectional segment form of fsb_sdpa_{fwd,bwd}) against the non-causal key-mask + dropout kernels on the
   padded [samples, S] tensors, and the FLOPs of a segment are 4 D H n^2 (every pair inside it). Device time per call (10 calls captured in one CUDA graph, replayed
   under CUDA events), alternated `--reps` times (medians and spread). TFLOP/s over the FLOPs the block-diagonal mask
   needs, counted from the lengths: forward 4 D H n (n + 1) / 2 per segment of n tokens (QK^T and PV over the causal
   pairs), backward 2.5 times that; the pad tail is not counted.
   mt5 (C5 head shape, 16 heads x 64, dropout 0.1): the three packed forms against what the padded batch runs today on
   [samples, 128] / [samples, 64]: the encoder (the biased segment form, bidirectional) against the bias + key-mask
   kernels, the decoder self-attention (the biased segment form, causal) against the causal bias kernels, and the
   cross-attention (the cross segment form) against the key-mask kernels; FLOPs counted from the real pairs.
2. The step, eager PretrainStep, `--samples` samples per micro-batch, padded against packed (fsb200/packing.py, rows of S).
   llama: Ziya width (hidden 5120, 40 heads, vocabulary 39424) at 4 layers, padded by the reference collator's dynamic
   padding to the longest sample. gpt2: GPT-2-110M (12 layers, hidden 768, vocabulary 50264) with the released dropout 0.1
   at all three sites, padded to 1024 as GPT2QADataset does. megatronbert: the C3 configuration (24 layers, hidden 2048,
   32 heads, vocabulary 21128, dropout 0.1, ZeRO-1), micro-batches of `--samples` documents padded to 512 against the
   same documents packed by pack_mlm_batch, with documents/s and MLM label tokens/s. Every micro-batch shape is warmed up first; then the two
   variants alternate `--reps` times (which goes first swapped each time), each timing its `--batches` micro-batches (one
   optimizer step each) between CUDA events. Label tokens/s, non-pad tokens/s (the padded batch's real tokens, the same
   count for both), peak allocated memory. mt5: Randeng-T5 width (d_model 1024, 16 heads x 64, d_ff 2816, vocabulary
   32128) at 4 encoder + 4 decoder layers, dropout 0.1, `--samples` samples per micro-batch.

  python tools/bench_packing.py [--model llama|gpt2|megatronbert|mt5] [--reps 5] [--rows 4] [--samples 8] [--batches 4] [--skip-attention]
                                [--skip-step] [--out DIR]

Prints one JSON line per measurement, the card's name, power limit and max SM clock first; --out also writes them to
DIR/bench_packing.jsonl."""
import argparse
import gc
import json
import math
import os
import statistics
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
from bench_int8 import card, graph_us  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.packing import first_fit, pack_causal_lm_batch, pack_mlm_batch, pack_seq2seq_batch  # noqa: E402

SEED = 20231018
# seq, length mix (median, sigma, prompt share), vocabulary, hidden, heads, head_dim, layers, eos (= pad), attention dropout
MODELS = {"llama": SimpleNamespace(seq=2048, median=320.0, sigma=0.9, prompt_share=0.4, V=39424, hidden=5120, heads=40,
                                   hd=128, layers=4, eos=2, p=0.0),
          "gpt2": SimpleNamespace(seq=1024, median=160.0, sigma=0.7, prompt_share=0.0, V=50264, hidden=768, heads=12, hd=64,
                                  layers=12, eos=50256, p=0.1),
          "megatronbert": SimpleNamespace(seq=512, median=200.0, sigma=0.6, prompt_share=0.0, V=21128, hidden=2048, heads=32,
                                          hd=64, layers=24, eos=0, p=0.1),
          "mt5": SimpleNamespace(seq=128, dec=64, median=75.0, sigma=0.4, prompt_share=0.0, V=32128, hidden=1024, heads=16,
                                 hd=64, layers=4, eos=0, p=0.1, ff=2816, pack=4)}
M = MODELS["llama"]


def lengths(n, seed=SEED):
    rs = np.random.RandomState(seed)
    return [int(x) for x in np.clip(np.round(rs.lognormal(math.log(M.median), M.sigma, size=n)), 2, M.seq)]


def sft_batch(lens, seed):
    """The padded batch the reference pipeline emits for samples of these lengths: llama the SFT collator's (to the longest
    sample, with position ids), gpt2 GPT2QADataset's (to max_seq_length, with the attention mask)."""
    rs = np.random.RandomState(seed)
    L = max(lens) if M is MODELS["llama"] else M.seq
    ids = np.full((len(lens), L), M.eos, dtype=np.int64)
    lab = np.full((len(lens), L), -100, dtype=np.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = rs.randint(3, M.eos if M.eos > 3 else M.V, size=n)
        p = max(1, min(n - 1, int(M.prompt_share * n))) if M.prompt_share else 0
        lab[i, p:n] = ids[i, p:n]
    out = {"input_ids": torch.from_numpy(ids), "labels": torch.from_numpy(lab)}
    if M is MODELS["llama"]:
        out["position_ids"] = torch.arange(L)[None].expand(len(lens), L).contiguous()
    else:
        out["attention_mask"] = torch.from_numpy((np.arange(L)[None] < np.array(lens)[:, None]).astype(np.int64))
    return out


def mlm_batch(lens, seed):
    """ErLangShenCollator's batch for documents of these lengths: [CLS] (101) first, ~15 % of the other tokens labelled,
    token types 0 then 1, padded to 512 with [PAD] (0), a sentence-order label per document."""
    rs = np.random.RandomState(seed)
    n, L = len(lens), M.seq
    ids = np.zeros((n, L), dtype=np.int64)
    tt = np.zeros((n, L), dtype=np.int64)
    lab = np.full((n, L), -100, dtype=np.int64)
    for i, m in enumerate(lens):
        ids[i, :m] = rs.randint(106, M.V, size=m)
        ids[i, 0] = 101
        tt[i, m // 2:m] = 1
        sel = rs.rand(m) < 0.15
        sel[0] = False
        lab[i, :m][sel] = ids[i, :m][sel]
    return {"input_ids": torch.from_numpy(ids), "token_type_ids": torch.from_numpy(tt), "labels": torch.from_numpy(lab),
            "attention_mask": torch.from_numpy((np.arange(L)[None] < np.array(lens)[:, None]).astype(np.int64)),
            "next_sentence_label": torch.from_numpy(rs.randint(0, 2, size=n).astype(np.int64))}


def attention(args, emit):
    lens_all = lengths(4096)
    SEQ, HEADS, HD = M.seq, M.heads, M.hd
    rows, t = [], 0
    while True:   # take samples in order until first fit needs more than `rows` rows
        trial = first_fit(lens_all[:t + 1], SEQ)
        if len(trial) > args.rows:
            break
        rows, t = trial, t + 1
    lens = lens_all[:t]
    seg = torch.zeros((args.rows, SEQ), dtype=torch.int64)
    for r, members in enumerate(rows):
        p = 0
        for k, i in enumerate(members):
            seg[r, p:p + lens[i]] = k
            p += lens[i]
        seg[r, p:] = len(members)
    bidir = M is MODELS["megatronbert"]
    real = sum(n * n if bidir else n * (n + 1) // 2 for n in lens)
    g = torch.Generator().manual_seed(0)

    def tensors(n):
        qkv = torch.randn(n, SEQ, HEADS, 3, HD, generator=g).to(torch.bfloat16).cuda()
        dout = torch.randn(n, SEQ, HEADS, HD, generator=g).to(torch.bfloat16).cuda()
        dqkv = torch.empty_like(qkv)
        return (qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]), dout, (dqkv[:, :, :, 0], dqkv[:, :, :, 1], dqkv[:, :, :, 2])
    (q, k, v), dout, (dq, dk, dv) = tensors(args.rows)
    st, en = ops.segment_bounds(seg.cuda())
    sc = 1.0 / math.sqrt(HD)
    drop = ops.Dropout(M.p, SEED, torch.zeros(1, dtype=torch.int64, device="cuda"), 1) if M.p > 0 else None
    o_s, l_s = ops.sdpa_segments_fwd(q, k, v, sc, st, en, drop=drop, causal=not bidir)
    if drop is None:   # llama: the causal kernel on the same packed rows
        base, (qc, kc, vc), doc, (dqc, dkc, dvc), mask = "causal", (q, k, v), dout, (dq, dk, dv), None
    else:              # gpt2: the padded batch, one sample per row under its key mask, as GPT2QADataset makes it
        base = "noncausal_keymask" if bidir else "causal_keymask"
        (qc, kc, vc), doc, (dqc, dkc, dvc) = tensors(len(lens))
        mask = (torch.arange(SEQ)[None] < torch.tensor(lens)[:, None]).to(torch.uint8).cuda()
    causal = not bidir
    o_c, l_c = ops.sdpa_fwd(qc, kc, vc, sc, causal, kv_mask=mask, drop=drop)
    seg_kind = "segments_bidirectional" if bidir else "segments"
    fns = {
        (seg_kind, "fwd"): lambda: ops.sdpa_segments_fwd(q, k, v, sc, st, en, out=o_s, drop=drop, causal=causal),
        (base, "fwd"): lambda: ops.sdpa_fwd(qc, kc, vc, sc, causal, kv_mask=mask, out=o_c, drop=drop),
        (seg_kind, "bwd"): lambda: ops.sdpa_segments_bwd(q, k, v, o_s, dout, l_s, sc, st, en, dq, dk, dv, drop=drop,
                                                         causal=causal),
        (base, "bwd"): lambda: ops.sdpa_bwd(qc, kc, vc, o_c, doc, l_c, sc, causal, dqc, dkc, dvc, kv_mask=mask, drop=drop),
    }
    times = {key: [] for key in fns}
    for rep in range(args.reps):
        order = list(fns) if rep % 2 == 0 else list(reversed(list(fns)))
        for key in order:
            times[key].append(graph_us(fns[key], calls=10, reps=10))
    for (kind, pas), ts in times.items():
        flops = (4 if pas == "fwd" else 10) * HD * HEADS * real
        med = statistics.median(ts)
        emit(dict(bench="attention", model=args.model, kernel=kind, pass_=pas,
                  rows=len(lens) if kind.endswith("keymask") else args.rows, seq=SEQ, heads=HEADS, head_dim=HD, dropout=M.p,
                  samples=len(lens), mean_len=round(sum(lens) / len(lens), 1), us_median=round(med, 1),
                  us_min=round(min(ts), 1), us_max=round(max(ts), 1),
                  tflops_block_diagonal=round(flops / med / 1e6, 1),
                  pairs_block_diagonal=real, pairs_causal=args.rows * SEQ * (SEQ + 1) // 2))


def step(args, emit):
    from fsb200.trainer import PretrainStep
    if M is MODELS["llama"]:
        from fsb200.models.llama import LlamaForCausalLM
        cfg = SimpleNamespace(vocab_size=M.V, hidden_size=M.hidden, num_hidden_layers=M.layers, num_attention_heads=M.heads,
                              rms_norm_epsilon=1e-6, max_position_embeddings=M.seq, rotary_emb_base=10000,
                              llama_mlp_multiple_of=256)
        model = LlamaForCausalLM(cfg, device="cuda")
    elif M is MODELS["megatronbert"]:
        from fsb200.models.bert import MegatronBertForPreTraining
        cfg = SimpleNamespace(vocab_size=M.V, hidden_size=M.hidden, num_hidden_layers=M.layers, num_attention_heads=M.heads,
                              intermediate_size=4 * M.hidden, max_position_embeddings=M.seq, type_vocab_size=2,
                              layer_norm_eps=1e-12, hidden_act="gelu", hidden_dropout_prob=M.p,
                              attention_probs_dropout_prob=M.p)
        model = MegatronBertForPreTraining(cfg, device="cuda", world_size=1)
    else:
        from fsb200.models.gpt2 import GPT2LMHeadModel
        cfg = SimpleNamespace(vocab_size=M.V, n_positions=M.seq, n_embd=M.hidden, n_layer=M.layers, n_head=M.heads,
                              layer_norm_epsilon=1e-5, initializer_range=0.02, resid_pdrop=M.p, embd_pdrop=M.p,
                              attn_pdrop=M.p, activation_function="gelu_new")
        model = GPT2LMHeadModel(cfg, device="cuda", world_size=1)
    mlm = M is MODELS["megatronbert"]
    st = PretrainStep(model, lambda s: 1e-5, lr=1e-5, betas=(0.9, 0.95), weight_decay=0.1, **({"stage": 1} if mlm else {}))
    SEQ, EOS = M.seq, M.eos
    lens = lengths(args.samples * args.batches, seed=SEED + 1)
    padded = [(mlm_batch if mlm else sft_batch)(lens[i * args.samples:(i + 1) * args.samples], seed=i)
              for i in range(args.batches)]
    pack = (lambda b: pack_mlm_batch(b, SEQ, EOS)) if mlm else (lambda b: pack_causal_lm_batch(b, SEQ, EOS))
    variants = {"padded": [{k: v.cuda() for k, v in b.items()} for b in padded],
                "packed": [{k: v.cuda() for k, v in pack(b).items() if k != "attention_mask"} for b in padded]}
    labels = sum(int((b["labels"][:, 0 if mlm else 1:] != -100).sum()) for b in padded)
    tokens = sum(lens)
    shapes = {k: [tuple(b["input_ids"].shape) for b in v] for k, v in variants.items()}
    for name, bs in variants.items():   # warm-up: every shape
        for b in bs:
            st.step_device([b])
    torch.cuda.synchronize()
    res = {k: {"s": [], "peak": 0} for k in variants}
    for rep in range(args.reps):
        for name in (["padded", "packed"] if rep % 2 == 0 else ["packed", "padded"]):
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for b in variants[name]:
                st.step_device([b])
            e1.record()
            torch.cuda.synchronize()
            res[name]["s"].append(e0.elapsed_time(e1) / 1e3)
            res[name]["peak"] = max(res[name]["peak"], torch.cuda.max_memory_allocated())
    for name, r in res.items():
        med = statistics.median(r["s"])
        emit(dict(bench="step", model=args.model, variant=name, layers=M.layers, hidden=M.hidden, dropout=M.p,
                  samples_per_microbatch=args.samples,
                  microbatches=args.batches, shapes=shapes[name], label_tokens=labels, nonpad_tokens=tokens,
                  label_tok_s_median=round(labels / med), nonpad_tok_s_median=round(tokens / med),
                  label_tok_s_min=round(labels / max(r["s"])), label_tok_s_max=round(labels / min(r["s"])),
                  documents_s_median=round(len(lens) / med, 1),
                  seconds=[round(x, 4) for x in r["s"]], peak_alloc_gib=round(r["peak"] / 2 ** 30, 2)))
    del st, model
    gc.collect()


def seq2seq_batch(lens, seed):
    """LCSTSDataset's batch for sources of these lengths: source padded to 128 under attention_mask 0, target 64 tokens
    with every position labelled (its pad ids included, as the reference leaves them)."""
    rs = np.random.RandomState(seed)
    n = len(lens)
    ids = np.zeros((n, M.seq), dtype=np.int64)
    for i, m in enumerate(lens):
        ids[i, :m] = rs.randint(2, M.V, size=m)
    return {"input_ids": torch.from_numpy(ids),
            "attention_mask": torch.from_numpy((np.arange(M.seq)[None] < np.array(lens)[:, None]).astype(np.int64)),
            "labels": torch.from_numpy(rs.randint(2, M.V, size=(n, M.dec)).astype(np.int64))}


def mt5_attention(args, emit):
    from fsb200.models.base import cross_segment_bounds
    lens = lengths(args.rows * M.pack * 4)
    packed = pack_seq2seq_batch(seq2seq_batch(lens, 0), M.pack * M.seq, M.pack * M.dec, 0)
    R = packed["input_ids"].shape[0]
    n, Se, Sd = len(lens), M.pack * M.seq, M.pack * M.dec
    H, HD = M.heads, M.hd
    g = torch.Generator().manual_seed(0)
    rnd = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    drop = ops.Dropout(M.p, SEED, torch.zeros(1, dtype=torch.int64, device="cuda"), 1)
    enc_b = ops.segment_bounds(packed["segment_ids"].cuda())
    dec_b = ops.segment_bounds(packed["decoder_segment_ids"].cuda())
    kvb, qb = cross_segment_bounds(packed["decoder_segment_ids"].cuda(), packed["segment_ids"].cuda())
    mask = (torch.arange(M.seq)[None] < torch.tensor(lens)[:, None]).to(torch.uint8).cuda()
    fns, flops = {}, {}
    for form, (Bp, Sqp, Skp, Bd, Sqd, Skd, real) in {
            "encoder": (R, Se, Se, n, M.seq, M.seq, sum(m * m for m in lens)),
            "decoder": (R, Sd, Sd, n, M.dec, M.dec, n * M.dec * (M.dec + 1) // 2),
            "cross": (R, Sd, Se, n, M.dec, M.seq, sum(M.dec * m for m in lens))}.items():
        for variant, (B, Sq, Sk) in (("packed", (Bp, Sqp, Skp)), ("padded", (Bd, Sqd, Skd))):
            q, k, v, do = rnd(B, Sq, H, HD), rnd(B, Sk, H, HD), rnd(B, Sk, H, HD), rnd(B, Sq, H, HD)
            dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            rel = torch.randn(H, Sq + Sk - 1, generator=g).cuda() if form != "cross" else None
            drel = torch.zeros_like(rel) if rel is not None else None
            if variant == "packed":
                kw = dict(causal=form == "decoder", rel_bias=rel) if form != "cross" else dict(causal=False, kv_bounds=qb)
                b = {"encoder": enc_b, "decoder": dec_b, "cross": kvb}[form]
                o, lse = ops.sdpa_segments_fwd(q, k, v, 1.0, *b, drop=drop, **kw)
                f = (lambda q=q, k=k, v=v, o=o, b=b, kw=kw: ops.sdpa_segments_fwd(q, k, v, 1.0, *b, out=o, drop=drop, **kw))
                bw = (lambda q=q, k=k, v=v, o=o, lse=lse, do=do, dq=dq, dk=dk, dv=dv, b=b, kw=kw, drel=drel:
                      ops.sdpa_segments_bwd(q, k, v, o, do, lse, 1.0, *b, dq, dk, dv, drop=drop, drel_bias=drel, **kw))
            else:
                causal, km = form == "decoder", None if form == "decoder" else mask
                o, lse = ops.sdpa_fwd(q, k, v, 1.0, causal, kv_mask=km, rel_bias=rel, drop=drop)
                f = (lambda q=q, k=k, v=v, o=o, causal=causal, km=km, rel=rel:
                     ops.sdpa_fwd(q, k, v, 1.0, causal, kv_mask=km, rel_bias=rel, out=o, drop=drop))
                bw = (lambda q=q, k=k, v=v, o=o, lse=lse, do=do, dq=dq, dk=dk, dv=dv, causal=causal, km=km, rel=rel, drel=drel:
                      ops.sdpa_bwd(q, k, v, o, do, lse, 1.0, causal, dq, dk, dv, kv_mask=km, rel_bias=rel, drel_bias=drel,
                                   drop=drop))
            fns[(form, variant, "fwd")], fns[(form, variant, "bwd")] = f, bw
            flops[(form, "fwd")], flops[(form, "bwd")] = 4 * HD * H * real, 10 * HD * H * real
    times = {key: [] for key in fns}
    for rep in range(args.reps):
        for key in (list(fns) if rep % 2 == 0 else list(reversed(list(fns)))):
            times[key].append(graph_us(fns[key], calls=10, reps=10))
    for (form, variant, pas), ts in times.items():
        med = statistics.median(ts)
        emit(dict(bench="attention", model="mt5", form=form, variant=variant, pass_=pas, rows=R if variant == "packed" else n,
                  heads=H, head_dim=HD, dropout=M.p, samples=n, mean_src_len=round(sum(lens) / n, 1),
                  us_median=round(med, 1), us_min=round(min(ts), 1), us_max=round(max(ts), 1),
                  tflops_real_pairs=round(flops[(form, pas)] / med / 1e6, 1)))


def mt5_step(args, emit):
    from fsb200.models.t5 import MT5ForConditionalGeneration
    from fsb200.trainer import PretrainStep
    cfg = SimpleNamespace(vocab_size=M.V, d_model=M.hidden, d_kv=M.hd, num_heads=M.heads, d_ff=M.ff, num_layers=M.layers,
                          num_decoder_layers=M.layers, layer_norm_epsilon=1e-6, relative_attention_num_buckets=32,
                          relative_attention_max_distance=128, pad_token_id=0, decoder_start_token_id=0,
                          dropout_rate=M.p, feed_forward_proj="gated-gelu", tie_word_embeddings=False)
    model = MT5ForConditionalGeneration(cfg, device="cuda", world_size=1)
    st = PretrainStep(model, lambda s: 1e-5, lr=1e-5, betas=(0.9, 0.95), weight_decay=0.1)
    lens = lengths(args.samples * args.batches, seed=SEED + 1)
    padded = [seq2seq_batch(lens[i * args.samples:(i + 1) * args.samples], seed=i) for i in range(args.batches)]
    variants = {"padded": [{k: v.cuda() for k, v in b.items()} for b in padded],
                "packed": [{k: v.cuda() for k, v in pack_seq2seq_batch(b, M.pack * M.seq, M.pack * M.dec, 0).items()
                            if k != "attention_mask"} for b in padded]}
    labels = sum(int((b["labels"] != -100).sum()) for b in padded)
    tokens = sum(lens) + labels
    shapes = {k: [(tuple(b["input_ids"].shape), tuple(b["labels"].shape)) for b in v] for k, v in variants.items()}
    for bs in variants.values():
        for b in bs:
            st.step_device([b])
    torch.cuda.synchronize()
    res = {k: {"s": [], "peak": 0} for k in variants}
    for rep in range(args.reps):
        for name in (["padded", "packed"] if rep % 2 == 0 else ["packed", "padded"]):
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for b in variants[name]:
                st.step_device([b])
            e1.record()
            torch.cuda.synchronize()
            res[name]["s"].append(e0.elapsed_time(e1) / 1e3)
            res[name]["peak"] = max(res[name]["peak"], torch.cuda.max_memory_allocated())
    for name, r in res.items():
        med = statistics.median(r["s"])
        emit(dict(bench="step", model="mt5", variant=name, layers=f"{M.layers}+{M.layers}", hidden=M.hidden, dropout=M.p,
                  samples_per_microbatch=args.samples, microbatches=args.batches, shapes=shapes[name],
                  label_tokens=labels, nonpad_tokens=tokens, label_tok_s_median=round(labels / med),
                  nonpad_tok_s_median=round(tokens / med), label_tok_s_min=round(labels / max(r["s"])),
                  label_tok_s_max=round(labels / min(r["s"])), seconds=[round(x, 4) for x in r["s"]],
                  peak_alloc_gib=round(r["peak"] / 2 ** 30, 2)))
    del st, model
    gc.collect()


def main():
    global M
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=sorted(MODELS), default="llama")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", type=int, default=4)
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    M = MODELS[args.model]
    if not torch.cuda.is_available():
        raise SystemExit("bench_packing: no CUDA device; the measurements need an H100")
    sink = open(os.path.join(args.out, f"bench_packing_{args.model}.jsonl" if args.model != "llama" else "bench_packing.jsonl"),
                "w") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")
    emit(dict(bench="card", **card()))
    if not args.skip_attention:
        (mt5_attention if args.model == "mt5" else attention)(args, emit)
    if not args.skip_step:
        (mt5_step if args.model == "mt5" else step)(args, emit)
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
