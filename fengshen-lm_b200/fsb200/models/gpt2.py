"""Wenzhong-GPT2 on the fsb200 kernels — drop-in for `transformers.GPT2LMHeadModel` as the reference uses it
(fengshen/examples/wenzhong_qa/finetune_wenzhong.py:56: `GPT2LMHeadModel.from_pretrained(...)`, training_step :89-113).

The arithmetic restated here lives in 3P `transformers` (gpt2/modeling_gpt2.py; SURVEY.md Appendix C):
pre-LN blocks `x + attn(ln_1(x))`, `x + mlp(ln_2(x))`, final `ln_f`; fused `c_attn` Conv1D with weight stored [in, out]
(q | k | v contiguous thirds); `gelu_new`; learned positions `wte[ids] + wpe[pos]`; LM head tied to `wte`; shifted mean
cross-entropy with ignore_index -100. State-dict keys follow HF (`transformer.h.N.attn.c_attn.weight`, ...).
Conv1D's [in, out] layout maps onto the GEMM layouts without any transpose: forward = NN, dgrad = NT, wgrad = TN.
Dropout (`embd_pdrop`, `attn_pdrop`, `resid_pdrop`, each in [0, 1) and independent) applies in training mode
(`model.training`, also under no_grad), at HF's sites: the embedding sum, the attention probabilities (inside the causal
attention kernels) and the attention / MLP `c_proj` outputs, dropped by the LayerNorm that adds them to the residual stream
(`ln_2`, the next block's `ln_1`, `ln_f`). Seed, stream counter and eval mode as in fsb200/models/base.py; `generate` in
training mode with a non-zero probability is rejected (HF would drop).
Packed rows (several samples per row, fsb200/packing.py) pass `segment_ids`, as LlamaForCausalLM does: attention stays
causal inside each segment, the attention-probability dropout included, and never crosses one.
Head widths 64 (Wenzhong-110M), 96 (the 3.5B Wenzhong / Yuyuan: 32 heads x 96) and 128 run; at 96 the KV-cache decode pads
each head to 128 columns (see generate).
fp8=True trains each block's c_attn, attn.c_proj, mlp.c_fc (bias, gelu_new and its pre-activation in the FP8 GEMM's
epilogue) and mlp.c_proj in FP8 (layers.Fp8Conv1D, include/fsb200.h fsb_gemm_fp8 / fsb_gemm_fp8_t): e4m3 activations and
weights, e5m2 gradients, per-tensor power-of-two scales from each tensor's amax just before its cast, fp32 accumulation. The
forward keeps the transposed e4m3 codes of ln_1's and ln_2's outputs and of the GELU output instead of the bf16 tensors;
attn.c_proj makes its input's codes from the attention output in the backward (attention keeps that output anyway). The
embeddings, the tied LM head, the LayerNorms, attention, dGELU with the c_fc bias gradient, the loss and the optimizer stay
bf16, as do the master weights and gradients; `generate` runs the bf16 projections.
load_in_8bit / load_in_4bit (`from_pretrained(..., load_in_8bit=True)`): an inference-only model whose four block
projections are held quantised (layers.QuantizedLinear: int8 per output channel, or int4 with a scale per row and group of
128 k) from the transposed [out, in] weight, their biases bf16; c_fc's bias and gelu_new run in the W8A16 / W4A16 GEMM's
epilogue (include/fsb200.h fsb_gemm_w8a16_bias). The no-grad forwards and `generate` run them; the embeddings, the tied LM
head and the LayerNorms stay bf16, without a gradient buffer. Training, save_pretrained and fp8=True raise.
"""
import math
from collections import namedtuple
from types import SimpleNamespace

import torch

from .. import generation
from .. import lib as L
from .. import ops
from ..decode_graph import DecodeGraphs
from ..flat import FlatSpec
from .base import FlatModel, _Holder, flat_ids, key_mask, learned_pos_emb_bwd, packed_segments, refuse_key_padding
from .layers import WQ, Fp8Conv1D, Linear, QuantizedLinear, apply_dropout, quantized_unsupported, residual_norm_bwd

_Block = namedtuple("_Block", "c_attn attn_proj c_fc mlp_proj")   # a block's projections


_QKEYS = (("c_attn", "attn.c_attn"), ("attn_proj", "attn.c_proj"), ("c_fc", "mlp.c_fc"), ("mlp_proj", "mlp.c_proj"))


class GPT2LMHeadModel(FlatModel):
    wq_transposed = True   # a checkpoint's Conv1D weights are [in, out]: quantised from their transpose

    def __init__(self, config, device=None, world_size=None, seed=0, fp8=False, load_in_8bit=False, load_in_4bit=False):
        """fp8: train the block projections in FP8; see the module docstring. The training and no-grad (validation)
        forwards both run FP8; results differ from bf16 by design. n_embd, the MLP's inner width and the tokens per
        micro-batch (batch x sequence length) must be multiples of 16 (checked at the first forward).

        load_in_8bit: an inference-only model. Each block's c_attn, attn.c_proj, mlp.c_fc and mlp.c_proj are held as int8
        q [out, in] + fp32 per-output-channel scales s [out], quantised from the transposed Conv1D weight, and run through
        the W8A16 GEMM with their bf16 bias (and gelu_new for c_fc) in its epilogue; wte, wpe (with the tied LM head), the
        LayerNorms and the biases stay bf16 in flat buffers without a gradient buffer. Training, save_pretrained and fp8=True
        raise. load_in_4bit: the same with int4 projections (a bf16 scale per row and group of 128 k); n_embd and the inner
        width must then be multiples of 128."""
        super().__init__(config)
        if load_in_8bit and load_in_4bit:
            raise ValueError("fsb200 GPT2LMHeadModel: load_in_8bit and load_in_4bit are mutually exclusive; pass one")
        if fp8 and (load_in_8bit or load_in_4bit):
            raise ValueError("fsb200 GPT2LMHeadModel: fp8=True trains in FP8; it cannot be combined with load_in_8bit or "
                             "load_in_4bit (inference-only weight formats)")
        self.fp8 = bool(fp8)
        self.weight_format = "int8" if load_in_8bit else "int4" if load_in_4bit else "bf16"
        self.load_in_8bit, self.load_in_4bit = self.weight_format == "int8", self.weight_format == "int4"
        quantized = self.weight_format != "bf16"
        g = lambda k, d=None: getattr(config, k, d)
        self.h, self.nl, self.nh = g("n_embd", g("hidden_size")), g("n_layer", g("num_hidden_layers")), \
            g("n_head", g("num_attention_heads"))
        self.V, self.npos = g("vocab_size"), g("n_positions", g("max_position_embeddings", 1024))
        self.eps = g("layer_norm_epsilon", 1e-5)
        self.inner = g("n_inner") or 4 * self.h
        self.p_embd, self.p_attn, self.p_resid = self._dropout_probs("GPT2", "embd_pdrop", "attn_pdrop", "resid_pdrop")
        if g("activation_function", "gelu_new") != "gelu_new":
            raise RuntimeError("fsb200 GPT2: only activation_function='gelu_new' is implemented")
        h, V = self.h, self.V
        self.hn = h // self.nh
        if self.hn not in (64, 96, 128) or V % 8 or h % 8:
            raise RuntimeError("fsb200 GPT2: head dim must be 64/96/128 and vocab/hidden multiples of 8 (pad the vocab)")
        if self.load_in_4bit and (h % 128 or self.inner % 128):
            raise RuntimeError(f"fsb200 GPT2LMHeadModel(load_in_4bit=True): n_embd ({h}) and the inner width ({self.inner}) "
                               "must be multiples of 128 (the int4 scale group)")

        spec = FlatSpec()
        spec.add("transformer.wte.weight", (V, h), "wte")
        spec.add("transformer.wpe.weight", (self.npos, h), "wte")
        for i in range(self.nl):
            p, bk = f"transformer.h.{i}.", f"layer{i}"
            for n, s in (("ln_1.weight", (h,)), ("ln_1.bias", (h,)), ("attn.c_attn.weight", (h, 3 * h)),
                         ("attn.c_attn.bias", (3 * h,)), ("attn.c_proj.weight", (h, h)), ("attn.c_proj.bias", (h,)),
                         ("ln_2.weight", (h,)), ("ln_2.bias", (h,)), ("mlp.c_fc.weight", (h, self.inner)),
                         ("mlp.c_fc.bias", (self.inner,)), ("mlp.c_proj.weight", (self.inner, h)),
                         ("mlp.c_proj.bias", (h,))):
                if not (quantized and n.endswith(".weight") and not n.startswith("ln_")):   # int8 / int4: held as q + s
                    spec.add(p + n, s, bk)
        spec.add("transformer.ln_f.weight", (h,), "wte")
        spec.add("transformer.ln_f.bias", (h,), "wte")
        self._bind_flat(spec, device, world_size, grads=not quantized)
        self.lm_head = _Holder()
        self.lm_head.weight = self.transformer.wte.weight  # tied (modeling_gpt2.py:646)
        self._head = Linear.of(self.lm_head.weight)
        if quantized:   # QuantizedLinear [n, k] = [out, in]: the Conv1D weight's transpose
            qlin = lambda m, n, k: QuantizedLinear(self.weight_format, n, k, self.flat.params.device, bias=m.bias.data,
                                                   model="GPT2LMHeadModel")
            self._proj = [_Block(qlin(b.attn.c_attn, 3 * h, h), qlin(b.attn.c_proj, h, h),
                                 qlin(b.mlp.c_fc, self.inner, h), qlin(b.mlp.c_proj, h, self.inner))
                          for b in self.transformer.h]
        else:
            conv1d = lambda m: Linear.of(m.weight, m.bias, conv1d=True)
            self._proj = [_Block(conv1d(b.attn.c_attn), conv1d(b.attn.c_proj), conv1d(b.mlp.c_fc), conv1d(b.mlp.c_proj))
                          for b in self.transformer.h]
        self._proj_generate = self._proj   # what generate runs: bf16 under fp8=True, the int8 / int4 projections if quantised
        if self.fp8:
            self._proj = [_Block(*(Fp8Conv1D(q) for q in pj)) for pj in self._proj]
        self.reset_parameters(seed)
        # dropout sites of one forward, in transformers' call order: 0 embeddings; for layer i, 1 + 3i attention probabilities,
        # 2 + 3i attention c_proj output, 3 + 3i MLP c_proj output. A site whose probability is 0 keeps its number.
        self._init_dropout(1 + 3 * self.nl, (self.p_embd, self.p_attn, self.p_resid))

    @torch.no_grad()
    def reset_parameters(self, seed=0):
        """HF GPT2 _init_weights: N(0, initializer_range) for Linear/Embedding, c_proj scaled by 1/sqrt(2*n_layer),
        LayerNorm weight 1 / bias 0, biases 0."""
        std = getattr(self.config, "initializer_range", 0.02)
        gen = torch.Generator(device=self.flat.params.device).manual_seed(seed)
        for name, prm in self.named_parameters():
            if name.endswith("bias"):
                prm.zero_()
            elif ".ln_" in name:
                prm.fill_(1.0)
            else:
                s = std / math.sqrt(2 * self.nl) if name.endswith("c_proj.weight") else std
                prm.normal_(0.0, s, generator=gen)
        if self.weight_format != "bf16":   # each quantised projection: drawn in bf16 on the device and quantised, one at a time
            for wq in self._wq:
                for key, (q, s) in wq.items():
                    tmp = torch.empty(self._weight_shape(q, s), dtype=torch.bfloat16, device=q.device)
                    tmp.normal_(0.0, std / math.sqrt(2 * self.nl) if key in ("attn_proj", "mlp_proj") else std, generator=gen)
                    WQ[self.weight_format][0](tmp, q, s)
                    del tmp

    # ---- int8 / int4 (load_in_8bit / load_in_4bit; loading and get_memory_footprint: FlatModel) -------------------------
    @property
    def _wq(self):
        """Per block {projection: (q, s)} of an int8 / int4 model, projections named as _Block names them."""
        return [{f: (getattr(pj, f).q, getattr(pj, f).s) for f, _ in _QKEYS} for pj in self._proj]

    def _wq_targets(self):
        """{state-dict key of a Conv1D weight: the (q, s) it quantises into}."""
        return {f"transformer.h.{i}.{key}.weight": (getattr(pj, f).q, getattr(pj, f).s)
                for i, pj in enumerate(self._proj) for f, key in _QKEYS}

    def save_pretrained(self, path, **kw):
        if self.weight_format != "bf16":
            raise quantized_unsupported("GPT2LMHeadModel", self.weight_format, f"save_pretrained ({self.weight_format} export)")
        return super().save_pretrained(path, **kw)

    # ---- forward ----------------------------------------------------------------------------------------------------
    def forward(self, input_ids=None, attention_mask=None, labels=None, position_ids=None, return_logits=False,
                segment_ids=None, **_):
        """segment_ids: optional integer [B, S] (host or device) for packed rows; a segment is a maximal run of equal
        consecutive values in a row. Every layer's attention is then causal inside each segment only, and the label of each
        segment's first token is ignored. Pass per-segment position_ids (fsb200/packing.py emits them). No key mask is used:
        the packer makes the pad tail a segment of its own, and an attention_mask with zeros is refused. None: one causal
        sequence per row under attention_mask, as before."""
        B, S = input_ids.shape
        if self.fp8:
            bad = [f"{name} ({v})" for name, v in (("n_embd", self.h), ("the inner width", self.inner),
                                                    (f"batch {B} x sequence length {S}", B * S)) if v % 16]
            if bad:
                raise ValueError(f"fsb200 GPT2LMHeadModel(fp8=True): {', '.join(bad)} not a multiple of 16 (the FP8 GEMM "
                                 "operands need 16-byte rows in both layouts)")
        dev = self.flat.params.device
        ids, lab = flat_ids(input_ids, dev), flat_ids(labels, dev)
        if self.weight_format != "bf16" and lab is not None and torch.is_grad_enabled():
            raise quantized_unsupported("GPT2LMHeadModel", self.weight_format, "a training forward (labels under grad mode)")
        pos = None if position_ids is None else flat_ids(position_ids.expand(B, S), dev)
        if segment_ids is None:
            seg, mask = (), key_mask(attention_mask, dev)
        else:
            refuse_key_padding(attention_mask, "GPT2LMHeadModel")
            bounds, lab = packed_segments(segment_ids, lab, B, S, dev)
            seg, mask = (bounds,), None
        loss, logits = self._step_or_forward(lab is not None, return_logits, ids, pos, mask, lab, B, S, *seg)
        return SimpleNamespace(loss=loss, logits=None if logits is None else logits.view(B, S, self.V),
                               past_key_values=None, hidden_states=None, attentions=None)

    def _forward_impl(self, ids, pos, mask, lab, B, S, seg=None, *, save, want_logits):
        """seg: None or the (seg_start, seg_end) bounds of packed rows (ops.segment_bounds); mask is then None."""
        scale = 1.0 / math.sqrt(self.hn)
        acts = [] if save else None
        base = self._dropout_base()

        def attend(i, q5):
            drop = self._drop(base, self.p_attn, 1 + 3 * i)
            if seg is not None:
                q, k, v = q5[:, :, 0], q5[:, :, 1], q5[:, :, 2]
                return ops.sdpa_segments_fwd(q, k, v, scale, *seg, drop=drop)
            return ops.sdpa_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], scale, True, kv_mask=mask, drop=drop)
        hf, stf, xf = self._stack(ids, pos, B, S, attend, acts, base)
        logits = self._head(hf)
        loss, ctx = None, None
        if lab is not None:
            keep = logits.clone() if (want_logits and save) else None
            loss, dlogits, _ = ops.softmax_xent(logits, lab, S, shift=1, grad_scale=self.loss_scale,
                                                dlogits="inplace" if save else None)
            if save:
                ctx = (acts, hf, stf, xf, dlogits, ids, pos, mask, B, S, base, seg)
                logits = keep
        return loss, (logits if want_logits else None), ctx

    def _stack(self, ids, pos, B, S, attend, acts=None, base=None, proj=None):
        """Embedding, the blocks and ln_f over ids [B * S] -> (hidden states, ln_f stats, residual stream). attend(i, q5) is
        block i's attention over the packed q|k|v view [B, S, 3, heads, head_dim] -> (out, lse), drawing its own probability
        mask; `acts`, when given, collects what the backward reads. base: the forward's dropout stream base (None: no
        dropout, as in generation's prefill and decode steps). proj: the blocks' projections (default self._proj)."""
        h, nh, hn = self.h, self.nh, self.hn
        tr = self.transformer
        pr = self.p_resid
        D = lambda p, site: self._drop(base, p, site)
        self._need("no_decay"); self._need("wte")
        x = apply_dropout(ops.embedding_fwd(ids, tr.wte.weight.data, pos=pos, P=tr.wpe.weight.data, seq_len=S),
                          D(self.p_embd, 0))
        prev_m = None
        save = acts is not None
        for i, (blk, pj) in enumerate(zip(tr.h, self._proj if proj is None else proj)):
            self._need(f"layer{i}")
            h1, st1, x = ops.layernorm_fwd(x if prev_m is None else prev_m, blk.ln_1.weight.data, blk.ln_1.bias.data,
                                           self.eps, residual=None if prev_m is None else x,
                                           drop=None if prev_m is None else D(pr, 3 * i))   # layer i-1's MLP output
            # h1s, h2s, fs: what the projections' backward reads of their inputs (the tensors themselves in bf16, their
            # transposed e4m3 codes and scales in FP8)
            qkv, h1s = pj.c_attn.forward(h1, save)
            o, lse = attend(i, qkv.view(B, S, 3, nh, hn))
            a = pj.attn_proj(o.view(B * S, h))
            h2, st2, x1 = ops.layernorm_fwd(a, blk.ln_2.weight.data, blk.ln_2.bias.data, self.eps, residual=x,
                                            drop=D(pr, 2 + 3 * i))
            pre = None if acts is None else torch.empty((B * S, self.inner), dtype=torch.bfloat16, device=x.device)
            f, h2s = pj.c_fc.forward(h2, save, epilogue=L.EPI_GELU_TANH, aux=pre)
            m, fs = pj.mlp_proj.forward(f, save)
            if acts is not None:
                acts.append((x, st1, h1s, qkv, o, lse, x1, st2, h2s, pre, fs))
            # free this block's temporaries before the next block allocates its own (the peak of a long prompt's prefill)
            del st1, h1, h1s, qkv, o, lse, a, st2, h2, h2s, pre, f, fs
            x, prev_m = x1, m
        return ops.layernorm_fwd(prev_m, tr.ln_f.weight.data, tr.ln_f.bias.data, self.eps, residual=x,
                                 drop=D(pr, 3 * self.nl))

    # ---- KV-cache generation -----------------------------------------------------------------------------------------
    # transformers' GenerationMixin on GPT-2 (wenzhong_qa/README.md:58-67: sampling with top_p, num_return_sequences,
    # return_dict_in_generate, output_scores). Prefill and decode steps run the training layer stack (`_stack`) with their
    # own attention: the prefill writes the prompt's keys / values into a pre-allocated cache, one [layers, rows, cap, 2,
    # heads, head_dim] allocation, and attends causally under the left-padding key mask; a decode step feeds one token per
    # row, appends its keys / values at the device-side slot kv_len - 1 (ops.kv_append) and attends with the split-KV decode
    # kernel (ops.attn_decode). The decode step is one CUDA-graph replay (fsb200/decode_graph.py); beam search gathers the
    # cache, key mask and positions into the twin (ops.kv_reorder). Position ids follow transformers 5.5.0
    # (generation/utils.py:716-720): cumsum(mask) - 1, pads at 0.
    # Head width 96 decodes on the head_dim 128 decode kernel over a zero-padded cache: the cache's last dimension is 128,
    # the prefill and ops.kv_append write its first 96 columns, and each step copies q into the first 96 columns of a
    # zero-padded [rows, heads, 128] buffer. The zero columns add nothing to q.k, the output's padded columns come out as
    # P.0, and its first 96 feed attn_proj. Beam reorder moves whole slots and is unchanged.
    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, **kwargs):
        """HF `generate` semantics (fsb200/generation.py lists what is implemented); prompts are LEFT-padded. Runs without
        dropout; in training mode with a non-zero dropout probability it raises (HF would drop)."""
        self._refuse_dropout_generate("GPT2", "embd_pdrop / attn_pdrop / resid_pdrop")
        dev = self.flat.params.device
        ids = input_ids.to(device=dev, dtype=torch.int64)
        B, S0 = ids.shape
        c = generation.resolve(self.config, kwargs, S0, False)
        if c.max_length > self.npos:
            raise ValueError(f"fsb200 GPT2 generate: max_length {c.max_length} exceeds n_positions {self.npos}")
        mask = generation.default_attention_mask(ids, c.pad, c.eos) if attention_mask is None else \
            attention_mask.to(device=dev, dtype=torch.int64)
        ids, mask = ids.repeat_interleave(c.expand, 0), mask.repeat_interleave(c.expand, 0)
        R = ids.shape[0]
        cap = (max(c.max_length, S0 + 1) + 63) // 64 * 64
        scale = 1.0 / math.sqrt(self.hn)
        hn, hc = self.hn, 128 if self.hn == 96 else self.hn   # head width, cached head width
        pad = (lambda t: t[..., :hn]) if hc != hn else (lambda t: t)   # the head's columns of a cache view
        q_pad = torch.zeros((R, self.nh, hc), dtype=torch.bfloat16, device=dev) if hc != hn else None
        # per cache: keys / values, key mask, next position id of every row
        st = [SimpleNamespace(cache=torch.zeros((self.nl, R, cap, 2, self.nh, hc), dtype=torch.bfloat16, device=dev),
                              kv_mask=torch.zeros((R, cap), dtype=torch.uint8, device=dev),
                              count=torch.zeros(R, dtype=torch.int64, device=dev))
              for _ in range(2 if c.num_beams > 1 else 1)]
        st[0].kv_mask[:, :S0] = mask.to(torch.uint8)
        st[0].count.copy_(mask.sum(-1))
        kv_len = torch.full((1,), S0, dtype=torch.int32, device=dev)

        def prefill():
            pos = (mask.cumsum(-1) - 1).masked_fill(mask == 0, 0)
            pre = None if bool(mask.all()) else st[0].kv_mask[:, :S0].contiguous()

            def attend(i, q5):
                pad(st[0].cache[i][:, :S0]).copy_(q5[:, :, 1:3])
                return ops.sdpa_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], scale, True, kv_mask=pre)
            return self._last_logits(ids.reshape(-1), pos.reshape(-1), R, S0, attend)

        def body(tok, index, a, b):
            if b is not a:
                ops.kv_reorder(a.cache, b.cache, index, kv_len)
                torch.index_select(a.kv_mask, 0, index, out=b.kv_mask)
                torch.index_select(a.count, 0, index, out=b.count)
            kv_len.add_(1)

            def attend(i, q5):   # the key mask is shared by the layers: the first one sets the new slot's bit
                kv = b.cache[i]
                ops.kv_append(q5[:, 0, 1], q5[:, 0, 2], pad(kv[:, :, 0]), pad(kv[:, :, 1]), kv_len,
                              kv_mask=b.kv_mask if i == 0 else None)
                if q_pad is None:
                    return ops.attn_decode(q5[:, 0, 0], kv[:, :, 0], kv[:, :, 1], kv_len, scale, kv_mask=b.kv_mask)
                q_pad[..., :hn].copy_(q5[:, 0, 0])
                o, lse = ops.attn_decode(q_pad, kv[:, :, 0], kv[:, :, 1], kv_len, scale, kv_mask=b.kv_mask)
                return o[..., :hn].contiguous(), lse
            logits = self._last_logits(tok, b.count, R, 1, attend)
            b.count.add_(1)
            return logits

        return generation.run(DecodeGraphs(self, R, st, body, prefill), ids, c)

    def _last_logits(self, ids, pos, B, S, attend):
        """fp32 logits [B, V] of the last position of every sequence."""
        hf, _, _ = self._stack(ids, pos, B, S, attend, proj=self._proj_generate)
        return self._head(hf.view(B, S, self.h)[:, -1].contiguous()).float()

    # ---- backward ---------------------------------------------------------------------------------------------------
    def _backward_impl(self, ctx, gloss):
        acts, hf, stf, xf, dlogits, ids, pos, mask, B, S, base, seg = ctx
        h, nh, hn = self.h, self.nh, self.hn
        T = B * S
        acc = self.accumulate_grads
        pr = self.p_resid
        D = lambda p, site: self._drop(base, p, site)
        self._begin_backward()
        tr = self.transformer
        scale = 1.0 / math.sqrt(hn)
        if gloss is not None:
            ops.scale_inplace(dlogits, gloss)  # upstream scalar; the kernel exits immediately when it is 1.0
        dhf = self._head.backward(dlogits, hf, acc)   # tied head: written first, the embedding adds later
        del dlogits
        # d(residual), d(last MLP output)
        dx, dm = residual_norm_bwd(dhf, xf, tr.ln_f.weight, tr.ln_f.bias, stf, D(pr, 3 * self.nl), acc)
        for i in reversed(range(self.nl)):
            blk, pj = tr.h[i], self._proj[i]
            x, st1, h1s, qkv, o, lse, x1, st2, h2s, pre, fs = acts[i]
            acts[i] = None
            df = pj.mlp_proj.backward(dm, fs, acc)
            dpre = ops.act_bwd_bias(L.ACT_GELU_TANH, df, pre, pj.c_fc.bias_grad, accumulate=acc)   # dGELU + c_fc bias grad
            dh2 = pj.c_fc.backward(dpre, h2s, acc, colsum=False)
            dx1, da = residual_norm_bwd(dh2, x1, blk.ln_2.weight, blk.ln_2.bias, st2, D(pr, 2 + 3 * i), acc, dres=dx)
            do = pj.attn_proj.backward(da, pj.attn_proj.saved_input(o.view(T, h)), acc)   # o is kept for attention anyway
            dqkv = torch.empty_like(qkv)
            q5, d5 = qkv.view(B, S, 3, nh, hn), dqkv.view(B, S, 3, nh, hn)
            if seg is not None:
                ops.sdpa_segments_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, S, nh, hn), lse, scale, *seg,
                                      d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], drop=D(self.p_attn, 1 + 3 * i))
            else:
                ops.sdpa_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, S, nh, hn), lse, scale, True,
                             d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], kv_mask=mask, drop=D(self.p_attn, 1 + 3 * i))
            dh1 = pj.c_attn.backward(dqkv, h1s, acc)
            # layer 0's LN had no residual (x = the embeddings); layer i's summed layer i-1's dropped MLP output into x
            dx, dm = residual_norm_bwd(dh1, x, blk.ln_1.weight, blk.ln_1.bias, st1, D(pr, 3 * i) if i > 0 else None, acc,
                                       dres=dx1)
            self._done(f"layer{i}")
        dx = apply_dropout(dx, D(self.p_embd, 0))
        ops.embedding_bwd(ids, dx, tr.wte.weight.main_grad)  # accumulates onto the LM-head wgrad (tied weights)
        learned_pos_emb_bwd(pos, dx, tr.wpe.weight.main_grad, B, S, acc)
        self._done("wte")
        self._done("no_decay")
