"""Ziya-LLaMA on the fsb200 kernels — drop-in for `fengshen.models.llama.modeling_llama.LlamaForCausalLM`.

Same constructor (`LlamaForCausalLM(config)`), same `forward(input_ids, attention_mask, position_ids, labels)` ->
`CausalLMOutputWithPast`-like result (reference: fengshen/models/llama/modeling_llama.py:272-351), same state-dict key
names (`llama.embed_in.word_embeddings.weight`, `llama.layers.N.attention.query_key_value.weight`, ...,
`embed_out.final_linear.weight`; utils/llama_convert/hf_to_fs.py:136-147), same per-head interleaved QKV weight layout
(layers/transformer.py:488-497). What differs is everything underneath:
  * activations stay [b, s, h] token-major — no [s, b, h] transposes (modeling_llama.py:201,222), no q/k/v repacking;
  * all parameters are views into one flat bf16 buffer, gradients go straight into the parallel flat grad buffer;
  * the whole network is ONE autograd node (fsb200/models/base.py): forward runs the hand-scheduled kernel sequence and keeps
    the activations it needs; `loss.backward()` runs the matching hand-written backward (dgrad / wgrad GEMMs, fused
    attention backward, norm backward with the residual-gradient add fused in).
The causal mask is implicit (flash path semantics, transformer.py:441-448: `attention_mask` is not applied; identical to
the `global` path when the mask is all ones — SURVEY.md Appendix B).
Packed rows (several documents per row, fsb200/packing.py) pass `segment_ids`: attention then stays causal inside each
segment and never crosses one (the varlen `cu_seqlens` semantics of the flash path, transformer.py:434-448).
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
from .base import FlatModel, _Holder, flat_ids, packed_segments
from .layers import WQ, Fp8Linear, GatedMLP, Linear, QuantizedLinear, quantized_unsupported


def llama_ff_dim(hidden_size, multiple_of=256):
    ff = int(2 * hidden_size * 4 / 3)  # layers/transformer.py:589-590
    return multiple_of * ((ff + multiple_of - 1) // multiple_of)


def _init_normal_(t, std, gen):
    t.copy_(torch.empty(t.shape, dtype=torch.float32).normal_(0.0, std, generator=gen).to(t.dtype))


# weight format -> (quantiser, q / s layout): the table layers.QuantizedLinear reads, shared with GPT-2
_WQ = WQ

_Layer = namedtuple("_Layer", "qkv dense mlp")   # a layer's projections: query_key_value, dense, the gated MLP (w1 | w3, w2)


def _quantized_unsupported(fmt, what):
    return quantized_unsupported("LlamaForCausalLM", fmt, what)


class LlamaForCausalLM(FlatModel):
    supports_gradient_checkpointing = True

    def __init__(self, config, device=None, world_size=None, seed=0, tp_group=None, load_in_8bit=False, load_in_4bit=False,
                 fp8=False, gradient_checkpointing=False):
        """tp_group: the tensor-model-parallel process group (mpu.get_model_parallel_group()) or None. With t = its size > 1
        this rank holds the shard the reference's `part_{rank}` checkpoints hold (utils/llama_convert/convert_fs_llama_tp.py
        :143-181): heads / ff columns / vocabulary rows split t ways (ColumnParallelLinear mpu/layers.py:261-360 for QKV,
        w1, w3 and the LM head; RowParallelLinear :363-470 for dense and w2; VocabParallelEmbedding :62-130), norms replicated.
        `world_size` is then the DATA-parallel size (ranks that share a tensor-parallel rank).

        load_in_8bit: an inference-only model (`from_pretrained(..., load_in_8bit=True)`, examples/ziya_inference/
        hf_quantizatin_inference.py:20-22). Each layer's four projections (query_key_value, dense, w1 | w3, w2) are held as
        int8 q [n, k] + fp32 per-row scales s [n] and run through the W8A16 GEMM; the embedding, the norm scales and the LM
        head stay bf16 in flat buffers without a gradient buffer. Training, tensor parallelism and save_pretrained raise.

        load_in_4bit: the same with int4 projections (examples/ziya_inference/hf_quantizatin_inference.py:3,16): q packed two
        per byte [n / 2, k] + bf16 scales [n, k / 128], one per row and group of 128 k, run through the W4A16 GEMM.
        hidden_size and the MLP width must then be multiples of 128.

        fp8: train in FP8 (include/fsb200.h, fsb_gemm_fp8). Each layer's four projections (query_key_value, dense, w1 | w3,
        w2) run as Fp8Linear: e4m3 activations and weights, e5m2 gradients, per-tensor power-of-two scales computed from each
        tensor's amax just before its cast, fp32 accumulation. The embedding, the LM head, the norms and attention stay bf16,
        as do the master weights, the gradients and the optimizer state, so checkpoints and resume are unchanged. The training
        and no-grad (validation) forwards run FP8; `generate` runs the bf16 layer stack on the same weights. Results differ from
        bf16 by design. hidden_size, the MLP width and the tokens per micro-batch must be multiples of 16 (checked at the first
        forward); tensor parallelism and load_in_8bit / load_in_4bit are refused.

        gradient_checkpointing: activation recompute (also `gradient_checkpointing_enable()` / `_disable()`). The training
        forward keeps only the residual stream entering each layer; the backward re-runs each layer's forward from it, up to
        what the layer's backward reads (not the w2 GEMM), just before that layer's backward. The gradients are bit-identical
        to those without it, at about one more forward of the layers; the activation memory of the layers drops from one
        saved set per layer to one bf16 [tokens, hidden] tensor per layer plus one saved set. The no-grad forward and
        `generate` keep nothing either way and are unaffected; so are int8 / int4 models, which do not train."""
        super().__init__(config)
        self.gradient_checkpointing = bool(gradient_checkpointing)
        import torch.distributed as dist
        if load_in_8bit and load_in_4bit:
            raise ValueError("fsb200 LlamaForCausalLM: load_in_8bit and load_in_4bit are mutually exclusive; pass one")
        if fp8 and (load_in_8bit or load_in_4bit):
            raise ValueError("fsb200 LlamaForCausalLM: fp8=True trains in FP8; it cannot be combined with load_in_8bit or "
                             "load_in_4bit (inference-only weight formats)")
        self.fp8 = bool(fp8)
        # the layer projections' weight format; load_in_8bit / load_in_4bit are kept as the public flags
        self.weight_format = "int8" if load_in_8bit else "int4" if load_in_4bit else "bf16"
        self.load_in_8bit = self.weight_format == "int8"
        self.load_in_4bit = self.weight_format == "int4"
        quantized = self.weight_format != "bf16"
        self.tp_group = tp_group
        self.tp = dist.get_world_size(tp_group) if tp_group is not None else 1
        self.tp_rank = dist.get_rank(tp_group) if tp_group is not None else 0
        if quantized and self.tp > 1:
            raise _quantized_unsupported(self.weight_format, "tensor parallelism")
        if self.fp8 and self.tp > 1:
            raise NotImplementedError("fsb200 LlamaForCausalLM: fp8=True under tensor parallelism is not implemented (the "
                                      "per-tensor scales of the shards differ from one GPU's)")
        h, V, nl, nh = config.hidden_size, config.vocab_size, config.num_hidden_layers, config.num_attention_heads
        self.h, self.V, self.nl, self.nh = h, V, nl, nh
        self.hn = h // nh
        self.ff = llama_ff_dim(h, getattr(config, "llama_mlp_multiple_of", 256))
        self.eps = getattr(config, "rms_norm_epsilon", 1e-6)
        if self.hn not in (64, 128):
            raise RuntimeError(f"fsb200: head dim {self.hn} unsupported (64 or 128)")
        if V % 8 or h % 8:
            raise RuntimeError("fsb200: vocab_size and hidden_size must be multiples of 8")
        t = self.tp
        if nh % t or self.ff % (8 * t) or V % (8 * t):
            raise RuntimeError(f"fsb200: heads {nh}, ff {self.ff} and vocab {V} must split evenly over tensor-parallel size {t}")
        if self.load_in_4bit and (h % 128 or self.ff % 128):
            raise RuntimeError(f"fsb200: an int4 model needs hidden_size ({h}) and the MLP width ({self.ff}) to be multiples "
                               "of 128 (the scale group)")
        # local (per tensor-parallel rank) extents
        self.nh_l, self.ff_l, self.V_l = nh // t, self.ff // t, V // t
        self.h_l = self.nh_l * self.hn
        self.tp_replicated_buckets = ("no_decay",)   # norms: identical on every tensor-parallel rank (counted once in the norm)

        spec = FlatSpec()
        spec.add("llama.embed_in.word_embeddings.weight", (self.V_l, h), "embed_in")
        for i in range(nl):
            p, bk = f"llama.layers.{i}.", f"layer{i}"
            spec.add(p + "input_layernorm.scale", (h,), bk)          # *.scale names match 'layernorm.' -> no-decay bucket
            if not quantized:
                spec.add(p + "attention.query_key_value.weight", (3 * self.h_l, h), bk)
                spec.add(p + "attention.dense.weight", (h, self.h_l), bk)
            spec.add(p + "post_attention_layernorm.scale", (h,), bk)
            if not quantized:
                spec.add(p + "mlp.w1.weight", (self.ff_l, h), bk)   # w1 | w3 adjacent: one [2ff, h] GEMM operand
                spec.add(p + "mlp.w3.weight", (self.ff_l, h), bk)
                spec.add(p + "mlp.w2.weight", (h, self.ff_l), bk)
        spec.add("llama.final_layer_norm.scale", (h,), "head")
        spec.add("embed_out.final_linear.weight", (self.V_l, h), "head")
        self._bind_flat(spec, device, world_size, tp=self.tp, grads=not quantized)
        if quantized:   # w1 | w3 is one [2ff, h] operand as in the bf16 layout
            qlin = lambda n, k: QuantizedLinear(self.weight_format, n, k, self.flat.params.device, model="LlamaForCausalLM")
            self._proj = [_Layer(qlin(3 * h, h), qlin(h, h), GatedMLP(qlin(2 * self.ff, h), qlin(h, self.ff), L.ACT_SILU))
                          for _ in range(nl)]
        else:
            self._proj = [_Layer(Linear.of(lyr.attention.query_key_value.weight), Linear.of(lyr.attention.dense.weight),
                                 GatedMLP(Linear.span(self.flat, f"llama.layers.{i}.mlp.w1.weight", 2 * self.ff_l, h),
                                          Linear.of(lyr.mlp.w2.weight), L.ACT_SILU))
                          for i, lyr in enumerate(self.llama.layers)]
        self._proj_bf16 = self._proj   # what generate runs
        if self.fp8:
            self._proj = [_Layer(Fp8Linear(lp.qkv), Fp8Linear(lp.dense),
                                 GatedMLP(Fp8Linear(lp.mlp.wi), Fp8Linear(lp.mlp.wo), L.ACT_SILU))
                          for lp in self._proj_bf16]
        self._head = Linear.of(self.embed_out.final_linear.weight)

        # RoPE tables exactly as RotaryEmbedding builds them (layers/positional_embeddings.py:38-52), fp32; inv_freq is also a
        # buffer of every layer in the reference's module tree (modeling_llama.py:97-127), hence in its state dict
        self._inv_freq = 1.0 / (getattr(config, "rotary_emb_base", 10000) ** (torch.arange(0, self.hn, 2).float() / self.hn))
        for lyr in self.llama.layers:
            if "attention" not in lyr._modules:    # int8 / int4: the projections live outside the flat buffers
                lyr.attention = _Holder()
            lyr.attention.rotary_emb = _Holder()
            lyr.attention.rotary_emb.register_buffer("inv_freq", self._inv_freq.clone().to(self.flat.params.device))
        self._rope_rows = 0
        self._ensure_rope(getattr(config, "max_position_embeddings", 2048))
        self.reset_parameters(seed)

    def _ensure_rope(self, n):
        """cos/sin tables with at least n rows. RotaryEmbedding regrows its cache when a longer sequence arrives
        (positional_embeddings.py:54-68); fsb_rope_inplace never reads past the table (rows beyond it become NaN)."""
        if n <= self._rope_rows:
            return
        dev = self.flat.params.device
        t = torch.arange(n, dtype=self._inv_freq.dtype)
        freqs = torch.einsum("i,j->ij", t, self._inv_freq)
        self._cos = freqs.cos().contiguous().to(dev)
        self._sin = freqs.sin().contiguous().to(dev)
        self._rope_rows = n

    # ---- init (layers/init_functions.py:121-142: small_init std sqrt(2/(5h)); wang_init std 2/(L*sqrt(h))) -------------
    @torch.no_grad()
    def reset_parameters(self, seed=0):
        h, nl = self.h, self.nl
        small = math.sqrt(2.0 / (5.0 * h))
        wang = 2.0 / (nl * math.sqrt(h))
        big = self.flat.total > 300_000_000  # billions of CPU randn take minutes: draw on the device instead
        gen = torch.Generator(device=self.flat.params.device if big else "cpu").manual_seed(seed + 7919 * self.tp_rank)
        for name, prm in self.named_parameters():
            if name.endswith(".scale"):
                prm.fill_(1.0)
                continue
            std = wang if (name.endswith("dense.weight") or name.endswith("w2.weight")) else small
            if big:
                prm.normal_(0.0, std, generator=gen)
            else:
                _init_normal_(prm.data, std, gen)
        if self.weight_format != "bf16":   # each quantised matrix: drawn in bf16 on the device and quantised, one at a time
            dgen = torch.Generator(device=self.flat.params.device).manual_seed(seed + 104729)
            for wq in self._wq:
                for key, (q, s) in wq.items():
                    tmp = torch.empty(self._weight_shape(q, s), dtype=torch.bfloat16, device=q.device)
                    tmp.normal_(0.0, wang if key in ("dense", "w2") else small, generator=dgen)
                    _WQ[self.weight_format][0](tmp, q, s)
                    del tmp

    # ---- int8 / int4 (load_in_8bit / load_in_4bit; loading and get_memory_footprint: FlatModel) -------------------------
    @property
    def _wq(self):
        """Per layer {projection: (q, s)} of an int8 / int4 model (w13: the w1 | w3 operand), as `_w8` / `_w4` name them."""
        return [{"qkv": (lp.qkv.q, lp.qkv.s), "dense": (lp.dense.q, lp.dense.s), "w13": (lp.mlp.wi.q, lp.mlp.wi.s),
                 "w2": (lp.mlp.wo.q, lp.mlp.wo.s)} for lp in self._proj]
    _w8 = _w4 = _wq

    @property
    def _w13(self):
        """Per layer the [2ff, h] w1 | w3 operand of a bf16 model."""
        return [lp.mlp.wi.weight for lp in self._proj_bf16]

    def _wq_targets(self):
        """{state-dict key: (q, s) it quantises into} of every quantised projection. w1 and w3 are the upper and lower
        halves of the w1 | w3 projection, in q (whose int4 rows pack two weight rows) as in s."""
        out = {}
        for i, (qkv, dense, mlp) in enumerate(self._proj):
            p = f"llama.layers.{i}."
            (q1, q3), (s1, s3) = mlp.wi.q.chunk(2), mlp.wi.s.chunk(2)
            out.update({p + "attention.query_key_value.weight": (qkv.q, qkv.s), p + "attention.dense.weight": (dense.q, dense.s),
                        p + "mlp.w1.weight": (q1, s1), p + "mlp.w3.weight": (q3, s3), p + "mlp.w2.weight": (mlp.wo.q, mlp.wo.s)})
        return out

    def save_pretrained(self, path, **kw):
        if self.weight_format != "bf16":
            raise _quantized_unsupported(self.weight_format, f"save_pretrained ({self.weight_format} export)")
        return super().save_pretrained(path, **kw)

    # ---- forward ----------------------------------------------------------------------------------------------------
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, labels=None, return_logits=False,
                segment_ids=None, **_):
        """segment_ids: optional integer [B, S] (host or device) for packed rows; a segment is a maximal run of equal
        consecutive values in a row. Every layer's attention is then causal inside each segment only, and the label of each
        segment's first token is ignored (its prediction would cross a document boundary). Pass per-segment position_ids
        (fsb200/packing.py emits them). None: one causal sequence per row, as before."""
        B, S = input_ids.shape
        dev = self.flat.params.device
        ids = flat_ids(input_ids, dev)
        if position_ids is None:
            self._ensure_rope(S)
            pos = torch.arange(S, device=dev, dtype=torch.int64).repeat(B)
        else:
            if not position_ids.is_cuda:   # host tensor (the collators emit CPU batches): exact bound, no device sync
                lo, hi = int(position_ids.min()), int(position_ids.max())
                if lo < 0:
                    raise ValueError(f"position_ids must be non-negative, got {lo}")
                self._ensure_rope(hi + 1)
            pos = position_ids.to(device=dev, dtype=torch.int64).expand(B, S).contiguous().view(-1)
            if position_ids.is_cuda:       # device tensor: asynchronous device-side check against the table size
                self._ensure_rope(S)
                torch._assert_async(((pos >= 0) & (pos < self._rope_rows)).all(),
                                    "fsb200 LlamaForCausalLM: position_ids outside [0, rope table rows); pass them on the "
                                    "host or raise config.max_position_embeddings")
        if self.fp8 and (self.h % 16 or self.ff % 16 or (B * S) % 16):
            raise ValueError(f"fsb200 LlamaForCausalLM(fp8=True): hidden_size ({self.h}), the MLP width ({self.ff}) and the "
                             f"tokens per micro-batch (batch {B} x sequence {S}) must be multiples of 16 (the FP8 GEMM "
                             "operands need 16-byte rows in both layouts)")
        lab = flat_ids(labels, dev)
        if self.weight_format != "bf16" and lab is not None and torch.is_grad_enabled():
            raise _quantized_unsupported(self.weight_format, "a training forward (labels under grad mode)")
        seg = ()
        if segment_ids is not None:
            bounds, lab = packed_segments(segment_ids, lab, B, S, dev)
            seg = (bounds,)
        loss, logits = self._step_or_forward(lab is not None, return_logits, ids, pos, lab, B, S, *seg)
        return SimpleNamespace(loss=loss, logits=None if logits is None else logits.view(B, S, self.V),
                               past_key_values=None, hidden_states=None, attentions=None)

    def _attend(self, seg):
        """The training attention over a layer's q|k|v view (see _stack): causal, or inside the segments of packed rows
        when seg holds their (seg_start, seg_end) bounds (ops.segment_bounds)."""
        scale = 1.0 / math.sqrt(self.hn)
        if seg is None:
            return lambda i, q5: ops.sdpa_fwd(q5[:, :, :, 0], q5[:, :, :, 1], q5[:, :, :, 2], scale, True)
        return lambda i, q5: ops.sdpa_segments_fwd(q5[:, :, :, 0], q5[:, :, :, 1], q5[:, :, :, 2], scale, *seg)

    def _forward_impl(self, ids, pos, lab, B, S, seg=None, *, save, want_logits):
        """seg: None or the (seg_start, seg_end) bounds of packed rows (ops.segment_bounds)."""
        acts = [] if save else None
        recompute = save and self.gradient_checkpointing   # fixed for this step: the backward reads it from ctx
        hf, rstdf, xf = self._stack(ids, pos, B, S, self._attend(seg), acts, checkpoints=recompute)
        logits = self._head(hf)
        logits = self._tp_gather_columns(logits)   # ParallelLinear(parallel_output=False): full-vocabulary logits on every rank
        loss = None
        ctx = None
        if lab is not None:
            keep = logits.clone() if (want_logits and save) else None
            loss, dlogits, _ = ops.softmax_xent(logits, lab, S, shift=1, grad_scale=self.loss_scale,
                                                dlogits="inplace" if save else None)
            if save:
                ctx = (acts, recompute, hf, rstdf, xf, dlogits, ids, pos, B, S, seg)
                logits = keep
        return loss, (logits if want_logits else None), ctx

    def _stack(self, ids, pos, B, S, attend, acts=None, proj=None, checkpoints=False):
        """Embedding, the layers and the final norm over ids [B * S] -> (hidden states, their rstd, residual stream).
        attend(i, q5) is layer i's attention over the per-head interleaved q|k|v view [B, S, heads, 3, head_dim] (rotary
        embedding applied) -> (out, lse); `acts`, when given, collects what the backward reads: per layer the saved tuple of
        `_layer`, or with `checkpoints` only the residual stream entering the layer, from which the backward recomputes the
        rest. proj: the layers' projections (default self._proj)."""
        save = acts is not None and not checkpoints
        self._need("no_decay"); self._need("embed_in")
        ids_l, emb_keep = self._local_ids(ids)
        x = ops.embedding_fwd(ids_l, self.llama.embed_in.word_embeddings.weight.data)
        if emb_keep is not None:      # VocabParallelEmbedding.forward (mpu/layers.py:104-130): foreign rows are zero, then all-reduce
            x.mul_(emb_keep)
            self._tp_all_reduce(x)
        m = None
        for i, lp in enumerate(self._proj if proj is None else proj):
            xs, x, m, saved = self._layer(i, lp, x, m, pos, B, S, attend, save)
            if acts is not None:
                acts.append(xs if checkpoints else saved)
            del xs, saved
        self._need("head")
        return ops.rmsnorm_fwd(m, self.llama.final_layer_norm.scale.data, self.eps, residual=x)

    def _layer(self, i, lp, x, m, pos, B, S, attend, save, out=True):
        """Layer i with projections lp over the residual stream x plus m, the previous layer's MLP output (None for the
        first layer, or when x already is that sum) -> (xs, x1, m', saved): xs = x + m, the layer's input; x1 = xs + the
        attention output; m' the MLP output; saved (with `save`) what the backward reads. Its temporaries are freed on
        return, before the next layer allocates its own (the peak of a long prompt's prefill). out=False (with save): stop
        before the w2 GEMM and its all-reduce, for a recompute whose m' nothing reads; m' is then None."""
        nh, hn, hl = self.nh_l, self.hn, self.h_l      # LOCAL heads under tensor parallelism
        lyr = self.llama.layers[i]
        self._need(f"layer{i}")
        # without a residual the kernel returns x itself; with one, the bf16-rounded sum, over which it takes the row
        # statistics: a recompute from the stored sum reproduces h1 and rstd1 bit for bit (csrc/norm.cu, norm_fwd_kernel)
        h1, rstd1, x = ops.rmsnorm_fwd(x if m is None else m, lyr.input_layernorm.scale.data, self.eps,
                                       residual=None if m is None else x)
        qkv, h1s = lp.qkv.forward(h1, save)   # h1s: what the QKV weight gradient reads of h1
        ops.rope_inplace(qkv, self._cos, self._sin, pos, nh, hn, 3 * hl, 3 * hn, offset=0)
        ops.rope_inplace(qkv, self._cos, self._sin, pos, nh, hn, 3 * hl, 3 * hn, offset=hn)
        o, lse = attend(i, qkv.view(B, S, nh, 3, hn))
        a, os_ = lp.dense.forward(o.view(B * S, hl), save)
        self._tp_all_reduce(a)        # RowParallelLinear: partial sums over the head shards (mpu/layers.py:451-470)
        h2, rstd2, x1 = ops.rmsnorm_fwd(a, lyr.post_attention_layernorm.scale.data, self.eps, residual=x)
        m, ms = lp.mlp(h2, save, out=out)
        if out:
            self._tp_all_reduce(m)    # RowParallelLinear (w2)
        return x, x1, m, ((x, rstd1, h1s, qkv, o, os_, lse, x1, rstd2, ms) if save else None)

    # ---- KV-cache inference (SURVEY.md §8f rank 4) -----------------------------------------------------------------------
    # The reference decodes through HF's GenerationMixin: `prepare_inputs_for_generation` (modeling_llama.py:353-377) feeds the
    # last token with position_ids = cumsum(attention_mask) - 1, every layer concatenates the new key / value onto `layer_past`
    # (layers/transformer.py:529-537) and `llama_generate.generate` (examples/ziya_llama/llama_generate.py:16-39) left-pads the
    # prompts. Here the cache is a pre-allocated [batch, max_length, heads, head_dim] pair per layer; prefill and decode steps
    # run the training layer stack (`_stack`), a decode step with one query row per sequence, the unused tail of the cache (and
    # the left padding) hidden by the key mask. Padded keys ARE masked (the reference's `global` attention path; its flash
    # path ignores the mask). The decode step keeps its position on the device (kv_len, the position ids; the new keys /
    # values land at slot kv_len - 1 through ops.kv_append) and runs as one CUDA-graph replay (fsb200/decode_graph.py).
    @property
    def device(self):
        return self.flat.params.device

    @torch.no_grad()
    def generate(self, input_ids, attention_mask=None, max_length=None, max_new_tokens=None, do_sample=False,
                 temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0, pad_token_id=None, eos_token_id=None,
                 generator=None, num_return_sequences=1, **_):
        """Greedy / sampling decode with a KV cache; the keyword surface `llama_generate.generate` passes to HF's
        `model.generate` (do_sample, top_p, top_k, max_length, repetition_penalty, temperature, pad_token_id, eos_token_id),
        plus num_return_sequences (sampling only; each prompt repeated in place, HF's `_expand_inputs_for_generation`), which
        hf_quantizatin_inference.py passes. Prompts are LEFT-padded (attention_mask 0 on the pads). Returns
        [batch * num_return_sequences, <= max_length] token ids, prompt included, finished rows filled with pad_token_id —
        HF's GenerationMixin conventions, selected by fsb200/generation.py."""
        if self.tp > 1:
            raise NotImplementedError("fsb200: KV-cache decoding under tensor parallelism is not implemented")
        nrs = int(num_return_sequences or 1)
        if nrs > 1 and not do_sample:
            raise ValueError("fsb200 generate: greedy search with `num_return_sequences` > 1 returns identical rows; "
                             "set do_sample=True")
        dev = self.device
        ids = input_ids.to(device=dev, dtype=torch.int64)
        B, S0 = ids.shape
        mask = torch.ones((B, S0), dtype=torch.uint8, device=dev) if attention_mask is None else \
            attention_mask.to(device=dev).to(torch.uint8)
        if nrs > 1:
            ids, mask = ids.repeat_interleave(nrs, 0), mask.repeat_interleave(nrs, 0)
            B *= nrs
        if max_length is None:
            max_length = S0 + (max_new_tokens if max_new_tokens is not None else 20)
        if max_length <= S0:
            return ids
        c = SimpleNamespace(num_beams=1, do_sample=do_sample, temperature=temperature, top_k=top_k, top_p=top_p,
                            repetition_penalty=repetition_penalty, max_length=max_length, output_scores=False,
                            return_dict=False, eos=None if eos_token_id is None else [eos_token_id],
                            pad=pad_token_id if pad_token_id is not None else (eos_token_id if eos_token_id is not None else 0))
        Lmax = (max_length + 63) // 64 * 64
        self._ensure_rope(max_length)
        scale = 1.0 / math.sqrt(self.hn)
        cache = [(torch.zeros((B, Lmax, self.nh, self.hn), dtype=torch.bfloat16, device=dev),
                  torch.zeros((B, Lmax, self.nh, self.hn), dtype=torch.bfloat16, device=dev)) for _ in range(self.nl)]
        kv_mask = torch.zeros((B, Lmax), dtype=torch.uint8, device=dev)
        kv_mask[:, :S0] = mask
        count = mask.long().sum(-1)                                             # real tokens so far = next position id
        kv_len = torch.full((1,), S0, dtype=torch.int32, device=dev)

        def prefill():
            # position_ids = cumsum(mask) - 1, pads -> 1 (prepare_inputs_for_generation, modeling_llama.py:360-366)
            pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
            pre = None if bool(mask.all()) else kv_mask[:, :S0].contiguous()

            def attend(i, q5):   # attend inside the prompt (causal + left-padding mask)
                kc, vc = cache[i]
                kc[:, :S0].copy_(q5[:, :, :, 1])
                vc[:, :S0].copy_(q5[:, :, :, 2])
                return ops.sdpa_fwd(q5[:, :, :, 0], q5[:, :, :, 1], q5[:, :, :, 2], scale, True, kv_mask=pre)
            return self._last_logits(ids.reshape(-1), pos.reshape(-1).contiguous(), B, S0, attend)

        def body(tok, *_):
            kv_len.add_(1)

            def attend(i, q5):   # one query row per sequence against the whole cache; unwritten slots are masked
                kc, vc = cache[i]
                ops.kv_append(q5[:, 0, :, 1], q5[:, 0, :, 2], kc, vc, kv_len, kv_mask=kv_mask if i == 0 else None)
                return ops.sdpa_fwd(q5[:, :, :, 0], kc, vc, scale, False, kv_mask=kv_mask)
            out = self._last_logits(tok, count, B, 1, attend)
            count.add_(1)
            return out

        return generation.run(DecodeGraphs(self, B, [cache], body, prefill), ids, c, generator)

    def _last_logits(self, ids, pos, B, S, attend):
        """fp32 logits [B, V] of the last position of every sequence."""
        hf, _, _ = self._stack(ids, pos, B, S, attend, proj=self._proj_bf16)   # fp8=True: generate runs in bf16
        last = hf.view(B, S, self.h)[:, -1].contiguous()                       # [B, h]
        rows = max(8, B)                                                        # the GEMM wants >= 8 aligned rows
        if rows != B:
            pad = torch.zeros((rows, self.h), dtype=last.dtype, device=last.device)
            pad[:B] = last
            last = pad
        return self._head(last)[:B].float()

    # ---- backward ---------------------------------------------------------------------------------------------------
    def _backward_impl(self, ctx, gloss):
        acts, recompute, hf, rstdf, xf, dlogits, ids, pos, B, S, seg = ctx
        nh, hn, hl = self.nh_l, self.hn, self.h_l
        T = B * S
        acc = self.accumulate_grads
        self._begin_backward()
        if gloss is not None:
            ops.scale_inplace(dlogits, gloss)  # upstream scalar; the kernel exits immediately when it is 1.0
        if self.tp > 1:   # this rank's vocabulary columns of dlogits (a strided view: the GEMMs take the row stride)
            dlogits = dlogits[:, self.tp_rank * self.V_l:(self.tp_rank + 1) * self.V_l]
        dhf = self._head.backward(dlogits, hf, acc)
        self._tp_all_reduce(dhf)          # backward of copy_to_model_parallel_region (mpu/mappings.py): sum the partial dgrads
        del dlogits
        self._done("head")
        fscale = self.llama.final_layer_norm.scale
        dx = ops.rmsnorm_bwd(dhf, xf, fscale.data, rstdf, fscale.main_grad, accumulate=acc)
        attend = self._attend(seg) if recompute else None
        for i in reversed(range(self.nl)):
            lyr, lp = self.llama.layers[i], self._proj[i]
            if recompute:   # layer i's forward again from its input, up to what its backward reads; the kernels are
                # deterministic, so these are the bits the forward computed. The parameters are already gathered (_need is a
                # no-op) and nothing here advances state (LLaMA has no dropout)
                x, rstd1, h1s, qkv, o, os_, lse, x1, rstd2, ms = self._layer(i, lp, acts[i], None, pos, B, S, attend,
                                                                             save=True, out=False)[3]
            else:
                x, rstd1, h1s, qkv, o, os_, lse, x1, rstd2, ms = acts[i]
            acts[i] = None
            # x_next = x1 + m  ->  dm = dx, residual gradient into x1 = dx
            dh2 = lp.mlp.backward(dx, ms, acc)
            self._tp_all_reduce(dh2)      # column-parallel w1|w3: dgrad partial sums
            s2 = lyr.post_attention_layernorm.scale
            dx1 = ops.rmsnorm_bwd(dh2, x1, s2.data, rstd2, s2.main_grad, accumulate=acc, dres=dx)
            # x1 = x + a  ->  da = dx1
            do = lp.dense.backward(dx1, os_, acc)
            dqkv = torch.empty_like(qkv)
            q5, d5 = qkv.view(B, S, nh, 3, hn), dqkv.view(B, S, nh, 3, hn)
            if seg is None:
                ops.sdpa_bwd(q5[:, :, :, 0], q5[:, :, :, 1], q5[:, :, :, 2], o, do.view(B, S, nh, hn), lse,
                             1.0 / math.sqrt(hn), True, d5[:, :, :, 0], d5[:, :, :, 1], d5[:, :, :, 2])
            else:
                ops.sdpa_segments_bwd(q5[:, :, :, 0], q5[:, :, :, 1], q5[:, :, :, 2], o, do.view(B, S, nh, hn), lse,
                                      1.0 / math.sqrt(hn), *seg, d5[:, :, :, 0], d5[:, :, :, 1], d5[:, :, :, 2])
            ops.rope_inplace(dqkv, self._cos, self._sin, pos, nh, hn, 3 * hl, 3 * hn, backward=True, offset=0)
            ops.rope_inplace(dqkv, self._cos, self._sin, pos, nh, hn, 3 * hl, 3 * hn, backward=True, offset=hn)
            dh1 = lp.qkv.backward(dqkv, h1s, acc)
            self._tp_all_reduce(dh1)      # column-parallel QKV: dgrad partial sums
            s1 = lyr.input_layernorm.scale
            dx = ops.rmsnorm_bwd(dh1, x, s1.data, rstd1, s1.main_grad, accumulate=acc, dres=dx1)
            # free this layer's activations and transients before the next layer's recompute allocates its own
            del x, rstd1, h1s, qkv, o, os_, lse, x1, rstd2, ms, dh2, dx1, do, dqkv, q5, d5, dh1
            self._done(f"layer{i}")
        W_in = self.llama.embed_in.word_embeddings.weight
        if not acc:
            W_in.main_grad.zero_()
        ids_l, emb_keep = self._local_ids(ids)
        if emb_keep is not None:
            dx = dx * emb_keep            # rows of foreign vocabulary shards contribute nothing here
        ops.embedding_bwd(ids_l, dx, W_in.main_grad)
        self._done("embed_in")
        self._done("no_decay")

    # ---- tensor-parallel exchanges (fengshen/models/megatron/mpu/mappings.py:29-192), NCCL on the compute stream -------------
    def _tp_all_reduce(self, t):
        if self.tp > 1:
            import torch.distributed as dist
            dist.all_reduce(t, group=self.tp_group)

    def _tp_gather_columns(self, t):
        """[rows, n/tp] on every rank -> [rows, n] (gather_from_model_parallel_region, last-dimension concatenation)."""
        if self.tp == 1:
            return t
        import torch.distributed as dist
        buf = torch.empty((self.tp,) + tuple(t.shape), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(buf, t.contiguous(), group=self.tp_group)
        return buf.permute(1, 0, 2).reshape(t.shape[0], self.tp * t.shape[1])

    def _local_ids(self, ids):
        """VocabParallelEmbedding index arithmetic (mpu/layers.py:104-121): ids of this rank's vocabulary range re-based to 0,
        foreign ids clamped (their rows are zeroed by the returned [rows, 1] bf16 mask). (ids, None) without tensor parallelism."""
        if self.tp == 1:
            return ids, None
        lo = self.tp_rank * self.V_l
        mine = (ids >= lo) & (ids < lo + self.V_l)
        return torch.where(mine, ids - lo, torch.zeros_like(ids)), mine.to(torch.bfloat16)[:, None]
