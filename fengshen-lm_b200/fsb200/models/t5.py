"""Randeng-T5 / mT5 on the fsb200 kernels — drop-in for `transformers.MT5ForConditionalGeneration` as the reference uses it
(fengshen/examples/pretrain_t5/pretrain_t5.py:57-59 builds it from an MT5Config; training_step :81-87 is
`self.model(input_ids=..., labels=...)`). BASELINE config 5.

The arithmetic restated here lives in 3P `transformers` (mt5/modeling_mt5.py; SURVEY.md Appendix C):
  * pre-RMSNorm sub-layers `x + f(norm(x))` (MT5LayerNorm :47-70 == the in-tree RMSNorm formula), final RMSNorm per stack;
  * attention WITHOUT the 1/sqrt(d) scale (:300) plus an additive relative-position bias `table[bucket(k - q), h]` (:181-235)
    owned by the FIRST self-attention layer of each stack and reused by every layer of that stack; fp32 softmax (:323);
    decoder cross-attention over the encoder's final hidden states with zero bias and the encoder padding mask;
  * gated-GeLU FFN `wo(gelu_new(wi_0 x) * wi_1 x)` (:96-123); nothing has a bias vector;
  * one shared token embedding for both stacks, `decoder_input_ids = shift_right(labels)` (start id = pad id, -100 -> pad;
    :592, :1123-1125), untied `lm_head` without the d^-0.5 rescale (:1143), CrossEntropyLoss(ignore_index=-100) over every
    decoder position (:1147-1150).
State-dict keys follow HF (`shared.weight`, `encoder.block.N.layer.0.SelfAttention.q.weight`, ...).

Kernel mapping: q|k|v (self), k|v (cross) and wi_0|wi_1 are adjacent in the flat buffer, so each is ONE GEMM; the bias reaches
the attention kernels as one fp32 vector per head over the offset k - q (`t5_bias.rel_bias_vector`), and its gradient comes
back the same way (deterministic diagonal sums inside the dQ kernel, csrc/attention_bwd.cu) and is scattered onto the
[buckets, heads] table on the host side of the step (`t5_bias.scatter_rel_grad`). The encoder-output gradient is the sum of
every decoder layer's K|V-projection dgrad: accumulated in fp32 by the GEMM epilogue, rounded to bf16 once.
Dropout (`dropout_rate`, in [0, 1)) applies in training mode (`model.training`, also under no_grad) at HF's sites, in HF's call
order: the embeddings of each stack, the attention probabilities, the attention-output and FFN-output branches before their
residual add, the gated activation before `wo`, and each stack's final-norm output. Seed, stream counter and eval mode as in
fsb200/models/base.py. A branch is dropped by the RMSNorm that adds it to the residual stream, the gated activation by its
kernel, the attention probabilities inside the attention kernels (the decoder's self-attention with the causal flag, at every
rate), the embeddings and final-norm outputs by the standalone dropout kernel. `generate` in training mode with a non-zero rate
is rejected (HF would drop).
Packed rows (several samples per row, fsb200/packing.py pack_seq2seq_batch) pass `segment_ids` and `decoder_segment_ids`:
the encoder's self-attention is then bidirectional inside each encoder segment, the decoder's causal inside each decoder
segment, both with the relative-position bias (it depends on k - q only, so a segment sees the scores it would see alone),
and each decoder segment's cross-attention reads only the encoder segment with the same id. The dropout sites are unchanged.
fp8=True trains the layer projections in FP8 (layers.Fp8Linear, include/fsb200.h fsb_gemm_fp8): the encoder's q|k|v, o,
wi_0|wi_1 and wo, and the decoder's q|k|v, o, cross q, cross k|v, cross o, wi_0|wi_1 and wo. e4m3 activations and weights, e5m2
gradients, per-tensor power-of-two scales from each tensor's amax just before its cast, fp32 accumulation. The encoder output,
which every decoder layer's cross k|v projection reads, is quantised once per forward and its codes shared; those projections'
data gradients (bf16, the FP8 GEMM's output) are summed in fp32 (ops.accumulate), as the bf16 GEMM sums them in bf16
training. The shared embedding, the LM head, the RMSNorms, the relative-bias attention and its bias gradient, the gated-GeLU
kernel and the loss stay bf16, as do the master weights, the gradients and the optimizer state; `generate` runs the bf16
projections.
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
from . import t5_bias as TB
from .base import FlatModel, _Holder, cross_segment_bounds, flat_ids, key_mask, refuse_key_padding
from .layers import Fp8Linear, GatedMLP, Linear, apply_dropout, residual_norm_bwd

_Enc = namedtuple("_Enc", "qkv o mlp")             # a layer's projections: self-attention q|k|v and o, the gated FFN
_Dec = namedtuple("_Dec", "qkv o cq ckv co mlp")   # ... and between them cross-attention q, k|v and o


def shift_right(labels, start_id, pad_id, seg_start=None):
    """MT5 _shift_right (:592): decoder_input_ids = [start] + labels[:-1], with -100 replaced by the pad id. seg_start
    (int32 [B, S], packed rows, ops.segment_bounds of the decoder segment ids): every decoder segment starts from the start
    id instead, so no sample sees the previous one's last label. Torch ops only (any device)."""
    dec = labels.new_zeros(labels.shape)
    dec[:, 1:] = labels[:, :-1]
    dec[:, 0] = start_id
    dec = dec.masked_fill(dec == -100, pad_id)
    if seg_start is not None:
        pos = torch.arange(labels.shape[1], dtype=seg_start.dtype, device=seg_start.device)
        dec = dec.masked_fill(seg_start == pos, start_id)
    return dec


class MT5ForConditionalGeneration(FlatModel):
    def __init__(self, config, device=None, world_size=None, seed=0, fp8=False):
        """fp8: train the layer projections in FP8; see the module docstring. The training and no-grad (validation) forwards
        both run FP8; results differ from bf16 by design. d_model, d_ff and the tokens per micro-batch on both sides
        (batch x source length, batch x target length) must be multiples of 16 (checked at the first forward)."""
        super().__init__(config)
        self.fp8 = bool(fp8)
        g = lambda k, d=None: getattr(config, k, d)
        self.d, self.dk, self.nh, self.ff = g("d_model"), g("d_kv"), g("num_heads"), g("d_ff")
        self.ne = g("num_layers")
        self.nd = g("num_decoder_layers") or self.ne
        self.V = g("vocab_size")
        self.eps = g("layer_norm_epsilon", 1e-6)
        self.nbuckets = g("relative_attention_num_buckets", 32)
        self.maxdist = g("relative_attention_max_distance", 128)
        self.pad_id = g("pad_token_id", 0)
        self.start_id = g("decoder_start_token_id", 0)
        if self.start_id is None:
            self.start_id = self.pad_id
        self.p_drop, = self._dropout_probs("MT5", "dropout_rate")
        if g("feed_forward_proj", "gated-gelu") != "gated-gelu":
            raise RuntimeError("fsb200 MT5: only feed_forward_proj='gated-gelu' (T5 v1.1 / mT5) is implemented")
        # transformers 5.x FORCES tie_word_embeddings=True for MT5 configs (configuration_mt5.py __post_init__: "we have to tie
        # always") and applies NO d^-0.5 rescale to the decoder output (modeling_mt5.py:1141-1143) — that is what the reference
        # script gets from `MT5ForConditionalGeneration(config)` with the installed library, and what the goldens pin. Older
        # releases honoured mT5's untied head; both are implemented, neither rescales.
        self.tied = bool(g("tie_word_embeddings", False))
        if self.dk not in (64, 128) or self.V % 8 or self.d % 8 or self.ff % 8:
            raise RuntimeError("fsb200 MT5: d_kv must be 64/128 and vocab/d_model/d_ff multiples of 8 (pad the vocab)")
        d, inner, ff, V = self.d, self.nh * self.dk, self.ff, self.V
        self.inner = inner

        spec = FlatSpec()
        spec.add("shared.weight", (V, d), "shared")
        for i in range(self.ne):
            p, bk = f"encoder.block.{i}.layer.", f"enc{i}"
            for n in ("q", "k", "v"):                               # adjacent: one [3*inner, d] GEMM operand
                spec.add(p + f"0.SelfAttention.{n}.weight", (inner, d), bk)
            spec.add(p + "0.SelfAttention.o.weight", (d, inner), bk)
            if i == 0:
                spec.add(p + "0.SelfAttention.relative_attention_bias.weight", (self.nbuckets, self.nh), bk)
            spec.add(p + "0.layer_norm.weight", (d,), bk)
            spec.add(p + "1.DenseReluDense.wi_0.weight", (ff, d), bk)   # wi_0 | wi_1 adjacent: one [2*ff, d] operand
            spec.add(p + "1.DenseReluDense.wi_1.weight", (ff, d), bk)
            spec.add(p + "1.DenseReluDense.wo.weight", (d, ff), bk)
            spec.add(p + "1.layer_norm.weight", (d,), bk)
        spec.add("encoder.final_layer_norm.weight", (d,), "head")
        for i in range(self.nd):
            p, bk = f"decoder.block.{i}.layer.", f"dec{i}"
            for n in ("q", "k", "v"):
                spec.add(p + f"0.SelfAttention.{n}.weight", (inner, d), bk)
            spec.add(p + "0.SelfAttention.o.weight", (d, inner), bk)
            if i == 0:
                spec.add(p + "0.SelfAttention.relative_attention_bias.weight", (self.nbuckets, self.nh), bk)
            spec.add(p + "0.layer_norm.weight", (d,), bk)
            spec.add(p + "1.EncDecAttention.q.weight", (inner, d), bk)
            spec.add(p + "1.EncDecAttention.k.weight", (inner, d), bk)  # k | v adjacent: one [2*inner, d] operand
            spec.add(p + "1.EncDecAttention.v.weight", (inner, d), bk)
            spec.add(p + "1.EncDecAttention.o.weight", (d, inner), bk)
            spec.add(p + "1.layer_norm.weight", (d,), bk)
            spec.add(p + "2.DenseReluDense.wi_0.weight", (ff, d), bk)
            spec.add(p + "2.DenseReluDense.wi_1.weight", (ff, d), bk)
            spec.add(p + "2.DenseReluDense.wo.weight", (d, ff), bk)
            spec.add(p + "2.layer_norm.weight", (d,), bk)
        spec.add("decoder.final_layer_norm.weight", (d,), "head")
        if not self.tied:
            spec.add("lm_head.weight", (V, d), "head")
        self._bind_flat(spec, device, world_size)
        if self.tied:
            self.lm_head = _Holder()
            self.lm_head.weight = self._p["shared.weight"]      # same Parameter object: named_parameters() lists it once
        self._head = Linear.of(self._p["shared.weight" if self.tied else "lm_head.weight"])
        lin = lambda name: Linear.of(self.P(name + ".weight"))
        span = lambda first, rows: Linear.span(self.flat, first + ".weight", rows, d)
        mlp = lambda p: GatedMLP(span(p + "DenseReluDense.wi_0", 2 * ff), lin(p + "DenseReluDense.wo"), L.ACT_GELU_TANH)
        self._enc = [_Enc(span(p + "0.SelfAttention.q", 3 * inner), lin(p + "0.SelfAttention.o"), mlp(p + "1."))
                     for p in (f"encoder.block.{i}.layer." for i in range(self.ne))]
        self._dec = [_Dec(span(p + "0.SelfAttention.q", 3 * inner), lin(p + "0.SelfAttention.o"), lin(p + "1.EncDecAttention.q"),
                          span(p + "1.EncDecAttention.k", 2 * inner), lin(p + "1.EncDecAttention.o"), mlp(p + "2."))
                     for p in (f"decoder.block.{i}.layer." for i in range(self.nd))]
        self._enc_bf16, self._dec_bf16 = self._enc, self._dec   # what generate runs
        if self.fp8:
            f8 = lambda pj: type(pj)(*(GatedMLP(Fp8Linear(q.wi), Fp8Linear(q.wo), q.act) if isinstance(q, GatedMLP)
                                       else Fp8Linear(q) for q in pj))
            self._enc, self._dec = [f8(pj) for pj in self._enc], [f8(pj) for pj in self._dec]

        self.reset_parameters(seed)
        # dropout sites of one forward. Encoder: 0 embeddings; layer i: 1 + 4i attention probabilities, 2 + 4i attention output,
        # 3 + 4i gated activation, 4 + 4i FFN output; 1 + 4 Le final-norm output. Decoder from E = 2 + 4 Le: E embeddings; layer
        # i: E + 1 + 6i self-attention probabilities, E + 2 + 6i its output, E + 3 + 6i cross-attention probabilities, E + 4 + 6i
        # its output, E + 5 + 6i gated activation, E + 6 + 6i FFN output; E + 1 + 6 Ld final-norm output.
        self.dec_site0 = 2 + 4 * self.ne
        self._init_dropout(4 + 4 * self.ne + 6 * self.nd, (self.p_drop,))

    @torch.no_grad()
    def reset_parameters(self, seed=0):
        """HF MT5PreTrainedModel._init_weights with initializer_factor 1 (mt5/modeling_mt5.py)."""
        d, dk, nh, ff = self.d, self.dk, self.nh, self.ff
        gen = torch.Generator(device=self.flat.params.device).manual_seed(seed)
        for name, prm in self._p.items():
            if name.endswith("layer_norm.weight"):
                prm.fill_(1.0)
                continue
            if name in ("shared.weight", "lm_head.weight"):
                std = 1.0
            elif name.endswith(".q.weight"):
                std = (d * dk) ** -0.5
            elif name.endswith(".k.weight") or name.endswith(".v.weight") or "relative_attention_bias" in name:
                std = d ** -0.5
            elif name.endswith("Attention.o.weight"):
                std = (nh * dk) ** -0.5
            elif "wi_" in name:
                std = d ** -0.5
            else:  # DenseReluDense.wo
                std = ff ** -0.5
            prm.normal_(0.0, std, generator=gen)

    # ---- forward ----------------------------------------------------------------------------------------------------
    def _shift_right(self, labels):
        """MT5 _shift_right (:592): decoder_input_ids = [start] + labels[:-1], with -100 replaced by the pad id."""
        return shift_right(labels, self.start_id, self.pad_id)

    def forward(self, input_ids=None, attention_mask=None, labels=None, decoder_input_ids=None, return_logits=False,
                segment_ids=None, decoder_segment_ids=None, **_):
        """segment_ids [B, Se] / decoder_segment_ids [B, Sd]: optional integer ids of packed rows (host or device; both or
        neither), non-decreasing along each row; encoder and decoder segments with the same id value are one sample
        (fsb200/packing.py numbers them 0..m-1 and gives each side's pad tail id m). head_dim (d_kv) 64 only. No key mask is
        used: an attention_mask with zeros is refused. decoder_input_ids derived from labels restart at every decoder
        segment with the start id, so no sample sees the previous one's last label; the loss covers every labelled decoder
        position, as without packing. segment_ids=None: one sample per row under attention_mask, as before."""
        dev = self.flat.params.device
        B, Se = input_ids.shape
        if (segment_ids is None) != (decoder_segment_ids is None):
            raise ValueError("fsb200 MT5: pass segment_ids and decoder_segment_ids together (packed rows need both)")
        packed = ()
        if segment_ids is not None:
            if self.dk != 64:
                raise ValueError(f"fsb200 MT5: segment_ids need d_kv 64 (the packed attention kernels), this config has "
                                 f"d_kv {self.dk}")
            refuse_key_padding(attention_mask, "MT5")
            packed = (self._packed_bounds(segment_ids, decoder_segment_ids, B, Se, dev),)
        if decoder_input_ids is None:
            if labels is None:
                raise ValueError("fsb200 MT5: pass labels or decoder_input_ids")
            # packed: each decoder segment starts from the start id, as its sample would alone
            decoder_input_ids = shift_right(labels.to(device=dev, dtype=torch.int64), self.start_id, self.pad_id,
                                            packed[0][1][0] if packed else None)
        Sd = decoder_input_ids.shape[1]
        if self.fp8:
            bad = [f"{name} ({v})" for name, v in (("d_model", self.d), ("d_ff", self.ff),
                                                    (f"batch {B} x source length {Se}", B * Se),
                                                    (f"batch {B} x target length {Sd}", B * Sd)) if v % 16]
            if bad:
                raise ValueError(f"fsb200 MT5ForConditionalGeneration(fp8=True): {', '.join(bad)} not a multiple of 16 (the "
                                 "FP8 GEMM operands need 16-byte rows in both layouts; d_model, d_ff and the tokens per "
                                 "micro-batch on both sides must be). With the span-corruption collator's target length "
                                 "of 114, the micro-batch must be a multiple of 8")
        ids, dec_ids, lab = flat_ids(input_ids, dev), flat_ids(decoder_input_ids, dev), flat_ids(labels, dev)
        mask = None if packed else key_mask(attention_mask, dev)
        loss, logits = self._step_or_forward(lab is not None, return_logits, ids, dec_ids, mask, lab, B, Se, Sd, *packed)
        return SimpleNamespace(loss=loss, logits=None if logits is None else logits.view(B, Sd, self.V),
                               past_key_values=None, encoder_last_hidden_state=None)

    @staticmethod
    def _packed_bounds(segment_ids, decoder_segment_ids, B, Se, dev):
        """-> (encoder (seg_start, seg_end), decoder (seg_start, seg_end), cross ((kv_start, kv_end), (q_start, q_end)))."""
        enc, dec = segment_ids, decoder_segment_ids
        if tuple(enc.shape) != (B, Se) or dec.dim() != 2 or dec.shape[0] != B:
            raise ValueError(f"fsb200 MT5: segment_ids must be [batch, source length] = [{B}, {Se}] and decoder_segment_ids "
                             f"[{B}, target length], got {tuple(enc.shape)} and {tuple(dec.shape)}")
        if enc.device != dec.device:
            enc, dec = enc.to(device=dev, non_blocking=True), dec.to(device=dev, non_blocking=True)
        # on the ids' own device: host ids are checked exactly, device ids without a synchronisation
        cross = tuple(tuple(t.to(device=dev, non_blocking=True) for t in side) for side in cross_segment_bounds(dec, enc))
        to_dev = lambda t: t.to(device=dev, non_blocking=True)
        return ops.segment_bounds(to_dev(enc)), ops.segment_bounds(to_dev(dec)), cross

    def _norm(self, prev, x, name, drop=None):
        """pre-norm with the pending residual add (of the branch `prev`, dropped by `drop`) fused in: returns (normed, rstd,
        residual stream)."""
        if prev is None:
            return ops.rmsnorm_fwd(x, self.P(name).data, self.eps)
        return ops.rmsnorm_fwd(prev, self.P(name).data, self.eps, residual=x, drop=drop)

    def _encode(self, ids, mask, B, Se, rel_e, save, base=None, seg=None, proj=None):
        """Encoder stack over ids [B * Se]; returns (saved activations, final hidden states (after their dropout), their rstd,
        residual stream). base: the forward's dropout stream base (None: no dropout). seg: the (seg_start, seg_end) bounds of
        packed rows (mask is then None). proj: the layers' projections (default self._enc)."""
        nh, dk, inner = self.nh, self.dk, self.inner
        P = self.P
        Te = B * Se
        D = lambda site: self._drop(base, self.p_drop, site)
        x, prev = apply_dropout(ops.embedding_fwd(ids, P("shared.weight").data), D(0)), None
        eacts = []
        for i, pj in enumerate(self._enc if proj is None else proj):
            p = f"encoder.block.{i}.layer."
            self._need(f"enc{i}")
            h1, r1, x = self._norm(prev, x, p + "0.layer_norm.weight", D(4 * i))   # layer i-1's FFN output
            # qs: what q|k|v's backward reads of h1 (h1 itself in bf16, its transposed e4m3 codes and scale in FP8)
            qkv, qs = pj.qkv.forward(h1, save)
            q5 = qkv.view(B, Se, 3, nh, dk)
            if seg is None:
                o, lse = ops.sdpa_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], 1.0, False, kv_mask=mask, rel_bias=rel_e,
                                      drop=D(1 + 4 * i))
            else:
                o, lse = ops.sdpa_segments_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], 1.0, *seg, drop=D(1 + 4 * i),
                                               causal=False, rel_bias=rel_e)
            a = pj.o(o.view(Te, inner))
            h2, r2, x1 = self._norm(a, x, p + "1.layer_norm.weight", D(2 + 4 * i))
            m, ms = pj.mlp(h2, save, drop=D(3 + 4 * i))
            if save:
                eacts.append((x, r1, qs, qkv, o, lse, x1, r2, ms))
            x, prev = x1, m
        self._need("head")
        enc_h, rfe, xfe = self._norm(prev, x, "encoder.final_layer_norm.weight", D(4 * self.ne))
        return eacts, apply_dropout(enc_h, D(1 + 4 * self.ne)), rfe, xfe

    def _decode(self, dec_ids, B, S, attend, cross_attend, acts=None, base=None, proj=None):
        """Decoder stack over dec_ids [B * S] -> (final hidden states (after their dropout), their rstd, residual stream).
        attend(i, q5) is layer i's self-attention over the packed q|k|v view [B, S, 3, heads, d_kv] -> (out, lse);
        cross_attend(i, qc) its cross-attention from the query projection [B * S, inner] -> (out, lse, the encoder's K|V or
        None); `acts`, when given, collects what the backward reads. base: the forward's dropout stream base (None: no
        dropout); the attention callbacks draw their own probability masks. proj: the layers' projections (default
        self._dec)."""
        nh, dk, inner = self.nh, self.dk, self.inner
        P = self.P
        T = B * S
        E = self.dec_site0
        D = lambda site: self._drop(base, self.p_drop, site)
        self._need("no_decay"); self._need("shared")
        y, prev = apply_dropout(ops.embedding_fwd(dec_ids, P("shared.weight").data), D(E)), None
        save = acts is not None
        for i, pj in enumerate(self._dec if proj is None else proj):
            p = f"decoder.block.{i}.layer."
            self._need(f"dec{i}")
            h1, r1, y = self._norm(prev, y, p + "0.layer_norm.weight", D(E + 6 * i))   # layer i-1's FFN output
            qkv, qs = pj.qkv.forward(h1, save)
            o, lse = attend(i, qkv.view(B, S, 3, nh, dk))
            a = pj.o(o.view(T, inner))
            h2, r2, y1 = self._norm(a, y, p + "1.layer_norm.weight", D(E + 2 + 6 * i))
            qc, h2s = pj.cq.forward(h2, save)
            oc, lsec, kvc = cross_attend(i, qc)
            ac = pj.co(oc.view(T, inner))
            h3, r3, y2 = self._norm(ac, y1, p + "2.layer_norm.weight", D(E + 4 + 6 * i))
            m, ms = pj.mlp(h3, save, drop=D(E + 5 + 6 * i))
            if save:
                acts.append((y, r1, qs, qkv, o, lse, y1, r2, h2s, qc, kvc, oc, lsec, y2, r3, ms))
            y, prev = y2, m
        self._need("head")
        hf, rfd, xfd = self._norm(prev, y, "decoder.final_layer_norm.weight", D(E + 6 * self.nd))
        return apply_dropout(hf, D(E + 1 + 6 * self.nd)), rfd, xfd

    # ---- KV-cache generation -----------------------------------------------------------------------------------------
    # transformers' GenerationMixin on MT5 (mt5_summary.py:41-49,131-139; finetune_t5.py:66-71). The encoder runs once; every
    # decoder layer projects its cross-attention K|V once from the encoder output; each step runs the training decoder stack
    # (`_decode`) on one token per row, appends its self-attention K|V at the device-side slot kv_len - 1 (ops.kv_append) of
    # a [layers, rows, cap, 2, heads, d_kv] cache and runs the split-KV decode kernel twice per layer: self-attention with
    # the relative-position bias at the query's slot, cross-attention under the encoder padding mask. Every decode step is
    # one CUDA-graph replay (fsb200/decode_graph.py); beam search gathers the self-attention cache into the twin
    # (ops.kv_reorder). The cross-attention K|V is the same for every beam of an item and is not reordered.
    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, **kwargs):
        """HF `generate` semantics (fsb200/generation.py lists what is implemented); sequences start with
        decoder_start_token_id. Runs without dropout; in training mode with dropout_rate > 0 it raises (HF would drop)."""
        self._refuse_dropout_generate("MT5", "dropout_rate")
        dev = self.flat.params.device
        nh, dk = self.nh, self.dk
        P = self.P
        ids = input_ids.to(device=dev, dtype=torch.int64).contiguous()
        B, Se = ids.shape
        c = generation.resolve(self.config, kwargs, 1, True)
        mask = generation.default_attention_mask(ids, c.pad, c.eos) if attention_mask is None else \
            attention_mask.to(device=dev, dtype=torch.int64)
        emask = None if bool(mask.all()) else mask.to(torch.uint8).contiguous()
        self._need("no_decay"); self._need("shared")
        rel_e = TB.rel_bias_vector(P("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight").data, Se, Se, True,
                                   self.nbuckets, self.maxdist)
        _, enc_h, _, _ = self._encode(ids.view(-1), emask, B, Se, rel_e, False, proj=self._enc_bf16)   # fp8=True: bf16
        R = B * c.expand
        cross = []
        for i in range(self.nd):
            self._need(f"dec{i}")
            kvc = self._dec_bf16[i].ckv(enc_h).view(B, Se, 2, nh, dk)
            cross.append(kvc.repeat_interleave(c.expand, 0) if c.expand > 1 else kvc)
        cmask = None if emask is None else emask.repeat_interleave(c.expand, 0).contiguous()
        cap = (max(c.max_length, 2) + 63) // 64 * 64
        rel_d = TB.rel_bias_vector(P("decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight").data, cap, cap,
                                   False, self.nbuckets, self.maxdist)
        enc_len = torch.full((1,), Se, dtype=torch.int32, device=dev)
        start = torch.full((R, 1), c.start, dtype=torch.int64, device=dev)
        caches = [torch.zeros((self.nd, R, cap, 2, nh, dk), dtype=torch.bfloat16, device=dev)
                  for _ in range(2 if c.num_beams > 1 else 1)]
        kv_len = torch.zeros(1, dtype=torch.int32, device=dev)

        def cross_attend(i, qc):
            oc, lsec = ops.attn_decode(qc.view(R, nh, dk), cross[i][:, :, 0], cross[i][:, :, 1], enc_len, 1.0, kv_mask=cmask)
            return oc, lsec, None

        def body(tok, index, a, b):
            if b is not a:
                ops.kv_reorder(a, b, index, kv_len)
            kv_len.add_(1)

            def attend(i, q5):
                kv = b[i]
                ops.kv_append(q5[:, 0, 1], q5[:, 0, 2], kv[:, :, 0], kv[:, :, 1], kv_len)
                return ops.attn_decode(q5[:, 0, 0], kv[:, :, 0], kv[:, :, 1], kv_len, 1.0, rel_bias=rel_d)
            hf, _, _ = self._decode(tok, R, 1, attend, cross_attend, proj=self._dec_bf16)
            return self._head(hf).float()

        graphs = DecodeGraphs(self, R, caches, body)
        graphs.tok.copy_(start.view(-1))      # the first step decodes the start token
        return generation.run(graphs, start, c)

    def _forward_impl(self, ids, dec_ids, mask, lab, B, Se, Sd, segs=None, *, save, want_logits):
        """segs: None or the bounds of packed rows (_packed_bounds); mask is then None."""
        nh, dk = self.nh, self.dk
        P = self.P
        self._need("no_decay"); self._need("shared")
        # relative-position bias vectors (fp32 [heads, 2S - 1]) from the two [buckets, heads] tables
        rel_e = TB.rel_bias_vector(P("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight").data, Se, Se, True,
                                   self.nbuckets, self.maxdist)
        rel_d = TB.rel_bias_vector(P("decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight").data, Sd, Sd, False,
                                   self.nbuckets, self.maxdist)
        base = self._dropout_base()
        E = self.dec_site0
        D = lambda site: self._drop(base, self.p_drop, site)
        enc_seg, dec_seg, cross = (None, None, None) if segs is None else segs
        eacts, enc_h, rfe, xfe = self._encode(ids, mask, B, Se, rel_e, save, base, enc_seg)
        # every decoder layer's cross k|v projection reads enc_h: under fp8 its codes are made once and shared, and what the
        # backward reads of it (enc_s) is kept once
        enc_codes = self._dec[0].ckv.quantize_input(enc_h, save) if self.fp8 and self.nd else None
        enc_s = enc_h if enc_codes is None else enc_codes[1:]

        def attend(i, q5):
            if dec_seg is not None:
                return ops.sdpa_segments_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], 1.0, *dec_seg, drop=D(E + 1 + 6 * i),
                                             rel_bias=rel_d)
            return ops.sdpa_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], 1.0, True, rel_bias=rel_d, drop=D(E + 1 + 6 * i))

        def cross_attend(i, qc):
            ckv = self._dec[i].ckv
            kvc = ckv(enc_h) if enc_codes is None else ckv.forward(enc_h, False, codes=enc_codes)[0]
            kv5 = kvc.view(B, Se, 2, nh, dk)
            if cross is not None:
                oc, lsec = ops.sdpa_segments_fwd(qc.view(B, Sd, nh, dk), kv5[:, :, 0], kv5[:, :, 1], 1.0, *cross[0],
                                                 drop=D(E + 3 + 6 * i), causal=False, kv_bounds=cross[1])
            else:
                oc, lsec = ops.sdpa_fwd(qc.view(B, Sd, nh, dk), kv5[:, :, 0], kv5[:, :, 1], 1.0, False, kv_mask=mask,
                                        drop=D(E + 3 + 6 * i))
            return oc, lsec, kvc
        dacts = [] if save else None
        hf, rfd, xfd = self._decode(dec_ids, B, Sd, attend, cross_attend, dacts, base)
        logits = self._head(hf)
        loss, ctx = None, None
        if lab is not None:
            keep = logits.clone() if (want_logits and save) else None
            loss, dlogits, _ = ops.softmax_xent(logits, lab, Sd, shift=0, grad_scale=self.loss_scale,
                                                dlogits="inplace" if save else None)
            if save:
                ctx = (eacts, dacts, enc_s, rfe, xfe, hf, rfd, xfd, dlogits, ids, dec_ids, mask, rel_e, rel_d, B, Se, Sd, base,
                       segs)
                logits = keep
        return loss, (logits if want_logits else None), ctx

    # ---- backward ---------------------------------------------------------------------------------------------------
    def _backward_impl(self, ctx, gloss):
        eacts, dacts, enc_s, rfe, xfe, hf, rfd, xfd, dlogits, ids, dec_ids, mask, rel_e, rel_d, B, Se, Sd, base, segs = ctx
        enc_seg, dec_seg, cross = (None, None, None) if segs is None else segs
        d, nh, dk, inner = self.d, self.nh, self.dk, self.inner
        P = self.P
        Te, Td = B * Se, B * Sd
        acc = self.accumulate_grads
        dev = self.flat.params.device
        E = self.dec_site0
        D = lambda site: self._drop(base, self.p_drop, site)

        self._begin_backward()
        if gloss is not None:
            ops.scale_inplace(dlogits, gloss)
        dhf = self._head.backward(dlogits, hf, acc)   # tied head: written first, the embeddings add later
        del dlogits
        self._done("head")                      # lm_head is the bucket's only decayed parameter (the norms are no-decay)
        dy, dm = residual_norm_bwd(apply_dropout(dhf, D(E + 1 + 6 * self.nd)), xfd, P("decoder.final_layer_norm.weight"), None,
                                   rfd, D(E + 6 * self.nd), acc)
        drel_e = torch.zeros_like(rel_e)
        drel_d = torch.zeros_like(rel_d)
        denc32 = torch.empty((Te, d), dtype=torch.float32, device=dev)   # sum over decoder layers of the K|V dgrads
        for i in reversed(range(self.nd)):
            p, pj = f"decoder.block.{i}.layer.", self._dec[i]
            y, r1, qs, qkv, o, lse, y1, r2, h2s, qc, kvc, oc, lsec, y2, r3, ms = dacts[i]
            dacts[i] = None
            dh3 = pj.mlp.backward(dm, ms, acc, drop=D(E + 5 + 6 * i))
            dy2, dac = residual_norm_bwd(dh3, y2, P(p + "2.layer_norm.weight"), None, r3, D(E + 4 + 6 * i), acc, dres=dy)
            # cross-attention
            doc = pj.co.backward(dac, pj.co.saved_input(oc.view(Td, inner)), acc)   # oc is kept for attention anyway
            dqc = torch.empty_like(qc)
            dkvc = torch.empty_like(kvc)
            kv5, dkv5 = kvc.view(B, Se, 2, nh, dk), dkvc.view(B, Se, 2, nh, dk)
            if cross is not None:
                ops.sdpa_segments_bwd(qc.view(B, Sd, nh, dk), kv5[:, :, 0], kv5[:, :, 1], oc, doc.view(B, Sd, nh, dk), lsec,
                                      1.0, *cross[0], dqc.view(B, Sd, nh, dk), dkv5[:, :, 0], dkv5[:, :, 1],
                                      drop=D(E + 3 + 6 * i), causal=False, kv_bounds=cross[1])
            else:
                ops.sdpa_bwd(qc.view(B, Sd, nh, dk), kv5[:, :, 0], kv5[:, :, 1], oc, doc.view(B, Sd, nh, dk), lsec, 1.0,
                             False, dqc.view(B, Sd, nh, dk), dkv5[:, :, 0], dkv5[:, :, 1], kv_mask=mask,
                             drop=D(E + 3 + 6 * i))
            dh2 = pj.cq.backward(dqc, h2s, acc)
            if self.fp8:   # the FP8 GEMM writes bf16: each layer's dgrad is rounded once, their sum is kept in fp32
                ops.accumulate(denc32, pj.ckv.backward(dkvc, enc_s, acc), overwrite=(i == self.nd - 1))
            else:
                pj.ckv.backward(dkvc, enc_s, acc, dx=denc32, dx_accumulate=(i != self.nd - 1))
            dy1, da = residual_norm_bwd(dh2, y1, P(p + "1.layer_norm.weight"), None, r2, D(E + 2 + 6 * i), acc, dres=dy2)
            # causal self-attention with the decoder's relative-position bias
            do = pj.o.backward(da, pj.o.saved_input(o.view(Td, inner)), acc)
            dqkv = torch.empty_like(qkv)
            q5, d5 = qkv.view(B, Sd, 3, nh, dk), dqkv.view(B, Sd, 3, nh, dk)
            if dec_seg is not None:
                ops.sdpa_segments_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, Sd, nh, dk), lse, 1.0, *dec_seg,
                                      d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], drop=D(E + 1 + 6 * i), rel_bias=rel_d,
                                      drel_bias=drel_d)
            else:
                ops.sdpa_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, Sd, nh, dk), lse, 1.0, True,
                             d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], rel_bias=rel_d, drel_bias=drel_d, drop=D(E + 1 + 6 * i))
            dh1 = pj.qkv.backward(dqkv, qs, acc)
            # layer 0's norm had no residual (y = the embeddings); layer i's summed layer i-1's dropped FFN output into y
            dy, dm = residual_norm_bwd(dh1, y, P(p + "0.layer_norm.weight"), None, r1, D(E + 6 * i) if i > 0 else None, acc,
                                       dres=dy1)
            if i == 0:
                self._table_grad("decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", drel_d, Sd, False, acc)
            self._done(f"dec{i}")
        ddec_emb = apply_dropout(dy, D(E))      # gradient w.r.t. the decoder's input embeddings
        # ---- encoder
        if self.nd > 0:
            denc = ops.cast_f32_to_bf16(denc32)
        else:
            denc = torch.zeros((Te, d), dtype=torch.bfloat16, device=dev)
        del denc32
        dx, dm = residual_norm_bwd(apply_dropout(denc, D(1 + 4 * self.ne)), xfe, P("encoder.final_layer_norm.weight"), None,
                                   rfe, D(4 * self.ne), acc)
        for i in reversed(range(self.ne)):
            p, pj = f"encoder.block.{i}.layer.", self._enc[i]
            x, r1, qs, qkv, o, lse, x1, r2, ms = eacts[i]
            eacts[i] = None
            dh2 = pj.mlp.backward(dm, ms, acc, drop=D(3 + 4 * i))
            dx1, da = residual_norm_bwd(dh2, x1, P(p + "1.layer_norm.weight"), None, r2, D(2 + 4 * i), acc, dres=dx)
            do = pj.o.backward(da, pj.o.saved_input(o.view(Te, inner)), acc)
            dqkv = torch.empty_like(qkv)
            q5, d5 = qkv.view(B, Se, 3, nh, dk), dqkv.view(B, Se, 3, nh, dk)
            if enc_seg is not None:
                ops.sdpa_segments_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, Se, nh, dk), lse, 1.0, *enc_seg,
                                      d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], drop=D(1 + 4 * i), causal=False,
                                      rel_bias=rel_e, drel_bias=drel_e)
            else:
                ops.sdpa_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, Se, nh, dk), lse, 1.0, False,
                             d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], kv_mask=mask, rel_bias=rel_e, drel_bias=drel_e,
                             drop=D(1 + 4 * i))
            dh1 = pj.qkv.backward(dqkv, qs, acc)
            dx, dm = residual_norm_bwd(dh1, x, P(p + "0.layer_norm.weight"), None, r1, D(4 * i) if i > 0 else None, acc,
                                       dres=dx1)
            if i == 0:
                self._table_grad("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", drel_e, Se, True, acc)
            self._done(f"enc{i}")
        dx = apply_dropout(dx, D(0))
        Wg = P("shared.weight").main_grad
        if not acc and not self.tied:
            Wg.zero_()
        ops.embedding_bwd(ids, dx, Wg)          # encoder inputs
        ops.embedding_bwd(dec_ids, ddec_emb, Wg)  # decoder inputs share the table
        self._done("shared")
        self._done("no_decay")

    def _table_grad(self, name, drel, S, bidirectional, acc):
        """[heads, 2S - 1] gradient of the bias vector -> [buckets, heads] gradient of the embedding table (fixed-index
        index_add: deterministic), written to the flat gradient buffer."""
        g = TB.scatter_rel_grad(drel, S, S, bidirectional, self.nbuckets, self.maxdist)
        mg = self.P(name).main_grad
        if acc:
            mg.copy_((mg.float() + g).to(mg.dtype))
        else:
            mg.copy_(g.to(mg.dtype))


def t5_flops_per_step(cfg, B, Se, Sd):
    """Algorithmic FLOPs of one forward + backward (3x forward) over B samples — SURVEY.md §8(d) C5 formula: matmul parameters
    touched per token x 6, plus attention (encoder full, decoder causal-counted, cross full)."""
    d, inner, ff, V = cfg["d_model"], cfg["num_heads"] * cfg["d_kv"], cfg["d_ff"], cfg["vocab_size"]
    Le, Ld = cfg["num_layers"], cfg.get("num_decoder_layers") or cfg["num_layers"]
    enc_mm = Le * (4 * d * inner + 3 * d * ff)
    dec_mm = Ld * (4 * d * inner + 2 * d * inner + 3 * d * ff) + V * d      # self + cross q/o + FFN + head, per decoder token
    cross_kv = Ld * 2 * d * inner                                            # per ENCODER token
    mm = 6.0 * B * (Se * (enc_mm + cross_kv) + Sd * dec_mm)
    attn = 3.0 * 4.0 * inner * B * (Le * Se * Se + Ld * Sd * Sd / 2 + Ld * Se * Sd)
    return mm + attn
