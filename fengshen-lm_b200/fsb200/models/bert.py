"""Erlangshen-BERT / Erlangshen-MegatronBERT on the fsb200 kernels — drop-ins for the two HF classes the reference's
MLM pretraining scripts instantiate:
    transformers.BertForMaskedLM            examples/pretrain_bert/pretrain_bert.py:135-137           (config 1)
    transformers.MegatronBertForPreTraining examples/pretrain_erlangshen_bert/pretrain_erlangshen.py:138-141 (config 3)
The arithmetic restated here lives in 3P `transformers` (SURVEY.md Appendix C):
  BERT          post-LN blocks  x = LN(x + W_o attn(x)); x = LN(x + W_2 act(W_1 x)); embeddings word+pos+type -> LN.
  MegatronBERT  pre-LN blocks   x + W_o attn(ln(x)); x + W_2 act(W_1 ln(x)); final encoder ln; embeddings WITHOUT LN;
                pooler tanh(W x[:,0]) + NSP head; loss = CE(mlm) + CE(nsp).
Both: separate q/k/v Linear(h,h)+bias (laid out adjacently -> one [3h,h] GEMM), softmax(QK^T/sqrt(hn) + padding mask),
LayerNorm eps 1e-12, MLM head = dense + act + LN + decoder tied to the word embeddings + bias, CE ignore_index -100.
State-dict keys follow HF.
Dropout (hidden_dropout_prob, attention_probs_dropout_prob; the two may differ) applies in training mode (`model.training`,
also under no_grad), at HF's sites: the embeddings (BERT: after the LN; MegatronBERT: the sum, no LN), the attention
probabilities, and the attention-output and FFN-output branches before their residual add — fused into the attention kernels
and the LayerNorms that add the branch to the residual. Seed, stream counter and eval mode as in fsb200/models/base.py.
"""
import math
from collections import namedtuple
from types import SimpleNamespace

import torch

from .. import lib as L
from .. import ops
from ..flat import FlatSpec
from .base import FlatModel, flat_ids, key_mask, learned_pos_emb_bwd
from .layers import Linear, apply_dropout, residual_norm_bwd

_Layer = namedtuple("_Layer", "qkv attn_out inter out")   # attention.self q|k|v, attention.output.dense, intermediate, output


class _BertFamily(FlatModel):
    PRE_LN = False

    def __init__(self, config, device=None, world_size=None, seed=0):
        super().__init__(config)
        g = lambda k, d=None: getattr(config, k, d)
        self.h, self.nl, self.nh, self.V = g("hidden_size"), g("num_hidden_layers"), g("num_attention_heads"), g("vocab_size")
        self.ff, self.npos, self.ntype = g("intermediate_size"), g("max_position_embeddings", 512), g("type_vocab_size", 2)
        self.eps = g("layer_norm_eps", 1e-12)
        self.p_hidden, self.p_attn = self._dropout_probs("BERT", "hidden_dropout_prob", "attention_probs_dropout_prob")
        act = g("hidden_act", "gelu")
        if act not in ("gelu", "gelu_new"):
            raise RuntimeError(f"fsb200 BERT: hidden_act={act!r} not implemented (gelu, gelu_new)")
        self.epi = L.EPI_GELU_ERF if act == "gelu" else L.EPI_GELU_TANH
        self.act = L.ACT_GELU_ERF if act == "gelu" else L.ACT_GELU_TANH
        h = self.h
        self.hn = h // self.nh
        if self.hn not in (64, 128) or self.V % 8 or h % 128:
            raise RuntimeError("fsb200 BERT: head dim must be 64/128, vocab a multiple of 8, hidden a multiple of 128")
        pre = self.PRE_LN
        spec = FlatSpec()
        E = "bert.embeddings."
        spec.add(E + "word_embeddings.weight", (self.V, h), "emb")
        spec.add(E + "position_embeddings.weight", (self.npos, h), "emb")
        spec.add(E + "token_type_embeddings.weight", (self.ntype, h), "emb")
        if not pre:
            spec.add(E + "LayerNorm.weight", (h,), "emb"); spec.add(E + "LayerNorm.bias", (h,), "emb")
        for i in range(self.nl):
            p, bk = f"bert.encoder.layer.{i}.", f"layer{i}"
            if pre:
                spec.add(p + "attention.ln.weight", (h,), bk); spec.add(p + "attention.ln.bias", (h,), bk)
            for n in ("query", "key", "value"):            # adjacent: one [3h, h] operand
                spec.add(p + f"attention.self.{n}.weight", (h, h), bk)
            for n in ("query", "key", "value"):            # adjacent in the no-decay bucket: one [3h] bias
                spec.add(p + f"attention.self.{n}.bias", (h,), bk)
            spec.add(p + "attention.output.dense.weight", (h, h), bk); spec.add(p + "attention.output.dense.bias", (h,), bk)
            if pre:
                spec.add(p + "ln.weight", (h,), bk); spec.add(p + "ln.bias", (h,), bk)
            else:
                spec.add(p + "attention.output.LayerNorm.weight", (h,), bk)
                spec.add(p + "attention.output.LayerNorm.bias", (h,), bk)
            spec.add(p + "intermediate.dense.weight", (self.ff, h), bk); spec.add(p + "intermediate.dense.bias", (self.ff,), bk)
            spec.add(p + "output.dense.weight", (h, self.ff), bk); spec.add(p + "output.dense.bias", (h,), bk)
            if not pre:
                spec.add(p + "output.LayerNorm.weight", (h,), bk); spec.add(p + "output.LayerNorm.bias", (h,), bk)
        if pre:
            spec.add("bert.encoder.ln.weight", (h,), "head"); spec.add("bert.encoder.ln.bias", (h,), "head")
            spec.add("bert.pooler.dense.weight", (h, h), "head"); spec.add("bert.pooler.dense.bias", (h,), "head")
        spec.add("cls.predictions.bias", (self.V,), "head")
        spec.add("cls.predictions.transform.dense.weight", (h, h), "head")
        spec.add("cls.predictions.transform.dense.bias", (h,), "head")
        spec.add("cls.predictions.transform.LayerNorm.weight", (h,), "head")
        spec.add("cls.predictions.transform.LayerNorm.bias", (h,), "head")
        if pre:
            spec.add("cls.seq_relationship.weight", (2, h), "head"); spec.add("cls.seq_relationship.bias", (2,), "head")
        self._bind_flat(spec, device, world_size)
        dev = self.flat.params.device
        P = self.P
        lin = lambda n: Linear.of(P(n + ".weight"), P(n + ".bias"))
        self._proj = [_Layer(Linear.span(self.flat, p + "attention.self.query.weight", 3 * h, h, p + "attention.self.query.bias"),
                             lin(p + "attention.output.dense"), lin(p + "intermediate.dense"), lin(p + "output.dense"))
                      for p in (f"bert.encoder.layer.{i}." for i in range(self.nl))]
        self._transform = lin("cls.predictions.transform.dense")
        self._decoder = Linear.of(P(E + "word_embeddings.weight"), P("cls.predictions.bias"))   # tied to the word embeddings
        if pre:
            self._pooler = lin("bert.pooler.dense")
            # NSP classifier padded to 8 outputs (pad logits = -30000 -> zero probability); parameters stay [2, h]
            self._nsp_w = torch.zeros(8, h, dtype=torch.bfloat16, device=dev)
            self._nsp_b = torch.full((8,), -30000.0, dtype=torch.bfloat16, device=dev)
        self.reset_parameters(seed)
        # dropout sites of one forward: 0 embeddings; for layer i, 1 + 3i attention probabilities, 2 + 3i attention output,
        # 3 + 3i FFN output
        self._init_dropout(1 + 3 * self.nl, (self.p_hidden, self.p_attn))

    @torch.no_grad()
    def reset_parameters(self, seed=0):
        std = getattr(self.config, "initializer_range", 0.02)
        gen = torch.Generator(device=self.flat.params.device).manual_seed(seed)
        for name, prm in self._p.items():
            if name.endswith("bias"):
                prm.zero_()
            elif "LayerNorm.weight" in name or name.endswith("ln.weight"):
                prm.fill_(1.0)
            else:
                prm.normal_(0.0, std, generator=gen)

    # ---- forward ----------------------------------------------------------------------------------------------------
    def forward(self, input_ids=None, attention_mask=None, token_type_ids=None, position_ids=None, labels=None,
                next_sentence_label=None, return_logits=False, **_):
        B, S = input_ids.shape
        dev = self.flat.params.device
        c = lambda t: flat_ids(t, dev)
        ids, tt, pos, lab = c(input_ids), c(token_type_ids), c(position_ids), c(labels)
        nsl = c(next_sentence_label)
        mask = key_mask(attention_mask, dev)
        loss, logits, nsp = self._step_or_forward(lab is not None, return_logits, ids, tt, pos, mask, lab, nsl, B, S)
        out = SimpleNamespace(loss=loss, logits=None if logits is None else logits.view(B, S, self.V),
                              hidden_states=None, attentions=None)
        out.prediction_logits = out.logits
        out.seq_relationship_logits = None if nsp is None else nsp[:, :2]
        return out

    def _forward_impl(self, ids, tt, pos, mask, lab, nsl, B, S, save, want_logits):
        h, nh, hn, pre = self.h, self.nh, self.hn, self.PRE_LN
        T = B * S
        P = self.P
        E = "bert.embeddings."
        scale = 1.0 / math.sqrt(hn)
        self._need("no_decay"); self._need("emb")
        base = self._dropout_base()
        ph, pa = self.p_hidden, self.p_attn
        D = lambda p, site: self._drop(base, p, site)
        emb = ops.embedding_fwd(ids, P(E + "word_embeddings.weight").data, pos=pos,
                                P=P(E + "position_embeddings.weight").data, token_type=tt,
                                T=P(E + "token_type_embeddings.weight").data, seq_len=S)
        acts = []
        if pre:
            x, prev_m, emb_ctx = emb, None, None
        else:
            x, st_e, _ = ops.layernorm_fwd(emb, P(E + "LayerNorm.weight").data, P(E + "LayerNorm.bias").data, self.eps)
            emb_ctx = (emb, st_e)
        x = apply_dropout(x, D(ph, 0))
        for i, pj in enumerate(self._proj):
            p = f"bert.encoder.layer.{i}."
            self._need(f"layer{i}")
            if pre:
                h1, st1, x = ops.layernorm_fwd(x if prev_m is None else prev_m, P(p + "attention.ln.weight").data,
                                               P(p + "attention.ln.bias").data, self.eps,
                                               residual=None if prev_m is None else x,
                                               drop=None if prev_m is None else D(ph, 3 * i))   # layer i-1's FFN output
                attn_in = h1
            else:
                attn_in = x
            qkv = pj.qkv(attn_in)
            q5 = qkv.view(B, S, 3, nh, hn)
            o, lse = ops.sdpa_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], scale, False, kv_mask=mask, drop=D(pa, 1 + 3 * i))
            a = pj.attn_out(o.view(T, h))
            if pre:
                h2, st2, x1 = ops.layernorm_fwd(a, P(p + "ln.weight").data, P(p + "ln.bias").data, self.eps, residual=x,
                                                drop=D(ph, 2 + 3 * i))
            else:
                h2, st2, x1 = ops.layernorm_fwd(a, P(p + "attention.output.LayerNorm.weight").data,
                                                P(p + "attention.output.LayerNorm.bias").data, self.eps, residual=x,
                                                drop=D(ph, 2 + 3 * i))
            prea = torch.empty((T, self.ff), dtype=torch.bfloat16, device=x.device) if save else None
            f = pj.inter(h2, epilogue=self.epi, aux=prea)
            m = pj.out(f)
            if pre:
                if save:
                    acts.append((x, st1, h1, qkv, o, lse, x1, st2, h2, prea, f))
                x, prev_m = x1, m
            else:
                xo, st3, s2 = ops.layernorm_fwd(m, P(p + "output.LayerNorm.weight").data,
                                                P(p + "output.LayerNorm.bias").data, self.eps, residual=h2,
                                                drop=D(ph, 3 + 3 * i))
                if save:
                    acts.append((x, qkv, o, lse, x1, st2, h2, prea, f, s2, st3))
                x = xo
        self._need("head")
        if pre:
            hf, stf, xf = ops.layernorm_fwd(prev_m, P("bert.encoder.ln.weight").data, P("bert.encoder.ln.bias").data,
                                            self.eps, residual=x, drop=D(ph, 3 * self.nl))
        else:
            hf, stf, xf = x, None, None
        # MLM head: dense + act + LN + tied decoder + bias (on every position)
        tpre = torch.empty((T, h), dtype=torch.bfloat16, device=hf.device) if save else None
        tf = self._transform(hf, epilogue=self.epi, aux=tpre)
        tn, stt, _ = ops.layernorm_fwd(tf, P("cls.predictions.transform.LayerNorm.weight").data,
                                       P("cls.predictions.transform.LayerNorm.bias").data, self.eps)
        logits = self._decoder(tn)
        loss, ctx, nsp_logits = None, None, None
        nsp_ctx = None
        if pre:
            first = hf.view(B, S, h)[:, 0, :]                     # strided [B, h] view, row stride S*h
            ppre = self._pooler(first)
            pooled = ops.act_fwd(L.ACT_TANH, ppre)
            self._nsp_w[:2].copy_(P("cls.seq_relationship.weight").data)
            self._nsp_b[:2].copy_(P("cls.seq_relationship.bias").data)
            nsp_logits = ops.gemm(L.GEMM_NT, pooled, self._nsp_w, bias=self._nsp_b)   # [B, 8]
            nsp_ctx = (first, ppre, pooled)
        if lab is not None:
            keep = logits.clone() if (want_logits and save) else None
            loss, dlogits, _ = ops.softmax_xent(logits, lab, S, shift=0, grad_scale=self.loss_scale,
                                                dlogits="inplace" if save else None)
            dnsp = None
            if pre and nsl is not None:
                keep_nsp = nsp_logits.clone()
                nloss, dnsp, _ = ops.softmax_xent(nsp_logits, nsl, 1, shift=0, grad_scale=self.loss_scale,
                                                  dlogits="inplace" if save else None)
                loss = loss + nloss                               # modeling_megatron_bert.py:776-779
                nsp_logits = keep_nsp
            if save:
                ctx = (acts, emb_ctx, hf, stf, xf, tpre, tf, stt, tn, dlogits, nsp_ctx, dnsp, ids, tt, pos, mask, B, S, base)
                logits = keep
        return loss, (logits if want_logits else None), nsp_logits, ctx

    # ---- backward ---------------------------------------------------------------------------------------------------
    def _backward_impl(self, ctx, gloss):
        acts, emb_ctx, hf, stf, xf, tpre, tf, stt, tn, dlogits, nsp_ctx, dnsp, ids, tt, pos, mask, B, S, base = ctx
        ph, pa = self.p_hidden, self.p_attn
        D = lambda p, site: self._drop(base, p, site)
        h, nh, hn, pre = self.h, self.nh, self.hn, self.PRE_LN
        T = B * S
        P = self.P
        acc = self.accumulate_grads
        self._begin_backward()
        E = "bert.embeddings."
        scale = 1.0 / math.sqrt(hn)
        if gloss is not None:
            ops.scale_inplace(dlogits, gloss)
            if dnsp is not None:
                ops.scale_inplace(dnsp, gloss)
        dtn = self._decoder.backward(dlogits, tn, acc)     # tied decoder: written first, the embedding adds later
        del dlogits
        lnw, lnb = P("cls.predictions.transform.LayerNorm.weight"), P("cls.predictions.transform.LayerNorm.bias")
        dtf = ops.layernorm_bwd(dtn, tf, lnw.data, stt, lnw.main_grad, lnb.main_grad, accumulate=acc)
        dtpre = ops.act_bwd(self.act, dtf, tpre)
        dhf = self._transform.backward(dtpre, hf, acc)
        if pre and dnsp is not None:
            first, ppre, pooled = nsp_ctx
            sw, sb = P("cls.seq_relationship.weight"), P("cls.seq_relationship.bias")
            dpooled = ops.gemm(L.GEMM_NN, dnsp, self._nsp_w)                     # [B, h]
            dw8 = ops.gemm(L.GEMM_TN, dnsp, pooled, out_dtype=torch.float32)     # [8, h]
            db8 = torch.zeros(8, dtype=torch.float32, device=dnsp.device)
            ops.colsum(dnsp, db8)
            if acc:
                sw.main_grad.add_(dw8[:2].to(sw.main_grad.dtype)); sb.main_grad.add_(db8[:2].to(sb.main_grad.dtype))
            else:
                sw.main_grad.copy_(dw8[:2]); sb.main_grad.copy_(db8[:2])
            dppre = ops.act_bwd(L.ACT_TANH, dpooled, ppre)
            self._pooler.backward(dppre, first, acc, dx=dhf.view(B, S, h)[:, 0, :], dx_accumulate=True)   # += into token 0 rows
        elif pre:
            for n in ("cls.seq_relationship.weight", "cls.seq_relationship.bias", "bert.pooler.dense.weight",
                      "bert.pooler.dense.bias"):
                if not acc:
                    P(n).main_grad.zero_()
        if pre:
            ew, eb = P("bert.encoder.ln.weight"), P("bert.encoder.ln.bias")
            dx, dmb = residual_norm_bwd(dhf, xf, ew, eb, stf, D(ph, 3 * self.nl), acc)
        else:
            dx = dhf
        self._done("head")          # after the final encoder LN: its weight gradient is in the head bucket
        for i in reversed(range(self.nl)):
            p, pj = f"bert.encoder.layer.{i}.", self._proj[i]
            if pre:
                x, st1, h1, qkv, o, lse, x1, st2, h2, prea, f = acts[i]
                dm, dres_in = dmb, dx                      # x_next = x1 + drop(m)
            else:
                x, qkv, o, lse, x1, st2, h2, prea, f, s2, st3 = acts[i]
                lw, lb = P(p + "output.LayerNorm.weight"), P(p + "output.LayerNorm.bias")
                dsum, dm = residual_norm_bwd(dx, s2, lw, lb, st3, D(ph, 3 + 3 * i), acc)   # d(h2 + drop(m)), d(m)
                dres_in = None
            acts[i] = None
            df = pj.out.backward(dm, f, acc)
            dprea = ops.act_bwd_bias(self.act, df, prea, pj.inter.bias_grad, accumulate=acc)   # dGELU + its bias grad
            if pre:
                dh2 = pj.inter.backward(dprea, h2, acc, colsum=False)
                lw, lb = P(p + "ln.weight"), P(p + "ln.bias")
                dx1, da = residual_norm_bwd(dh2, x1, lw, lb, st2, D(ph, 2 + 3 * i), acc, dres=dres_in)
            else:
                pj.inter.backward(dprea, h2, acc, dx=dsum, dx_accumulate=True, colsum=False)   # dh2 = d(h2+m) + dgrad(fc1)
                lw, lb = P(p + "attention.output.LayerNorm.weight"), P(p + "attention.output.LayerNorm.bias")
                dsum, da = residual_norm_bwd(dsum, x1, lw, lb, st2, D(ph, 2 + 3 * i), acc)       # d(x + drop(a)), d(a)
            do = pj.attn_out.backward(da, o.view(T, h), acc)
            dqkv = torch.empty_like(qkv)
            q5, d5 = qkv.view(B, S, 3, nh, hn), dqkv.view(B, S, 3, nh, hn)
            ops.sdpa_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o, do.view(B, S, nh, hn), lse, scale, False,
                         d5[:, :, 0], d5[:, :, 1], d5[:, :, 2], kv_mask=mask, drop=D(pa, 1 + 3 * i))
            if pre:
                dh1 = pj.qkv.backward(dqkv, h1, acc)
                lw, lb = P(p + "attention.ln.weight"), P(p + "attention.ln.bias")
                # layer 0's LN had no residual (x = the embeddings); layer i's summed layer i-1's dropped FFN output into x
                dx, dmb = residual_norm_bwd(dh1, x, lw, lb, st1, D(ph, 3 * i) if i > 0 else None, acc, dres=dx1)
            else:
                dx = pj.qkv.backward(dqkv, x, acc, dx=dsum, dx_accumulate=True)   # dx_in = d(x+a) + dgrad(qkv)
            self._done(f"layer{i}")
        dx = apply_dropout(dx, D(ph, 0))
        if not pre:
            emb, st_e = emb_ctx
            lw, lb = P(E + "LayerNorm.weight"), P(E + "LayerNorm.bias")
            dx = ops.layernorm_bwd(dx, emb, lw.data, st_e, lw.main_grad, lb.main_grad, accumulate=acc)
        ops.embedding_bwd(ids, dx, P(E + "word_embeddings.weight").main_grad)   # adds onto the tied decoder's weight gradient
        learned_pos_emb_bwd(pos, dx, P(E + "position_embeddings.weight").main_grad, B, S, acc)
        wtt = P(E + "token_type_embeddings.weight")
        # token types: dT = onehot(tt)^T dx as a (tiny-M) GEMM; all-zero types reduce to a column sum
        if tt is None:
            ops.colsum(dx, wtt.main_grad[0], accumulate=acc)
            if not acc:
                wtt.main_grad[1:].zero_()
        else:
            onehot = torch.zeros(T, 8, dtype=torch.bfloat16, device=dx.device)
            onehot.scatter_(1, tt.view(-1, 1), 1.0)
            d8 = ops.gemm(L.GEMM_TN, onehot, dx, out_dtype=torch.float32)
            if acc:
                wtt.main_grad.add_(d8[:self.ntype].to(wtt.main_grad.dtype))
            else:
                wtt.main_grad.copy_(d8[:self.ntype])
        self._done("emb")
        self._done("no_decay")


class BertForMaskedLM(_BertFamily):
    PRE_LN = False


class MegatronBertForPreTraining(_BertFamily):
    PRE_LN = True
