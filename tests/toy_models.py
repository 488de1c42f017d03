"""TEST DOUBLES — torch-CPU stand-ins for the fsb200 model classes, with the SAME engine-facing surface (flat bucketed storage,
`grad_hook` / `param_hook` / `backward_begin_hook`, `accumulate_grads`, `loss_scale`, HF-named parameters, autograd entry through
one Function) and a deliberately trivial network (embedding -> tied output projection). They let `-m "not gpu"` tests drive the
whole host side — fsb200.launch, fsb200.hf rebinding, the compat Trainer, ZeroEngine (with tests/cpu_kernels.py), checkpoints,
resume, export — without a GPU. Never importable from the product package: they live under tests/."""
from types import SimpleNamespace

import torch
from torch import nn

from fsb200.flat import FlatBuffers, FlatSpec
from fsb200.models.base import bind_flat_parameters


class _ToyBase(nn.Module):
    H = 16

    def _spec(self, V, h):
        raise NotImplementedError

    def __init__(self, config, device=None, world_size=None, seed=0):
        super().__init__()
        self.config = config
        self.V = config.vocab_size
        if world_size is None:   # as the real models: the initialised process group decides
            import torch.distributed as dist
            world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.flat = FlatBuffers(self._spec(self.V, self.H), "cpu", world_size=world_size)
        bind_flat_parameters(self, self.flat)
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, prm in self._p.items():
                prm.copy_((torch.randn(prm.shape, generator=g) * 0.02).to(torch.bfloat16))
                if name.endswith("layer_norm.weight"):
                    prm.fill_(1.0)
        self.accumulate_grads, self.loss_scale, self.grad_hook = False, 1.0, None

    def load_reference_state_dict(self, sd):
        with torch.no_grad():
            for k, v in sd.items():
                self._p[k].copy_(v.to(torch.bfloat16))

    def save_pretrained(self, path, **_):
        from fsb200.models.export import save_pretrained
        save_pretrained(self, path)

    def cuda(self, device=None):
        return self

    def _loss(self, w, batch):
        raise NotImplementedError

    def forward(self, **batch):
        batch = {k: v for k, v in batch.items() if isinstance(v, torch.Tensor)}
        hook = getattr(self, "param_hook", None)
        if hook is not None:
            for b, _, _, _ in self.flat.buckets:
                hook(b)
        if torch.is_grad_enabled() and batch.get("labels") is not None:
            anchor = next(iter(self._p.values()))
            loss, logits = _ToyStep.apply(self, batch, anchor)
        else:
            with torch.no_grad():
                loss, logits = self._loss({k: p.detach().float() for k, p in self._p.items()}, batch)
        return SimpleNamespace(loss=loss, logits=logits, prediction_logits=logits)


class _ToyStep(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, batch, _anchor):
        with torch.enable_grad():
            leaves = {k: p.detach().float().requires_grad_() for k, p in model._p.items()}
            loss, logits = model._loss(leaves, batch)
        ctx.model, ctx.graph = model, (loss, leaves)
        out_logits = logits.detach().to(torch.bfloat16)
        ctx.mark_non_differentiable(out_logits)
        return loss.detach().clone(), out_logits

    @staticmethod
    def backward(ctx, gloss, _gl):
        model = ctx.model
        loss, leaves = ctx.graph
        ctx.graph = None
        names = list(leaves)
        grads = torch.autograd.grad(loss, [leaves[n] for n in names], gloss * model.loss_scale, allow_unused=True)
        gmap = dict(zip(names, grads))
        begin = getattr(model, "backward_begin_hook", None)
        if begin is not None:
            begin()
        fb = model.flat
        for b, start, length, _ in reversed(fb.buckets):     # a bucket's gradients are complete before it is reported
            for name, (off, _) in fb.offsets.items():
                if start <= off < start + length:
                    g = gmap[name]
                    gv = model._p[name].main_grad
                    g16 = torch.zeros_like(gv) if g is None else g.to(torch.bfloat16)
                    if model.accumulate_grads:
                        gv.copy_((gv.float() + g16.float()).to(torch.bfloat16))
                    else:
                        gv.copy_(g16)
            if model.grad_hook is not None:
                model.grad_hook(b)
        return None, None, None


class ToyMegatronBert(_ToyBase):
    """MLM over a tied embedding + a sentence-order head on the mean token embedding (keys named as in MegatronBERT)."""

    def _spec(self, V, h):
        s = FlatSpec()
        s.add("bert.embeddings.word_embeddings.weight", (V, h), "emb")
        s.add("bert.embeddings.token_type_embeddings.weight", (2, h), "emb")
        s.add("cls.predictions.bias", (V,), "head")
        s.add("cls.seq_relationship.weight", (2, h), "head")
        s.add("cls.seq_relationship.bias", (2,), "head")
        return s

    def _loss(self, w, batch):
        E = w["bert.embeddings.word_embeddings.weight"]
        x = E[batch["input_ids"]] + w["bert.embeddings.token_type_embeddings.weight"][batch["token_type_ids"]]
        # one step of context mixing, so that masked positions can be predicted from their neighbours
        am = batch["attention_mask"].float().unsqueeze(-1)
        ctxv = (x * am).sum(1, keepdim=True) / am.sum(1, keepdim=True).clamp(min=1)
        hid = x + ctxv
        logits = hid @ E.t() + w["cls.predictions.bias"]
        loss = nn.functional.cross_entropy(logits.view(-1, self.V), batch["labels"].view(-1), ignore_index=-100)
        if batch.get("next_sentence_label") is not None:
            nsp = ctxv[:, 0] @ w["cls.seq_relationship.weight"].t() + w["cls.seq_relationship.bias"]
            loss = loss + nn.functional.cross_entropy(nsp, batch["next_sentence_label"].view(-1))
        return loss, logits


class ToyGPT2(_ToyBase):
    """Next-token prediction from the current token + position through a tied embedding (keys named as in GPT-2)."""

    def _spec(self, V, h):
        s = FlatSpec()
        s.add("transformer.wte.weight", (V, h), "wte")
        s.add("transformer.wpe.weight", (getattr(self.config, "n_positions", 128), h), "wte")
        s.add("transformer.ln_f.bias", (h,), "head")
        return s

    def _loss(self, w, batch):
        E = w["transformer.wte.weight"]
        ids = batch["input_ids"]
        S = ids.shape[1]
        hid = E[ids] + w["transformer.wpe.weight"][:S] + w["transformer.ln_f.bias"]
        logits = hid @ E.t()
        loss = None
        if batch.get("labels") is not None:
            loss = nn.functional.cross_entropy(logits[:, :-1].reshape(-1, self.V), batch["labels"][:, 1:].reshape(-1),
                                               ignore_index=-100)
        return loss, logits


class ToyMT5(_ToyBase):
    """Decoder token + mean encoder embedding -> tied output projection (keys named as in mT5 with a tied head)."""

    def _spec(self, V, h):
        s = FlatSpec()
        s.add("shared.weight", (V, h), "shared")
        s.add("decoder.final_layer_norm.weight", (h,), "head")
        return s

    def _loss(self, w, batch):
        E = w["shared.weight"]
        labels = batch.get("labels")
        dec = batch.get("decoder_input_ids")
        if dec is None:
            dec = torch.zeros_like(labels)
            dec[:, 1:] = labels[:, :-1]
            dec = dec.masked_fill(dec == -100, 0)
        hid = (E[dec] + E[batch["input_ids"]].mean(1, keepdim=True)) * w["decoder.final_layer_norm.weight"]
        logits = hid @ E.t()
        loss = None if labels is None else nn.functional.cross_entropy(logits.view(-1, self.V), labels.reshape(-1),
                                                                      ignore_index=-100)
        return loss, logits
