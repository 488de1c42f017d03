"""What the fsb200 model classes share with the ZeRO engine (fsb200/engine.py) and with each other, so that a model file holds
only its own maths:
  * parameters are views into one flat bf16 buffer (fsb200/flat.py), registered under the HF dotted names of the class the
    model stands in for, each with `.main_grad` over its slice of the flat gradient buffer;
  * the engine drives a model through `param_hook` / `grad_hook` / `backward_begin_hook`, `accumulate_grads` and `loss_scale`;
  * a training forward is ONE autograd node: it runs the model's `_forward_impl(save=True)` and `loss.backward()` runs its
    hand-written `_backward_impl`, which writes every gradient into the flat gradient buffer."""
import torch
from torch import nn

from .. import ops
from ..flat import FlatBuffers
from . import export
from .layers import WQ


class _Holder(nn.Module):
    """Bare container so that named_parameters() / state_dict() reproduce the reference's key names."""


def bind_flat_parameters(module, flat):
    """Register every entry of `flat` on `module`, in flat-layout order, as an nn.Parameter over its view with `.main_grad`
    over its gradient view (when `flat` has a gradient buffer), under its dotted name: `a.b.weight` becomes module.a.b.weight,
    and an integer component an nn.ModuleList entry (`transformer.h.3.*` -> module.transformer.h[3]). The parameters are also
    kept by name in module._p."""
    module._p = {}
    for name in flat.offsets:
        prm = nn.Parameter(flat.view(name), requires_grad=flat.grads is not None)
        if flat.grads is not None:
            prm.main_grad = flat.view(name, grad=True)
        module._p[name] = prm
        parts = name.split(".")
        mod = module
        for part, nxt in zip(parts[:-1], parts[1:]):
            if part not in mod._modules:   # a ModuleList's entries are named "0", "1", ...: they arrive in index order
                mod.add_module(part, nn.ModuleList() if nxt.isdigit() else _Holder())
            mod = mod._modules[part]
        setattr(mod, parts[-1], prm)


def flat_ids(t, dev):
    """Integer inputs (token ids, labels, position or token-type ids) as contiguous int64 [B * S] on `dev`; None stays None."""
    return None if t is None else t.to(device=dev, dtype=torch.int64).contiguous().view(-1)


def key_mask(attention_mask, dev):
    """The attention kernels' key-padding mask: uint8 [B, S] on `dev`, or None when there is no mask or no padding."""
    if attention_mask is None or bool(attention_mask.all()):
        return None
    return attention_mask.to(device=dev, dtype=torch.uint8).contiguous()


def packed_segments(segment_ids, lab, B, S, dev):
    """Packed-row inputs: segment_ids, integer [B, S] (host or device; a segment is a maximal run of equal consecutive values
    in a row), and the flat labels `lab` of a causal LM (int64 [B * S] or None). Returns ((seg_start, seg_end), labels): the
    attention bounds of ops.segment_bounds, and the labels with each segment's first token ignored (its prediction would
    cross a document boundary). Models whose targets are not shifted (the MLM encoders) pass lab=None."""
    if tuple(segment_ids.shape) != (B, S):
        raise ValueError(f"segment_ids must be [batch, seq] = [{B}, {S}], got {tuple(segment_ids.shape)}")
    seg_start, seg_end = ops.segment_bounds(segment_ids.to(device=dev, non_blocking=True))
    if lab is not None:   # a segment's first token is not a target of the previous segment's last
        first = (seg_start == torch.arange(S, dtype=torch.int32, device=dev)).view(-1)
        lab = lab.masked_fill(first, -100)
    return (seg_start, seg_end), lab


def cross_segment_bounds(dec_ids, enc_ids):
    """Cross-attention bounds of packed encoder-decoder rows (ops.sdpa_segments_fwd kv_bounds form): decoder segment x of
    row b attends to the encoder segment of row b with the same id value. dec_ids: integer [B, Sd], enc_ids: integer
    [B, Se], on one device, each non-decreasing along the row (so a segment is the run of one id). Returns
    ((kv_start, kv_end), (q_start, q_end)), contiguous int32 [B, Sd] and [B, Se]: the encoder positions each decoder token
    sees and the decoder positions that see each encoder token. An id with no match on the other side gets an empty range.
    Torch ops only, no host synchronisation (capturable in a CUDA graph): decreasing ids are refused exactly for host
    tensors and with an asynchronous device-side assert for device tensors."""
    for t, n in ((dec_ids, "decoder segment ids"), (enc_ids, "encoder segment ids")):
        if t.dim() != 2 or t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
            raise ValueError(f"{n} must be an integer [batch, seq] tensor, got {t.dtype} {tuple(t.shape)}")
    if dec_ids.shape[0] != enc_ids.shape[0] or dec_ids.device != enc_ids.device:
        raise ValueError(f"decoder and encoder segment ids must share batch and device, got {tuple(dec_ids.shape)} on "
                         f"{dec_ids.device} and {tuple(enc_ids.shape)} on {enc_ids.device}")
    dec, enc = dec_ids.to(torch.int64).contiguous(), enc_ids.to(torch.int64).contiguous()
    ordered = (dec[:, 1:] >= dec[:, :-1]).all() & (enc[:, 1:] >= enc[:, :-1]).all()
    msg = "segment ids must be non-decreasing along each row (samples placed in order)"
    if dec.is_cuda:
        torch._assert_async(ordered, msg)
    elif not bool(ordered):
        raise ValueError(msg)
    i32 = lambda t: t.to(torch.int32).contiguous()
    kv = (i32(torch.searchsorted(enc, dec, right=False)), i32(torch.searchsorted(enc, dec, right=True)))
    q = (i32(torch.searchsorted(dec, enc, right=False)), i32(torch.searchsorted(dec, enc, right=True)))
    return kv, q


def refuse_key_padding(attention_mask, model):
    """Packed rows carry no key mask: an attention_mask with zeros together with segment_ids is refused, exactly on the host
    and with an asynchronous device-side assert on the device (no synchronisation, so a CUDA-graph step stays capturable).
    `model` names the class in the message."""
    if attention_mask is None:
        return
    if attention_mask.is_cuda:
        torch._assert_async((attention_mask != 0).all(),
                            f"fsb200 {model}: attention_mask has zeros together with segment_ids; packed rows "
                            "need no key mask (the pad tail is a segment of its own)")
    elif not bool((attention_mask != 0).all()):
        raise ValueError(f"fsb200 {model}: attention_mask has zeros together with segment_ids; packed rows need no "
                         "key mask (the pad tail is a segment of its own)")


def learned_pos_emb_bwd(pos, dx, grad, B, S, accumulate):
    """Gradient of a learned absolute position table ([positions, h], `grad` = its main_grad) from the gradient dx [B * S, h]
    of the embedding sum. Without position ids row s is sum_b dx[b, s] (a column sum of dx viewed as [B, S * h]); with them,
    a scatter-add by id. Rows no token used are zeroed unless gradients accumulate."""
    if pos is None:
        ops.colsum(dx.view(B, S * grad.shape[1]), grad[:S].reshape(-1), accumulate=accumulate)
        if not accumulate and S < grad.shape[0]:
            grad[S:].zero_()
    else:
        if not accumulate:
            grad.zero_()
        ops.embedding_bwd(pos, dx, grad)


class FlatModel(nn.Module):
    """Base of the fsb200 model classes. A subclass parses its config, builds its FlatSpec, calls `_bind_flat`, and implements
    `_forward_impl(*inputs, save, want_logits) -> (loss, *outputs, saved)` and `_backward_impl(saved, gloss)`."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.accumulate_grads = False   # set by the engine for micro-batches after the first
        self.loss_scale = 1.0           # 1 / (gradient_accumulation_steps * world_size), folded into dlogits
        self.grad_hook = None           # engine callback: grad_hook(bucket) when a bucket's gradients are final

    def _bind_flat(self, spec, device=None, world_size=None, tp=1, grads=True):
        """Allocate the flat buffers for `spec` and bind every entry. `world_size` is the data-parallel size the buckets are
        padded for: by default the initialised process group's size over the tensor-parallel size `tp`. grads=False: no
        gradient buffer (inference-only models)."""
        if world_size is None:   # laid out for the job's data-parallel world (the scripts build the model in setup())
            import torch.distributed as dist
            world_size = (dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1) // tp
        dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}"
                           if torch.cuda.is_available() else "cuda")
        if dev.type != "cuda":
            raise RuntimeError(f"fsb200 {type(self).__name__} runs on CUDA only (no CPU fallback on the product path)")
        self.flat = FlatBuffers(spec, dev, world_size=world_size, grads=grads)
        bind_flat_parameters(self, self.flat)

    def P(self, name):
        return self._p[name]

    # ---- activation recompute (HF PreTrainedModel's gradient-checkpointing names) --------------------------------------
    supports_gradient_checkpointing = False   # a subclass that recomputes sets it and reads self.gradient_checkpointing
    gradient_checkpointing = False

    @property
    def is_gradient_checkpointing(self):
        return self.gradient_checkpointing

    def gradient_checkpointing_enable(self, gradient_checkpointing_kwargs=None):
        """Recompute activations in the backward instead of keeping them. gradient_checkpointing_kwargs (HF passes them on to
        torch.utils.checkpoint, e.g. use_reentrant) are accepted and ignored: the recompute is the model's own."""
        if not self.supports_gradient_checkpointing:
            raise NotImplementedError(f"fsb200 {type(self).__name__}: activation recompute (gradient checkpointing) is not "
                                      "implemented for this model; it keeps every layer's activations")
        self.gradient_checkpointing = True

    def gradient_checkpointing_disable(self):
        self.gradient_checkpointing = False

    # The reference scripts call `.from_pretrained(..., torch_dtype=torch.half).cuda()`; parameters here are views into the
    # flat bf16 CUDA buffer and must never be re-allocated by nn.Module._apply.
    def cuda(self, device=None):
        return self

    def half(self):
        return self

    def bfloat16(self):
        return self

    def to(self, *args, **kwargs):
        return self

    @torch.no_grad()
    def load_reference_state_dict(self, sd):
        """Copy a reference state dict (HF key names; fp32 / fp16 / bf16 tensors on any device) into the parameters. Every
        parameter's key must be present with its shape; other keys (tied aliases, buffers) are ignored. An int8 / int4
        model quantises each projection on the device as it arrives (_load_quantized_shard)."""
        if self.weight_format != "bf16":
            missing = (set(self._p) | set(self._wq_targets())) - set(sd)
            if missing:
                raise KeyError(f"missing key in state dict: {sorted(missing)[0]}")
            self._load_quantized_shard(sd, set())
            return
        for k, prm in self._p.items():
            if k not in sd:
                raise KeyError(f"missing key in state dict: {k}")
            if tuple(sd[k].shape) != tuple(prm.shape):
                raise ValueError(f"shape mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(prm.shape)}")
        for k, prm in self._p.items():
            prm.copy_(sd[k].to(device=prm.device, dtype=prm.dtype))

    def save_pretrained(self, path, **_):
        """HF-style export (config.json + pytorch_model.bin with this class's HF key names): fsb200/models/export.py."""
        export.save_pretrained(self, path)

    # ---- int8 / int4 inference-only models (load_in_8bit / load_in_4bit: LLaMA, GPT-2) -----------------------------------
    # Such a model holds its layer projections as layers.QuantizedLinear (q + s) outside the flat buffers and lists them in
    # `_wq` (per layer {projection: (q, s)}) and `_wq_targets()` ({state-dict key: (q, s) it quantises into}).
    weight_format = "bf16"   # "int8" / "int4" for those models
    wq_transposed = False    # the checkpoint stores the projections [in, out] (GPT-2's Conv1D), the transpose of [n, k]

    @staticmethod
    def _weight_shape(q, s):
        """[n, k] of the bf16 weight that (q, s) holds: s has one row per weight row in both formats, q the k columns."""
        return s.shape[0], q.shape[1]

    @torch.no_grad()
    def _load_quantized_shard(self, sd, loaded):
        """Load the keys of `sd` (a whole state dict or one checkpoint shard) this int8 / int4 model holds: bf16 parameters
        are copied, projections quantised on the device (one bf16 temporary at a time, transposed first when the checkpoint
        stores them [in, out]). The shard's shapes are checked before anything is written. Adds the loaded keys to the set
        `loaded` and returns the keys it does not yet hold."""
        targets = self._wq_targets()
        for k, v in sd.items():
            want = None
            if k in self._p:
                want = tuple(self._p[k].shape)
            elif k in targets:
                want = tuple(self._weight_shape(*targets[k]))
                want = want[::-1] if self.wq_transposed else want
            if want is not None and tuple(v.shape) != want:
                raise ValueError(f"shape mismatch for {k}: {tuple(v.shape)} vs {want}")
        for k, v in sd.items():
            v = v if v.dtype == torch.bfloat16 else v.to(torch.bfloat16)   # converted where it lies: one bf16 copy on the device
            if k in self._p:
                self._p[k].copy_(v)
            elif k in targets:
                q, s = targets[k]
                tmp = v.to(q.device)
                tmp = (tmp.t() if self.wq_transposed else tmp).contiguous()
                WQ[self.weight_format][0](tmp, q, s)
                del tmp
            else:
                continue
            loaded.add(k)
        return (set(self._p) | set(targets)) - loaded

    def get_memory_footprint(self):
        """Bytes held by the model's tensors: parameters (and their gradient buffer, if any), int8 / int4 weights and scales, and
        buffers (transformers' `PreTrainedModel.get_memory_footprint`, which hf_quantizatin_inference.py prints)."""
        n = self.flat.params.numel() * self.flat.params.element_size()
        if self.flat.grads is not None:
            n += self.flat.grads.numel() * self.flat.grads.element_size()
        for wq in self._wq if self.weight_format != "bf16" else ():
            n += sum(q.numel() * q.element_size() + s.numel() * s.element_size() for q, s in wq.values())
        return n + sum(b.numel() * b.element_size() for b in self.buffers())

    # ---- engine hooks -----------------------------------------------------------------------------------------------
    def _need(self, bucket):
        """Forward is about to read this bucket's parameters (the engine may still be all-gathering them)."""
        hook = getattr(self, "param_hook", None)
        if hook is not None:
            hook(bucket)

    def _done(self, bucket):
        """This bucket's gradients are final. A bucket the layout lacks (mT5's "head" with a tied LM head) is skipped."""
        if self.grad_hook is not None and bucket in self.flat.bucket_index:
            self.grad_hook(bucket)

    def _begin_backward(self):
        hook = getattr(self, "backward_begin_hook", None)
        if hook is not None:
            hook()

    # ---- dropout ----------------------------------------------------------------------------------------------------
    # Masks come from Philox (include/fsb200.h): a seed drawn once from torch.default_generator at construction (only when a
    # probability is > 0) and a device stream counter that every training forward advances by its number of sites, so eager
    # runs and replayed CUDA graphs draw the same fresh masks. In eval mode, or with every probability 0, the forward and
    # backward run the dropout-free kernels.
    def _dropout_probs(self, model, *keys):
        """The config's dropout probabilities `keys` (absent or None: 0), each checked to lie in [0, 1)."""
        probs = tuple(float(getattr(self.config, k, 0.0) or 0.0) for k in keys)
        for k, v in zip(keys, probs):
            if not 0.0 <= v < 1.0:
                raise RuntimeError(f"fsb200 {model}: {k}={v} outside [0, 1)")
        return probs

    def _init_dropout(self, sites, probs):
        """`sites` dropout sites per forward; the seed and the stream counter when one of `probs` is > 0, else None."""
        self.dropout_sites = sites
        self.dropout_seed, self.dropout_counter = None, None
        if max(probs) > 0:
            self.dropout_seed = int(torch.randint(0, 2 ** 63 - 1, (1,), generator=torch.default_generator).item())
            self.dropout_counter = torch.zeros(1, dtype=torch.int64, device=self.flat.params.device)

    def _dropout_base(self):
        """The stream base of this forward's masks, advancing the counter; None (no dropout) unless training with a seed."""
        if not self.training or self.dropout_seed is None:
            return None
        return ops.dropout_advance(self.dropout_counter, self.dropout_sites)

    def _drop(self, base, p, site):
        """The Dropout of one site of the forward whose stream base is `base` (None: no dropout in that forward)."""
        return None if base is None or p == 0.0 else ops.Dropout(p, self.dropout_seed, base, site)

    def _refuse_dropout_generate(self, model, keys):
        """generate runs without dropout: in training mode with a probability > 0 it raises (HF would drop)."""
        if self.training and self.dropout_seed is not None:
            raise RuntimeError(f"fsb200 {model}: generate in training mode with {keys} > 0 would drop; call model.eval() first")

    # ---- forward ----------------------------------------------------------------------------------------------------
    def _step_or_forward(self, has_labels, want_logits, *inputs):
        """-> (loss, *outputs). With labels under grad mode, the step node: `loss.backward()` then runs `_backward_impl`.
        Otherwise a forward that keeps no activations (and always returns the logits)."""
        if has_labels and torch.is_grad_enabled():
            return _Step.apply(self, want_logits, next(iter(self._p.values())), *inputs)
        return self._forward_impl(*inputs, save=False, want_logits=True)[:-1]


class _Step(torch.autograd.Function):
    """The whole network as one autograd node. `anchor`, a parameter, makes the node differentiable; its .grad is never
    materialised: the kernels write the gradients into model.flat.grads."""

    @staticmethod
    def forward(ctx, model, want_logits, anchor, *inputs):
        loss, *outputs, saved = model._forward_impl(*inputs, save=True, want_logits=want_logits)
        ctx.model, ctx.saved, ctx.n_args = model, saved, 3 + len(inputs)
        ctx.mark_non_differentiable(*[t for t in outputs if t is not None])
        return (loss, *outputs)

    @staticmethod
    def backward(ctx, gloss, *_):
        saved, ctx.saved = ctx.saved, None
        ctx.model._backward_impl(saved, gloss)
        return (None,) * ctx.n_args
