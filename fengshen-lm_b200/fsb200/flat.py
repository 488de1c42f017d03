"""Flat, bucketed parameter / gradient storage shared by the models and the ZeRO engine.

All 16-bit parameters live in ONE contiguous bf16 buffer (gradients in a parallel buffer) — the layout DeepSpeed's
ZeRO-1/2 optimizer creates by flattening (SURVEY.md Appendix D) — cut into BUCKETS (one per transformer layer, plus
embeddings, LM head and one bucket for every no-weight-decay parameter). Each bucket is padded to a multiple of
world_size*ALIGN so that data-parallel rank r owns the r-th equal slice of EVERY bucket:
  * a bucket's gradients can be reduce-scattered the moment its layer's backward finishes (overlap with backward);
  * the rank's optimizer state is the concatenation of its bucket slices (a contiguous local fp32 shard);
  * after the update each bucket is re-assembled with one in-place all-gather.
A bucket is homogeneous in weight decay (the grouping BY NAME of fengshen/models/model_utils.py:39-47), so the fused
AdamW kernel runs once per bucket slice.
"""
import torch

NO_DECAY_SUBSTRINGS = ['bias', 'LayerNorm.bias', 'LayerNorm.weight', 'layer_norm.', 'layernorm.']  # model_utils.py:40
ALIGN = 128  # elements: every parameter starts 256-byte aligned (TMA needs 16 B, vector kernels 16 B)
NO_DECAY_BUCKET = "no_decay"


def is_no_decay(name):
    return any(nd in name for nd in NO_DECAY_SUBSTRINGS)


def _numel(shape):
    n = 1
    for s in shape:
        n *= s
    return n


class FlatSpec:
    """Ordered list of (name, shape, bucket). Entries of one bucket are laid out adjacently in registration order."""

    def __init__(self):
        self.entries = []

    def add(self, name, shape, bucket):
        self.entries.append((name, tuple(shape), NO_DECAY_BUCKET if is_no_decay(name) else bucket))

    def plan(self, world_size=1):
        """-> (offsets {name: (offset, shape)}, buckets [(bucket, start, length, weight_decay_on)], total)."""
        order = []
        for _, _, b in self.entries:
            if b not in order and b != NO_DECAY_BUCKET:
                order.append(b)
        if any(b == NO_DECAY_BUCKET for _, _, b in self.entries):
            order.append(NO_DECAY_BUCKET)
        gran = world_size * ALIGN
        offsets, buckets, cur = {}, [], 0
        for b in order:
            start = cur
            for name, shape, bb in self.entries:
                if bb != b:
                    continue
                offsets[name] = (cur, shape)
                cur += (_numel(shape) + ALIGN - 1) // ALIGN * ALIGN
            cur = start + (cur - start + gran - 1) // gran * gran
            buckets.append((b, start, cur - start, b != NO_DECAY_BUCKET))
        return offsets, buckets, cur


class FlatBuffers:
    """Owns the flat bf16 parameter and gradient buffers and hands out views. grads=False allocates no gradient buffer
    (`grads` is None): a model that only runs inference (an int8 LLaMA) then holds its parameters alone."""

    def __init__(self, spec, device, world_size=1, grad_dtype=torch.bfloat16, grads=True):
        self.offsets, self.buckets, self.total = spec.plan(world_size)
        self.world_size = world_size
        self.params = torch.zeros(self.total, dtype=torch.bfloat16, device=device)
        self.grads = torch.zeros(self.total, dtype=grad_dtype, device=device) if grads else None
        self.bucket_index = {b: i for i, (b, _, _, _) in enumerate(self.buckets)}
        # gradient-space layout: identical to the parameter layout until compact_grads() folds the per-layer buckets
        # onto rotating slots (ZeRO-2: a full-size gradient buffer never exists)
        self.grad_bucket_start = [start for _, start, _, _ in self.buckets]
        self.grad_total = self.total
        self.rot_group = [None] * len(self.buckets)   # bucket -> (group name, slot) when its gradients live in a rotating slot
        self._grad_views = []                         # (tensor, parameter-space offset, shape) of every grad view handed out
        # local shard layout: concatenation of this rank's slice of every bucket
        self.shard_offsets, cur = [], 0
        for _, _, length, _ in self.buckets:
            self.shard_offsets.append(cur)
            cur += length // world_size
        self.shard_numel = cur

    def _bucket_of(self, off):
        for i, (_, start, length, _) in enumerate(self.buckets):
            if start <= off < start + length:
                return i
        raise ValueError(f"offset {off} outside the flat buffer")

    def _grad_off(self, off):
        i = self._bucket_of(off)
        return self.grad_bucket_start[i] + (off - self.buckets[i][1])

    def _grad_view(self, off, shape):
        if self.grads is None:
            raise RuntimeError("fsb200: these flat buffers were built without a gradient buffer")
        g = self._grad_off(off)
        t = self.grads[g:g + _numel(shape)].view(shape)
        self._grad_views.append((t, off, tuple(shape)))
        return t

    def view(self, name, grad=False):
        off, shape = self.offsets[name]
        if grad:
            return self._grad_view(off, shape)
        return self.params[off:off + _numel(shape)].view(shape)

    def span(self, first_name, rows, cols, grad=False):
        """[rows, cols] view starting at `first_name` and covering the adjacent entries after it (fused GEMM operand)."""
        off, _ = self.offsets[first_name]
        covered, cur = 0, off
        for name, (o, shape) in sorted(self.offsets.items(), key=lambda kv: kv[1][0]):
            if o < off or covered >= rows * cols:
                continue
            if o != cur:
                raise ValueError(f"span({first_name}): entries are not contiguous at {name} (padding in between)")
            covered += _numel(shape)
            cur = o + _numel(shape)
        if covered != rows * cols:
            raise ValueError(f"span({first_name}): {rows}x{cols} does not end on a parameter boundary")
        if grad:
            return self._grad_view(off, (rows, cols))
        return self.params[off:off + rows * cols].view(rows, cols)

    def bucket_slice(self, i, rank, grad=False):
        """Rank `rank`'s slice of bucket i inside the flat buffer."""
        _, start, length, _ = self.buckets[i]
        per = length // self.world_size
        if grad:
            start = self.grad_bucket_start[i]
        buf = self.grads if grad else self.params
        return buf[start + rank * per: start + (rank + 1) * per]

    def bucket_view(self, i, grad=False):
        _, start, length, _ = self.buckets[i]
        if grad:
            start = self.grad_bucket_start[i]
        buf = self.grads if grad else self.params
        return buf[start:start + length]

    # ---- ZeRO-2 gradient storage ------------------------------------------------------------------------------------
    def compact_grads(self, slots=2, min_group=3):
        """Fold every family of equally sized per-layer buckets (`layer0..layerN`, `enc0..`, `dec0..`) onto `slots` rotating
        gradient slots: bucket k of a family writes slot k % slots. The engine reduce-scatters a slot before backward reaches
        the layer that reuses it, so gradients of at most `slots` layers of a family exist at any time — DeepSpeed ZeRO-2's
        "gradients are partitioned as they are produced" (SURVEY.md Appendix D) instead of a full-size buffer. Every grad view
        handed out so far (prm.main_grad, fused-operand spans) is re-pointed in place. A tensor derived from such a view
        (`.view(-1)`, a slice) is not re-pointed and keeps writing the released buffer, so a model must not keep one across
        construction: it keeps the view and derives at the point of use. Returns the bytes released."""
        import re
        if self.grads is None:
            return 0
        fam = {}
        for i, (name, _, length, _) in enumerate(self.buckets):
            m = re.fullmatch(r"(.*?)(\d+)", name)
            if m:
                fam.setdefault((m.group(1), length), []).append((int(m.group(2)), i))
        starts, cur = [None] * len(self.buckets), 0
        rot = [None] * len(self.buckets)
        fam_base = {}
        for i, (name, _, length, _) in enumerate(self.buckets):
            key = next((k for k, v in fam.items() if any(bi == i for _, bi in v) and len(v) >= min_group), None)
            if key is None:
                starts[i] = cur
                cur += length
                continue
            if key not in fam_base:
                fam_base[key] = cur
                cur += slots * length
            k = next(idx for idx, bi in fam[key] if bi == i)
            rot[i] = (key[0], k % slots)
            starts[i] = fam_base[key] + (k % slots) * length
        if not fam_base:
            return 0
        new = torch.zeros(cur, dtype=self.grads.dtype, device=self.grads.device)
        self.grad_bucket_start, self.grad_total, self.rot_group = starts, cur, rot
        old_bytes = self.grads.numel() * self.grads.element_size()
        self.grads = new
        for t, off, shape in self._grad_views:
            g = self._grad_off(off)
            t.set_(new.untyped_storage(), g, shape)
        return old_bytes - cur * new.element_size()
