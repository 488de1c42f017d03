"""Packed batches for causal-LM fine-tuning: several samples per row instead of one padded sample per row.

The Ziya-LLaMA SFT recipe (examples/ziya_llama/finetune_ziya_llama.py:36-85, `LlamaSFTCollator`) pads every micro-batch to
its longest sample; the pads carry label -100 and cost a full forward and backward each. `pack_causal_lm_batch` takes that
collator's output and places the samples one after another into rows of exactly `max_seq_length` tokens, first fit in sample
order, with `segment_ids` that keep attention inside each sample (LlamaForCausalLM.forward(segment_ids=...)) and position ids
that restart at 0 in each sample, so every sample sees the RoPE positions it had in the padded batch.

The Wenzhong-GPT2 QA recipe's batches have the same format: `GPT2QADataset.encode` pads every question + answer to
`max_seq_length` with eos (its pad), labels -100 on every pad, and `default_collate` adds the `question` / `answer` strings,
which the packer ignores. An eos inside the text is unlabelled there too, and stays an input. Packed, they feed
GPT2LMHeadModel.forward(segment_ids=...), whose learned position embeddings then see each sample's own positions 0, 1, ...

`PackingCollator(inner, max_seq_length, pad_id)` wraps any collator that emits that format (`default_collate` for the GPT-2
dataset), so a script's own collator runs unchanged inside it. The number of rows varies from batch to batch; the samples handed to the collator do not change, so
consumed-sample accounting is unaffected.
"""
import torch

IGNORE_INDEX = -100


def _kept_prefix(ids, labels, max_seq_length):
    """The tokens of one padded row that can influence its loss: up to and including its last labelled token (under causal
    attention nothing after it reaches a loss term), at most max_seq_length of them. None when no token is labelled."""
    ids, labels = ids[:max_seq_length], labels[:max_seq_length]
    where = (labels != IGNORE_INDEX).nonzero()
    if where.numel() == 0:
        return None
    n = int(where[-1]) + 1
    return ids[:n], labels[:n]


def first_fit(lengths, max_seq_length):
    """Rows for samples of the given lengths (each <= max_seq_length), first fit in sample order: each sample goes into the
    first row with room left, else into a new row. Returns a list of rows, each a list of sample indices."""
    rows, free = [], []
    for i, n in enumerate(lengths):
        for r, room in enumerate(free):
            if n <= room:
                rows[r].append(i)
                free[r] -= n
                break
        else:
            rows.append([i])
            free.append(max_seq_length - n)
    return rows


def pack_causal_lm_batch(batch, max_seq_length, pad_id):
    """batch: `input_ids` and `labels` [n, L] (tensors or nested lists), pad-filled, labels -100 on prompts and pads.
    Returns a dict of [rows, max_seq_length] tensors: `input_ids` (pad_id after the last sample of a row), `labels` (-100 on
    segment starts and pads), `attention_mask` (ones), `position_ids` (0, 1, ... in each segment), `segment_ids` (0, 1, ...
    per row; the pad tail is a segment of its own). Rows without a labelled token are dropped; a batch with none left packs
    into one all-pad row whose labels are all ignored. LlamaForCausalLM gives such a batch a loss of exactly 0 and zero
    gradients (its cross-entropy divides by max(labelled targets, 1)), so a training step on it changes the weights only
    through AdamW's momentum and weight decay, as a padded batch without labels would."""
    ids = torch.as_tensor(batch["input_ids"], dtype=torch.int64)
    labels = torch.as_tensor(batch["labels"], dtype=torch.int64)
    if ids.dim() != 2 or ids.shape != labels.shape:
        raise ValueError(f"input_ids and labels must be [n, L] of one shape, got {tuple(ids.shape)} and {tuple(labels.shape)}")
    if max_seq_length <= 0:
        raise ValueError(f"max_seq_length must be positive, got {max_seq_length}")
    kept = [p for p in (_kept_prefix(i, l, max_seq_length) for i, l in zip(ids, labels)) if p is not None]
    rows = first_fit([len(p[0]) for p in kept], max_seq_length) or [[]]
    R, S = len(rows), max_seq_length
    out_ids = torch.full((R, S), pad_id, dtype=torch.int64)
    out_lab = torch.full((R, S), IGNORE_INDEX, dtype=torch.int64)
    out_pos = torch.zeros((R, S), dtype=torch.int64)
    out_seg = torch.zeros((R, S), dtype=torch.int64)
    for r, members in enumerate(rows):
        t = 0
        for k, i in enumerate(members):
            pi, pl = kept[i]
            n = len(pi)
            out_ids[r, t:t + n] = pi
            out_lab[r, t:t + n] = pl
            out_lab[r, t] = IGNORE_INDEX          # predicted from the previous segment's last token: not a target
            out_pos[r, t:t + n] = torch.arange(n)
            out_seg[r, t:t + n] = k
            t += n
        if t < S:                                  # pad tail: its own segment, positions from 0, no labels
            out_pos[r, t:] = torch.arange(S - t)
            out_seg[r, t:] = len(members)
    return {"input_ids": out_ids, "labels": out_lab, "attention_mask": torch.ones((R, S)),
            "position_ids": out_pos, "segment_ids": out_seg}


class PackingCollator:
    """collate(samples) = pack_causal_lm_batch(inner(samples), max_seq_length, pad_id)."""

    def __init__(self, inner, max_seq_length, pad_id):
        self.inner, self.max_seq_length, self.pad_id = inner, int(max_seq_length), int(pad_id)

    def __call__(self, samples):
        return pack_causal_lm_batch(self.inner(samples), self.max_seq_length, self.pad_id)
