"""Packed batches: several samples per row instead of one padded sample per row, for causal-LM fine-tuning and for BERT /
MegatronBERT MLM + sentence-order pretraining.

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

The Erlangshen MLM recipe (`ErLangShenCollator` / `FastErLangShenCollator`, fengshen/data/data_utils/collators.py) pads every
document to `max_seq_length` (512 for MegatronBERT-1.3B). `pack_mlm_batch` keeps each sample's whole non-pad prefix (attention
is bidirectional, so every token of a sample matters, labelled or not), places the samples first fit into rows of exactly
`max_seq_length`, and adds the `cls_positions` of each sample's [CLS] for the sentence-order head
(MegatronBertForPreTraining.forward(segment_ids=..., cls_positions=...)). `MLMPackingCollator` wraps those collators.

The mT5 / Randeng-T5 fine-tuning recipes pad both sides: `LCSTSDataset.encode` (fengshen/data/task_dataloader/
task_datasets.py) pads the source to `max_enc_length` and the summary to `max_dec_length` with `padding='max_length'`, and
`TaskT5Dataset.encode` (t5_datasets.py, used by finetune_t5.py and qa_t5) pads the source to `max_seq_length` and the target
to 16. `pack_seq2seq_batch` keeps each sample's source (its non-pad prefix) and target (its labels up to the last labelled
one) and places the samples first fit into encoder rows of `max_source_length` and decoder rows of `max_target_length` at
once, sample k of a row being segment k on both sides (MT5ForConditionalGeneration.forward(segment_ids=...,
decoder_segment_ids=...)). `Seq2SeqPackingCollator` wraps those collators. Both reference datasets leave their target pad
ids LABELLED (`labels[target == pad_token_id] = -100` compares a Python list with an int, which is False, and assigns nothing),
so every target keeps its full padded length and the loss covers those pads. The packer keeps that loss unchanged: it removes
only the source pads, and only when the rows are wider than the padded ones (with max_target_length equal to the padded
target length every decoder row holds one sample and nothing is gained). tools/bench_packing.py --model mt5 measures the
result on an LCSTS-like mix. Span-corruption pretraining
(`UnsuperviseT5Dataset`) emits rows of exactly the target length without pads, so packing gains it nothing.
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


def pack_mlm_batch(batch, max_seq_length, pad_id):
    """batch: an MLM collator's `input_ids`, `attention_mask`, `token_type_ids`, `labels` [n, L] (tensors or nested lists) and
    optionally `next_sentence_label` [n]. Each sample is its non-pad prefix (attention_mask must be ones then zeros; at most
    max_seq_length tokens), kept whole, and every sample is kept, labelled or not. Returns a dict of [rows, max_seq_length]
    tensors: `input_ids` (pad_id after the last sample of a row), `token_type_ids` and `labels` as given (0 and -100 on the
    pad tail), `attention_mask` (ones), `position_ids` (0, 1, ... in each sample), `segment_ids` (0, 1, ... per row; the pad
    tail is a segment of its own); and, when the batch has them, `next_sentence_label` [n] in sample order with
    `cls_positions` [n], the flat index row * max_seq_length + start of each sample's first token ([CLS])."""
    ids = torch.as_tensor(batch["input_ids"], dtype=torch.int64)
    mask = torch.as_tensor(batch["attention_mask"], dtype=torch.int64)
    tt = torch.as_tensor(batch["token_type_ids"], dtype=torch.int64)
    labels = torch.as_tensor(batch["labels"], dtype=torch.int64)
    if ids.dim() != 2 or not ids.shape == mask.shape == tt.shape == labels.shape:
        raise ValueError(f"input_ids, attention_mask, token_type_ids and labels must be [n, L] of one shape, got "
                         f"{tuple(ids.shape)}, {tuple(mask.shape)}, {tuple(tt.shape)} and {tuple(labels.shape)}")
    if max_seq_length <= 0:
        raise ValueError(f"max_seq_length must be positive, got {max_seq_length}")
    nsl = batch.get("next_sentence_label")
    if nsl is not None:
        nsl = torch.as_tensor(nsl, dtype=torch.int64).view(-1)
        if nsl.numel() != ids.shape[0]:
            raise ValueError(f"next_sentence_label has {nsl.numel()} entries for {ids.shape[0]} samples")
    lengths = (mask != 0).sum(1)
    if not bool(((mask != 0) == (torch.arange(ids.shape[1]) < lengths[:, None])).all()):
        raise ValueError("attention_mask must be a prefix of ones per sample (pads only at the end)")
    if bool((lengths == 0).any()):
        raise ValueError("a sample has no tokens (attention_mask all zero)")
    if bool((lengths > max_seq_length).any()):
        raise ValueError(f"a sample has {int(lengths.max())} tokens, more than max_seq_length = {max_seq_length}")
    lengths = lengths.tolist()
    rows = first_fit(lengths, max_seq_length)
    R, S = len(rows), max_seq_length
    out_ids = torch.full((R, S), pad_id, dtype=torch.int64)
    out_tt = torch.zeros((R, S), dtype=torch.int64)
    out_lab = torch.full((R, S), IGNORE_INDEX, dtype=torch.int64)
    out_pos = torch.zeros((R, S), dtype=torch.int64)
    out_seg = torch.zeros((R, S), dtype=torch.int64)
    cls = torch.zeros(len(lengths), dtype=torch.int64)
    for r, members in enumerate(rows):
        t = 0
        for k, i in enumerate(members):
            n = lengths[i]
            out_ids[r, t:t + n] = ids[i, :n]
            out_tt[r, t:t + n] = tt[i, :n]
            out_lab[r, t:t + n] = labels[i, :n]
            out_pos[r, t:t + n] = torch.arange(n)
            out_seg[r, t:t + n] = k
            cls[i] = r * S + t
            t += n
        if t < S:                                  # pad tail: its own segment, positions from 0, type 0, no labels
            out_pos[r, t:] = torch.arange(S - t)
            out_seg[r, t:] = len(members)
    out = {"input_ids": out_ids, "attention_mask": torch.ones((R, S), dtype=torch.int64), "token_type_ids": out_tt,
           "labels": out_lab, "position_ids": out_pos, "segment_ids": out_seg}
    if nsl is not None:
        out["next_sentence_label"] = nsl.clone()
        out["cls_positions"] = cls
    return out


class MLMPackingCollator:
    """collate(samples) = pack_mlm_batch(inner(samples), max_seq_length, pad_id), for ErLangShenCollator /
    FastErLangShenCollator (or any collator with their output format)."""

    def __init__(self, inner, max_seq_length, pad_id):
        self.inner, self.max_seq_length, self.pad_id = inner, int(max_seq_length), int(pad_id)

    def __call__(self, samples):
        return pack_mlm_batch(self.inner(samples), self.max_seq_length, self.pad_id)


def first_fit_pairs(lengths, budgets):
    """first_fit for samples with two lengths (source, target) and two row budgets: a sample goes into the first row where
    both fit, else into a new row. Returns a list of rows, each a list of sample indices."""
    rows, free = [], []
    for i, (ns, nt) in enumerate(lengths):
        for r, (rs, rt) in enumerate(free):
            if ns <= rs and nt <= rt:
                rows[r].append(i)
                free[r] = (rs - ns, rt - nt)
                break
        else:
            rows.append([i])
            free.append((budgets[0] - ns, budgets[1] - nt))
    return rows


def pack_seq2seq_batch(batch, max_source_length, max_target_length, pad_id):
    """batch: an encoder-decoder collator's `input_ids` and `attention_mask` [n, Le] (the mask a prefix of ones per sample)
    and `labels` [n, Ld] (-100 ignored), tensors or nested lists; other keys (the strings LCSTSDataset adds) are ignored. A
    sample's source is its non-pad prefix (at most max_source_length tokens) and its target its labels up to and including
    the last one != -100 (at most max_target_length; pad-id targets that a dataset labels stay targets, so the loss is the
    padded batch's). Samples without a labelled target are dropped; a batch with none left packs into one row of pads whose
    labels are all ignored (MT5ForConditionalGeneration gives it a loss of exactly 0 and zero gradients). Returns a dict:
    `input_ids` (pad_id after the last source of a row), `attention_mask` (ones) and `segment_ids` [R, max_source_length];
    `labels` (-100 after the last target) and `decoder_segment_ids` [R, max_target_length]. Segment ids are 0..m-1 for the m
    samples of a row on both sides, and each side's pad tail gets id m, so the two tails pair with each other."""
    ids = torch.as_tensor(batch["input_ids"], dtype=torch.int64)
    mask = torch.as_tensor(batch["attention_mask"], dtype=torch.int64)
    labels = torch.as_tensor(batch["labels"], dtype=torch.int64)
    if ids.dim() != 2 or ids.shape != mask.shape or labels.dim() != 2 or labels.shape[0] != ids.shape[0]:
        raise ValueError(f"input_ids and attention_mask must be [n, Le] of one shape and labels [n, Ld], got "
                         f"{tuple(ids.shape)}, {tuple(mask.shape)} and {tuple(labels.shape)}")
    if max_source_length <= 0 or max_target_length <= 0:
        raise ValueError(f"max_source_length and max_target_length must be positive, got {max_source_length} and "
                         f"{max_target_length}")
    src_len = (mask != 0).sum(1)
    if not bool(((mask != 0) == (torch.arange(ids.shape[1]) < src_len[:, None])).all()):
        raise ValueError("attention_mask must be a prefix of ones per sample (pads only at the end)")
    if bool((src_len == 0).any()):
        raise ValueError("a sample has no source tokens (attention_mask all zero)")
    if bool((src_len > max_source_length).any()):
        raise ValueError(f"a sample has {int(src_len.max())} source tokens, more than max_source_length = "
                         f"{max_source_length}")
    labelled = labels != IGNORE_INDEX
    pos = torch.arange(labels.shape[1])
    tgt_len = torch.where(labelled, pos + 1, 0).max(1).values   # one past the last labelled position, 0 when none
    if bool((tgt_len > max_target_length).any()):
        raise ValueError(f"a sample has {int(tgt_len.max())} target tokens, more than max_target_length = "
                         f"{max_target_length}")
    kept = [i for i in range(ids.shape[0]) if int(tgt_len[i]) > 0]
    rows = first_fit_pairs([(int(src_len[i]), int(tgt_len[i])) for i in kept], (max_source_length, max_target_length))
    rows = [[kept[j] for j in r] for r in rows] or [[]]
    R, Se, Sd = len(rows), max_source_length, max_target_length
    out_ids = torch.full((R, Se), pad_id, dtype=torch.int64)
    out_seg = torch.zeros((R, Se), dtype=torch.int64)
    out_lab = torch.full((R, Sd), IGNORE_INDEX, dtype=torch.int64)
    out_dseg = torch.zeros((R, Sd), dtype=torch.int64)
    for r, members in enumerate(rows):
        s = t = 0
        for k, i in enumerate(members):
            ns, nt = int(src_len[i]), int(tgt_len[i])
            out_ids[r, s:s + ns] = ids[i, :ns]
            out_seg[r, s:s + ns] = k
            out_lab[r, t:t + nt] = labels[i, :nt]
            out_dseg[r, t:t + nt] = k
            s, t = s + ns, t + nt
        out_seg[r, s:] = len(members)          # pad tails: id m on both sides
        out_dseg[r, t:] = len(members)
    return {"input_ids": out_ids, "attention_mask": torch.ones((R, Se), dtype=torch.int64), "segment_ids": out_seg,
            "labels": out_lab, "decoder_segment_ids": out_dseg}


class Seq2SeqPackingCollator:
    """collate(samples) = pack_seq2seq_batch(inner(samples), max_source_length, max_target_length, pad_id), for the T5
    fine-tuning collators (LCSTSDataset / TaskT5Dataset items through default_collate, or any collator with that format)."""

    def __init__(self, inner, max_source_length, max_target_length, pad_id):
        self.inner, self.pad_id = inner, int(pad_id)
        self.max_source_length, self.max_target_length = int(max_source_length), int(max_target_length)

    def __call__(self, samples):
        return pack_seq2seq_batch(self.inner(samples), self.max_source_length, self.max_target_length, self.pad_id)
