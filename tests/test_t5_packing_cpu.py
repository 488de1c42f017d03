"""CPU: packed seq2seq batches for mT5 / Randeng-T5 fine-tuning (fsb200/packing.py pack_seq2seq_batch,
Seq2SeqPackingCollator) and the cross-attention bounds of packed rows (fsb200/models/base.py cross_segment_bounds)."""
import random

import pytest
import torch

import os

import numpy as np

from fsb200 import ops
from fsb200.models.base import cross_segment_bounds
from fsb200.models.t5 import shift_right
from fsb200.packing import Seq2SeqPackingCollator, first_fit, first_fit_pairs, pack_seq2seq_batch

PAD = 0


def _padded(n, seed, le=128, ld=64, max_src=60, max_tgt=30):
    """LCSTSDataset.encode-shaped samples (source and target padded to max length, labels -100 on the target pads), with an
    empty summary, a full-length source and target, and a labelled pad id inside a target (TaskT5Dataset keeps those)."""
    rng = random.Random(seed)
    ids = torch.full((n, le), PAD, dtype=torch.int64)
    mask = torch.zeros((n, le), dtype=torch.int64)
    labels = torch.full((n, ld), -100, dtype=torch.int64)
    for i in range(n):
        ns = le if i == 2 else rng.randint(1, max_src)
        nt = 0 if i == 1 else ld if i == 2 else rng.randint(1, max_tgt)
        ids[i, :ns] = torch.tensor([rng.randrange(2, 500) for _ in range(ns)])
        mask[i, :ns] = 1
        labels[i, :nt] = torch.tensor([rng.randrange(2, 500) for _ in range(nt)], dtype=torch.int64)
        if i == 3 and nt > 3:
            labels[i, nt - 2] = PAD
            labels[i, 1] = -100                    # an ignored position inside the target stays ignored
    return {"input_ids": ids, "attention_mask": mask, "labels": labels, "text": [f"t{i}" for i in range(n)]}


def _unpack(packed):
    """Every (source, target labels) pair of a packed batch, in row order, tails left out."""
    out = []
    for r in range(packed["input_ids"].shape[0]):
        e, d = packed["segment_ids"][r], packed["decoder_segment_ids"][r]
        m = max(int(e[-1]), int(d[-1]))
        for k in range(m + 1):
            src, tgt = packed["input_ids"][r][e == k], packed["labels"][r][d == k]
            if len(tgt) and (tgt != -100).any():
                out.append((src.tolist(), tgt.tolist()))
    return out


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_packer_recovers_every_sample_exactly(seed):
    batch = _padded(24, seed)
    packed = pack_seq2seq_batch(batch, 128, 64, PAD)
    R = packed["input_ids"].shape[0]
    assert R < 24
    for k, shape in (("input_ids", (R, 128)), ("attention_mask", (R, 128)), ("segment_ids", (R, 128)),
                     ("labels", (R, 64)), ("decoder_segment_ids", (R, 64))):
        assert tuple(packed[k].shape) == shape and packed[k].dtype == torch.int64, k
    assert bool((packed["attention_mask"] == 1).all())
    want = []
    for i in range(24):
        ns = int(batch["attention_mask"][i].sum())
        lab = batch["labels"][i]
        where = (lab != -100).nonzero()
        if where.numel() == 0:
            continue                                     # no labelled target: dropped
        want.append((batch["input_ids"][i, :ns].tolist(), lab[:int(where[-1]) + 1].tolist()))
    got = _unpack(packed)
    assert sorted(got) == sorted(want)
    # each row's ids are 0..m-1 then the tail id m on both sides, non-decreasing; the pads carry pad_id / -100
    for r in range(R):
        for seg in (packed["segment_ids"][r], packed["decoder_segment_ids"][r]):
            assert bool((seg[1:] >= seg[:-1]).all()) and int(seg[0]) == 0
        e, d = packed["segment_ids"][r], packed["decoder_segment_ids"][r]
        m = int(max(e.max(), d.max()))
        assert set(e.tolist()) | set(d.tolist()) <= set(range(m + 1))
    # the loss is unchanged: the same labelled targets, in the same number
    assert int((packed["labels"] != -100).sum()) == int((batch["labels"] != -100).sum())


def test_placement_is_first_fit_on_both_budgets():
    lengths = [(60, 10), (60, 50), (10, 10), (8, 40), (50, 4)]
    # sample 1 fits row 0 on both sides; sample 2's source does not (120 + 10 > 128); sample 3's source would fit row 0
    # but its target not (60 + 40 > 64), so it joins row 1; sample 4's source does not fit row 0 (120 + 50 > 128)
    assert first_fit_pairs(lengths, (128, 64)) == [[0, 1], [2, 3, 4]]
    # with one budget wide open, the pairs reduce to first_fit over the other lengths
    rng = random.Random(4)
    ls = [rng.randint(1, 100) for _ in range(50)]
    assert first_fit_pairs([(n, 1) for n in ls], (128, 10 ** 6)) == first_fit(ls, 128)


def test_batch_without_targets_packs_one_ignored_row():
    batch = _padded(4, 5)
    batch["labels"][:] = -100
    packed = pack_seq2seq_batch(batch, 128, 64, PAD)
    assert packed["input_ids"].shape[0] == 1
    assert bool((packed["input_ids"] == PAD).all()) and bool((packed["labels"] == -100).all())
    assert bool((packed["segment_ids"] == 0).all()) and bool((packed["decoder_segment_ids"] == 0).all())


def test_collator_wraps_the_inner_collator():
    seen = []

    def inner(samples):
        seen.append(len(samples))
        return _padded(len(samples), 7)
    out = Seq2SeqPackingCollator(inner, 128, 64, PAD)(list(range(10)))
    assert seen == [10] and set(out) == {"input_ids", "attention_mask", "segment_ids", "labels", "decoder_segment_ids"}


def test_packer_refusals():
    b = _padded(3, 8)
    with pytest.raises(ValueError, match="more than max_source_length"):
        pack_seq2seq_batch(b, 64, 64, PAD)
    with pytest.raises(ValueError, match="more than max_target_length"):
        pack_seq2seq_batch(b, 128, 32, PAD)
    bad = dict(b, attention_mask=b["attention_mask"].clone())
    bad["attention_mask"][0, 0] = 0
    with pytest.raises(ValueError, match="prefix of ones"):
        pack_seq2seq_batch(bad, 128, 64, PAD)


def _brute(dec, enc):
    B, Sd = dec.shape
    Se = enc.shape[1]
    kv_s = torch.zeros(B, Sd, dtype=torch.int32)
    kv_e = torch.zeros(B, Sd, dtype=torch.int32)
    q_s = torch.zeros(B, Se, dtype=torch.int32)
    q_e = torch.zeros(B, Se, dtype=torch.int32)
    for b in range(B):
        for t in range(Sd):
            ks = [k for k in range(Se) if enc[b, k] == dec[b, t]]
            # an empty range sits where the id would be inserted (the kernels need only start >= end)
            pos = sum(1 for k in range(Se) if enc[b, k] < dec[b, t])
            kv_s[b, t], kv_e[b, t] = (ks[0], ks[-1] + 1) if ks else (pos, pos)
        for k in range(Se):
            qs = [t for t in range(Sd) if dec[b, t] == enc[b, k]]
            pos = sum(1 for t in range(Sd) if dec[b, t] < enc[b, k])
            q_s[b, k], q_e[b, k] = (qs[0], qs[-1] + 1) if qs else (pos, pos)
    return (kv_s, kv_e), (q_s, q_e)


@pytest.mark.parametrize("seed", range(4))
def test_cross_segment_bounds_against_brute_force(seed):
    g = torch.Generator().manual_seed(seed)
    B, Sd, Se = 3, 37, 23
    dec = torch.sort(torch.randint(0, 6, (B, Sd), generator=g), dim=1).values     # ids with gaps: some unmatched
    enc = torch.sort(torch.randint(0, 6, (B, Se), generator=g), dim=1).values
    got = cross_segment_bounds(dec, enc)
    want = _brute(dec, enc)
    for gs, ws in zip(got, want):
        for gt, wt in zip(gs, ws):
            assert gt.dtype == torch.int32 and gt.is_contiguous() and torch.equal(gt, wt)


def test_cross_segment_bounds_of_a_packed_batch_pair_every_sample():
    packed = pack_seq2seq_batch(_padded(24, 3), 128, 64, PAD)
    (kv_s, kv_e), (q_s, q_e) = cross_segment_bounds(packed["decoder_segment_ids"], packed["segment_ids"])
    for r in range(packed["input_ids"].shape[0]):
        e, d = packed["segment_ids"][r], packed["decoder_segment_ids"][r]
        for t in range(64):
            ks = (e == d[t]).nonzero().flatten()
            if len(ks):
                assert (int(kv_s[r, t]), int(kv_e[r, t])) == (int(ks[0]), int(ks[-1]) + 1)
            else:                                           # a decoder tail whose encoder row is full
                assert int(kv_s[r, t]) == int(kv_e[r, t])


def test_cross_segment_bounds_refusals():
    with pytest.raises(ValueError, match="non-decreasing"):
        cross_segment_bounds(torch.tensor([[0, 1, 0]]), torch.tensor([[0, 1]]))
    with pytest.raises(ValueError, match="non-decreasing"):
        cross_segment_bounds(torch.tensor([[0, 1]]), torch.tensor([[1, 0]]))
    with pytest.raises(ValueError, match="integer"):
        cross_segment_bounds(torch.zeros(1, 4), torch.zeros(1, 4, dtype=torch.int64))
    with pytest.raises(ValueError, match="share batch"):
        cross_segment_bounds(torch.zeros(2, 4, dtype=torch.int64), torch.zeros(1, 4, dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ decoder inputs
def test_decoder_inputs_restart_at_every_segment_against_a_loop():
    """shift_right with the decoder segment starts (what MT5ForConditionalGeneration.forward derives from the labels of
    packed rows): the start id at every segment start, the previous label elsewhere, -100 as the pad id."""
    start, pad = 7, 0
    packed = pack_seq2seq_batch(_padded(24, 4), 128, 64, PAD)
    labels = packed["labels"]
    seg_start, _ = ops.segment_bounds(packed["decoder_segment_ids"])
    got = shift_right(labels, start, pad, seg_start)
    want = torch.empty_like(labels)
    for r in range(labels.shape[0]):
        d = packed["decoder_segment_ids"][r].tolist()
        for t in range(labels.shape[1]):
            if t == 0 or d[t] != d[t - 1]:
                want[r, t] = start
            else:
                want[r, t] = pad if int(labels[r, t - 1]) == -100 else int(labels[r, t - 1])
    assert torch.equal(got, want)
    assert torch.equal(shift_right(labels, start, pad), shift_right(labels, start, pad, torch.zeros_like(seg_start)))


# ------------------------------------------------------------------------------------------------ reference batches
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "t5_finetune_batches.npz")


def _golden(case):
    z = np.load(GOLDEN)
    batch = {k: torch.from_numpy(z[f"{case}/{k}"]) for k in ("input_ids", "attention_mask", "labels")}
    return batch, int(z[f"{case}/max_source_length"]), int(z[f"{case}/max_target_length"])


@pytest.mark.parametrize("case", ["lcsts", "task_t5"])
def test_packer_on_the_reference_datasets_batches(case):
    """Batches of the unmodified LCSTSDataset.encode / TaskT5Dataset.encode (oracle/make_golden_t5_finetune.py: cut
    sources and summaries, an empty summary, full-length targets). Both datasets leave their target pad ids labelled, so
    every target keeps its full padded length and the loss is that of the padded batch: with rows as long as the padded
    ones every decoder row holds one sample (nothing is gained), and only wider rows remove the source pads."""
    batch, le, ld = _golden(case)
    n = batch["input_ids"].shape[0]
    assert bool((batch["labels"] != -100).all())                  # the reference labels every target position
    same = pack_seq2seq_batch(batch, le, ld, PAD)
    assert same["input_ids"].shape[0] == n
    for k in (2, 4):
        packed = pack_seq2seq_batch(batch, k * le, k * ld, PAD)
        assert packed["input_ids"].shape[0] == -(-n // k)
        want = [(batch["input_ids"][i, :int(batch["attention_mask"][i].sum())].tolist(), batch["labels"][i].tolist())
                for i in range(n)]
        assert sorted(_unpack(packed)) == sorted(want)
        assert int((packed["labels"] != -100).sum()) == int((batch["labels"] != -100).sum()) == n * ld
        assert int((packed["input_ids"] != PAD).sum()) == int((batch["input_ids"] != PAD).sum())
