"""CPU: pack_causal_lm_batch on the Wenzhong-GPT2 QA format. Real GPT2QADataset items (the compat restatement of the
reference's medicalQADataset.py) over an offline byte-level tokenizer, collated by torch's default_collate as the
reference's DataLoader does: pad == eos, labels -100 on every pad, so an eos inside the text is unlabelled too, and the
`question` / `answer` strings ride along."""
import argparse
import os
import sys

import torch
from torch.utils.data import default_collate

import hf_fixtures as F

sys.path.insert(0, os.path.join(F.ROOT, "fengshen-lm_b200", "compat"))
from fengshen.data.task_dataloader.medicalQADataset import GPT2QADataset  # noqa: E402
from fsb200.packing import pack_causal_lm_batch  # noqa: E402

MAX = 64


def _dataset(tmp_path, rows):
    F.gpt2_tokenizer_dir(tmp_path / "tok")
    path = tmp_path / "train.txt"
    with open(path, "w", encoding="utf8") as f:
        f.writelines(repr(r) + "\n" for r in rows)
    args = argparse.Namespace(pretrained_model_path=str(tmp_path / "tok"), max_seq_length=MAX)
    return GPT2QADataset(str(path), "train", args)


def test_packing_gpt2_qa_batches(tmp_path):
    rows = [{"Question": "q1: headache?", "answer": " rest."},
            {"Question": "x" * 40, "answer": "y" * 40},                            # fills max_seq_length: no pad
            {"Question": "before<|endoftext|>after?", "answer": " ok."},           # an eos inside the text
            {"Question": "q3?", "answer": " water, sleep."},
            {"Question": "q4: fever", "answer": " see a doctor"}]
    ds = _dataset(tmp_path, rows)
    tok = ds.tokenizer
    assert tok.pad_token_id == tok.eos_token_id
    eos = tok.eos_token_id
    items = [ds[i] for i in range(len(rows))]
    batch = default_collate(items)
    assert isinstance(batch["question"], list)                               # string fields ride along
    assert batch["input_ids"].shape == (len(rows), MAX)
    full = items[1]
    assert bool((full["attention_mask"] == 1).all()) and bool((full["labels"] != -100).all())
    inner = items[2]
    at = (inner["input_ids"] == eos) & (inner["attention_mask"] == 1)
    assert int(at.sum()) == 1 and bool((inner["labels"][at] == -100).all())  # the reference leaves it unlabelled

    packed = pack_causal_lm_batch(batch, MAX, eos)
    ids, lab, pos, seg = (packed[k] for k in ("input_ids", "labels", "position_ids", "segment_ids"))
    assert ids.shape[1] == MAX and ids.shape[0] < len(rows)
    assert bool((packed["attention_mask"] == 1).all())
    # the sample that fills a row stands alone in it, one segment, positions 0 .. MAX - 1
    r_full = next(r for r in range(ids.shape[0]) if torch.equal(ids[r], full["input_ids"]))
    assert bool((seg[r_full] == 0).all()) and torch.equal(pos[r_full], torch.arange(MAX))
    assert lab[r_full, 0] == -100 and torch.equal(lab[r_full, 1:], full["labels"][1:])
    # every other sample: cut after its last labelled token, placed whole, positions from 0, its start label ignored
    found = 0
    for it in items:
        n = int((it["labels"] != -100).nonzero()[-1]) + 1
        for r in range(ids.shape[0]):
            for s in range(MAX - n + 1):
                if torch.equal(ids[r, s:s + n], it["input_ids"][:n]) and (s == 0 or seg[r, s] != seg[r, s - 1]):
                    assert torch.equal(pos[r, s:s + n], torch.arange(n))
                    assert bool((seg[r, s:s + n] == seg[r, s]).all())
                    assert s + n == MAX or seg[r, s + n] != seg[r, s]
                    assert lab[r, s] == -100 and torch.equal(lab[r, s + 1:s + n], it["labels"][1:n])
                    found += 1
                    break
            else:
                continue
            break
    assert found == len(items)
    # the eos inside the text is an input, unlabelled; the pad tails are eos, unlabelled, a segment of their own
    r_in = next(r for r in range(ids.shape[0]) if any(torch.equal(ids[r, s:s + 5], inner["input_ids"][:5])
                                                        for s in range(MAX - 4)))
    assert bool(((ids[r_in] == eos) & (lab[r_in] == -100)).any())
    for r in range(ids.shape[0]):
        tail = seg[r] == seg[r, -1]
        if lab[r][tail].eq(-100).all() and r != r_full:
            assert bool((ids[r][tail] == eos).all())
            assert torch.equal(pos[r][tail], torch.arange(int(tail.sum())))
