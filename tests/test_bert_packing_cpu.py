"""CPU: MLM + sentence-order packing (fsb200/packing.py pack_mlm_batch / MLMPackingCollator) on the batches of the unmodified
reference ErLangShenCollator (tests/golden/bert_collator.json) and of FastErLangShenCollator: every sample recovered exactly
from the packed rows, [CLS] at cls_positions, first-fit rows with the pad tail a segment of its own, the refusals, and the
example's --pack_sequences flag around both collators."""
import os
import sys

import numpy as np
import pytest
import torch

import hf_fixtures as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
for p in ("fengshen-lm_b200", os.path.join("fengshen-lm_b200", "compat")):
    if os.path.join(ROOT, p) not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, p))

from fsb200.packing import MLMPackingCollator, first_fit, pack_mlm_batch  # noqa: E402


def _cls_id():
    import bert_collator_cases as C
    return C.build_vocab().index("[CLS]")


def _golden_batches():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "bert_collator.json"), encoding="utf8") as fh:
        return json.load(fh)["batches"]


def _tokenizer(tmp_path):
    import bert_collator_cases as C
    from transformers import BertTokenizer
    with open(tmp_path / "vocab.txt", "w", encoding="utf8") as fh:
        fh.write("\n".join(C.build_vocab()) + "\n")
    return BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)


def _fast_batches(tmp_path):
    import bert_collator_cases as C
    from fengshen.data.data_utils.collators import FastErLangShenCollator
    tok = _tokenizer(tmp_path)
    docs = [{"text": t} for t in C.TEXTS] + [{"text": C.TEXTS[0] + C.TEXTS[2] + C.TEXTS[5]}]
    out = []
    for L in (32, 64, 128):
        c = FastErLangShenCollator(tokenizer=tok, max_seq_length=L)
        c.setup()
        c.np_rng = np.random.RandomState(L)
        out.append((c(docs), L, tok.pad_token_id))
    return out


def _check_packed(batch, packed, L, pad_id):
    """Every sample of `batch` recovered exactly from `packed`, and the row layout rules."""
    ids, am = torch.as_tensor(batch["input_ids"]), torch.as_tensor(batch["attention_mask"])
    tt, lab = torch.as_tensor(batch["token_type_ids"]), torch.as_tensor(batch["labels"])
    nsl = torch.as_tensor(batch["next_sentence_label"]).view(-1)
    n = ids.shape[0]
    R, S = packed["input_ids"].shape
    assert S == L
    assert set(packed) == {"input_ids", "attention_mask", "token_type_ids", "labels", "position_ids", "segment_ids",
                           "next_sentence_label", "cls_positions"}
    assert torch.equal(packed["attention_mask"], torch.ones(R, S, dtype=torch.int64))
    assert torch.equal(packed["next_sentence_label"], nsl)
    cls = packed["cls_positions"]
    assert cls.dtype == torch.int64 and cls.shape == (n,) and len(set(cls.tolist())) == n
    flat = {k: packed[k].view(-1) for k in ("input_ids", "token_type_ids", "labels", "position_ids", "segment_ids")}
    lengths = am.sum(1).tolist()
    used = torch.zeros(R * S, dtype=torch.bool)
    for i, m in enumerate(lengths):
        c = int(cls[i])
        r, s = divmod(c, S)
        assert s + m <= S
        sl = slice(c, c + m)
        assert torch.equal(flat["input_ids"][sl], ids[i, :m])
        assert torch.equal(flat["token_type_ids"][sl], tt[i, :m])
        assert torch.equal(flat["labels"][sl], lab[i, :m])
        assert torch.equal(flat["position_ids"][sl], torch.arange(m))
        seg = flat["segment_ids"][sl]
        assert bool((seg == seg[0]).all())
        assert s == 0 or flat["segment_ids"][c - 1] != seg[0]               # a segment of its own
        assert s + m == S or flat["segment_ids"][c + m] != seg[0]
        used[sl] = True
    assert torch.equal(packed["input_ids"].view(-1)[cls], torch.full((n,), _cls_id()))   # [CLS] at cls_positions
    # rows: the existing first fit, in sample order; samples packed back to back from position 0
    rows = first_fit(lengths, S)
    assert R == len(rows)
    for r, members in enumerate(rows):
        t = 0
        for k, i in enumerate(members):
            assert int(cls[i]) == r * S + t
            assert int(packed["segment_ids"][r, t]) == k
            t += lengths[i]
        if t < S:                  # the pad tail: one more segment, positions from 0, pads, type 0, no labels
            assert bool((packed["segment_ids"][r, t:] == len(members)).all())
            assert torch.equal(packed["position_ids"][r, t:], torch.arange(S - t))
            assert bool((packed["input_ids"][r, t:] == pad_id).all())
            assert bool((packed["token_type_ids"][r, t:] == 0).all())
            assert bool((packed["labels"][r, t:] == -100).all())
    assert int(used.sum()) == sum(lengths)


def test_pack_reference_collator_batches():
    batches = _golden_batches()
    assert len(batches) == 6
    for b in batches:
        L = len(b["input_ids"][0])
        packed = pack_mlm_batch(b, L, 0)
        _check_packed(b, packed, L, 0)


def test_pack_reference_batches_into_longer_rows_shares_rows():
    """The same samples into rows of 4x the collator's length: several samples per row, still recovered exactly."""
    shared = 0
    for b in _golden_batches():
        L = len(b["input_ids"][0])
        packed = pack_mlm_batch(b, 4 * L, 0)
        _check_packed(b, packed, 4 * L, 0)
        shared += packed["input_ids"].shape[0] < len(b["input_ids"])
    assert shared > 0


def test_pack_native_collator_batches(tmp_path):
    for batch, L, pad in _fast_batches(tmp_path):
        packed = pack_mlm_batch(batch, L, pad)
        _check_packed(batch, packed, L, pad)
        assert packed["input_ids"].shape[0] <= batch["input_ids"].shape[0]


def test_samples_without_mlm_labels_are_kept():
    b = {k: torch.as_tensor(v) for k, v in _golden_batches()[0].items()}
    b["labels"][0] = -100
    packed = pack_mlm_batch(b, b["input_ids"].shape[1], 0)
    _check_packed(b, packed, b["input_ids"].shape[1], 0)


def test_collator_wraps_the_inner_collator():
    b = _golden_batches()[1]
    L = len(b["input_ids"][0])
    seen = []

    def inner(samples):
        seen.append(samples)
        return b
    out = MLMPackingCollator(inner, L, 0)(["x", "y"])
    assert seen == [["x", "y"]]
    _check_packed(b, out, L, 0)
    assert "cls_positions" not in pack_mlm_batch({k: v for k, v in b.items() if k != "next_sentence_label"}, L, 0)


def test_refusals():
    b = {k: torch.as_tensor(v) for k, v in _golden_batches()[0].items()}
    L = b["input_ids"].shape[1]
    hole = dict(b, attention_mask=b["attention_mask"].clone())
    hole["attention_mask"][0, 1] = 0                      # ones, a zero, ones: not a prefix
    with pytest.raises(ValueError, match="prefix"):
        pack_mlm_batch(hole, L, 0)
    empty = dict(b, attention_mask=b["attention_mask"].clone())
    empty["attention_mask"][0] = 0
    with pytest.raises(ValueError, match="no tokens"):
        pack_mlm_batch(empty, L, 0)
    with pytest.raises(ValueError, match="more than max_seq_length"):
        pack_mlm_batch(b, int(b["attention_mask"].sum(1).max()) - 1, 0)
    with pytest.raises(ValueError, match="one shape"):
        pack_mlm_batch(dict(b, labels=b["labels"][:, :-1]), L, 0)
    with pytest.raises(ValueError, match="next_sentence_label"):
        pack_mlm_batch(dict(b, next_sentence_label=b["next_sentence_label"][:-1]), L, 0)
    with pytest.raises(ValueError, match="positive"):
        pack_mlm_batch(b, 0, 0)


@pytest.mark.parametrize("native", [False, True])
def test_example_pack_sequences_wraps_both_collators(tmp_path, native):
    import runpy
    import hf_recipes
    from fengshen.data.data_utils.collators import ErLangShenCollator, FastErLangShenCollator
    F.bert_dir(tmp_path / "m")
    corpus = F.bert_corpus(tmp_path / "train.json", n=8)
    ns = runpy.run_path(hf_recipes.EXAMPLE, run_name="example_not_main")
    base = ["--model_path", str(tmp_path / "m"), "--train_file", str(corpus), "--max_seq_length", "64"] + \
        (["--native_collator"] if native else [])
    tok = _tokenizer(tmp_path)
    plain = ns["parse_args"](base)
    assert plain.pack_sequences is False
    assert not isinstance(ns["build_data"](plain, tok).collate_fn, MLMPackingCollator)
    args = ns["parse_args"](base + ["--pack_sequences"])
    assert args.pack_sequences is True
    dm = ns["build_data"](args, tok)
    col = dm.collate_fn
    assert isinstance(col, MLMPackingCollator) and col.max_seq_length == 64 and col.pad_id == tok.pad_token_id
    assert type(col.inner) is (FastErLangShenCollator if native else ErLangShenCollator)
    import json
    docs = [json.loads(line) for line in open(corpus, encoding="utf8")]
    packed = col(docs)
    assert {"segment_ids", "position_ids", "cls_positions", "next_sentence_label"} <= set(packed)
    assert packed["input_ids"].shape[1] == 64
    assert torch.equal(packed["input_ids"].view(-1)[packed["cls_positions"]],
                       torch.full((len(docs),), tok.cls_token_id))
