"""CPU: the packing collator (fsb200/packing.py) and the segment-bounds helper (ops.segment_bounds).

The packed batch must carry every labelled sample intact (tokens and labels contiguous and unchanged), restart the position
ids at 0 in every segment, ignore the labels of segment starts and pads, and place the samples first fit in sample order."""
import os
import random

import pytest
import torch

from fsb200 import ops
from fsb200.packing import PackingCollator, first_fit, pack_causal_lm_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAD = 2


def _sft_batch(rows, pad=PAD):
    """The padded format of the Ziya SFT collator: per sample (prompt tokens, output tokens), labels -100 on the prompt,
    eos-padded to the longest row, labels -100 on pads."""
    ids, labs = [], []
    for turns in rows:
        i, l = [], []
        for prompt, output in turns:
            i += prompt + output
            l += [-100] * len(prompt) + output
        ids.append(i)
        labs.append(l)
    L = max(len(i) for i in ids)
    return {"input_ids": torch.tensor([i + [pad] * (L - len(i)) for i in ids]),
            "labels": torch.tensor([l + [-100] * (L - len(l)) for l in labs]),
            "attention_mask": torch.ones((len(ids), L))}


def _kept(ids, labs, max_len):
    """Plain restatement: the prefix of each row up to its last labelled token (rows without labels dropped)."""
    out = []
    for i, l in zip(ids.tolist(), labs.tolist()):
        i, l = i[:max_len], l[:max_len]
        last = max((t for t, x in enumerate(l) if x != -100), default=-1)
        if last >= 0:
            out.append((i[:last + 1], l[:last + 1]))
    return out


def _check_packed(batch, packed, max_len, pad=PAD):
    kept = _kept(batch["input_ids"], batch["labels"], max_len)
    ids, lab, pos, seg = (packed[k] for k in ("input_ids", "labels", "position_ids", "segment_ids"))
    R, S = ids.shape
    assert S == max_len and lab.shape == pos.shape == seg.shape == (R, S)
    assert torch.equal(packed["attention_mask"], torch.ones((R, S)))
    for r in range(R):
        for k, (s, e) in enumerate(_runs(seg[r].tolist())):
            assert seg[r, s].item() == k                               # segment ids 0, 1, ... per row
            assert pos[r, s:e].tolist() == list(range(e - s))          # positions restart at 0 and step by 1
            assert lab[r, s].item() == -100                            # segment starts are not targets
    # row r holds the kept samples first_fit puts there, in order, contiguous, tokens and labels unchanged (the first label
    # ignored), then at most a pad tail of pad tokens without labels
    rows = first_fit([len(k[0]) for k in kept], max_len) or [[]]
    assert R == len(rows)
    for r, members in enumerate(rows):
        runs = list(_runs(seg[r].tolist()))
        assert len(runs) - len(members) in (0, 1)
        for (s, e), i in zip(runs, members):
            assert ids[r, s:e].tolist() == kept[i][0] and lab[r, s + 1:e].tolist() == kept[i][1][1:]
        if len(runs) > len(members):
            s, e = runs[-1]
            assert e == S and all(x == pad for x in ids[r, s:e].tolist()) and all(x == -100 for x in lab[r, s:e].tolist())


def _runs(row):
    s = 0
    for t in range(1, len(row) + 1):
        if t == len(row) or row[t] != row[t - 1]:
            yield s, t
            s = t


def test_first_fit_hand_worked():
    # exact fit: 6 + 4 fills a row of 10; 7 opens a row; 3 fits into that row; a sample of exactly 10 takes its own row
    assert first_fit([6, 4, 7, 3, 10, 1], 10) == [[0, 1], [2, 3], [4], [5]]
    # first fit, not next fit: 2 goes back into the first row with room
    assert first_fit([5, 8, 2, 3], 10) == [[0, 2, 3], [1]]
    assert first_fit([], 10) == []


def test_pack_hand_worked_rows():
    P, O = [7, 7, 7], [5, 5]
    batch = _sft_batch([
        [(P, O)],                      # 5 tokens
        [([8], [9, 9, 9, 9])],         # 5 tokens: exact fit with the first
        [([1] * 4, [])],               # no labelled token: dropped
        [(P, [6] * 7)],                # 10 tokens: exactly max_seq_length
        [([3, 3], [4, 4]), ([3], [4])],  # two turns, 7 tokens
    ])
    packed = pack_causal_lm_batch(batch, 10, PAD)
    assert packed["input_ids"].tolist() == [
        [7, 7, 7, 5, 5, 8, 9, 9, 9, 9],
        [7, 7, 7, 6, 6, 6, 6, 6, 6, 6],
        [3, 3, 4, 4, 3, 4, PAD, PAD, PAD, PAD]]
    assert packed["labels"].tolist() == [
        [-100, -100, -100, 5, 5, -100, 9, 9, 9, 9],
        [-100, -100, -100, 6, 6, 6, 6, 6, 6, 6],
        [-100, -100, 4, 4, -100, 4, -100, -100, -100, -100]]
    assert packed["segment_ids"].tolist() == [[0] * 5 + [1] * 5, [0] * 10, [0] * 6 + [1] * 4]
    assert packed["position_ids"].tolist() == [[0, 1, 2, 3, 4, 0, 1, 2, 3, 4], list(range(10)), [0, 1, 2, 3, 4, 5, 0, 1, 2, 3]]
    _check_packed(batch, packed, 10)


def test_pack_drops_the_tail_after_the_last_label_and_truncates():
    # row 0's labels stop before its end (a prompt-only second turn): the unlabelled tail is dropped.
    # row 1 is longer than max_seq_length: cut at max_seq_length (inside its output), then at its last label.
    batch = _sft_batch([[([1, 1], [2, 2]), ([3, 3, 3], [])], [([4] * 3, [5] * 9)]])
    packed = pack_causal_lm_batch(batch, 8, PAD)
    assert packed["input_ids"].tolist() == [[1, 1, 2, 2, PAD, PAD, PAD, PAD], [4, 4, 4, 5, 5, 5, 5, 5]]
    assert packed["labels"].tolist() == [[-100, -100, 2, 2, -100, -100, -100, -100], [-100, -100, -100, 5, 5, 5, 5, 5]]
    # a cut inside the prompt leaves no label: the sample is dropped; nothing left packs into one ignored pad row
    empty = pack_causal_lm_batch(_sft_batch([[([4] * 9, [5])]]), 8, PAD)
    assert empty["input_ids"].tolist() == [[PAD] * 8] and empty["labels"].tolist() == [[-100] * 8]


def test_packing_collator_wraps_the_inner_collator():
    rows = [[([1, 2], [3, 4])], [([5], [6, 7, 8])]]
    col = PackingCollator(lambda samples: _sft_batch(samples), 16, PAD)
    got = col(rows)
    want = pack_causal_lm_batch(_sft_batch(rows), 16, PAD)
    assert all(torch.equal(got[k], want[k]) for k in want)


def test_pack_random_sft_batches():
    rng = random.Random(0)
    for trial in range(30):
        max_len = rng.choice([16, 33, 64])
        rows = []
        for _ in range(rng.randint(1, 9)):
            turns = [([rng.randint(3, 50) for _ in range(rng.randint(0, 12))],
                      [rng.randint(3, 50) for _ in range(rng.randint(0, 12))]) for _ in range(rng.randint(1, 3))]
            rows.append(turns)
        batch = _sft_batch(rows)
        packed = pack_causal_lm_batch(batch, max_len, PAD)
        _check_packed(batch, packed, max_len)


def _bounds_python(row):
    S = len(row)
    start, end = [0] * S, [0] * S
    s = 0
    for t in range(1, S + 1):
        if t == S or row[t] != row[t - 1]:
            for u in range(s, t):
                start[u], end[u] = s, t
            s = t
    return start, end


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.int16])
def test_segment_bounds_matches_python(dtype):
    g = torch.Generator().manual_seed(1)
    for S in (1, 2, 7, 64, 129):
        ids = torch.randint(0, 3, (4, S), generator=g).to(dtype)    # few values: runs, repeats, non-monotonic ids
        ids[0] = 5
        start, end = ops.segment_bounds(ids)
        assert start.dtype == end.dtype == torch.int32 and start.is_contiguous() and end.is_contiguous()
        for b in range(4):
            ws, we = _bounds_python(ids[b].tolist())
            assert start[b].tolist() == ws and end[b].tolist() == we


def test_segment_bounds_refuses_non_integer_input():
    with pytest.raises(RuntimeError, match="integer"):
        ops.segment_bounds(torch.zeros((2, 4)))
    with pytest.raises(RuntimeError, match="integer"):
        ops.segment_bounds(torch.zeros(4, dtype=torch.int64))


def test_pack_reference_collator_batches():
    """tests/golden/ziya_sft_collator.npz: batches of the unmodified reference LlamaSFTCollator
    (oracle/make_golden_llama_sft.py): multi-turn samples, a cut inside an output, cuts inside a prompt."""
    import numpy as np
    g = np.load(os.path.join(ROOT, "tests", "golden", "ziya_sft_collator.npz"))
    for name in ("multi_turn", "cut_in_output", "cut_in_prompt"):
        batch = {"input_ids": torch.from_numpy(g[name + "/input_ids"]), "labels": torch.from_numpy(g[name + "/labels"])}
        max_len, eos = int(g[name + "/max_seq_length"]), int(g[name + "/eos"])
        packed = pack_causal_lm_batch(batch, max_len, eos)
        _check_packed(batch, packed, max_len, pad=eos)
        labelled = int((batch["labels"] != -100).sum())
        starts = len(_kept(batch["input_ids"], batch["labels"], max_len))
        # every labelled token survives; only the segment starts lose theirs, and those are prompt tokens here
        assert int((packed["labels"] != -100).sum()) == labelled
        assert starts == sum(1 for row in batch["labels"].tolist() if any(x != -100 for x in row))
    # the row cut inside its first prompt has no labelled token and is dropped; the row cut inside its second prompt keeps
    # its first turn
    lab = torch.from_numpy(g["cut_in_prompt/labels"])
    assert (lab[1] != -100).sum() == 0 and (lab[0] != -100).sum() > 0
