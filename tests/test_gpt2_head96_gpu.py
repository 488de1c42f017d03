"""GPU: GPT-2 at head width 96, the shape of the 3.5B Wenzhong / Yuyuan models (30 layers, 32 heads x 96, hidden 3072).

A small 96-head model (n_embd 384, 4 heads, 2 layers, V 512) against transformers fp32 at the bars of test_gpt2_gpu.py;
dropout, packing, the CUDA-graph step and the Wenzhong recipe through the tests of test_gpt2_dropout_gpu.py and
test_gpt2_packing_gpu.py, run on their config with n_embd 384 (so head width 96); KV-cache generation on the padded
decode cache; and 2 layers at full width (3072, 32 heads, seq 1024, V 50304) against transformers, with the fp64 launch
census and the write-footprint census of one such step at dropout 0.1."""
import gc
import os
import sys

import pytest
import torch

import footprint as F
import test_gpt2_dropout_gpu as GD
import test_gpt2_packing_gpu as GP
import test_generate_graph_gpu as GG
import test_generate_hf_gpu as GH
from test_gpt2_dropout_gpu import launched  # noqa: F401  (the recipe's fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

from fsb200.models.gpt2 import GPT2LMHeadModel  # noqa: E402

SMALL96 = dict(H.GPT2_SMALL, n_embd=384)   # 4 heads x 96


def _grad_check(mine, ref, cos_min=0.998, ratio_tol=0.03):
    refp = dict(ref.named_parameters())
    n = 0
    for name, prm in mine.named_parameters():
        got, want = prm.main_grad.float().cpu().flatten(), refp[name].grad.flatten()
        cos = torch.dot(got, want) / (got.norm() * want.norm() + 1e-30)
        assert cos.item() >= cos_min, (name, cos.item())
        assert abs(got.norm().item() / (want.norm().item() + 1e-30) - 1.0) <= ratio_tol, name
        n += 1
    assert n == len(refp)


def _pair(cfg, seed=0):
    ref = H.build_gpt2(cfg, seed=seed)
    mine = GPT2LMHeadModel(ref.config, device="cuda")
    mine.load_reference_state_dict(ref.state_dict())
    assert mine.hn == 96
    return ref, mine


@pytest.mark.parametrize("padded", [False, True], ids=["full", "padding_mask"])
def test_small_96_head_model_vs_transformers(padded):
    ref, mine = _pair(SMALL96)
    batch = H.make_lm_batch(SMALL96["vocab_size"], 2, 96, seed=1234)
    kw = {}
    if padded:
        am = torch.ones(2, 96, dtype=torch.int64)
        am[1, 70:] = 0
        batch["labels"][1, 70:] = -100
        kw["attention_mask"] = am
    out_ref = ref(input_ids=batch["input_ids"], labels=batch["labels"], **kw)
    out_ref.loss.backward()
    out = mine(input_ids=batch["input_ids"].cuda(), labels=batch["labels"].cuda(), return_logits=True,
               **{k: v.cuda() for k, v in kw.items()})
    assert abs(out.loss.item() - out_ref.loss.item()) <= 3e-3, (out.loss.item(), out_ref.loss.item())
    tol = 4 * 2.0 ** -8 * out_ref.logits.abs().max().item()
    live = (batch["labels"] != -100) if padded else torch.ones(2, 96, dtype=torch.bool)
    assert (out.logits.float().cpu() - out_ref.logits.detach())[live].abs().max().item() <= tol
    out.loss.backward()
    torch.cuda.synchronize()
    _grad_check(mine, ref)


def test_head_widths_other_than_64_96_128_are_refused():
    for n_embd in (4 * 80, 4 * 112):
        with pytest.raises(RuntimeError, match="64/96/128"):
            GPT2LMHeadModel(H.build_gpt2(dict(SMALL96, n_embd=n_embd)).config, device="cuda")
    with pytest.raises(RuntimeError, match="multiples of 8"):
        GPT2LMHeadModel(H.build_gpt2(dict(SMALL96, vocab_size=510)).config, device="cuda")


# ------------------------------------------------------------------------------------------------ dropout, packing, graphs
@pytest.fixture
def width96():
    """The config of test_gpt2_dropout_gpu.py / test_gpt2_packing_gpu.py (shared dict) at n_embd 384: 4 heads x 96."""
    saved = dict(GD.CFG)
    GD.CFG["n_embd"] = 384
    assert GD._mine(GD._hf(0.0, 0.0, 0.0)).hn == 96
    yield
    GD.CFG.clear()
    GD.CFG.update(saved)


@pytest.mark.parametrize("probs", [(0.1, 0.2, 0.05), (0.1, 0.0, 0.1)], ids=["distinct", "attn0"])
def test_dropout_parity_with_replayed_masks(width96, probs):
    with pytest.MonkeyPatch.context() as mp:
        GD.test_model_parity_with_replayed_masks(probs, mp)


def test_packed_rows_with_dropout_vs_transformers(width96):
    with pytest.MonkeyPatch.context() as mp:
        GP.test_packed_parity_with_transformers_on_replayed_masks(mp)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_zero_segment_ids_is_the_unsegmented_path_bit_for_bit(width96, p):
    GP.test_zero_segment_ids_is_the_unsegmented_path_bit_for_bit(p)


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_equals_eager_with_dropout_and_ga2(width96, stage):
    (l0, p0, c0, sites), (l1, p1, c1, _) = GD._graph_vs_eager(stage, 2, 0.1)
    assert c0 == c1 == 5 * 2 * sites
    assert max(abs(a - b) for a, b in zip(l0, l1)) < 1e-5, (l0, l1)
    assert torch.equal(p0, p1), (p0.float() - p1.float()).abs().max()


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_equals_eager_on_packed_batches(width96, stage):
    GP.test_cuda_graph_step_equals_eager_on_packed_batches_with_dropout(stage)


def test_every_launch_of_a_packed_dropout_step_against_fp64(width96):
    with pytest.MonkeyPatch.context() as mp:
        GP.test_every_launch_of_a_packed_dropout_step_against_fp64(mp)


def test_wenzhong_recipe_trains_at_head_width_96(launched, tmp_path, monkeypatch):  # noqa: F811
    import hf_fixtures as HF
    monkeypatch.setitem(HF.GPT2_CFG, "n_embd", 384)
    GD.test_wenzhong_recipe_with_dropout_trains(launched, tmp_path, monkeypatch)


# ------------------------------------------------------------------------------------------------ generation
def _gen_pair(seed=0):
    """test_generate_hf_gpu.py's GPT-2 pair at n_embd 384 (4 heads x 96)."""
    import transformers
    torch.manual_seed(seed)
    cfg = transformers.GPT2Config(vocab_size=GH.V, n_positions=256, n_embd=384, n_layer=2, n_head=4, bos_token_id=3,
                                  eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
    ref = transformers.GPT2LMHeadModel(cfg).eval()
    with torch.no_grad():
        ref.transformer.ln_f.weight.mul_(8.0)
    ref.load_state_dict(GH._bf16_exact(ref.state_dict()))
    ours = GPT2LMHeadModel(cfg, device="cuda", world_size=1)
    ours.load_reference_state_dict(ref.state_dict())
    assert ours.hn == 96
    return ref, ours


def test_greedy_matches_transformers_and_cached_logits_match_uncached_forward():
    """Greedy ids equal transformers' until the oracle's top-2 margin first drops below GH.MARGIN; at every step the cached
    logits equal transformers' logits on the same prefix and the model's own uncached forward, within the bf16 tolerance."""
    ref, ours = _gen_pair()
    ids = torch.randint(4, GH.V, (2, 40), generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        want = ref.generate(input_ids=ids, max_new_tokens=30, return_dict_in_generate=True, output_scores=True)
    got = ours.generate(input_ids=ids.cuda(), max_new_tokens=30, return_dict_in_generate=True, output_scores=True)
    seq = got.sequences.cpu()
    assert torch.equal(seq[:, :40], ids)
    assert GH._decisive_compare(seq, want.sequences, want.scores, 40) >= 1
    cached = torch.stack(got.scores, 1)
    with torch.no_grad():
        oracle = ref(input_ids=seq[:, :-1]).logits[:, 39:]
    assert (cached.cpu() - oracle).abs().max().item() <= GH._tol(oracle)
    full = ours(input_ids=got.sequences[:, :-1]).logits.float()[:, 39:]
    assert (cached - full).abs().max().item() <= GH._tol(full)


def test_left_padding_gives_the_row_alone_continuation():
    """A left-padded row decodes as the row alone: the same tokens and, at every step, the same logits within the bf16
    tolerance; the padding is visible to the check (the oracle with the padding not masked gives different logits)."""
    ref, ours = _gen_pair(seed=2)
    g = torch.Generator().manual_seed(3)
    a = torch.randint(4, GH.V, (1, 37), generator=g)
    b = torch.randint(4, GH.V, (1, 22), generator=g)
    ids = torch.full((2, 37), 3, dtype=torch.int64)
    ids[0], ids[1, 15:] = a[0], b[0]
    mask = (torch.arange(37)[None] >= torch.tensor([[0], [15]])).long()
    kw = dict(max_new_tokens=12, return_dict_in_generate=True, output_scores=True)
    out = ours.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), **kw)
    alone_a = ours.generate(input_ids=a.cuda(), **kw)
    alone_b = ours.generate(input_ids=b.cuda(), **kw)
    assert torch.equal(out.sequences[0, 37:], alone_a.sequences[0, 37:])
    assert torch.equal(out.sequences[1, 37:], alone_b.sequences[0, 22:])
    padded, single = torch.stack(out.scores, 1)[1], torch.stack(alone_b.scores, 1)[0]
    assert (padded - single).abs().max().item() <= GH._tol(single)
    with torch.no_grad():
        seen = ref(input_ids=ids[1:], attention_mask=torch.ones_like(ids[1:])).logits[0, -1]
        hidden = ref(input_ids=b).logits[0, -1]
    assert (seen - hidden).abs().max().item() > 10 * GH._tol(hidden)


def test_decode_cache_is_padded_to_128_columns_and_the_padding_stays_zero(monkeypatch):
    """The cache generate allocates is [layers, rows, cap, 2, heads, 128]; after a run the columns past 96 are still zero."""
    _, ours = _gen_pair()
    seen = []
    real = torch.zeros

    def zeros(*shape, **kw):
        t = real(*shape, **kw)
        if len(t.shape) == 6:
            seen.append(t)
        return t
    monkeypatch.setattr(torch, "zeros", zeros)
    ids = torch.randint(4, GH.V, (2, 24), generator=torch.Generator().manual_seed(3)).cuda()
    ours.generate(input_ids=ids, max_new_tokens=10, num_beams=2)
    monkeypatch.undo()
    assert seen and all(t.shape[-1] == 128 and t.shape[-2] == 4 for t in seen)
    assert any(t[..., :96].abs().sum().item() > 0 for t in seen)
    assert all(not t[..., 96:].any().item() for t in seen)


def _gpt2_96(seed=0):
    import transformers
    cfg = transformers.GPT2Config(vocab_size=GG.V, n_positions=256, n_embd=384, n_layer=2, n_head=4, bos_token_id=3,
                                  eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
    m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=seed)
    with torch.no_grad():
        m.transformer.ln_f.weight.mul_(8.0)
    return m


GRAPH_CASES = {
    "greedy": dict(max_new_tokens=20),
    "beam2": dict(max_new_tokens=16, num_beams=2, return_dict_in_generate=True, output_scores=True),
    # the Wenzhong README's sampling call
    "readme_sampling": dict(max_length=60, do_sample=True, top_p=0.9, num_return_sequences=5, return_dict_in_generate=True,
                            output_scores=True, eos_token_id=3, pad_token_id=0),
}


@pytest.mark.parametrize("case", sorted(GRAPH_CASES))
def test_graph_decode_equals_eager_decode(case, monkeypatch):
    m = _gpt2_96()
    ids = torch.randint(4, GG.V, (3, 24), generator=torch.Generator().manual_seed(7)).cuda()
    a, b = GG._both(monkeypatch, lambda: m.generate(input_ids=ids, **GRAPH_CASES[case]))
    GG._assert_same(a, b)


def test_left_padding_graph_equals_eager(monkeypatch):
    m = _gpt2_96(seed=1)
    ids, mask = GG._left_padded(4, 30, 3, seed=8)
    for kw in (dict(max_new_tokens=18, return_dict_in_generate=True, output_scores=True),
               dict(max_new_tokens=12, num_beams=3, return_dict_in_generate=True, output_scores=True)):
        a, b = GG._both(monkeypatch, lambda: m.generate(input_ids=ids, attention_mask=mask, **kw))
        GG._assert_same(a, b)


# ------------------------------------------------------------------------------------------------ full width
FULL = dict(vocab_size=50304, n_positions=1024, n_embd=3072, n_layer=2, n_head=32)


def test_full_width_two_layers_vs_transformers():
    """2 layers of the 3.5B shape (hidden 3072, 32 heads x 96) at seq 1024, as test_baseline_shapes_gpu.py does for C2."""
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    ref, mine = _pair(FULL, seed=0)
    batch = H.make_lm_batch(FULL["vocab_size"], 1, 1024, seed=77)
    out_ref = ref(input_ids=batch["input_ids"], labels=batch["labels"])
    out_ref.loss.backward()
    out = mine(input_ids=batch["input_ids"].cuda(), labels=batch["labels"].cuda(), return_logits=True)
    assert abs(out.loss.item() - out_ref.loss.item()) <= 3e-3, (out.loss.item(), out_ref.loss.item())
    tol = 4 * 2.0 ** -8 * out_ref.logits.abs().max().item()
    assert (out.logits.float().cpu() - out_ref.logits.detach()).abs().max().item() <= tol
    out.loss.backward()
    torch.cuda.synchronize()
    _grad_check(mine, ref)
    del ref, mine, out, out_ref
    gc.collect(); torch.cuda.empty_cache()


def _full_width_workload(monkeypatch):
    """bench's gpt2-110m workload at the 3.5B width (3072, 32 heads x 96, V 50304), 4 sequences of 1024."""
    import bench
    real = bench.workload

    def workload(name):
        w = dict(real(name))
        if name == "gpt2-110m":
            w.update(n_embd=3072, n_head=32, vocab_size=50304, per_gpu=4, micro=4)
        return w
    monkeypatch.setattr(bench, "workload", workload)


def test_every_launch_of_a_full_width_dropout_step_against_fp64():
    with pytest.MonkeyPatch.context() as mp:
        _full_width_workload(mp)
        GD.test_every_launch_of_a_gpt2_dropout_step_against_fp64(mp)


def test_write_footprint_of_every_launch_of_a_full_width_dropout_step():
    import launch_census
    import launch_refs as LR
    stats = F.Stats()
    with pytest.MonkeyPatch.context() as mp:
        _full_width_workload(mp)
        mp.setattr(LR, "CHECKERS", F.footprint_checkers(stats))
        GD.test_every_launch_of_a_gpt2_dropout_step_against_fp64(mp)
    assert {"sdpa_fwd", "sdpa_bwd"} <= set(stats.checked), sorted(stats.checked)
    assert launch_census is not None
