"""GPU: KV-cache generation of the HF-backed models, `MT5ForConditionalGeneration.generate` and `GPT2LMHeadModel.generate`,
on the split-KV decode kernel. Token ids are an integer output: the greedy continuation must equal transformers' CPU fp32
`generate` on the same bf16-exact weights wherever the oracle's own top-2 margin is larger than the bf16 noise of the logits.
The cached step logits must match fsb200's own uncached forward over the same prefix within the bf16 logits tolerance of
tests/test_t5_gpu.py (4 * 2^-8 of the largest logit).

The random-init fixtures are shaped so that these checks can see attention. Scaling the TIED embedding would make each model
echo its input token with a huge margin, so the logits are sharpened through the final norm instead. In mT5 the token
embedding is scaled down (the residual stream then carries the layers' outputs rather than the input token), the decoder's
self-attention values are scaled up (the history drives the logits) and the decoder's relative-position bias table is scaled
to the O(1-10) range of a trained T5 (the bias moves the logits by far more than the tolerance). Every scale is a power of
two, so the weights stay bf16-exact. `_assert_nontrivial` checks that the oracle's continuations are not constant echoes."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))

from fsb200.models.gpt2 import GPT2LMHeadModel  # noqa: E402
from fsb200.models.t5 import MT5ForConditionalGeneration  # noqa: E402

V = 512
MARGIN = 0.4          # logits; above the bf16 noise of the logits


def _bf16_exact(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def _tol(logits):
    return 4 * 2.0 ** -8 * logits.abs().max().item()


def _pair_t5(seed=0, self_attn_gain=4.0):
    import transformers
    torch.manual_seed(seed)
    cfg = transformers.MT5Config(vocab_size=V, d_model=256, d_kv=64, d_ff=512, num_layers=2, num_heads=4,
                                 relative_attention_num_buckets=32, dropout_rate=0.0, pad_token_id=0, eos_token_id=1,
                                 decoder_start_token_id=0)
    ref = transformers.MT5ForConditionalGeneration(cfg).eval()
    with torch.no_grad():
        ref.shared.weight.mul_(1.0 / 16)
        ref.decoder.final_layer_norm.weight.mul_(8.0)
        for blk in ref.decoder.block:
            blk.layer[0].SelfAttention.v.weight.mul_(self_attn_gain)
        ref.decoder.block[0].layer[0].SelfAttention.relative_attention_bias.weight.mul_(32.0)
    ref.load_state_dict(_bf16_exact(ref.state_dict()))
    ours = MT5ForConditionalGeneration(cfg, device="cuda", world_size=1)
    ours.load_reference_state_dict(ref.state_dict())
    return ref, ours


def _pair_gpt2(seed=0):
    import transformers
    torch.manual_seed(seed)
    cfg = transformers.GPT2Config(vocab_size=V, n_positions=256, n_embd=256, n_layer=2, n_head=4, bos_token_id=3,
                                  eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
    ref = transformers.GPT2LMHeadModel(cfg).eval()
    with torch.no_grad():
        ref.transformer.ln_f.weight.mul_(8.0)
    ref.load_state_dict(_bf16_exact(ref.state_dict()))
    ours = GPT2LMHeadModel(cfg, device="cuda", world_size=1)
    ours.load_reference_state_dict(ref.state_dict())
    return ref, ours


def _assert_nontrivial(gen, last_in):
    """Each row of the oracle's continuation has at least 3 distinct tokens and is not a repeat of the last input token."""
    for b, row in enumerate(gen.tolist()):
        assert len(set(row)) >= 3 and any(t != int(last_in[b]) for t in row), (b, row)


def _decisive_steps(scores):
    """[rows] number of leading steps whose oracle top-2 margin is at least MARGIN."""
    m = torch.stack([s.topk(2, -1).values.diff(dim=-1).abs()[:, 0] for s in scores], 1)
    return (m >= MARGIN).int().cumprod(1).sum(1)


def _decisive_compare(got, want, scores, start):
    """Rows must agree token by token until the oracle's top-2 margin first drops below MARGIN."""
    n = _decisive_steps(scores)
    for b in range(want.shape[0]):
        k = int(n[b])
        assert torch.equal(got[b, start:start + k], want[b, start:start + k]), b
    return int(n.sum())


def _enc_batch(B=3, S=29, seed=5):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, V, (B, S), generator=g)
    mask = torch.ones_like(ids)
    mask[1, 20:] = 0
    ids[1, 20:] = 0
    return ids, mask


def test_mt5_greedy_matches_transformers_and_cached_logits_match_uncached_forward():
    ref, ours = _pair_t5()
    ids, mask = _enc_batch()
    with torch.no_grad():
        want = ref.generate(input_ids=ids, attention_mask=mask, max_new_tokens=24, return_dict_in_generate=True,
                            output_scores=True)
    _assert_nontrivial(want.sequences[:, 1:], torch.zeros(3, dtype=torch.int64))
    got = ours.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), max_new_tokens=24, return_dict_in_generate=True,
                        output_scores=True)
    seq = got.sequences.cpu()
    assert torch.equal(seq[:, 0], torch.zeros(3, dtype=torch.int64))
    assert _decisive_compare(seq, want.sequences, want.scores, 1) >= 8
    # every cached step's logits == the training-path forward over decoder_input_ids = the generated prefix; the decoder's
    # self-attention sees distinct histories and a position bias that moves the logits by far more than the tolerance
    steps = len(got.scores)
    full = ours(input_ids=ids.cuda(), attention_mask=mask.cuda(), decoder_input_ids=got.sequences[:, :steps]).logits.float()
    cached = torch.stack(got.scores, 1)
    assert (cached - full).abs().max().item() <= _tol(full)
    # and the same logits against the fp32 oracle, teacher-forced on the same tokens
    with torch.no_grad():
        oracle = ref(input_ids=ids, attention_mask=mask, decoder_input_ids=seq[:, :steps]).logits
    assert (cached.cpu() - oracle).abs().max().item() <= _tol(oracle)


class _Jitter:
    """Uniform noise of +-amp on the processed scores: a bf16-sized perturbation of the oracle's search."""

    def __init__(self, seed, amp):
        self.g, self.amp = torch.Generator().manual_seed(seed), amp

    def __call__(self, input_ids, scores):
        return scores + (torch.rand(scores.shape, generator=self.g) * 2 - 1) * self.amp


def _stable_beam_rows(ref, ids, mask, want, kw, runs=4, amp=0.25):
    """Rows whose oracle beam result survives `runs` jittered searches: only there must a bf16 search agree."""
    from transformers import LogitsProcessorList
    keep = torch.ones(want.shape[0], dtype=torch.bool)
    for r in range(runs):
        with torch.no_grad():
            alt = ref.generate(input_ids=ids, attention_mask=mask, logits_processor=LogitsProcessorList([_Jitter(r, amp)]),
                               **kw)
        n = min(alt.shape[1], want.shape[1])
        keep &= (alt[:, :n] == want[:, :n]).all(1)
    return [b for b in range(want.shape[0]) if keep[b]]


def test_mt5_beam_search_matches_transformers_on_stable_rows():
    ref, ours = _pair_t5(seed=2)
    ids, mask = _enc_batch(seed=7)
    kw = dict(max_length=20, num_beams=2, repetition_penalty=2.5, length_penalty=1.0, early_stopping=True)
    with torch.no_grad():
        want = ref.generate(input_ids=ids, attention_mask=mask, **kw)
    _assert_nontrivial(want[:, 1:], torch.zeros(3, dtype=torch.int64))
    stable = _stable_beam_rows(ref, ids, mask, want, kw)
    assert stable, "no row of the oracle's beam search is stable under bf16-sized noise"
    got = ours.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), **kw).cpu()
    assert got.shape[0] == 3 and torch.equal(got[:, 0], torch.zeros(3, dtype=torch.int64))
    for b in stable:
        n = min(got.shape[1], want.shape[1])
        assert torch.equal(got[b, :n], want[b, :n]), b
    two = ours.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), num_return_sequences=2, **kw).cpu()
    assert two.shape[0] == 6 and torch.equal(two[0::2, :got.shape[1]], got)   # the best hypothesis comes first


def test_gpt2_greedy_matches_transformers_and_cached_logits_match_uncached_forward():
    ref, ours = _pair_gpt2()
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(4, V, (2, 40), generator=g)
    with torch.no_grad():
        want = ref.generate(input_ids=ids, max_new_tokens=30, return_dict_in_generate=True, output_scores=True)
    _assert_nontrivial(want.sequences[:, 40:], ids[:, -1])
    got = ours.generate(input_ids=ids.cuda(), max_new_tokens=30, return_dict_in_generate=True, output_scores=True)
    seq = got.sequences.cpu()
    assert torch.equal(seq[:, :40], ids)
    assert _decisive_compare(seq, want.sequences, want.scores, 40) >= 8
    steps = len(got.scores)
    full = ours(input_ids=got.sequences[:, :40 + steps - 1]).logits.float()[:, 39:]
    cached = torch.stack(got.scores, 1)
    assert (cached - full).abs().max().item() <= _tol(full)


def test_gpt2_left_padding_gives_the_row_alone_continuation():
    """A left-padded row must decode exactly as the row alone: the same tokens and, at every step, the same logits within the
    bf16 tolerance. The padding is visible to the check: the oracle with the padding NOT masked gives different logits."""
    ref, ours = _pair_gpt2(seed=2)
    g = torch.Generator().manual_seed(3)
    a = torch.randint(4, V, (1, 37), generator=g)
    b = torch.randint(4, V, (1, 22), generator=g)
    ids = torch.full((2, 37), 3, dtype=torch.int64)
    ids[0], ids[1, 15:] = a[0], b[0]
    mask = (torch.arange(37)[None] >= torch.tensor([[0], [15]])).long()
    kw = dict(max_new_tokens=12, return_dict_in_generate=True, output_scores=True)
    out = ours.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), **kw)
    alone_a = ours.generate(input_ids=a.cuda(), **kw)
    alone_b = ours.generate(input_ids=b.cuda(), **kw)
    assert torch.equal(out.sequences[0, 37:], alone_a.sequences[0, 37:])
    assert torch.equal(out.sequences[1, 37:], alone_b.sequences[0, 22:])
    _assert_nontrivial(alone_b.sequences[:, 22:].cpu(), b[:, -1])
    padded, single = torch.stack(out.scores, 1)[1], torch.stack(alone_b.scores, 1)[0]
    assert (padded - single).abs().max().item() <= _tol(single)
    with torch.no_grad():
        seen = ref(input_ids=ids[1:], attention_mask=torch.ones_like(ids[1:])).logits[0, -1]
        hidden = ref(input_ids=b).logits[0, -1]
    assert (seen - hidden).abs().max().item() > 10 * _tol(hidden)
    with pytest.raises(ValueError, match="n_positions"):
        ours.generate(input_ids=a.cuda(), max_length=300)


def test_seeded_sampling_is_reproducible():
    _, ours = _pair_gpt2()
    prompt = torch.randint(4, V, (2, 16), generator=torch.Generator().manual_seed(1)).cuda()
    kw = dict(return_dict_in_generate=True, output_scores=True, max_length=60, do_sample=True, top_p=0.9, eos_token_id=3,
              pad_token_id=0, num_return_sequences=5)
    torch.manual_seed(0)
    s1 = ours.generate(input_ids=prompt, **kw)
    torch.manual_seed(0)
    s2 = ours.generate(input_ids=prompt, **kw)
    assert torch.equal(s1.sequences, s2.sequences) and s1.sequences.shape[0] == 10
    assert len(s1.scores) == s1.sequences.shape[1] - 16
    assert len({tuple(r) for r in s1.sequences[:5].tolist()}) > 1      # the draws differ between return sequences
    _, t5 = _pair_t5()
    ids, mask = _enc_batch()
    torch.manual_seed(4)
    a = t5.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), do_sample=True, top_k=20, max_length=16)
    torch.manual_seed(4)
    b = t5.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), do_sample=True, top_k=20, max_length=16)
    assert torch.equal(a, b)


def test_mt5_summary_predict_step_through_trainer_predict():
    import pytorch_lightning as pl
    ref, ours = _pair_t5()
    ids, mask = _enc_batch()

    class Summary(pl.LightningModule):
        def __init__(self):
            super().__init__()
            self.model = ours
            self.args = type("A", (), {"max_dec_length": 12})()

        # fengshen/examples/mt5_summary/mt5_summary.py:131-139, restated unchanged
        def predict_step(self, batch, batch_idx):
            text = batch['text']
            summary = batch['summary']
            generated_ids = self.model.generate(
                input_ids=batch['input_ids'],
                attention_mask=batch['attention_mask'],
                max_length=self.args.max_dec_length
            )
            return {"pred": generated_ids, "text": text, "summary": summary}

    class Data(pl.LightningDataModule):
        def predict_dataloader(self):
            return [{"input_ids": ids.cuda(), "attention_mask": mask.cuda(), "text": ["t"] * 3, "summary": ["s"] * 3}]

    out = pl.Trainer(devices=1).predict(Summary(), datamodule=Data())
    assert len(out) == 1 and out[0]["text"] == ["t"] * 3
    with torch.no_grad():
        want = ref.generate(input_ids=ids, attention_mask=mask, max_length=12, return_dict_in_generate=True,
                            output_scores=True)
    _assert_nontrivial(want.sequences[:, 1:], torch.zeros(3, dtype=torch.int64))
    pred = out[0]["pred"].cpu()
    assert pred.shape[0] == 3 and pred.shape[1] <= 12
    decisive = [b for b, n in enumerate(_decisive_steps(want.scores).tolist()) if n == len(want.scores)]
    assert decisive, "no fully decisive row"
    n = min(pred.shape[1], want.sequences.shape[1])
    for b in decisive:
        assert torch.equal(pred[b, :n], want.sequences[b, :n]), b


def _captured_step(model, monkeypatch, **kw):
    """The step function `generate` hands to the controller (fsb200/generation.py), captured before any token is chosen."""
    from fsb200 import generation
    got = {}

    def capture(step, seqs, c, generator=None):
        got.update(step=step, seqs=seqs)
        return seqs

    monkeypatch.setattr(generation, "run", capture)
    model.generate(**kw)
    monkeypatch.undo()
    return got["step"], got["seqs"]


@pytest.mark.parametrize("kind", ["t5", "gpt2"])
def test_cache_rows_follow_the_beam_reorder(kind, monkeypatch):
    """Beam search hands each step a gather of the rows: every new beam continues some old beam of its batch item. Feed
    random tokens under random gathers and compare every cached step with the uncached forward of the gathered histories,
    within the bf16 logits tolerance."""
    g = torch.Generator().manual_seed(11)
    if kind == "t5":
        _, ours = _pair_t5()
        ids, mask = _enc_batch()
        step, hist = _captured_step(ours, monkeypatch, input_ids=ids.cuda(), attention_mask=mask.cuda(), num_beams=3,
                                    max_length=16)
        enc, emask = ids.repeat_interleave(3, 0).cuda(), mask.repeat_interleave(3, 0).cuda()
        full = lambda h: ours(input_ids=enc, attention_mask=emask, decoder_input_ids=h).logits[:, -1].float()  # noqa
    else:
        _, ours = _pair_gpt2()
        ids = torch.randint(4, V, (3, 20), generator=g)
        step, hist = _captured_step(ours, monkeypatch, input_ids=ids.cuda(), num_beams=3, max_new_tokens=10)
        full = lambda h: ours(input_ids=h).logits[:, -1].float()  # noqa: E731
    R = hist.shape[0]
    assert R == 9
    logits = step(None, None)
    for t in range(8):
        f = full(hist)
        assert (logits - f).abs().max().item() <= _tol(f), t
        # as beam search does: every new beam of a batch item continues some beam of the same item (repeats allowed)
        reorder = ((torch.arange(R) // 3) * 3 + torch.randint(0, 3, (R,), generator=g)).cuda()
        tokens = torch.randint(4, V, (R,), generator=g).cuda()
        hist = torch.cat([hist[reorder], tokens[:, None]], 1)
        logits = step(tokens, reorder)
