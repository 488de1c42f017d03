"""CPU: the generation controller (fsb200/generation.py) against transformers' own `generate` (HF 5.5.0).

`step` wraps a tiny fp32 transformers MT5 or GPT-2 together with its own `past_key_values`, so both sides see the same
logits and only the token-selection loop differs: greedy, sampling (same torch seed => the same draws), beam search
(HF's `_beam_search`, processors on log-probabilities), eos / pad filling and the length limits. The decode loops of the
fsb200 models themselves are GPU-tested in tests/test_generate_hf_gpu.py."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))

from fsb200 import generation as G  # noqa: E402

V = 96


@pytest.fixture(scope="module")
def t5():
    from transformers import MT5Config, MT5ForConditionalGeneration
    torch.manual_seed(0)
    cfg = MT5Config(vocab_size=V, d_model=32, d_kv=8, d_ff=64, num_layers=2, num_heads=4, relative_attention_num_buckets=8,
                    dropout_rate=0.0, pad_token_id=0, eos_token_id=1, decoder_start_token_id=0)
    m = MT5ForConditionalGeneration(cfg).eval()
    with torch.no_grad():
        # sharper distributions through the final norm, not the tied embedding (that would make the model echo its input):
        # a small token embedding lets the layers' outputs, and so the history, decide the next token
        m.shared.weight.mul_(1.0 / 16)
        m.decoder.final_layer_norm.weight.mul_(8.0)
        for blk in m.decoder.block:
            blk.layer[0].SelfAttention.v.weight.mul_(4.0)
    return m


@pytest.fixture(scope="module")
def gpt2():
    from transformers import GPT2Config, GPT2LMHeadModel
    torch.manual_seed(1)
    cfg = GPT2Config(vocab_size=V, n_positions=64, n_embd=32, n_layer=2, n_head=4, bos_token_id=3, eos_token_id=3,
                     resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
    m = GPT2LMHeadModel(cfg).eval()
    with torch.no_grad():
        m.transformer.ln_f.weight.mul_(8.0)
    return m


def _enc_inputs():
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(2, V, (2, 9), generator=g)
    mask = torch.ones_like(ids)
    mask[1, 6:] = 0
    ids[1, 6:] = 0
    return ids, mask


def _dec_inputs():
    g = torch.Generator().manual_seed(8)
    ids = torch.randint(4, V, (2, 7), generator=g)
    mask = torch.ones_like(ids)
    ids[1, :3] = 3        # left padding with the pad (= eos) id
    mask[1, :3] = 0
    return ids, mask


def _t5_generate(model, ids, mask, **kw):
    """fsb200's controller driving the transformers MT5 through its own cache."""
    c = G.resolve(model.config, kw, 1, True)
    ids, mask = ids.repeat_interleave(c.expand, 0), mask.repeat_interleave(c.expand, 0)
    enc = model.get_encoder()(input_ids=ids, attention_mask=mask)
    st = {"past": None, "tok": torch.full((ids.shape[0], 1), c.start, dtype=torch.int64)}

    def step(tokens, reorder):
        if tokens is not None:
            if reorder is not None:
                st["past"].reorder_cache(reorder)
            st["tok"] = tokens[:, None]
        out = model(encoder_outputs=enc, attention_mask=mask, decoder_input_ids=st["tok"], past_key_values=st["past"],
                    use_cache=True)
        st["past"] = out.past_key_values
        return out.logits[:, -1].float()

    with torch.no_grad():
        return G.run(step, st["tok"].clone(), c)


def _gpt2_generate(model, ids, mask, **kw):
    c = G.resolve(model.config, kw, ids.shape[1], False)
    ids, mask = ids.repeat_interleave(c.expand, 0), mask.repeat_interleave(c.expand, 0)
    st = {"past": None, "mask": mask}

    def step(tokens, reorder):
        if tokens is None:
            pos = (mask.cumsum(-1) - 1).masked_fill(mask == 0, 0)
            out = model(input_ids=ids, attention_mask=mask, position_ids=pos, use_cache=True)
        else:
            if reorder is not None:
                st["past"].reorder_cache(reorder)
                st["mask"] = st["mask"][reorder]
            st["mask"] = torch.cat([st["mask"], torch.ones_like(st["mask"][:, :1])], 1)
            pos = st["mask"].sum(-1, keepdim=True) - 1
            out = model(input_ids=tokens[:, None], attention_mask=st["mask"], position_ids=pos,
                        past_key_values=st["past"], use_cache=True)
        st["past"] = out.past_key_values
        return out.logits[:, -1].float()

    with torch.no_grad():
        return G.run(step, ids.clone(), c)


def _both(model, kind, seed=None, **kw):
    ids, mask = _enc_inputs() if kind == "t5" else _dec_inputs()
    if seed is not None:
        torch.manual_seed(seed)
    with torch.no_grad():
        want = model.generate(input_ids=ids, attention_mask=mask, **kw)
    if seed is not None:
        torch.manual_seed(seed)
    got = (_t5_generate if kind == "t5" else _gpt2_generate)(model, ids, mask, **kw)
    return got, want


def _seqs(x):
    return x if isinstance(x, torch.Tensor) else x.sequences


@pytest.mark.parametrize("kind", ["t5", "gpt2"])
def test_greedy_sequences_and_scores(kind, t5, gpt2):
    model = t5 if kind == "t5" else gpt2
    got, want = _both(model, kind, max_new_tokens=12, return_dict_in_generate=True, output_scores=True)
    assert torch.equal(got.sequences, want.sequences)
    assert len(got.scores) == len(want.scores)
    for a, b in zip(got.scores, want.scores):
        assert torch.allclose(a, b, atol=1e-6, rtol=0)
    g2, w2 = _both(model, kind, max_length=14, repetition_penalty=2.5)
    assert torch.equal(g2, w2)


@pytest.mark.parametrize("num_beams", [2, 4])
@pytest.mark.parametrize("length_penalty", [0.6, 1.0, 2.0])
@pytest.mark.parametrize("early_stopping", [True, False])
def test_beam_search_matches_transformers_t5(num_beams, length_penalty, early_stopping, t5):
    kw = dict(num_beams=num_beams, length_penalty=length_penalty, early_stopping=early_stopping, repetition_penalty=2.5,
              num_return_sequences=2, max_length=16, return_dict_in_generate=True, output_scores=True)
    got, want = _both(t5, "t5", **kw)
    assert torch.equal(got.sequences, want.sequences)
    assert torch.allclose(got.sequences_scores, want.sequences_scores, atol=1e-6, rtol=0)
    assert len(got.scores) == len(want.scores)


@pytest.mark.parametrize("early_stopping", [True, False, "never"])
def test_beam_search_matches_transformers_gpt2(early_stopping, gpt2):
    kw = dict(num_beams=3, early_stopping=early_stopping, num_return_sequences=3, max_new_tokens=10,
              return_dict_in_generate=True, output_scores=True)
    got, want = _both(gpt2, "gpt2", **kw)
    assert torch.equal(got.sequences, want.sequences)
    assert torch.allclose(got.sequences_scores, want.sequences_scores, atol=1e-6, rtol=0)
    assert torch.equal(_both(gpt2, "gpt2", num_beams=2, max_new_tokens=6)[0], _both(gpt2, "gpt2", num_beams=2,
                                                                                    max_new_tokens=6)[1])


@pytest.mark.parametrize("kind", ["t5", "gpt2"])
@pytest.mark.parametrize("kw", [dict(top_p=0.9), dict(top_k=7), dict(temperature=0.7, top_k=0),
                                dict(repetition_penalty=1.3, top_p=0.8, temperature=1.4),
                                dict(top_p=0.9, num_return_sequences=3)])
def test_sampling_draws_identical_tokens(kind, kw, t5, gpt2):
    model = t5 if kind == "t5" else gpt2
    got, want = _both(model, kind, seed=1234, do_sample=True, max_new_tokens=10, return_dict_in_generate=True,
                      output_scores=True, **kw)
    assert torch.equal(got.sequences, want.sequences)
    for a, b in zip(got.scores, want.scores):
        assert torch.equal(torch.isinf(a), torch.isinf(b))
        assert torch.allclose(a[torch.isfinite(a)], b[torch.isfinite(b)], atol=1e-5, rtol=0)


def test_eos_stops_rows_and_pads_the_finished_ones(t5, gpt2):
    # pick as eos a token the greedy continuation of row 0 emits early, so row 0 stops and row 1 runs on
    free = _both(gpt2, "gpt2", max_new_tokens=10, eos_token_id=None)[1]
    eos = int(free[0, 7 + 2])
    pad = 0 if eos != 0 else 1
    got, want = _both(gpt2, "gpt2", max_new_tokens=10, eos_token_id=eos, pad_token_id=pad)
    assert torch.equal(got, want)
    row = got[0, 7:].tolist()
    i = row.index(eos)
    assert all(t == pad for t in row[i + 1:])
    freet = _both(t5, "t5", max_length=12)[1]
    eos = int(freet[1, 3])
    got, want = _both(t5, "t5", max_length=12, eos_token_id=eos)
    assert torch.equal(got, want)
    got, want = _both(t5, "t5", max_length=12, eos_token_id=[eos, int(freet[0, 5])], num_beams=2)
    assert torch.equal(got, want)


def test_max_new_tokens_and_max_length(t5, gpt2):
    g, w = _both(gpt2, "gpt2", max_new_tokens=5)
    assert torch.equal(g, w) and g.shape[1] == 7 + 5
    g, w = _both(gpt2, "gpt2", max_length=9)
    assert torch.equal(g, w) and g.shape[1] == 9
    g, w = _both(t5, "t5", max_new_tokens=4, max_length=30)   # max_new_tokens wins, as in HF
    assert torch.equal(g, w) and g.shape[1] <= 1 + 4
    g, w = _both(t5, "t5")                                     # default max_length 20
    assert torch.equal(g, w)


@pytest.mark.parametrize("kw", [dict(force_words_ids=[[5]]), dict(num_beam_groups=2), dict(no_repeat_ngram_size=3),
                                dict(num_beams=2, do_sample=True)])
def test_unsupported_keywords_raise(kw, t5):
    name = next(iter(kw)) if "do_sample" not in kw else "do_sample"
    with pytest.raises(NotImplementedError, match=name):
        G.resolve(t5.config, kw, 1, True)
    G.resolve(t5.config, dict(num_beam_groups=1, no_repeat_ngram_size=0, force_words_ids=None), 1, True)


def test_fixtures_are_not_echoes(t5, gpt2):
    """The parity cases above only test something when the fixtures' continuations depend on their input: greedy rows that
    are not a repeat of their last input token and several distinct tokens per batch, beams whose scores are not 0 (a certain continuation), and sampling distributions that
    spread their mass over more than one token."""
    for model, kind in ((t5, "t5"), (gpt2, "gpt2")):
        ids, mask = _enc_inputs() if kind == "t5" else _dec_inputs()
        start = 1 if kind == "t5" else ids.shape[1]
        with torch.no_grad():
            g = model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=12)
            b = model.generate(input_ids=ids, attention_mask=mask, num_beams=4, num_return_sequences=2, max_length=16,
                               repetition_penalty=2.5, return_dict_in_generate=True, output_scores=True)
            s = model.generate(input_ids=ids, attention_mask=mask, do_sample=True, max_new_tokens=6,
                               return_dict_in_generate=True, output_scores=True)
        gen = g[:, start:]
        assert bool((gen != ids[:, -1:]).any(1).all()) and len(set(gen.flatten().tolist())) >= 3, (kind, g)
        assert bool((b.sequences_scores < -0.05).all()), (kind, b.sequences_scores)
        top = torch.stack([torch.softmax(x, -1).max(-1).values for x in s.scores])
        assert float(top.median()) < 0.9, (kind, top)
