"""CPU: the token selection of `generate` (repetition penalty -> temperature -> top-k -> top-p -> sample), as the controller
fsb200/generation.py runs it for every model, against transformers' own logits processors — what the reference's
`model.generate(**generate_kwargs)` applies (fengshen/examples/ziya_llama/llama_generate.py:33-34 with the kwargs of :52-61).
Same processed distribution => the same token from the same torch generator. The decode loop itself (KV cache, left
padding) is GPU-tested in tests/test_generate_gpu.py."""
import os
import sys
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))


def _select(logits, seqs, do_sample, temperature, top_k, top_p, penalty, generator):
    """The token generation.run appends after one step that returns `logits` for the rows `seqs`."""
    from fsb200 import generation
    c = SimpleNamespace(num_beams=1, do_sample=do_sample, temperature=temperature, top_k=top_k, top_p=top_p,
                        repetition_penalty=penalty, max_length=seqs.shape[1] + 1, output_scores=False, return_dict=False,
                        eos=None, pad=0)
    out = generation.run(lambda tokens, reorder: logits, seqs, c, generator)
    assert out.shape == (seqs.shape[0], seqs.shape[1] + 1) and torch.equal(out[:, :-1], seqs)
    return out[:, -1]


@pytest.mark.parametrize("temperature,top_k,top_p,penalty", [(0.8, 0, 1.0, 1.0), (1.0, 50, 1.0, 1.0), (0.7, 0, 0.85, 1.0),
                                                             (1.3, 40, 0.9, 1.2), (1.0, 0, 1.0, 1.5), (0.5, 1, 0.3, 1.0)])
def test_controller_selection_matches_transformers_logits_processors(temperature, top_k, top_p, penalty):
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    g = torch.Generator().manual_seed(0)
    B, V = 6, 503
    for trial in range(8):
        logits = torch.randn(B, V, generator=g) * 3.0
        seqs = torch.randint(0, V, (B, 17), generator=g)
        want = logits.clone()
        if penalty != 1.0:
            want = RepetitionPenaltyLogitsProcessor(penalty)(seqs, want)
        if temperature != 1.0:
            want = TemperatureLogitsWarper(temperature)(seqs, want)
        if top_k > 0:
            want = TopKLogitsWarper(top_k)(seqs, want)
        if top_p < 1.0:
            want = TopPLogitsWarper(top_p)(seqs, want)
        g_ref, g_ours = torch.Generator().manual_seed(100 + trial), torch.Generator().manual_seed(100 + trial)
        expect = torch.multinomial(torch.softmax(want, -1), 1, generator=g_ref).squeeze(1)
        got = _select(logits.clone(), seqs, True, temperature, top_k, top_p, penalty, g_ours)
        assert torch.equal(got, expect), (trial, got, expect)
        # greedy: arg-max of the penalised logits, no warpers
        greedy = _select(logits.clone(), seqs, False, temperature, top_k, top_p, penalty, None)
        base = RepetitionPenaltyLogitsProcessor(penalty)(seqs, logits.clone()) if penalty != 1.0 else logits
        assert torch.equal(greedy, base.argmax(-1))
