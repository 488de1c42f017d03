"""GPU parity at the real widths of the two BASELINE configs test_baseline_shapes_gpu.py does not cover, against the
transformers classes the reference trains, on CPU in fp32 with bf16-exact weights:

  C3  Erlangshen-MegatronBERT-1.3B: h 2048, 32 heads x 64, ff 8192, seq 512, V 21128, with 2 layers at batch 2 (MLM + SOP)
      against transformers.MegatronBertForPreTraining.
  C5  Randeng-T5-784M: d 1024, 16 heads x 64 with relative bias, gated-GeLU d_ff 2816, encoder and decoder 512, V 32600,
      tied head, with 2 + 2 layers at batch 2 against transformers.MT5ForConditionalGeneration.

Criteria as in test_baseline_shapes_gpu.py: loss 3e-3 (4e-3 for the BERT pair; mT5 adds 5e-4 relative, its random-init
loss is O(100), test_t5_gpu._loss_close), logits within 4 * 2^-8 * max|logit|, every parameter gradient at cosine >= 0.998
with its norm within 3 %.
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)


def _check_grads(mine_named, ref_grads, cos_min=0.998, ratio_tol=0.03, qk_cos_min=None):
    """The per-parameter criteria. A self-attention key bias adds q . b_k to every score of a query row, which the softmax
    ignores: its gradient is zero in exact arithmetic. transformers' fp32 gives 1e-8. Ours is the residue of
    delta = rowsum(dO O) formed from the bf16 O: with delta off by e_q, sum_k dS[q, k] = -e_q instead of 0, so the key-bias
    gradient is -scale sum_q e_q q, a coherent sum. Measured on one H100 80GB HBM3 (700 W): 3.3e-4 against a query-bias
    gradient of 2.9e-3 in MegatronBERT's layer 1. It is held below 25 % of the same layer's query-bias gradient instead of
    being compared by direction.
    The query and key projections of MegatronBERT at h 2048 are held to cosine >= 0.99 instead of 0.998: measured on one
    H100 80GB HBM3 (700 W), layer 1's query weight reaches 0.9948. At this width the random-init attention is close to
    uniform, so dS = P (dP - delta) is a small difference, and the bf16 O that delta is formed from (as in every flash-style
    backward) leaves a larger relative error in it than in the other gradients. The attention backward itself is held
    elementwise to its derived fp64 bound at this shape (B 32, 32 heads x 64, seq 512) by
    test_workload_launches_gpu.py[megatronbert-1.3b]."""
    checked = 0
    for name, prm in mine_named:
        qk = cos_min if qk_cos_min is None or not any(f"attention.self.{p}." in name for p in ("query", "key")) else qk_cos_min
        if name.endswith("attention.self.key.bias"):
            live = ref_grads[name.replace(".key.", ".query.")].norm().item()
            got, want = prm.main_grad.float().norm().item(), ref_grads[name].norm().item()
            assert got <= 0.25 * live and want <= 0.25 * live, (name, got, want, live)
            checked += 1
            continue
        got = prm.main_grad.float().cpu().flatten()
        want = ref_grads[name]
        if want is None or want.norm().item() < 1e-9:
            assert got.norm().item() < 1e-4, name
            continue
        want = want.flatten()
        cos = (torch.dot(got, want) / (got.norm() * want.norm() + 1e-30)).item()
        assert cos >= qk, (name, cos)
        assert abs(got.norm().item() / want.norm().item() - 1.0) <= ratio_tol, (name, got.norm().item(), want.norm().item())
        checked += 1
    return checked


def test_erlangshen_megatronbert_1_3b_real_width_vs_transformers():
    from fsb200.models.bert import MegatronBertForPreTraining
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    cfg = dict(vocab_size=21128, hidden_size=2048, num_hidden_layers=2, num_attention_heads=32, intermediate_size=8192,
               max_position_embeddings=512, type_vocab_size=2)
    ref = H.build_megatron_bert(cfg)
    batch = H.make_mlm_batch(cfg["vocab_size"], 2, 512, seed=31, nsp=True)     # BASELINE configs[2]: seq 512
    out_ref = ref(**batch)
    out_ref.loss.backward()
    mine = MegatronBertForPreTraining(ref.config, device="cuda")
    mine.load_reference_state_dict(ref.state_dict())
    out = mine(**{k: v.cuda() for k, v in batch.items()}, return_logits=True)
    assert abs(out.loss.item() - out_ref.loss.item()) <= 4e-3, (out.loss.item(), out_ref.loss.item())
    ref_logits = out_ref.prediction_logits
    tol = 4 * 2.0 ** -8 * ref_logits.abs().max().item()
    assert (out.logits.float().cpu() - ref_logits).abs().max().item() <= tol
    out.loss.backward()
    torch.cuda.synchronize()
    refg = {n: p.grad for n, p in ref.named_parameters()}
    assert _check_grads([(n, p) for n, p in mine.named_parameters() if n in refg], refg, qk_cos_min=0.99) > 0


def test_randeng_t5_784m_real_width_vs_transformers():
    from fsb200.models.t5 import MT5ForConditionalGeneration
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    cfg = dict(vocab_size=32600, d_model=1024, d_kv=64, d_ff=2816, num_layers=2, num_decoder_layers=2, num_heads=16,
               relative_attention_num_buckets=32, relative_attention_max_distance=128)
    ref = H.build_mt5(cfg)
    batch = H.make_t5_batch(cfg["vocab_size"], 2, 512, 512, seed=41)            # BASELINE configs[4]: enc 512 / dec 512
    out_ref = ref(**batch)
    out_ref.loss.backward()
    mine = MT5ForConditionalGeneration(ref.config, device="cuda")
    mine.load_reference_state_dict(ref.state_dict())
    out = mine(**{k: v.cuda() for k, v in batch.items()}, return_logits=True)
    want = out_ref.loss.item()
    assert abs(out.loss.item() - want) <= 3e-3 + 5e-4 * abs(want), (out.loss.item(), want)
    tol = 4 * 2.0 ** -8 * out_ref.logits.abs().max().item()
    assert (out.logits.float().cpu() - out_ref.logits).abs().max().item() <= tol
    out.loss.backward()
    torch.cuda.synchronize()
    refg = {n: p.grad for n, p in ref.named_parameters()}
    # every parameter of the HF model has a counterpart (embed_tokens / the tied lm_head are aliases of shared.weight)
    assert _check_grads(mine.named_parameters(), refg) == len(refg)
