"""GPU: FP8 training of mT5 / Randeng-T5 (`MT5ForConditionalGeneration(config, fp8=True)`).

Against transformers fp32 on the small config of test_t5_gpu.py: loss and logits at init, every parameter's gradient cosine,
and the 20-step loss curve beside bf16's distance from fp32. Bit identity with itself: the CUDA-graph step equals eager under
ZeRO-1 and ZeRO-2 with GA 2 at dropout 0.1, packed dropout steps repeat run to run, the no-grad forward equals the training
forward, and `generate` equals the bf16 model's on the same weights. The fp64 and write-footprint censuses of one FP8 step at
Randeng-T5 width (2 + 2 layers). Refusals and `from_pretrained(path, fp8=True)`."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

import fp8_epilogue_refs as E
from test_t5_dropout_gpu import _hf
from test_t5_packing_gpu import PAD, SD, SE, _padded

from fsb200 import lib as L, ops
from fsb200.engine import ZeroEngine
from fsb200.models.t5 import MT5ForConditionalGeneration
from fsb200.packing import pack_seq2seq_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

C5 = dict(vocab_size=32600, d_model=1024, d_kv=64, d_ff=2816, num_heads=16)


def _mine(ref, fp8=True, config=None):
    m = MT5ForConditionalGeneration(config or ref.config, device="cuda", fp8=fp8)
    m.load_reference_state_dict(ref.state_dict())
    return m


def _cuda(b):
    return {k: v.cuda() for k, v in b.items()}


def _grads(m):
    return {n: q.main_grad.float().cpu().flatten().clone() for n, q in m.named_parameters()}


def _cos(a, b):
    return (torch.dot(a, b) / (a.norm() * b.norm() + 1e-30)).item()


# -------------------------------------------------------------------------------------------- against transformers
def test_loss_logits_and_gradients_vs_transformers():
    """The small config (d_model 256, d_ff 512, 2 + 2 layers) on the batch of test_t5_gpu.py (2 x 96 / 48, 13 encoder pads).
    HF's init draws the tied embedding from N(0, 1), so the logits are O(100) and the loss O(150). Measured on an H100 80GB
    HBM3 (700 W): loss 167.783 against fp32's 167.436 (2.07e-3 relative; test_t5_gpu.py holds bf16 to 3e-3 + 5e-4
    relative, 5.2e-4 here), logits within 2.53e-2 of the largest logit (bf16's bar: 1.56e-2), worst gradient cosine 0.9792
    (encoder layer 1's query weight; bf16 holds 0.998). The bars: loss within 4e-3 relative, logits within 4e-2 of the
    largest, every gradient cosine >= 0.97."""
    ref = H.build_mt5(H.MT5_SMALL)
    batch = H.make_t5_batch(H.MT5_SMALL["vocab_size"], 2, 96, 48, seed=7, pad_tail=13)
    out_ref = ref(**batch)
    out_ref.loss.backward()
    mine = _mine(ref)
    assert all(type(pj.qkv).__name__ == "Fp8Linear" for pj in mine._enc + mine._dec)
    out = mine(**_cuda(batch), return_logits=True)
    out.loss.backward()
    torch.cuda.synchronize()
    rel = abs(out.loss.item() - out_ref.loss.item()) / abs(out_ref.loss.item())
    lmax = out_ref.logits.abs().max().item()
    ldiff = (out.logits.float().cpu() - out_ref.logits).abs().max().item() / lmax
    refp = dict(ref.named_parameters())
    worst = (1.0, None)
    for name, got in _grads(mine).items():
        c = _cos(got, refp[name].grad.flatten())
        worst = min(worst, (c, name))
    print(f"[t5 fp8] loss {out.loss.item():.4f} vs {out_ref.loss.item():.4f} (rel {rel:.2e}); logits max diff "
          f"{ldiff:.3e} of max |logit|; worst gradient cosine {worst}")
    assert rel <= 4e-3, (out.loss.item(), out_ref.loss.item())
    assert ldiff <= 4e-2, ldiff
    assert worst[0] >= 0.97, worst


def test_loss_curve_within_bf16_noise():
    """20 AdamW steps on the small config against transformers fp32 (relative distance, the curve runs from ~160 down to
    ~20). Measured on an H100 80GB HBM3 (700 W): FP8 2.36e-2 against bf16's 4.73e-3, 5.0x, outside LLaMA's 2.5x bar; the
    FP8 curve still falls from 159 to 19 with fp32's. Why mT5 lands further out than LLaMA or BERT is not established. One
    unverified guess: its N(0, 1) embeddings and unscaled attention put wide-ranging values through the e4m3 casts. The
    bars: at most 8x bf16's distance and at most 4e-2 relative."""
    steps, lr = 20, 1e-3
    V = H.MT5_SMALL["vocab_size"]
    batches = [H.make_t5_batch(V, 2, 64, 32, seed=40 + i) for i in range(4)]
    ref = H.build_mt5(H.MT5_SMALL)
    opt = torch.optim.AdamW(ref.parameters(), lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    want = []
    for it in range(steps):
        opt.zero_grad()
        out = ref(**batches[it % 4])
        out.loss.backward()
        opt.step()
        want.append(out.loss.item())
    want = np.array(want)
    curves = {}
    for fp8 in (False, True):
        mine = _mine(H.build_mt5(H.MT5_SMALL), fp8=fp8)
        eng = ZeroEngine(mine, lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
        c = []
        for it in range(steps):
            out = mine(**_cuda(batches[it % 4]))
            out.loss.backward()
            eng.backward_done()
            eng.step()
            c.append(out.loss.item())
        curves[fp8] = np.array(c)
    err8 = (np.abs(curves[True] - want) / np.abs(want)).max()
    err16 = (np.abs(curves[False] - want) / np.abs(want)).max()
    print(f"[t5 fp8] 20-step curve: |fp8 - fp32| / fp32 = {err8:.3e}, |bf16 - fp32| / fp32 = {err16:.3e}; "
          f"fp8 {curves[True][0]:.2f} -> {curves[True][-1]:.2f}")
    assert np.isfinite(curves[True]).all() and curves[True][-1] < 0.5 * curves[True][0]
    assert err8 <= 8 * err16 and err8 <= 4e-2, (err8, err16)


# ------------------------------------------------------------------------------------------------------------ paths
def _graph_vs_eager(stage):
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        model = _mine(_hf(0.1))
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2,
                          stage=stage, cuda_graph=graph)
        losses = []
        for it in range(4):
            # no attention_mask: a device mask is inspected on the host, which a captured step cannot do
            mbs = [{k: v.cuda() for k, v in H.make_t5_batch(H.MT5_SMALL["vocab_size"], 2, 64, 32, seed=300 + 2 * it + m)
                    .items() if k != "attention_mask"} for m in range(2)]
            losses.append(float(st.step_device(mbs)))
        runs.append((losses, model.flat.params.clone()))
    return runs


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_equals_eager_ga2_dropout(stage):
    (l0, p0), (l1, p1) = _graph_vs_eager(stage)
    assert all(math.isfinite(x) for x in l0)
    assert l0 == l1, (l0, l1)
    assert torch.equal(p0, p1)


def test_packed_dropout_steps_repeat_and_graph_equals_eager():
    """Packed rows (segment_ids + decoder_segment_ids) at dropout 0.1: two eager runs give the same bits, and the CUDA-graph
    step equals them."""
    from fsb200.trainer import PretrainStep
    p = pack_seq2seq_batch(_padded(16, seed=21), SE, SD, PAD)
    packed = {k: v[:2].cuda() for k, v in p.items() if k != "attention_mask"}
    runs = []
    for graph in (False, False, True):
        torch.manual_seed(3)
        model = _mine(_hf(0.1))
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, weight_decay=0.01, ga_steps=1, cuda_graph=graph)
        losses = [float(st.step_device([packed])) for _ in range(3)]
        runs.append((losses, model.flat.params.clone()))
    assert all(math.isfinite(x) for x in runs[0][0])
    for losses, params in runs[1:]:
        assert losses == runs[0][0] and torch.equal(params, runs[0][1])


def test_no_grad_forward_equals_grad_forward():
    mine = _mine(H.build_mt5(H.MT5_SMALL))
    b = _cuda(H.make_t5_batch(H.MT5_SMALL["vocab_size"], 2, 96, 48, seed=8, pad_tail=13))
    out = mine(**b, return_logits=True)
    with torch.no_grad():
        out2 = mine(**b, return_logits=True)
    assert out.loss.item() == out2.loss.item()
    assert torch.equal(out.logits, out2.logits)


def test_generate_equals_the_bf16_model():
    """generate runs the bf16 projections: greedy and beam search of an fp8=True model equal the bf16 model's."""
    ref = H.build_mt5(H.MT5_SMALL, seed=4)
    m8, m16 = _mine(ref, fp8=True), _mine(ref, fp8=False)
    ids = torch.randint(2, H.MT5_SMALL["vocab_size"], (3, 40), generator=torch.Generator().manual_seed(2)).cuda()
    for kw in (dict(max_length=12, do_sample=False), dict(max_length=8, num_beams=3, do_sample=False)):
        assert torch.equal(m8.generate(ids, **kw), m16.generate(ids, **kw)), kw


def test_refusals():
    """A width or token count that is not a multiple of 16 is named, and only the values that fail are."""
    V = H.MT5_SMALL["vocab_size"]
    m = _mine(H.build_mt5(dict(H.MT5_SMALL, d_ff=520)))
    with pytest.raises(ValueError, match=r"fp8=True\): d_ff \(520\) not a multiple of 16") as e:
        m(**_cuda(H.make_t5_batch(V, 2, 64, 32, seed=1)))
    assert "d_model (" not in str(e.value) and "x source length" not in str(e.value)
    m = _mine(H.build_mt5(H.MT5_SMALL))
    with pytest.raises(ValueError, match=r"fp8=True\): batch 3 x target length 114 \(342\) not a multiple of 16.*"
                                         r"micro-batch must be a multiple of 8") as e:
        m(**_cuda(H.make_t5_batch(V, 3, 64, 114, seed=1)))
    assert "source length" not in str(e.value) and "d_ff (" not in str(e.value)
    with pytest.raises(ValueError, match=r"fp8=True\): batch 3 x source length 40 \(120\) not a multiple of 16") as e:
        m(**_cuda(H.make_t5_batch(V, 3, 40, 32, seed=1)))
    assert "x target length" not in str(e.value)
    with pytest.raises(ValueError, match=r"batch 3 x source length 40 \(120\), batch 3 x target length 30 \(90\) not"):
        m(**_cuda(H.make_t5_batch(V, 3, 40, 30, seed=1)))
    out = m(**_cuda(H.make_t5_batch(V, 8, 64, 114, seed=1)))   # micro-batch 8 at 114 is fine
    assert math.isfinite(out.loss.item())
    with pytest.raises(NotImplementedError):
        m.gradient_checkpointing_enable()


def test_from_pretrained_forwards_fp8(tmp_path):
    import fsb200.hf as hf
    ref = H.build_mt5(H.MT5_SMALL, seed=5)
    _mine(ref, fp8=False).save_pretrained(str(tmp_path / "m"))
    m = hf.MT5ForConditionalGeneration.from_pretrained(str(tmp_path / "m"), fp8=True, device="cuda")
    assert m.fp8 and all(type(pj.ckv).__name__ == "Fp8Linear" for pj in m._dec)
    back = hf.MT5ForConditionalGeneration.from_pretrained(str(tmp_path / "m"), device="cuda")
    assert not back.fp8 and torch.equal(back.flat.params, m.flat.params)


# ---------------------------------------------------------------------------------------------------------- censuses
def _c5_fp8_census(monkeypatch, checkers):
    """One FP8 training step at Randeng-T5 width (d_model 1024, d_ff 2816, 16 heads), 2 encoder and 2 decoder layers,
    micro-batch 8 at 512 / 512, GA 2, ZeRO-2, every op launch recorded and its first call of each signature checked."""
    from types import SimpleNamespace
    from launch_census import Recorder
    from fsb200.trainer import PretrainStep
    torch.manual_seed(0)
    cfg = SimpleNamespace(num_layers=2, num_decoder_layers=2, relative_attention_num_buckets=32,
                          relative_attention_max_distance=128, dropout_rate=0.1, feed_forward_proj="gated-gelu",
                          tie_word_embeddings=True, layer_norm_epsilon=1e-6, pad_token_id=0, decoder_start_token_id=0, **C5)
    model = MT5ForConditionalGeneration(cfg, device="cuda", seed=1, fp8=True)
    st = PretrainStep(model, lambda s_: 1e-4, lr=1e-4, betas=(0.9, 0.999), weight_decay=0.1, grad_clip=1.0, ga_steps=2)
    mbs = [_cuda(H.make_t5_batch(C5["vocab_size"], 8, 512, 512, seed=60 + m)) for m in range(2)]
    for mb in mbs:
        mb.pop("attention_mask")
    rec = Recorder(checkers)
    rec.install(monkeypatch)
    c0 = L.launch_count
    try:
        loss = st.step_device(mbs)
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    assert {"fp8_quantize", "gemm_fp8"} <= {key[0] for key in rec.calls}
    assert L.launch_count - c0 - rec.extra_launches == rec.wrapped_launches
    assert math.isfinite(float(loss.item()))
    return rec


def test_every_launch_of_a_c5_width_fp8_step_against_fp64(monkeypatch):
    import launch_refs as LR
    checkers = dict(LR.CHECKERS)
    checkers["gemm_fp8"] = E.check_gemm_fp8
    rec = _c5_fp8_census(monkeypatch, checkers)
    # the cross k|v data gradients are summed into the encoder-output gradient [8 * 512, 1024] in fp32
    assert any(k[0] == "accumulate" and dict(k[1])["x16"][1] == (8 * 512, C5["d_model"]) for k in rec.checked)


def test_write_footprint_of_every_launch_of_a_c5_width_fp8_step(monkeypatch):
    import footprint as F
    stats = F.Stats()
    monkeypatch.setitem(F.WRITES, "gemm_fp8", F._gemm)
    _c5_fp8_census(monkeypatch, F.footprint_checkers(stats))
    assert "gemm_fp8" in stats.checked


# ---------------------------------------------------------------------------------------------------- bf16 unchanged
def test_fp8_false_launch_sequence_matches_the_bf16_record(monkeypatch):
    """fp8=False launches exactly what the model launched before it had an FP8 path: every kernel, in order, with its
    integer arguments (sizes, strides, flags, dropout sites, scratch sizes; device pointers and the stream left out), over two
    micro-batches of a dropout-0.1 step with GA 2 and the optimizer step, a packed step, a no-grad forward and a greedy
    generate. tests/golden/t5_bf16_launches.json holds that sequence, recorded on an H100 80GB HBM3 from the model as it
    was before fp8 existed, with the attention rows since translated to the current entry names fsb_sdpa_fwd /
    fsb_sdpa_bwd (the integer arguments the old entries did not take inserted at the values the model passes)."""
    from transformers import MT5Config
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "t5_bf16_launches.json")))
    got = []
    real = L.call

    def spy(name, *a, **k):
        # the stream is the last argument of every call; pointers are above 2^40
        got.append([name] + [x for x in a if isinstance(x, int) and abs(x) < 1 << 40][:-1])
        return real(name, *a, **k)
    monkeypatch.setattr(L, "call", spy)
    # the library's scratch buffers grow with the largest request a process has made, and their sizes are kernel
    # arguments: start from none, as the recording did
    monkeypatch.setattr(ops, "_ws_cache", {})
    torch.manual_seed(0)
    cfg = MT5Config(dropout_rate=0.1, feed_forward_proj="gated-gelu", decoder_start_token_id=0, pad_token_id=0,
                    **dict(H.MT5_SMALL, num_decoder_layers=3))
    m = MT5ForConditionalGeneration(cfg, device="cuda", seed=1)
    eng = ZeroEngine(m, lr=1e-3, ga_steps=2)
    b = _cuda(H.make_t5_batch(512, 2, 96, 48, seed=7, pad_tail=13))
    for _ in range(2):
        out = m(**b)
        out.loss.backward()
        eng.backward_done()
    eng.step()
    out = m(**_cuda(pack_seq2seq_batch(_padded(10, seed=1), 128, 64, 0)))
    out.loss.backward()
    eng.backward_done()
    with torch.no_grad():
        m(**b)
    m.eval()
    m.generate(b["input_ids"], max_length=10, do_sample=False)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert not any("fp8" in g[0] for g in got)
    assert len(got) == len(want), (len(got), len(want))
    first = next((i for i, (g, w) in enumerate(zip(got, want)) if g != w), None)
    assert first is None, (first, got[first], want[first])
