"""GPU: the gradient every model hands to AdamW through the ZeRO engine, checked exactly, at a depth where ZeRO-2 folds the
per-layer gradient buckets onto rotating slots (`FlatBuffers.compact_grads` needs at least 3 equally sized layer buckets; every
model here has 4 layers per stack).

The reference is a twin model with the same parameters and no engine, run with loss_scale = 1 / GA: its bf16 gradients of each
micro-batch, g0 and g1, are what the engine must hand to AdamW (`ZeroEngine._grad_seg`):
  * GA 1, ZeRO-1 or ZeRO-2: g0, bit for bit (the same deterministic kernels on the same inputs);
  * ZeRO-2, GA 2: the fp32 accumulator holds g0.float() + g1.float() bit for bit (the accumulate kernel is one fp32 add per
    element);
  * ZeRO-1, GA 2: the wgrad epilogues accumulate the bf16 buffer in place, so the engine's gradient is bit for bit what the twin
    gets by accumulating in place itself, and each element lies within two bf16 roundings of g0 + g1 (see `_check_stage1_ga2`).
"""
from types import SimpleNamespace

import pytest
import torch
from torch import nn

from fsb200.engine import ZeroEngine
from fsb200.flat import FlatBuffers
from fsb200.models.bert import BertForMaskedLM, MegatronBertForPreTraining
from fsb200.models.gpt2 import GPT2LMHeadModel
from fsb200.models.layers import GatedMLP, Linear
from fsb200.models.llama import LlamaForCausalLM
from fsb200.models.t5 import MT5ForConditionalGeneration
from fsb200.trainer import PretrainStep

pytestmark = pytest.mark.gpu

V, H = 512, 256
_BERT = dict(vocab_size=V, hidden_size=H, num_hidden_layers=4, num_attention_heads=4, intermediate_size=512,
             max_position_embeddings=128, type_vocab_size=2)
_LLAMA = dict(vocab_size=V, hidden_size=H, num_hidden_layers=4, rms_norm_epsilon=1e-6, max_position_embeddings=128,
              rotary_emb_base=10000, llama_mlp_multiple_of=256)
MODELS = {
    "gpt2": (GPT2LMHeadModel, dict(vocab_size=V, n_positions=128, n_embd=H, n_layer=4, n_head=4)),
    "bert": (BertForMaskedLM, _BERT),
    "megatronbert": (MegatronBertForPreTraining, _BERT),
    "mt5": (MT5ForConditionalGeneration, dict(vocab_size=V, d_model=H, d_kv=64, d_ff=512, num_layers=4, num_decoder_layers=4,
                                              num_heads=4, relative_attention_num_buckets=32,
                                              relative_attention_max_distance=128, tie_word_embeddings=True)),
    "llama_hd64": (LlamaForCausalLM, dict(_LLAMA, num_attention_heads=4)),
    "llama_hd128": (LlamaForCausalLM, dict(_LLAMA, num_attention_heads=2)),
}
# (ZeRO stage, gradient-accumulation steps)
CONFIGS = [(1, 1), (2, 1), (1, 2), (2, 2)]
B, S, S_DEC, PAD = 2, 64, 32, 11


def _model(name):
    cls, cfg = MODELS[name]
    return cls(SimpleNamespace(**cfg), device="cuda", seed=0)


def _batch(name, seed, mask=True):
    """One micro-batch; the last row's tail is padding (masked keys and ignored labels) wherever the model takes a mask."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, V, (B, S), generator=g)
    am = torch.ones_like(ids)
    am[-1, S - PAD:] = 0
    if name == "mt5":
        ids[-1, S - PAD:] = 0
        labels = torch.randint(2, V, (B, S_DEC), generator=g)
        labels[:, -3:] = -100
        b = dict(input_ids=ids, attention_mask=am, labels=labels)
    elif name in ("bert", "megatronbert"):
        labels = torch.where(torch.rand(B, S, generator=g) < 0.15, ids, torch.full_like(ids, -100))
        labels[-1, S - PAD:] = -100
        tt = torch.zeros_like(ids)
        tt[:, S // 2:] = 1
        b = dict(input_ids=ids, attention_mask=am, token_type_ids=tt, labels=labels)
        if name == "megatronbert":
            b["next_sentence_label"] = torch.randint(0, 2, (B,), generator=g)
    else:   # causal LMs: GPT-2 masks padded keys; LLaMA takes no mask and only ignores the padded labels
        labels = ids.clone()
        labels[-1, S - PAD:] = -100
        b = dict(input_ids=ids, attention_mask=am, labels=labels) if name == "gpt2" else dict(input_ids=ids, labels=labels)
    if not mask:
        b.pop("attention_mask", None)
    return {k: v.cuda() for k, v in b.items()}


def _batches(name, ga, seed, mask=True):
    return [_batch(name, seed + m, mask) for m in range(ga)]


def _slices(flat):
    """(name, slice of the flat parameter layout) of every parameter."""
    return [(n, slice(off, off + torch.Size(shape).numel())) for n, (off, shape) in flat.offsets.items()]


def _reference(model, twin, batches, ga, accumulate=False):
    """The twin's bf16 gradient after each micro-batch, from model's current parameters. accumulate: the twin accumulates its
    later micro-batches in place (the wgrad epilogues' ZeRO-1 path) instead of overwriting."""
    twin.flat.params.copy_(model.flat.params)
    twin.loss_scale = 1.0 / ga
    grads = []
    for m, b in enumerate(batches):
        twin.accumulate_grads = accumulate and m > 0
        twin(**b).loss.backward()
        grads.append(twin.flat.grads.clone())
    twin.accumulate_grads = False
    return grads


def _engine_micro_batches(model, eng, batches):
    for b in batches:
        model(**b).loss.backward()
        eng.backward_done()


def _engine_grad(eng):
    """The gradient AdamW is about to consume, in the flat parameter layout (one rank: a bucket's shard is the bucket)."""
    f = eng.flat
    out = torch.zeros(f.total, dtype=eng._grad_seg(0).dtype, device=f.params.device)
    for i, (_, start, length, _) in enumerate(f.buckets):
        out[start:start + length] = eng._grad_seg(i)
    return out


def _oracle(g, ga):
    """The exact gradient the step should consume, fp32: g0, or the fp32 sum g0 + g1."""
    return g[0].float() if ga == 1 else g[0].float() + g[1].float()


def _check_stage1_ga2(flat, got, g, acc_twin):
    """ZeRO-1, GA 2. The wgrad epilogues add micro-batch 1's fp32 partial s1 into the bf16 buffer holding g0, so
    got = bf16(g0 + s1), while the twin's g1 = bf16(s1): two bf16 roundings. Round-to-nearest with 8 significant bits is within
    2^-8 |r| of the value it rounds to r, so |got - (g0 + g1)| <= 2^-8 (|g1| + |got|), and got is exactly 0 where g0 and g1 both
    are. (2^-8 (|g0| + |g1|) does not bound it: with g0 small against g1 both roundings can approach 2^-8 |g1|, and about 1% of
    the elements of every parameter exceed it.)
    A tied embedding table is written k times per micro-batch (the LM head's GEMM, then one scatter-add per embedding lookup),
    rounding once per write, and the writes can cancel, so no element-wise bound relative to the result holds for it. Its 2k
    roundings are bounded in norm instead, by 2k * 2^-8 of the norm of |g0| + |g1| (measured: about 2.5e-3 of it). A dropped
    accumulation leaves an error of |g0|, far beyond either bound. The exact comparison with the twin that accumulates in place
    covers every parameter."""
    bad = [n for n, s in _slices(flat) if not torch.equal(got[s], acc_twin[s])]
    assert not bad, f"engine gradient differs from the twin accumulating in place in: {bad}"
    assert torch.equal(got, acc_twin), "engine gradient differs in the padding between parameters"
    g0, g1, gf = g[0].float(), g[1].float(), got.float()
    err = (gf - (g0 + g1)).abs()
    bound = 2.0 ** -8 * (g1.abs() + gf.abs())
    tied = _tied_writes(flat)
    over = {}
    for n, s in _slices(flat):
        if n in tied:
            continue
        if bool((err[s] > bound[s]).any()):
            i = int((err[s] - bound[s]).argmax())
            over[n] = (float(g0[s][i]), float(g1[s][i]), float(gf[s][i]))
    assert not over, f"beyond two bf16 roundings of g0 + g1 (g0, g1, engine) at the worst element: {over}"
    for n, k in tied.items():
        s = dict(_slices(flat))[n]
        e, scale = float(err[s].norm()), float((g0[s].abs() + g1[s].abs()).norm())
        assert e <= 2 * k * 2.0 ** -8 * scale, f"{n}: |engine - (g0 + g1)| = {e:.4g}, {e / scale:.3g} of |g0| + |g1|"


# tied embedding table -> gradient writes per micro-batch (LM-head GEMM + embedding scatter-adds)
_TIED = {"transformer.wte.weight": 2, "bert.embeddings.word_embeddings.weight": 2, "shared.weight": 3}


def _tied_writes(flat):
    return {n: k for n, k in _TIED.items() if n in flat.offsets}


def _tensors(obj, path, seen):
    """(attribute path, tensor) of every tensor reachable from obj through attributes (of modules, flat buffers and the
    models' projections), lists, tuples, dicts and a parameter's .main_grad."""
    if id(obj) in seen:
        return
    seen.add(id(obj))
    if isinstance(obj, torch.Tensor):
        yield path, obj
        mg = getattr(obj, "main_grad", None)
        if mg is not None:
            yield from _tensors(mg, path + ".main_grad", seen)
        return
    if isinstance(obj, dict):
        items = [(f"{path}[{k!r}]", v) for k, v in obj.items()]
    elif isinstance(obj, (list, tuple)):
        items = [(f"{path}[{i}]", v) for i, v in enumerate(obj)]
    elif isinstance(obj, (nn.Module, FlatBuffers, Linear, GatedMLP)):
        items = [(f"{path}.{k}", v) for k, v in vars(obj).items()]
    else:
        return
    for p, v in items:
        yield from _tensors(v, p, seen)


# ---- A: no tensor of the model stays on the gradient buffer ZeRO-2 released ---------------------------------------------------
@pytest.mark.parametrize("name", list(MODELS))
def test_zero2_compaction_leaves_no_stale_gradient_alias(name):
    model = _model(name)
    old = model.flat.grads.untyped_storage()     # held: its address cannot be handed out again while the walk runs
    ZeroEngine(model, stage=2, ga_steps=2)
    assert model.flat.grads.numel() < model.flat.total, "the layer buckets were not folded onto rotating gradient slots"
    stale = [p for p, t in _tensors(model, "model", set()) if t.untyped_storage().data_ptr() == old.data_ptr()]
    assert not stale, f"still on the released gradient buffer: {stale}"
    # every gradient view the flat buffers handed out is held where the walk sees it, not only by the flat buffers' own list
    reached = {id(model.flat)}
    for _ in _tensors(model, "model", reached):
        pass
    unseen = [(off, shape) for t, off, shape in model.flat._grad_views if id(t) not in reached]
    assert not unseen, f"gradient views the walk does not reach outside the flat buffers (offset, shape): {unseen}"


# ---- B: the gradient the engine hands to AdamW, exactly --------------------------------------------------------------------
@pytest.mark.parametrize("stage,ga", CONFIGS)
@pytest.mark.parametrize("name", list(MODELS))
def test_engine_gradient_equals_twin_gradients(name, stage, ga):
    model, twin = _model(name), _model(name)
    batches = _batches(name, ga, seed=10)
    g = _reference(model, twin, batches, ga)
    eng = ZeroEngine(model, stage=stage, ga_steps=ga)
    if stage == 2 and ga == 2:
        assert model.flat.grads.numel() < model.flat.total       # rotating slots in use
    _engine_micro_batches(model, eng, batches)
    got = _engine_grad(eng)
    ref = _oracle(g, ga)
    frozen = [n for n, s in _slices(model.flat) if bool(ref[s].ne(0).any()) and not bool(got[s].ne(0).any())]
    assert not frozen, f"the reference gradient is non-zero, the engine's is all zero: {frozen}"
    if stage == 1 and ga == 2:
        _check_stage1_ga2(model.flat, got, g, _reference(model, twin, batches, ga, accumulate=True)[-1])
        return
    want = g[0] if ga == 1 else ref
    assert got.dtype == want.dtype
    bad = [n for n, s in _slices(model.flat) if not torch.equal(got[s], want[s])]
    assert not bad, f"engine gradient is not bit-identical to the reference in: {bad}"
    assert torch.equal(got, want), "engine gradient differs in the padding between parameters"


# ---- C: every parameter with a gradient trains, and the clipping norm is the oracle's ----------------------------------------
@pytest.mark.parametrize("stage,ga", CONFIGS)
@pytest.mark.parametrize("name", list(MODELS))
def test_every_parameter_with_a_gradient_trains(name, stage, ga):
    """Two clipped AdamW steps without weight decay: a parameter moves only through its gradient, and AdamW's first steps move
    an element by about lr whenever its gradient is non-zero, so a frozen parameter shows however small its gradient."""
    model, twin = _model(name), _model(name)
    eng = ZeroEngine(model, lr=1e-3, weight_decay=0.0, grad_clip=1.0, stage=stage, ga_steps=ga)
    for step in range(2):
        batches = _batches(name, ga, seed=20 + 10 * step)
        ref = _oracle(_reference(model, twin, batches, ga), ga)
        _engine_micro_batches(model, eng, batches)
        # the bit-exact configurations clip by the oracle's norm; ZeRO-1 with GA 2 by the norm of its own bf16 sum
        want_norm = float((ref if ga == 1 or stage == 2 else _engine_grad(eng).float()).double().norm())
        before = eng.master.clone()
        eng.step()
        moved = eng.master != before         # one rank: the fp32 master shard is the flat parameter layout
        frozen = [n for n, s in _slices(model.flat) if bool(ref[s].ne(0).any()) and not bool(moved[s].any())]
        assert not frozen, f"step {step + 1}: parameters with a non-zero gradient did not move: {frozen}"
        got_norm = float(eng.grad_norm)
        assert abs(got_norm - want_norm) <= 1e-5 * want_norm, (step + 1, got_norm, want_norm)


# ---- D: a replayed CUDA-graph step equals the eager step ---------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MODELS))
def test_cuda_graph_step_equals_eager_zero2_ga2(name):
    """ZeRO-2 with GA 2: the graph replays the rotating-slot reduction and fp32 accumulation. No attention_mask: the forward
    decides on the host whether a padding mask is needed, which a capture cannot do."""
    steps = [PretrainStep(_model(name), lambda s_: 1e-3, lr=1e-3, weight_decay=0.01, grad_clip=1.0, ga_steps=2, stage=2,
                          cuda_graph=graph) for graph in (False, True)]
    eager, graph = (st.engine for st in steps)
    flat = eager.flat
    for step in range(2):
        batches = _batches(name, 2, seed=40 + 10 * step, mask=False)
        losses = [st.step_device(batches) for st in steps]
        diff = [b for i, (b, _, _, _) in enumerate(flat.buckets)
                if not torch.equal(eager._seg(eager.acc32, i), graph._seg(graph.acc32, i))]
        assert not diff, f"step {step + 1}: fp32 gradient accumulator differs, first in bucket {diff[0]} (all: {diff})"
        bad = [n for n, s in _slices(flat) if not torch.equal(eager.flat.params[s], graph.flat.params[s])]
        assert not bad, f"step {step + 1}: parameters differ, first {bad[0]} ({len(bad)} in all)"
        assert torch.equal(losses[0], losses[1]), (step + 1, float(losses[0]), float(losses[1]))
