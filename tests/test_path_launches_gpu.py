"""Census of the shipped paths the benchmark step does not take: every launch of dropout training, FP8 LLaMA training and
KV-cache generation, checked against fp64 (tests/launch_refs.py) through the recorder of tests/launch_census.py.

Every case runs at full width with 2 layers (T5: 2 encoder and 2 decoder layers); training cases use the benchmark's
micro-batch and ZeRO stage with ga = min(bench ga, 2), as tests/test_workload_launches_gpu.py does.
- Dropout steps (bert-base, megatronbert-1.3b, randeng-t5-784m) at the released rate 0.1, the stream counter preset to
  2^32 - 5 so that base + site carries from the low stream word into the high one. The recorder keys each masked call by
  its site as well, so every site is value-checked once, and logs every stream drawn: the sites under each
  dropout_advance(n) are exactly range(n), the second base is the first plus n, and every (base, site) is drawn by one
  forward and one backward of one mask kind with one p, seed and mask shape (launch_census.dropout_stream_problems).
- The FP8 step: ziya-llama-13b with fp8=True.
- Generation with the decode step eager (FSB_GENERATE_GRAPH=0), model build and weight quantisation inside the census:
  GPT-2 at bench width (greedy, 4 beams), mT5 at Randeng width (padded encoder rows, 4 beams) and LLaMA at Ziya width in
  bf16, int8 and int4 (left-padded prompts of about 1000 tokens, sampling). attn_decode, kv_append and kv_reorder depend on
  the device-held kv_len, so every call of theirs is checked, and the test asserts that attn_decode ran over more than one
  split of its keys. LLaMA decodes with sdpa_fwd over its kv_mask-ed cache instead, so there every sdpa_fwd is checked.

Asserted for every case, as in the benchmark census: every op has a checker, lib.launch_count grew by exactly the launches
of the wrapped calls, every checked call is within its bound, and the loss (training) is finite. `-s` prints the census.
"""
import gc
import math
import os
import sys
import time
from types import SimpleNamespace

import pytest
import torch

import launch_refs as R
from launch_census import DropoutLog, Recorder, dropout_stream_problems, free_gib, print_table, site_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (read only: WORKLOADS, build_model, make_host_batches)

from fsb200 import lib as L, ops  # noqa: E402

P_DROP = 0.1                      # the released Erlangshen-BERT, MegatronBERT, mT5 and Randeng dropout rate
COUNTER_PRESET = 2 ** 32 - 5      # base + site crosses into the high stream word inside the first forward
DECODE_OPS = ("attn_decode", "kv_append", "kv_reorder")
# device memory (GiB) each case needs, its fp64 checks included: the peak allocated on one H100 80GB HBM3 at 700 W (dropout
# BERT-base 1.8, MegatronBERT 9.0, Randeng-T5 7.7; FP8 LLaMA 25.2; generate GPT-2 greedy 0.9, 4 beams 1.1, mT5 1.0, LLaMA
# bf16 7.2, int8 5.7, int4 5.4) plus 2 GiB for the allocator's rounding
NEED_GIB = {"dropout-bert-base": 4, "dropout-megatronbert-1.3b": 11, "dropout-randeng-t5-784m": 10, "fp8-ziya-llama-13b": 28,
            "generate-gpt2-greedy": 3, "generate-gpt2-beam4": 4, "generate-mt5-beam4": 3, "generate-llama-bf16": 10,
            "generate-llama-int8": 8, "generate-llama-int4": 8}


def _two_layers(w):
    w = dict(w)
    for k in ("n_layer", "num_hidden_layers", "num_layers"):
        if k in w:
            w[k] = 2
    return w


def _need(case):
    need = NEED_GIB[case]
    gc.collect(); torch.cuda.empty_cache()     # what earlier tests left in torch's cache counts as free here
    if free_gib() < need:
        pytest.skip(f"{case} at full width with 2 layers and its fp64 checks needs about {need} GiB free; "
                    f"{free_gib():.1f} GiB are")
    torch.cuda.reset_peak_memory_stats()


def _dropout_model(w, dev):
    """bench.build_model's BERT / mT5 at the released dropout rates (bench.build_model itself builds them at 0)."""
    if w["family"] == "bert":
        from fsb200.models.bert import BertForMaskedLM, MegatronBertForPreTraining
        cfg = SimpleNamespace(vocab_size=w["vocab_size"], hidden_size=w["hidden_size"],
                              num_hidden_layers=w["num_hidden_layers"], num_attention_heads=w["num_attention_heads"],
                              intermediate_size=w["intermediate_size"], hidden_act=w["hidden_act"],
                              max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                              hidden_dropout_prob=P_DROP, attention_probs_dropout_prob=P_DROP, initializer_range=0.02)
        cls = MegatronBertForPreTraining if w["variant"] == "megatron" else BertForMaskedLM
        return cls(cfg, device=dev, world_size=1)
    from fsb200.models.t5 import MT5ForConditionalGeneration
    cfg = SimpleNamespace(vocab_size=w["vocab_size"], d_model=w["d_model"], d_kv=w["d_kv"], d_ff=w["d_ff"],
                          num_layers=w["num_layers"], num_decoder_layers=w["num_layers"], num_heads=w["num_heads"],
                          relative_attention_num_buckets=32, relative_attention_max_distance=128, dropout_rate=P_DROP,
                          feed_forward_proj="gated-gelu", tie_word_embeddings=True, layer_norm_epsilon=1e-6,
                          pad_token_id=0, decoder_start_token_id=0)
    return MT5ForConditionalGeneration(cfg, device=dev, world_size=1)


def _finish(case, rec, growth, t0):
    print_table(case, rec, time.time() - t0, max(rec.peak, torch.cuda.max_memory_allocated()))
    assert growth - rec.extra_launches == rec.wrapped_launches, \
        (f"lib.launch_count grew by {growth - rec.extra_launches} (checker re-runs excluded) but the wrapped ops calls "
         f"launched {rec.wrapped_launches}: a kernel was reached without going through fsb200.ops")


def _run(monkeypatch, rec, fn):
    """fn() under the recorder, the patches undone afterwards. A failure is re-raised without the traceback that holds the
    model, so the next case finds the device memory free."""
    msg = None
    try:
        rec.install(monkeypatch)
        torch.cuda.synchronize()
        c0 = L.launch_count
        try:
            out = fn()
            torch.cuda.synchronize()
        finally:
            monkeypatch.undo()
        return out, L.launch_count - c0
    except AssertionError as e:
        msg = str(e)
    gc.collect(); torch.cuda.empty_cache()
    raise AssertionError(msg)


def _train_step(w, model, rec, monkeypatch):
    from fsb200.schedules import polynomial_lr
    from fsb200.trainer import PretrainStep
    w["micro"] = min(w["micro"], w["per_gpu"])
    ga = min(w["per_gpu"] // w["micro"], 2)
    dev = model.flat.params.device
    stepper = PretrainStep(model, lambda s_: polynomial_lr(s_, w["lr"], 10, 1000, 1e-7), lr=w["lr"], betas=w["betas"],
                           weight_decay=w["wd"], grad_clip=w["clip"], ga_steps=ga, stage=w.get("stage", 2),
                           cuda_graph=False)
    batches = [{k: v.to(dev) for k, v in b.items()} for b in bench.make_host_batches(w, ga, 0)]
    return _run(monkeypatch, rec, lambda: stepper.step_device(batches)), ga


# ------------------------------------------------------------------------------------------------------ dropout steps
@pytest.mark.parametrize("name", ["bert-base", "megatronbert-1.3b", "randeng-t5-784m"])
def test_every_launch_of_a_dropout_step_against_fp64(name, monkeypatch):
    case = f"dropout-{name}"
    _need(case)
    t0 = time.time()
    torch.manual_seed(0)
    w = _two_layers(bench.workload(name))
    dev = torch.device("cuda", torch.cuda.current_device())
    model = _dropout_model(w, dev)
    model.dropout_counter.fill_(COUNTER_PRESET)
    log = DropoutLog()
    rec = Recorder(R.CHECKERS, extra_key=site_of, observe=log.observe)
    (loss, growth), ga = _train_step(w, model, rec, monkeypatch)
    _finish(case, rec, growth, t0)
    assert math.isfinite(float(loss.item())), f"{case}: loss {loss.item()}"
    n = model.dropout_sites
    assert len(log.advances) == ga and log.advances[0] == (COUNTER_PRESET, n), \
        f"{case}: dropout_advance calls {log.advances}, want {ga} starting at the preset {COUNTER_PRESET} with n = {n}"
    assert any(b + s >= 2 ** 32 for _, b, s, *_ in log.uses) and any(b + s < 2 ** 32 for _, b, s, *_ in log.uses), \
        f"{case}: the streams drawn do not straddle 2^32, so the high stream word was not exercised"
    problems = dropout_stream_problems(log.advances, log.uses)
    assert not problems, f"{case}: " + "; ".join(problems[:5])
    checked_sites = {k[1][-1][1] for k in rec.checked if k[1] and k[1][-1][0] == "extra" and k[1][-1][1] is not None}
    assert checked_sites == set(range(n)), f"{case}: value-checked sites {sorted(checked_sites)}, want range({n})"
    del model, loss
    gc.collect(); torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------- the FP8 step
def test_every_launch_of_the_fp8_llama_step_against_fp64(monkeypatch):
    case = "fp8-ziya-llama-13b"
    _need(case)
    t0 = time.time()
    torch.manual_seed(0)
    w = _two_layers(bench.workload("ziya-llama-13b"))
    from fsb200.models.llama import LlamaForCausalLM
    cfg = SimpleNamespace(vocab_size=w["vocab_size"], hidden_size=w["hidden_size"],
                          num_hidden_layers=w["num_hidden_layers"], num_attention_heads=w["num_attention_heads"],
                          rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                          llama_mlp_multiple_of=256)
    model = LlamaForCausalLM(cfg, device=torch.device("cuda", torch.cuda.current_device()), world_size=1, fp8=True)
    rec = Recorder(R.CHECKERS)
    (loss, growth), _ = _train_step(w, model, rec, monkeypatch)
    _finish(case, rec, growth, t0)
    assert math.isfinite(float(loss.item())), f"{case}: loss {loss.item()}"
    for op in ("fp8_quantize", "gemm_fp8"):
        assert any(k[0] == op for k in rec.checked), f"{case}: fp8=True made no {op} call"
    del model, loss
    gc.collect(); torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------------------- generation
class DecodeSplits:
    """Records (batch, heads, head_dim, cap, kv_len) of every attn_decode call (a Recorder `observe`)."""

    def __init__(self):
        self.calls = []

    def observe(self, op, a, ret):
        if op == "attn_decode":
            B, H, D = a["q"].shape
            self.calls.append((B, H, D, a["k_cache"].shape[1], int(a["kv_len"].item())))

    def chunks_used(self):
        """The largest number of key chunks one call covered. The split plan (attention_decode.cu decode_plan) depends on
        (batch, heads, cap) and the SM count only; the number of splits it gives is cross-checked against the workspace
        the library asks for."""
        sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        most = 0
        for B, H, D, cap, kv_len in self.calls:
            want = max(1, min(-(-4 * sms // (B * H)), -(-cap // 64)))
            chunk = -(-(-(-cap // want)) // 64) * 64
            splits = int(L.load().fsb_attn_decode_workspace_bytes(B, H, D, cap)) // (B * H * (D + 2) * 4)
            assert splits == -(-cap // chunk), f"split plan of attn_decode {B}x{H}x{D} cap {cap}: {splits} splits"
            most = max(most, -(-min(kv_len, cap) // chunk))
        return most


def _generate_census(case, monkeypatch, build, run, llama=False):
    """LLaMA decodes with sdpa_fwd over its whole cache, the unwritten slots masked by the kv_mask kv_append fills in: its
    result depends on that device-held mask, so every sdpa_fwd call is checked, and there is no split-KV call to count."""
    _need(case)
    t0 = time.time()
    torch.manual_seed(0)
    monkeypatch.setenv("FSB_GENERATE_GRAPH", "0")
    splits = DecodeSplits()
    rec = Recorder(R.CHECKERS, check_all=DECODE_OPS + (("sdpa_fwd",) if llama else ()), observe=splits.observe)

    def go():
        if llama:
            # llama._WQ holds the quantisers themselves, bound at import: point it at the recorder's wrappers
            from fsb200.models import llama as llama_module
            wq = llama_module._WQ
            for fmt, name in (("int8", "quantize_w8"), ("int4", "quantize_w4")):
                monkeypatch.setitem(wq, fmt, (getattr(ops, name), wq[fmt][1]))
        model = build()
        return run(model)
    out, growth = _run(monkeypatch, rec, go)
    _finish(case, rec, growth, t0)
    for op in ("kv_append", "sdpa_fwd" if llama else "attn_decode"):
        assert any(k[0] == op for k in rec.checked), f"{case}: no {op} call"
    if not llama:
        used = splits.chunks_used()
        assert used > 1, f"{case}: attn_decode covered at most {used} key chunk per call; the split-KV merge was not run"
    del out
    gc.collect(); torch.cuda.empty_cache()
    return rec


def _gpt2_bench():
    import transformers
    from fsb200.models.gpt2 import GPT2LMHeadModel
    w = bench.workload("gpt2-110m")
    cfg = transformers.GPT2Config(vocab_size=w["vocab_size"], n_positions=w["n_positions"], n_embd=w["n_embd"], n_layer=2,
                                  n_head=w["n_head"], bos_token_id=3, eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0,
                                  attn_pdrop=0.0, activation_function="gelu_new")
    return GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=0)


@pytest.mark.parametrize("mode", ["greedy", "beam4"])
def test_every_launch_of_gpt2_generate_against_fp64(mode, monkeypatch):
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(4, 50000, (2, 400), generator=g).cuda()
    kw = dict(max_new_tokens=12) if mode == "greedy" else dict(max_new_tokens=10, num_beams=4)
    rec = _generate_census(f"generate-gpt2-{mode}", monkeypatch, _gpt2_bench,
                           lambda m: m.generate(input_ids=ids, **kw))
    if mode == "beam4":
        assert any(k[0] == "kv_reorder" for k in rec.checked), "beam search made no kv_reorder call"


def test_every_launch_of_mt5_generate_against_fp64(monkeypatch):
    from fsb200.models.t5 import MT5ForConditionalGeneration
    w = bench.workload("randeng-t5-784m")

    def build():
        import transformers
        cfg = transformers.MT5Config(vocab_size=w["vocab_size"], d_model=w["d_model"], d_kv=w["d_kv"], d_ff=w["d_ff"],
                                     num_layers=2, num_decoder_layers=2, num_heads=w["num_heads"],
                                     relative_attention_num_buckets=32, dropout_rate=0.0, feed_forward_proj="gated-gelu",
                                     tie_word_embeddings=True, pad_token_id=0, eos_token_id=1, decoder_start_token_id=0)
        return MT5ForConditionalGeneration(cfg, device="cuda", world_size=1, seed=0)
    B, S = 2, 512
    ids = torch.randint(2, w["vocab_size"], (B, S), generator=torch.Generator().manual_seed(5))
    mask = torch.ones_like(ids)
    ids[1, S - 77:], mask[1, S - 77:] = 0, 0        # a right-padded encoder row, as the summary recipe feeds them
    ids, mask = ids.cuda(), mask.cuda()
    rec = _generate_census("generate-mt5-beam4", monkeypatch, build,
                           lambda m: m.generate(input_ids=ids, attention_mask=mask, max_length=10, num_beams=4))
    assert any(k[0] == "kv_reorder" for k in rec.checked), "beam search made no kv_reorder call"


@pytest.mark.parametrize("fmt", ["bf16", "int8", "int4"])
def test_every_launch_of_llama_generate_against_fp64(fmt, monkeypatch):
    from fsb200.models.llama import LlamaForCausalLM
    w = bench.workload("ziya-llama-13b")

    def build():
        cfg = SimpleNamespace(vocab_size=w["vocab_size"], hidden_size=w["hidden_size"], num_hidden_layers=2,
                              num_attention_heads=w["num_attention_heads"], rms_norm_epsilon=1e-6,
                              max_position_embeddings=2048, rotary_emb_base=10000, llama_mlp_multiple_of=256)
        return LlamaForCausalLM(cfg, device="cuda", seed=0, load_in_8bit=fmt == "int8", load_in_4bit=fmt == "int4")
    B, S = 2, 1000
    ids = torch.randint(4, w["vocab_size"], (B, S), generator=torch.Generator().manual_seed(6))
    mask = torch.ones_like(ids)
    ids[1, :37], mask[1, :37] = 2, 0                # a left-padded prompt
    ids, mask = ids.cuda(), mask.cuda()

    def run(m):
        g = torch.Generator(device="cuda").manual_seed(0)
        return m.generate(ids, attention_mask=mask, max_new_tokens=8, do_sample=True, top_k=50, top_p=0.9,
                          temperature=0.8, eos_token_id=2, pad_token_id=2, generator=g)
    rec = _generate_census(f"generate-llama-{fmt}", monkeypatch, build, run, llama=True)
    if fmt != "bf16":
        q = "quantize_w8" if fmt == "int8" else "quantize_w4"
        assert any(k[0] == q for k in rec.checked), f"loading the {fmt} model made no {q} call"
