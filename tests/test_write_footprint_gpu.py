"""Where every kernel launch writes: outputs fully written, nothing outside them touched, workspaces exactly the declared
size (tests/footprint.py gives the contract and the check).

a. The launch censuses of tests/test_workload_launches_gpu.py, tests/test_path_launches_gpu.py,
   tests/test_gpt2_dropout_gpu.py and tests/test_llama_packing_gpu.py run again with check_footprint as the checker of
   every op: the benchmark steps, the dropout steps, the FP8 and packed LLaMA steps and KV-cache generation. Their own
   builders and assertions are reused as they are (their `launch_refs.CHECKERS` is swapped for the footprint checkers).
b. Targeted cases for what those runs never reach: ragged rows, strided outputs, packed rope, a middle bucket of a real
   flat layout, duplicate embedding ids, odd vocabularies, quantisation into row slices, the KV cache edges, the dbias
   batch splits and separate segment gradients. Every operand of a case lies in one sentinel-filled arena, and every call
   is checked for its footprint and, through launch_refs' checkers, against fp64.
c. Every fsb_*_workspace_bytes at every plan: the C entry the ops wrapper formed is replayed with a workspace of exactly
   the returned size between guards, and with 16 bytes less, which must be refused without a launch (every byte of every
   operand unchanged).

`-s` prints one table per census run: op, signatures, calls, footprint-checked calls and bytes verified unchanged.
"""
import gc
import math
import time

import pytest
import torch

import footprint as F
import launch_census
import launch_refs as R
import test_gpt2_dropout_gpu as GD
import test_llama_packing_gpu as LP
import test_path_launches_gpu as PL
import test_workload_launches_gpu as WL
from fsb200 import lib as L, ops

pytestmark = pytest.mark.gpu

COVERED = F.Stats()      # every footprint-checked call of this file, censuses and targeted cases together
RUNS_SKIPPED = []

# --------------------------------------------------------------------------------------------------- a. the censuses
# device memory (GiB) each census run needs with its storage snapshots: the peak allocated on one H100 80GB HBM3 at 700 W
# (gpt2-110m 9.3, bert-base 1.1, megatronbert-1.3b 7.4, randeng-t5-784m 6.7, ziya-llama-13b 37.6 against 25.2 for the fp64
# census; dropout BERT-base 1.1, MegatronBERT 7.9, Randeng-T5 6.7, GPT-2 9.3; FP8 LLaMA 37.6; packed LLaMA 0.1; generate
# GPT-2 greedy 0.5, 4 beams 0.6, mT5 0.8, LLaMA bf16 6.8, int8 2.9, int4 2.7) plus 2 GiB for the allocator's rounding; `-s`
# prints it as "peak"
NEED_GIB = {"gpt2-110m": 12, "bert-base": 4, "megatronbert-1.3b": 10, "randeng-t5-784m": 9, "ziya-llama-13b": 40,
            "dropout-bert-base": 4, "dropout-megatronbert-1.3b": 10, "dropout-randeng-t5-784m": 9, "dropout-gpt2-110m": 12,
            "fp8-ziya-llama-13b": 40, "packed-llama": 3, "generate-gpt2-greedy": 3, "generate-gpt2-beam4": 3,
            "generate-mt5-beam4": 3, "generate-llama-bf16": 9, "generate-llama-int8": 5, "generate-llama-int4": 5}

CASES = {**{name: (lambda mp, name=name: WL.test_every_launch_of_the_step_against_fp64(name, mp)) for name in WL.bench.WORKLOADS},
         **{f"dropout-{name}": (lambda mp, name=name: PL.test_every_launch_of_a_dropout_step_against_fp64(name, mp))
            for name in ("bert-base", "megatronbert-1.3b", "randeng-t5-784m")},
         "dropout-gpt2-110m": GD.test_every_launch_of_a_gpt2_dropout_step_against_fp64,
         "fp8-ziya-llama-13b": PL.test_every_launch_of_the_fp8_llama_step_against_fp64,
         "packed-llama": LP.test_every_launch_of_a_packed_step_against_fp64,
         **{f"generate-gpt2-{mode}": (lambda mp, mode=mode: PL.test_every_launch_of_gpt2_generate_against_fp64(mode, mp))
            for mode in ("greedy", "beam4")},
         "generate-mt5-beam4": PL.test_every_launch_of_mt5_generate_against_fp64,
         **{f"generate-llama-{fmt}": (lambda mp, fmt=fmt: PL.test_every_launch_of_llama_generate_against_fp64(fmt, mp))
            for fmt in ("bf16", "int8", "int4")}}


def _table(case, rec, stats, secs, peak):
    rows = {}
    for (op, _), n in rec.calls.items():
        r = rows.setdefault(op, [0, 0])
        r[0] += 1; r[1] += n
    print(f"\n[footprint] {case}: {sum(r[0] for r in rows.values())} signatures, {sum(r[1] for r in rows.values())} calls, "
          f"{sum(stats.checked.values())} checked, {secs:.1f} s wall, peak {peak / 2 ** 30:.1f} GiB")
    print(f"[footprint] {'op':<22} {'signatures':>10} {'calls':>6} {'checked':>7} {'bytes verified':>15}")
    for op in sorted(rows):
        print(f"[footprint] {op:<22} {rows[op][0]:>10} {rows[op][1]:>6} {stats.checked.get(op, 0):>7} "
              f"{stats.guard_bytes.get(op, 0):>15}")


@pytest.mark.parametrize("case", list(CASES))
def test_footprint_of_every_launch(case, monkeypatch):
    gc.collect(); torch.cuda.empty_cache()
    if launch_census.free_gib() < NEED_GIB[case]:
        RUNS_SKIPPED.append(case)
        pytest.skip(f"{case} with its storage snapshots needs about {NEED_GIB[case]} GiB free; "
                    f"{launch_census.free_gib():.1f} GiB are")
    torch.cuda.reset_peak_memory_stats()
    stats, recs = F.Stats(), []

    class Kept(launch_census.Recorder):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            recs.append(self)
    checkers = F.footprint_checkers(stats)
    t0 = time.time()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(R, "CHECKERS", checkers)
        for mod in (launch_census, WL, PL):
            mp.setattr(mod, "Recorder", Kept)
        for op in ("segment_bounds", "sdpa_segments_fwd", "sdpa_segments_bwd"):
            mp.setattr(LP, f"check_{op}", checkers[op])
        try:
            CASES[case](monkeypatch)
        except pytest.skip.Exception:
            RUNS_SKIPPED.append(case)
            raise
    torch.cuda.synchronize()
    peak = max([torch.cuda.max_memory_allocated()] + [r.peak for r in recs])
    _table(case, recs[0], stats, time.time() - t0, peak)
    for op, n in stats.checked.items():
        COVERED.add(op, stats.guard_bytes[op]); COVERED.checked[op] += n - 1
    assert stats.checked, f"{case}: no call was footprint-checked"
    gc.collect(); torch.cuda.empty_cache()


def test_the_census_names_an_op_without_write_entry(monkeypatch):
    a = torch.ones(64, dtype=torch.bfloat16, device="cuda")
    monkeypatch.delitem(F.WRITES, "add")
    rec = launch_census.Recorder(F.footprint_checkers(F.Stats()))
    rec.install(monkeypatch)
    with pytest.raises(AssertionError, match=r"ops\.add has no write-footprint entry"):
        ops.add(a, a)


# --------------------------------------------------------------------------------------------- b. targeted cases
class Arena:
    """The operands of one case inside one allocation of 0x5a bytes, 512 bytes apart and 256-byte aligned: a stray write
    between operands or into another operand changes the arena outside every declared write."""

    def __init__(self, nbytes=96 << 20):
        self.buf = torch.full((nbytes,), 0x5A, dtype=torch.uint8, device="cuda")
        self.off = 512

    def take(self, shape, dtype, init=None):
        n = math.prod(shape) * torch.empty(0, dtype=dtype).element_size()
        t = self.buf[self.off:self.off + n].view(dtype).view(shape)
        self.off = (self.off + n + 512 + 255) // 256 * 256
        assert self.off <= self.buf.numel(), "arena too small"
        if init is not None:
            t.copy_(init)
        return t

    def randn(self, shape, dtype=torch.bfloat16, scale=1.0, gen=None):
        return self.take(shape, dtype, torch.randn(shape, generator=gen, device="cuda") * scale)


def run(op, *args, checker=None, **kwargs):
    """ops.<op>(*args, **kwargs), footprint-checked and value-checked (launch_refs' checker unless one is given)."""
    chk = checker or R.CHECKERS[op]
    return chk(lambda *a, **k: F.check_footprint(op, getattr(ops, op), a, k, COVERED), R.Bound(op), *args, **kwargs)


@pytest.fixture
def gen():
    return torch.Generator(device="cuda").manual_seed(1234)


def _drop(A, p=0.1, site=3):
    counter = A.take((1,), torch.int64, torch.tensor([2 ** 32 - 2], device="cuda"))
    base = run("dropout_advance", counter, 8)
    return ops.Dropout(p, 77, base, site)


@pytest.mark.parametrize("rows", [1, 37, 259])
def test_ragged_rows_of_the_norm_and_pointwise_kernels(rows, gen):
    A, cols = Arena(), 264
    x, res, dy = (A.randn((rows, cols), gen=gen) for _ in range(3))
    w, beta = A.randn((cols,), gen=gen), A.randn((cols,), gen=gen)
    d = _drop(A)
    for drop in (None, d):
        _, rstd, xs = run("rmsnorm_fwd", x, w, 1e-6, residual=res, drop=drop)
        dw = A.take((cols,), torch.float32, torch.zeros(cols, device="cuda"))
        if drop is None:
            run("rmsnorm_bwd", dy, xs, w, rstd, dw, dres=res)
        else:
            run("rmsnorm_bwd_dropout", dy, xs, w, rstd, dw, drop, accumulate=True, dres=res)
        _, stats, xs = run("layernorm_fwd", x, w, beta, 1e-5, residual=res, drop=drop)
        dg, db = A.randn((cols,), torch.float32, gen=gen), A.randn((cols,), torch.float32, gen=gen)
        if drop is None:
            run("layernorm_bwd", dy, xs, w, stats, dg, db, accumulate=True)
        else:
            run("layernorm_bwd_dropout", dy, xs, w, stats, dg, db, drop, dres=res)
    up2 = A.randn((rows, 2 * cols + 16), gen=gen)                  # gate | up: column halves of one strided output
    gate, up = up2[:, :cols], up2[:, cols:2 * cols]
    dgu = A.take((rows, 2 * cols + 24), torch.bfloat16)
    for act in (0, 1, 2):
        for drop in (None, d):
            run("glu_fwd", act, gate, up, drop=drop)
            run("glu_bwd", act, dy, gate, up, dgu[:, :cols], dgu[:, cols + 8:2 * cols + 8], drop=drop)
    for act in (1, 2):
        run("act_fwd", act, x)
        run("act_bwd", act, dy, x)
        dbias = A.randn((cols,), torch.float32, gen=gen)
        run("act_bwd_bias", act, dy, x, dbias, accumulate=act == 1)
    out = A.take((rows, cols), torch.bfloat16)
    run("add", x, res, out=out)
    run("add", x, res)
    acc = A.randn((rows * cols,), torch.float32, gen=gen)
    run("accumulate", acc, x.reshape(-1), scale=0.5)
    run("accumulate", acc, x.reshape(-1), scale=2.0, overwrite=True)
    run("cast_f32_to_bf16", acc, out=out.reshape(-1))
    run("scale_inplace", out, A.take((1,), torch.float32, torch.tensor([0.5], device="cuda")).reshape(()))
    run("dropout", x, d, out=out)
    run("dropout", x, d)
    wide = A.randn((rows, cols + 40), gen=gen)[:, :cols]             # ld > cols
    for dt in (torch.bfloat16, torch.float32):
        o = A.randn((cols,), dt, gen=gen)
        run("colsum", wide, o)
        run("colsum", wide, o, accumulate=True)
    V, P = 1000, 64
    W, Pw = A.randn((V, cols), gen=gen), A.randn((P, cols), gen=gen)
    ids = A.take((rows,), torch.int64, torch.randint(0, V, (rows,), generator=gen, device="cuda"))
    run("embedding_fwd", ids, W, P=Pw, seq_len=min(rows, P))


def test_rope_on_the_q_then_the_k_heads_of_a_packed_buffer(gen):
    A, t, H, D, max_pos = Arena(), 45, 5, 128, 64
    x = A.randn((t, H, 3, D), gen=gen)
    ang = torch.arange(max_pos, device="cuda")[:, None] * 10000.0 ** (-torch.arange(D // 2, device="cuda") / (D // 2))
    cos, sin = A.take((max_pos, D // 2), torch.float32, ang.cos()), A.take((max_pos, D // 2), torch.float32, ang.sin())
    pos = A.take((t,), torch.int64, torch.randint(0, max_pos, (t,), generator=gen, device="cuda"))
    for backward in (False, True):
        for offset in (0, D):                                           # q heads, then k heads; v never changes
            run("rope_inplace", x.reshape(-1), cos, sin, pos, H, D, 3 * H * D, 3 * D, backward=backward, offset=offset)


@pytest.mark.parametrize("world", [1, 4])
def test_adamw_and_sumsq_on_a_middle_bucket_of_a_flat_layout(world, gen):
    from fsb200.flat import FlatBuffers, FlatSpec
    spec = FlatSpec()
    for i, shape in enumerate([(33, 40), (77,), (129, 8), (5, 5), (300,), (64, 24)]):
        spec.add(f"layer{i // 2}.w{i}", shape, f"b{i // 2}")
    fb = FlatBuffers(spec, "cuda", world_size=world, grad_dtype=torch.float32)
    fb.params.copy_(torch.randn(fb.total, generator=gen, device="cuda"))
    fb.grads.copy_(torch.randn(fb.total, generator=gen, device="cuda"))
    shard = [torch.randn(fb.shard_numel, generator=gen, device="cuda") for _ in range(2)] + \
            [torch.rand(fb.shard_numel, generator=gen, device="cuda")]
    i, rank = 1, world - 1
    n = fb.buckets[i][2] // world
    seg = slice(fb.shard_offsets[i], fb.shard_offsets[i] + n)
    g = fb.bucket_slice(i, rank, grad=True)
    ss = torch.full((4,), 3.0, device="cuda")
    run("sumsq", g, ss[1:2])
    run("sumsq", fb.bucket_slice(i, rank), ss[1:2], accumulate=True)
    run("clip_coef", ss[1:2], 1.0, ss[2:3], norm_out=ss[3:4])
    hyper = torch.tensor([1e-3, 1 - 0.9 ** 3, (1 - 0.95 ** 3) ** 0.5], device="cuda")
    for kw in ({}, {"grad_scale": ss[2:3], "hyper": hyper}):
        run("adamw_flat", *(s[seg] for s in shard), g, fb.bucket_slice(i, rank), 1e-3, 0.9, 0.95, 1e-8, 0.1, 3, **kw)


def test_embedding_bwd_into_a_flat_gradient_view(gen):
    from fsb200.flat import FlatBuffers, FlatSpec
    spec = FlatSpec()
    for name, shape in (("wte", (500, 64)), ("wpe", (50, 64)), ("ln.weight", (64,))):
        spec.add(name, shape, "b0")
    fb = FlatBuffers(spec, "cuda")
    fb.grads.copy_(torch.randn(fb.total, generator=gen, device="cuda").bfloat16())
    dout = torch.randn((300, 64), generator=gen, device="cuda").bfloat16()
    ids = torch.randint(0, 8, (300,), generator=gen, device="cuda")                  # heavy duplicates
    ids[::7] = 499
    run("embedding_bwd", ids, dout, fb.view("wte", grad=True))
    run("embedding_bwd", None, dout, fb.view("wpe", grad=True), idx_mod=50)         # row t % 50


@pytest.mark.parametrize("V", [1000, 4104])
def test_softmax_xent_in_place_and_separate_with_ignored_rows(V, gen):
    A, rows, seq = Arena(), 24, 12
    lg = A.randn((rows, V + 24), scale=3.0, gen=gen)[:, :V]
    labels = torch.randint(0, V, (rows,), generator=gen, device="cuda")
    labels[[2, 5, 13]] = -100
    labels = A.take((rows,), torch.int64, labels)
    dl = A.take((rows, V + 24), torch.bfloat16)[:, :V]
    run("softmax_xent", lg, labels, seq, grad_scale=0.5, dlogits=dl)
    run("softmax_xent", lg, labels, seq, dlogits=None)
    run("softmax_xent", lg, labels, seq)
    bad = A.take((rows, V), torch.bfloat16)            # contiguous: row stride V, where the logits' is V + 24
    before = A.buf.clone()
    with pytest.raises(RuntimeError, match="dlogits must be bf16"):
        ops.softmax_xent(lg, labels, seq, dlogits=bad)
    assert torch.equal(A.buf, before), "the refused softmax_xent wrote into the arena"


def test_quantisers_into_row_slices_and_strided_quantised_gemm_outputs(gen):
    A, n, k = Arena(), 256, 384
    w = A.randn((n, k + 16), gen=gen)[:, :k]
    q8, s8 = A.take((3 * n, k), torch.int8), A.take((3 * n,), torch.float32)
    q8s, s8s = run("quantize_w8", w, q=q8[n:2 * n], s=s8[n:2 * n])
    q4, s4 = A.take((3 * n // 2, k), torch.uint8), A.take((3 * n, k // 128), torch.bfloat16)
    q4s, s4s = run("quantize_w4", w, q=q4[n // 2:n], s=s4[n:2 * n])
    run("quantize_w8", w)
    run("quantize_w4", w)
    for m in (1, 9, 70):
        a = A.randn((m, k + 8), gen=gen)[:, :k]
        out = A.take((m, n + 24), torch.bfloat16)[:, 8:n + 8]          # ld > n, a 16-byte aligned column offset
        run("gemm_w8a16", a, q8s, s8s, out=out)
        run("gemm_w4a16", a, q4s, s4s, out=out)
    x = A.randn((96, k + 32), gen=gen)[:, :k]
    for fmt in ("e4m3", "e5m2"):
        for rowwise, colwise in ((True, False), (False, True), (True, True)):
            run("fp8_quantize", x, fmt, rowwise=rowwise, colwise=colwise)
    ya, _, sa = run("fp8_quantize", x, "e5m2")
    yb, _, sb = run("fp8_quantize", A.randn((n, k), gen=gen), "e4m3")
    out = A.randn((96, n + 16), gen=gen)[:, :n]
    run("gemm_fp8", ya, sa, yb, sb, out=out)
    run("gemm_fp8", ya, sa, yb, sb, out=out, accumulate=True)


@pytest.mark.parametrize("kv_len", ["1", "cap", "cap+1"])
def test_kv_append_at_the_cache_edges_and_kv_reorder_of_a_live_prefix(kv_len, gen):
    A, B, H, D, cap = Arena(), 3, 4, 64, 40
    cache = A.randn((B, cap, 2, H, D), gen=gen)
    new = A.randn((B, 3, H, D), gen=gen)
    mask = A.take((B, cap), torch.uint8, torch.zeros(B, cap, dtype=torch.uint8, device="cuda"))
    n = {"1": 1, "cap": cap, "cap+1": cap + 1}[kv_len]
    kl = A.take((1,), torch.int32, torch.tensor([n], dtype=torch.int32, device="cuda"))
    run("kv_append", new[:, 1], new[:, 2], cache[:, :, 0], cache[:, :, 1], kl, kv_mask=mask)
    run("kv_append", new[:, 1], new[:, 2], cache[:, :, 0], cache[:, :, 1], kl)
    src, dst = A.randn((2, B, cap, 2 * H * D), gen=gen), A.randn((2, B, cap, 2 * H * D), gen=gen)
    idx = A.take((B,), torch.int64, torch.tensor([2, 0, 2], device="cuda"))
    live = A.take((1,), torch.int32, torch.tensor([min(n, cap - 3)], dtype=torch.int32, device="cuda"))
    run("kv_reorder", src, dst, idx, live)


@pytest.mark.parametrize("B", [1, 3, 17])
def test_sdpa_bwd_with_bias_and_mask_at_every_dbias_batch_split(B, gen):
    A, S, H, D = Arena(), 100, 2, 64
    qkv = A.randn((B, S, 3, H, D), gen=gen)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    mask = torch.ones(B, S, dtype=torch.uint8, device="cuda")
    mask[B // 2, S - 30:] = 0
    mask = A.take((B, S), torch.uint8, mask)
    rel = A.randn((H, 2 * S - 1), torch.float32, gen=gen)
    o = A.take((B, S, H, D), torch.bfloat16)
    _, lse = run("sdpa_fwd", q, k, v, 0.125, False, kv_mask=mask, out=o, rel_bias=rel)
    dout = A.randn((B, S, H, D), gen=gen)
    dqkv = A.take((B, S, 3, H, D), torch.bfloat16)
    drel = A.randn((H, 2 * S - 1), torch.float32, gen=gen)
    run("sdpa_bwd", q, k, v, o, dout, lse, 0.125, False, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], kv_mask=mask,
        rel_bias=rel, drel_bias=drel)


def test_sdpa_segments_into_separate_gradients(gen):
    A, B, S, H, D = Arena(), 2, 200, 2, 128
    q, k, v, dout = (A.randn((B, S, H, D), gen=gen) for _ in range(4))
    ids = torch.zeros(B, S, dtype=torch.int64, device="cuda")
    ids[0, 70:] = 1; ids[0, 71:] = 2; ids[1, 150:] = 5
    st, en = run("segment_bounds", A.take((B, S), torch.int64, ids), checker=LP.check_segment_bounds)
    o, lse = run("sdpa_segments_fwd", q, k, v, 0.088, st, en, out=A.take((B, S, H, D), torch.bfloat16),
                 checker=LP.check_sdpa_segments_fwd)
    dq, dk, dv = (A.take((B, S, H, D), torch.bfloat16) for _ in range(3))
    run("sdpa_segments_bwd", q, k, v, o, dout, lse, 0.088, st, en, dq, dk, dv, checker=LP.check_sdpa_segments_bwd)


def test_wrappers_refuse_an_output_smaller_than_what_the_kernel_addresses(gen):
    """Where a C entry addresses an output from a pointer and sizes, the ops wrapper refuses a tensor whose extent differs,
    and nothing is written."""
    A = Arena()
    x, y = A.randn((16, 64), gen=gen), A.randn((16, 64), gen=gen)
    short = A.take((16, 56), torch.bfloat16)
    flat_short = A.take((16 * 64 - 8,), torch.bfloat16)
    d = _drop(A)
    w = A.randn((64, 64), gen=gen)
    qkv = A.randn((2, 64, 3, 2, 64), gen=gen)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    o, lse = ops.sdpa_fwd(q, k, v, 0.125, True)
    cos = A.take((64, 32), torch.float32, torch.ones(64, 32, device="cuda"))
    pos = A.take((16,), torch.int64, torch.arange(16, device="cuda"))
    cases = {
        "gemm aux": lambda: ops.gemm(L.GEMM_NT, x, w, bias=w[0], epilogue=L.EPI_GELU_TANH, aux=short),
        "dropout out": lambda: ops.dropout(x, d, out=flat_short),
        "add out": lambda: ops.add(x, y, out=flat_short),
        "cast out": lambda: ops.cast_f32_to_bf16(x.float(), out=flat_short),
        "colsum out": lambda: ops.colsum(x, A.take((56,), torch.float32)),
        "glu_bwd dup": lambda: ops.glu_bwd(0, x, x, y, A.take((16, 64), torch.bfloat16), short),
        "sdpa_fwd out": lambda: ops.sdpa_fwd(q, k, v, 0.125, True, out=A.take((2, 63, 2, 64), torch.bfloat16)),
        "sdpa_bwd dv": lambda: ops.sdpa_bwd(q, k, v, o, o, lse, 0.125, True, qkv[:, :, 0], qkv[:, :, 1],
                                            A.take((2, 63, 2, 64), torch.bfloat16)),
        "rope heads": lambda: ops.rope_inplace(x[:8].reshape(-1), cos, cos, pos, 1, 64, 64, 64),
        "embedding_bwd dW": lambda: ops.embedding_bwd(None, x, short, idx_mod=8),
        "adamw m": lambda: ops.adamw_flat(*(A.take((64,), torch.float32) for _ in range(2)), A.take((60,), torch.float32),
                                          A.take((64,), torch.float32), None, 1e-3, 0.9, 0.95, 1e-8, 0.0, 1),
    }
    torch.cuda.synchronize()
    before = A.buf.clone()
    for what, call in cases.items():
        with pytest.raises(RuntimeError, match="must|shape|!="):
            call()
        torch.cuda.synchronize()
        assert torch.equal(A.buf, before), f"{what}: the refused call wrote into the arena"


def test_attn_decode_and_gemm_outputs_in_an_arena(gen):
    A, B, H, D, cap = Arena(), 2, 3, 128, 70
    cache = A.randn((B, cap, 2, H, D), gen=gen)
    q = A.randn((B, 3, H, D), gen=gen)[:, 0]
    kl = A.take((1,), torch.int32, torch.tensor([cap - 5], dtype=torch.int32, device="cuda"))
    run("attn_decode", q, cache[:, :, 0], cache[:, :, 1], kl, 0.1, out=A.take((B, H, D), torch.bfloat16))
    a, b = A.randn((77, 136), gen=gen), A.randn((200, 136), gen=gen)
    out = A.take((77, 216), torch.float32)[:, 8:208]
    run("gemm", L.GEMM_NT, a, b, out=out, out_dtype=torch.float32)
    run("gemm", L.GEMM_NT, a, b, out=out, out_dtype=torch.float32, accumulate=True)
    aux = A.take((77, 208), torch.bfloat16)[:, :200]
    run("gemm", L.GEMM_NT, a, b, bias=A.randn((200,), gen=gen), epilogue=L.EPI_GELU_TANH, aux=aux)


# ------------------------------------------------------------------------------------- c. every workspace at every plan
class Replay:
    """Runs one ops call with its workspace recorded, then replays the C entry it formed with a workspace of exactly
    `nbytes` between 4 KiB guards, and with 16 bytes less. The short call must be refused without a launch: every output
    is poisoned before it and must still hold the poison, bit for bit, afterwards."""

    def __init__(self, op, args, kwargs):
        self.op, self.args, self.kwargs = op, args, kwargs
        self.calls, self.ws = [], []
        fresh = F._Fresh()
        real_call, saved = L.call, (ops.torch, ops.workspace)

        def ws(nbytes, device, tag="default"):
            t = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)[:int(nbytes)]
            self.ws.append(t)
            return t

        def call(name, *a, tag=None):
            self.calls.append((name, a))
            return real_call(name, *a, tag=tag)
        L.call, ops.torch, ops.workspace = call, fresh, ws
        try:
            self.ret = getattr(ops, op)(*args, **kwargs)
        finally:
            L.call, (ops.torch, ops.workspace) = real_call, saved
        torch.cuda.synchronize()
        self.keep = fresh.allocs                     # the op's own temporaries stay alive for the replays
        self.operands = [t for t in list(args) + list(kwargs.values()) + fresh.allocs if isinstance(t, torch.Tensor)]

    def check(self, nbytes):
        assert len(self.calls) == 1 and len(self.ws) == 1, f"{self.calls}: want one entry and one workspace"
        name, a = self.calls[0]
        i = a.index(self.ws[0].data_ptr())
        assert a[i + 1] == nbytes, f"{name}: the wrapper passed {a[i + 1]} workspace bytes, the size function says {nbytes}"
        buf = torch.full((F.WS_GUARD + nbytes + F.WS_GUARD,), F.WS_SENTINEL, dtype=torch.uint8, device="cuda")
        L.call(name, *a[:i], buf[F.WS_GUARD:].data_ptr(), nbytes, *a[i + 2:])
        torch.cuda.synchronize()
        for side, g in (("before", buf[:F.WS_GUARD]), ("after", buf[F.WS_GUARD + nbytes:])):
            changed = int((g != F.WS_SENTINEL).sum())
            assert changed == 0, f"{name}: {changed} guard bytes {side} the exact {nbytes}-byte workspace changed"
        if nbytes >= 16:
            for w in F.WRITES[self.op](F.bound_arguments(self.op, self.args, self.kwargs)):
                F.poison(w.view)
            for t in self.keep:
                F.poison(t)
            snaps = [F.storage_bytes(t).clone() for t in self.operands]
            with pytest.raises(RuntimeError, match="workspace"):
                L.call(name, *a[:i], buf[F.WS_GUARD:].data_ptr(), nbytes - 16, *a[i + 2:])
            torch.cuda.synchronize()
            for t, s in zip(self.operands, snaps):
                assert torch.equal(F.storage_bytes(t), s), f"{name}: the refused call wrote into an operand"
        return name


def _ws_case(op, size, *args, **kwargs):
    """The call through ops under check_footprint (exact workspace, guards, fp64 values), then the C-entry replays."""
    run(op, *args, **kwargs)
    Replay(op, args, kwargs).check(int(size))


def _splits_of(nbytes, m, n):
    return nbytes // (m * n * 4)


@pytest.mark.parametrize("reserved", [0, 16])
def test_gemm_split_k_workspace_at_a_power_of_two_and_another_split(reserved, gen):
    lib = L.load()
    ops.set_reserved_sms(reserved)
    try:
        found = {}
        for M in (64, 128, 256, 384, 512, 768, 1024):
            for N in (64, 128, 256, 384, 768):
                for K in (4096, 8192, 12288, 16384, 24576, 32768):   # 12288 = 12 x 1024: 12 splits
                    s = _splits_of(int(lib.fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K)), M, N)
                    if s > 1:
                        found.setdefault("pow2" if s & (s - 1) == 0 else "other", (M, N, K, s))
        assert set(found) == {"pow2", "other"}, f"split plans found at {reserved} reserved SMs: {found}"
        for M, N, K, s in found.values():
            a, b = (torch.randn((K, d), generator=gen, device="cuda").bfloat16() for d in (M, N))
            for dt in (torch.bfloat16, torch.float32):
                _ws_case("gemm", lib.fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K), L.GEMM_TN, a, b, out_dtype=dt)
    finally:
        ops.set_reserved_sms(0)


@pytest.mark.parametrize("m", [1, 9, 17, 33, 65])
@pytest.mark.parametrize("fmt", ["w8", "w4"])
def test_weight_only_gemm_workspace_split_and_one_pass(m, fmt, gen):
    lib = L.load()
    size = lib.fsb_gemm_w8a16_workspace_bytes if fmt == "w8" else lib.fsb_gemm_w4a16_workspace_bytes
    plans = {}
    for n in (128, 512, 2048, 8192, 32768):
        for k in (1024, 4096, 8192):
            plans.setdefault(int(size(m, n, k)) > 0, (n, k))
    assert set(plans) == {True, False}, f"m = {m}: plans found {plans}"
    for split, (n, k) in plans.items():
        w = torch.randn((n, k), generator=gen, device="cuda").bfloat16()
        q, s = (ops.quantize_w8 if fmt == "w8" else ops.quantize_w4)(w)
        a = torch.randn((m, k), generator=gen, device="cuda").bfloat16()
        op = f"gemm_{fmt}a16"
        if split:
            _ws_case(op, size(m, n, k), a, q, s)
        else:
            run(op, a, q, s)           # one pass: the size function says 0 and the call takes no workspace


@pytest.mark.parametrize("layer", ["rmsnorm", "layernorm"])
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("rows, cols", [(37, 264), (4096, 1024), (300, 5120)])
def test_norm_bwd_workspace(layer, dropout, rows, cols, gen):
    A = Arena(160 << 20)
    x, dy, res = (A.randn((rows, cols), gen=gen) for _ in range(3))
    w, beta = A.randn((cols,), gen=gen), A.randn((cols,), gen=gen)
    d = _drop(A) if dropout else None
    size = L.load().fsb_norm_bwd_workspace_bytes(rows, cols, int(layer == "layernorm"))
    if layer == "rmsnorm":
        _, st, xs = run("rmsnorm_fwd", x, w, 1e-6, residual=res, drop=d)
        dw = A.take((cols,), torch.float32)
        if d is None:
            _ws_case("rmsnorm_bwd", size, dy, xs, w, st, dw, dres=res)
        else:
            _ws_case("rmsnorm_bwd_dropout", size, dy, xs, w, st, dw, d, dres=res)
    else:
        _, st, xs = run("layernorm_fwd", x, w, beta, 1e-5, residual=res, drop=d)
        dg, db = A.take((cols,), torch.bfloat16), A.take((cols,), torch.bfloat16)
        if d is None:
            _ws_case("layernorm_bwd", size, dy, xs, w, st, dg, db, dres=res)
        else:
            _ws_case("layernorm_bwd_dropout", size, dy, xs, w, st, dg, db, d, dres=res)


@pytest.mark.parametrize("rows, cols", [(5, 8), (37, 264), (4096, 768), (20000, 3072)])
def test_colsum_act_bwd_bias_and_sumsq_workspaces(rows, cols, gen):
    lib = L.load()
    A = Arena(max(96 << 20, 3 * rows * cols * 2 + (16 << 20)))
    x, dy = A.randn((rows, cols), gen=gen), A.randn((rows, cols), gen=gen)
    out = A.take((cols,), torch.float32)
    _ws_case("colsum", lib.fsb_colsum_workspace_bytes(rows, cols), x, out)
    _ws_case("act_bwd_bias", lib.fsb_act_bwd_bias_workspace_bytes(rows, cols), 1, dy, x, out)
    _ws_case("sumsq", lib.fsb_sumsq_workspace_bytes(), x.reshape(-1), A.take((1,), torch.float32))


@pytest.mark.parametrize("B, S", [(1, 64), (5, 200), (17, 128)])
def test_attention_dbias_workspace(B, S, gen):
    A, H, D = Arena(), 2, 64
    q, k, v, dout = (A.randn((B, S, H, D), gen=gen) for _ in range(4))
    rel = A.randn((H, 2 * S - 1), torch.float32, gen=gen)
    o, lse = run("sdpa_fwd", q, k, v, 0.125, True, rel_bias=rel)
    dq, dk, dv = (A.take((B, S, H, D), torch.bfloat16) for _ in range(3))
    drel = A.take((H, 2 * S - 1), torch.float32, torch.zeros(H, 2 * S - 1, device="cuda"))
    _ws_case("sdpa_bwd", L.load().fsb_sdpa_bwd_workspace_bytes(B, S, S, H), q, k, v, o, dout, lse, 0.125, True,
             dq, dk, dv, rel_bias=rel, drel_bias=drel)


def test_every_op_was_footprint_checked(request):
    """Every public ops function is footprint-checked by this file. The targeted cases alone reach every op, so the census
    runs a small GPU cannot hold do not matter; the check runs whenever every test function of the file was selected
    (it is the last one), and otherwise skips naming the functions left out and the ops not reached."""
    missing = [op for op in launch_census.ops_functions() if op not in COVERED.checked]
    ran = {item.originalname for item in request.session.items if item.module is request.module}
    left_out = sorted(n for n, f in vars(request.module).items() if n.startswith("test_") and callable(f) and n not in ran)
    if left_out:
        pytest.skip(f"not every test of the file was selected ({left_out}); ops not footprint-checked so far: {missing}")
    assert not missing, f"never footprint-checked: {missing}"
