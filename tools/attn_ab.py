"""A/B tool for the attention kernels: save every output of every form of fsb_sdpa_fwd / fsb_sdpa_bwd over a fixed seeded
case matrix, compare two such saves byte for byte, or time the forward and backward at the benchmark workloads' shapes.

    python tools/attn_ab.py --save DIR              # one .npy per output per case (needs a GPU)
    python tools/attn_ab.py --compare DIR_A DIR_B   # byte-equal check of two saves (CPU only); exit 1 on any difference
    python tools/attn_ab.py --time [--reps N]       # per-call times by CUDA-graph replay, one JSON line per shape

The case matrix: causal and bidirectional, ragged key masks, the relative bias with its gradient, dropout 0.1, the causal /
bidirectional / bias / cross segment forms, head_dim 64 and 128, and sequence lengths that are not multiples of 128."""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))

SEED, BASE, SITE = 0x2468_ACE0_1357_9BDF, (1 << 32) + 9, 5


def _torch():
    import torch
    from fsb200 import ops
    return torch, ops


def _inputs(torch, B, Sq, Skv, H, D, gen):
    """q, k, v, dout as strided views of packed buffers (the layout the models pass)."""
    qkv = torch.randn((B, Sq, 3, H, D), generator=gen).to("cuda", torch.bfloat16)
    kv = qkv if Sq == Skv else torch.randn((B, Skv, 3, H, D), generator=gen).to("cuda", torch.bfloat16)
    dout = torch.randn((B, Sq, H, D), generator=gen).to("cuda", torch.bfloat16)
    return qkv[:, :, 0], kv[:, :, 1], kv[:, :, 2], dout


def _ragged_mask(torch, B, S, gen):
    """uint8 [B, S]: row b keeps a ragged prefix, plus a few holes inside it."""
    m = torch.zeros((B, S), dtype=torch.uint8)
    for b in range(B):
        n = max(1, S - 37 * b - 11)
        m[b, :n] = 1
        m[b, torch.randint(0, n, (n // 9,), generator=gen)] = 0
        m[b, 0] = 1
    return m.cuda()


def _seg_ids(torch, B, S, gen):
    """Non-decreasing segment ids [B, S]: ragged segment lengths, a different layout per row."""
    ids = torch.zeros((B, S), dtype=torch.int64)
    for b in range(B):
        t, sid = 0, 0
        while t < S:
            n = int(torch.randint(1, 150, (1,), generator=gen))
            ids[b, t:t + n] = sid
            t, sid = t + n, sid + 1
    return ids


def _cases():
    """(name, spec) over the whole matrix. spec keys: entry ('plain' | 'seg'), D, causal, mask, bias, p, form, Sq, Skv."""
    S = 333
    for D in (64, 128):
        for causal in (True, False):
            for mask in (False, True):
                for bias in (False, True):
                    for p in (0.0, 0.1):
                        yield (f"plain_d{D}_c{int(causal)}_m{int(mask)}_b{int(bias)}_p{int(p * 10)}",
                               dict(entry="plain", D=D, causal=causal, mask=mask, bias=bias, p=p, Sq=S, Skv=S))
    for D, p in ((64, 0.0), (64, 0.1), (128, 0.0)):   # causal segments: dropout at head_dim 64 only
        yield f"seg_causal_d{D}_p{int(p * 10)}", dict(entry="seg", form="causal", D=D, p=p, Sq=S, Skv=S)
    for p in (0.0, 0.1):
        yield f"seg_bidir_p{int(p * 10)}", dict(entry="seg", form="bidir", D=64, p=p, Sq=S, Skv=S)
        yield f"seg_bias_causal_p{int(p * 10)}", dict(entry="seg", form="bias_causal", D=64, p=p, Sq=S, Skv=S)
        yield f"seg_bias_bidir_p{int(p * 10)}", dict(entry="seg", form="bias_bidir", D=64, p=p, Sq=S, Skv=S)
        yield f"seg_cross_p{int(p * 10)}", dict(entry="seg", form="cross", D=64, p=p, Sq=200, Skv=S)


def _run_case(torch, ops, spec, seed):
    from fsb200.models.base import cross_segment_bounds
    gen = torch.Generator().manual_seed(seed)
    B, H, D, Sq, Skv = 3, 3, spec["D"], spec["Sq"], spec["Skv"]
    q, k, v, dout = _inputs(torch, B, Sq, Skv, H, D, gen)
    sc = 1.0 / math.sqrt(D)
    drop = ops.Dropout(spec["p"], SEED, torch.tensor([BASE], dtype=torch.int64, device="cuda"), SITE) if spec["p"] else None
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    bias_form = spec.get("bias") or spec.get("form", "").startswith("bias")
    rel = drel = None
    if bias_form:
        rel = (torch.randn((H, Sq + Skv - 1), generator=gen) * 2).cuda()
        drel = (torch.randn((H, Sq + Skv - 1), generator=gen) * 1e-2).cuda()   # accumulated into
    if spec["entry"] == "plain":
        mask = _ragged_mask(torch, B, Skv, gen) if spec["mask"] else None
        out, lse = ops.sdpa_fwd(q, k, v, sc, spec["causal"], kv_mask=mask, rel_bias=rel, drop=drop)
        ops.sdpa_bwd(q, k, v, out, dout, lse, sc, spec["causal"], dq, dk, dv, kv_mask=mask, rel_bias=rel, drel_bias=drel,
                     drop=drop)
    else:
        form = spec["form"]
        kw = dict(drop=drop)
        if form == "cross":
            (ss, se), kvb = cross_segment_bounds(_seg_ids(torch, B, Sq, gen).cuda(), _seg_ids(torch, B, Skv, gen).cuda())
            kw.update(causal=False, kv_bounds=kvb)
        else:
            ss, se = ops.segment_bounds(_seg_ids(torch, B, Sq, gen).cuda())
            kw.update(causal=form in ("causal", "bias_causal"), rel_bias=rel)
        out, lse = ops.sdpa_segments_fwd(q, k, v, sc, ss, se, **kw)
        ops.sdpa_segments_bwd(q, k, v, out, dout, lse, sc, ss, se, dq, dk, dv, drel_bias=drel, **kw)
    res = dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)
    if drel is not None:
        res["drel_bias"] = drel
    return res


def _np(torch, t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int16).numpy() if t.dtype == torch.bfloat16 else t.numpy()   # bf16 kept as its raw bits


def save(out_dir):
    torch, ops = _torch()
    os.makedirs(out_dir, exist_ok=True)
    n = 0
    for i, (name, spec) in enumerate(_cases()):
        for key, t in _run_case(torch, ops, spec, 1000 + i).items():
            np.save(os.path.join(out_dir, f"{name}.{key}.npy"), _np(torch, t))
            n += 1
    torch.cuda.synchronize()
    print(json.dumps({"saved": n, "dir": out_dir}))


def compare(dir_a, dir_b):
    fa, fb = sorted(f for f in os.listdir(dir_a) if f.endswith(".npy")), sorted(f for f in os.listdir(dir_b) if f.endswith(".npy"))
    if fa != fb:
        print(json.dumps({"equal": False, "only_a": sorted(set(fa) - set(fb)), "only_b": sorted(set(fb) - set(fa))}))
        return 1
    diff = [f for f in fa if open(os.path.join(dir_a, f), "rb").read() != open(os.path.join(dir_b, f), "rb").read()]
    print(json.dumps({"equal": not diff, "files": len(fa), "different": diff}))
    return 1 if diff else 0


# Timed shapes: C2 = Wenzhong-GPT2-110M (bench.py's default workload), C3 = MegatronBERT-1.3B with its key-padding mask,
# C5 = Randeng-T5-784M's encoder self-attention with the relative bias. Per layer and micro-batch, as the step launches them.
SHAPES = {
    "C2": dict(B=32, S=1024, H=12, D=64, causal=True, mask=False, bias=False),
    "C3": dict(B=32, S=512, H=32, D=64, causal=False, mask=True, bias=False),
    "C5_enc": dict(B=32, S=512, H=16, D=64, causal=False, mask=False, bias=True),
}


def _graph_time(torch, fn, n, reps):
    """Seconds per call: n calls captured in one CUDA graph, replayed reps times between two events."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            for _ in range(n):
                fn()
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e-3 / (n * reps)


def time_shapes(reps):
    torch, ops = _torch()
    gen = torch.Generator().manual_seed(0)
    for name, c in SHAPES.items():
        B, S, H, D = c["B"], c["S"], c["H"], c["D"]
        q, k, v, dout = _inputs(torch, B, S, S, H, D, gen)
        mask = _ragged_mask(torch, B, S, gen) if c["mask"] else None
        rel = torch.randn((H, 2 * S - 1), generator=gen).cuda() if c["bias"] else None
        drel = torch.zeros_like(rel) if c["bias"] else None
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        sc = 1.0 / math.sqrt(D)
        out, lse = ops.sdpa_fwd(q, k, v, sc, c["causal"], kv_mask=mask, rel_bias=rel)
        t_f = _graph_time(torch, lambda: ops.sdpa_fwd(q, k, v, sc, c["causal"], kv_mask=mask, rel_bias=rel), 10, reps)
        t_b = _graph_time(torch, lambda: ops.sdpa_bwd(q, k, v, out, dout, lse, sc, c["causal"], dq, dk, dv, kv_mask=mask,
                                                      rel_bias=rel, drel_bias=drel), 10, reps)
        # FLOPs: 2 GEMMs forward, 5 backward (the algorithm's count, not the 7 the kernels issue); causal counts half
        fl = 4 * B * H * S * S * D * (0.5 if c["causal"] else 1.0)
        print(json.dumps({"shape": name, **c, "fwd_ms": round(t_f * 1e3, 4), "bwd_ms": round(t_b * 1e3, 4),
                          "fwd_tflops": round(fl / t_f / 1e12, 1), "bwd_tflops": round(2.5 * fl / t_b / 1e12, 1)}))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--save", metavar="DIR")
    g.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    g.add_argument("--time", action="store_true")
    ap.add_argument("--reps", type=int, default=20, help="graph replays per timing (--time)")
    a = ap.parse_args()
    if a.save:
        save(a.save)
    elif a.compare:
        sys.exit(compare(*a.compare))
    else:
        time_shapes(a.reps)


if __name__ == "__main__":
    main()
