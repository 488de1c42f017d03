"""Time of one validation batch (no-grad forward, as `Trainer.fit` runs `validation_step`) against one training micro-batch
(forward + backward) on one GPU, with CUDA events, at the C2 shape (GPT-2 110M, 32 x 1024) and the C5 shape (Randeng-T5-784M,
32 x encoder 512 / decoder 114). pretrain_randeng_t5_large.sh validates every 1 % of an epoch, so this ratio is the cost of
its validation per batch. The algorithmic ratio is about 1/3 (2 N_mm against 6 N_mm FLOPs per token).

  python tools/bench_validation.py [--iters 20] [--warmup 5] [--out DIR]

Prints one JSON line per shape, with the card's name and power limit; --out also writes them to DIR/bench_validation.json."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (workload table, model builder, synthetic batches)

SHAPES = {"C2": ("gpt2-110m", {}), "C5": ("randeng-t5-784m", {"seq_dec": 114})}


def card():
    # by PCI bus id: torch's device index is relative to CUDA_VISIBLE_DEVICES, nvidia-smi's is not
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", bus],
                       capture_output=True, text=True, check=True)
    name, power = (s.strip() for s in q.stdout.strip().split(","))
    return name, power


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(key, iters, warmup):
    name, over = SHAPES[key]
    w = bench.workload(name)
    w.update(over)
    model = bench.build_model(w, "cuda", 1)
    b = {k: v.cuda() for k, v in bench.make_host_batches(w, 1, 0)[0].items()}

    def train_micro():
        model(**b).loss.backward()

    def val_batch():
        with torch.no_grad():
            model(**b)

    train = time_ms(train_micro, iters, warmup)
    val = time_ms(val_batch, iters, warmup)
    out = {"shape": key, "workload": name, "micro_batch": w["micro"], "seq": w["seq"], "train_micro_batch_ms": round(train, 3),
           "validation_batch_ms": round(val, 3), "ratio": round(val / train, 4)}
    if w["family"] == "t5":
        out["seq_dec"] = w["seq_dec"]
    del model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_validation: needs a CUDA device")
    gpu, power = card()
    rows = []
    for key in SHAPES:
        r = measure(key, args.iters, args.warmup)
        r.update(gpu=gpu, power_limit=power)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_validation.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
