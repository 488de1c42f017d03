"""Dev tool: print the max |delta| between the bf16 GPU 20-step loss curve and the reference's fp32 CPU curve (goldens)."""
import importlib.util, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.chdir(ROOT)
for d in ("tests", "fengshen-lm_b200", "oracle", ""):
    sys.path.insert(0, os.path.join(ROOT, d))
spec = importlib.util.spec_from_file_location("t", os.path.join(ROOT, "tests", "test_llama_gpu.py"))
t = importlib.util.module_from_spec(spec); spec.loader.exec_module(t)
for path in t.GOLDEN[:2]:
    g = np.load(path)
    model, sd, (V, h, L, nh, B, S) = t._build(g)
    lr, b1, b2, eps, wd, warm, lr_end = (float(x) for x in g["train_hparams"])
    steps = len(g["loss_curve"])
    eng = t.ZeroEngine(model, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    batches = [t.O.make_batch(V, B, S, seed=1234 + i) for i in range(4)]
    curve = []
    for it in range(steps):
        b = batches[it % 4]
        out = model(input_ids=b["input_ids"].cuda(), position_ids=b["position_ids"].cuda(), labels=b["labels"].cuda())
        out.loss.backward(); eng.backward_done()
        eng.step(lr=t.O.polynomial_lr(it, lr, warm * steps, steps, lr_end))
        curve.append(out.loss.item())
    d = np.abs(np.array(curve) - g["loss_curve"])
    print(os.path.basename(path), "max|d| %.5f  mean|d| %.5f  rel max %.2e   loss %.3f -> %.3f (ref %.3f -> %.3f)" %
          (d.max(), d.mean(), (d / g["loss_curve"]).max(), curve[0], curve[-1], g["loss_curve"][0], g["loss_curve"][-1]))
