"""TEST INFRASTRUCTURE — golden items of the UNMODIFIED reference `BlendableDataset`
(fengshen/data/megatron_dataloader/blendable_dataset.py and the utils.py it imports, loaded by path) running on the reference's own C++ helpers compiled into
oracle/_ref/ (oracle/build_ref.sh): three datasets of 70 / 20 / 10 (name, index) items blended with weights 7 : 2 : 1, all 100
items in order. torch.distributed is initialised single-process because the reference calls get_rank() unconditionally.
tests/test_index_builders_cpu.py checks the compat BlendableDataset against tests/golden/blendable_dataset.json.
Run with a checkout of the reference:
    FSB_REFERENCE_ROOT=<reference tree> sh oracle/build_ref.sh && FSB_REFERENCE_ROOT=<reference tree> python oracle/make_golden_blendable_dataset.py"""
import importlib.util
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ["FSB_REFERENCE_ROOT"]
SIZES = (("a", 70), ("b", 20), ("c", 10))
WEIGHTS = (7, 2, 1)


def main():
    sys.path.insert(0, HERE)
    from make_golden_index_builders import load_reference_helpers, quiet_stdout
    helpers = load_reference_helpers()
    if helpers is None:
        raise SystemExit("oracle/_ref/helpers*.so missing: run `sh oracle/build_ref.sh` first")
    for pkg in ("fengshen", "fengshen.data", "fengshen.data.megatron_dataloader"):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m
    sys.modules["fengshen.data.megatron_dataloader.helpers"] = helpers
    sys.modules["fengshen.data.megatron_dataloader"].helpers = helpers
    for name in ("utils", "blendable_dataset"):   # blendable_dataset imports print_rank_0 from the reference's utils
        spec = importlib.util.spec_from_file_location(f"fengshen.data.megatron_dataloader.{name}",
                                                      os.path.join(REF, "fengshen/data/megatron_dataloader", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        spec.loader.exec_module(mod)
        assert mod.__file__.startswith(REF)
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:29632", rank=0, world_size=1)
    try:
        parts = [[(name, i) for i in range(n)] for name, n in SIZES]
        with quiet_stdout():
            ds = mod.BlendableDataset(parts, list(WEIGHTS))
        items = [list(ds[i]) for i in range(len(ds))]
    finally:
        dist.destroy_process_group()
    out = os.path.join(ROOT, "tests", "golden", "blendable_dataset.json")
    with open(out, "w") as fh:
        json.dump({"sizes": [list(s) for s in SIZES], "weights": list(WEIGHTS), "items": items}, fh, separators=(",", ":"))
    print(len(items), "items,", os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
