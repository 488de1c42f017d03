"""TEST INFRASTRUCTURE — golden batches of the UNMODIFIED reference script fengshen/examples/ziya_llama/finetune_ziya_llama.py:
its module body is run as written (fsb200.launch puts the compat surface in front of sys.path, as for a user), and ITS
`LlamaSFTCollator` turns the samples below into padded batches through a deterministic tokenizer double (one id per character,
eos = 2). tests/test_packing_cpu.py packs these batches and checks that every kept sample survives intact. Cases: multi-turn
samples, a sample cut at max_seq_length inside an output, one cut inside its second prompt, and one cut inside its first prompt
(no labelled token left). Run with a checkout of the reference:
  FSB_REFERENCE_ROOT=<reference tree> python oracle/make_golden_llama_sft.py"""
import os
import runpy
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ["FSB_REFERENCE_ROOT"]
SCRIPT = os.path.join(REF, "fengshen", "examples", "ziya_llama", "finetune_ziya_llama.py")
EOS, VOCAB = 2, 512


class CharTokenizer:
    """`tokenizer(text, add_special_tokens=False).input_ids` and `eos_token_id`, all the collator uses."""
    eos_token_id = EOS

    def __call__(self, text, add_special_tokens=True):
        return SimpleNamespace(input_ids=[3 + ord(c) % (VOCAB - 3) for c in text])


CASES = {
    # (max_seq_length, samples)
    "multi_turn": (96, [
        {"task": "qa", "prompt": ["hi", "and then?"], "output": ["hello there", "more"]},
        {"task": "qa", "prompt": ["one turn only"], "output": ["ok"]},
        {"task": "qa", "prompt": ["a", "b", "c"], "output": ["x", "yy", "zzz"]},
    ]),
    "cut_in_output": (40, [
        {"task": "qa", "prompt": ["short"], "output": ["a rather long answer that runs past the end of the row"]},
        {"task": "qa", "prompt": ["q"], "output": ["fits"]},
    ]),
    "cut_in_prompt": (48, [
        {"task": "qa", "prompt": ["first", "a second prompt long enough to be cut"], "output": ["answer", "never seen"]},
        {"task": "qa", "prompt": ["a first prompt so long that the row ends inside it, before any output"], "output": ["lost"]},
        {"task": "qa", "prompt": ["p"], "output": ["o"]},
    ]),
}


def main():
    sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))
    import fsb200.launch as launch
    launch.prepare(SCRIPT)
    sys.path.insert(0, os.path.dirname(SCRIPT))   # the script imports its sibling llama_generate
    ns = runpy.run_path(SCRIPT, run_name="reference_not_main")
    out = {}
    for name, (max_len, samples) in CASES.items():
        batch = ns["LlamaSFTCollator"](tokenizer=CharTokenizer(), max_seq_length=max_len)(samples)
        for k, v in batch.items():
            out[f"{name}/{k}"] = v.numpy()
        out[f"{name}/max_seq_length"] = np.int64(max_len)
        out[f"{name}/eos"] = np.int64(EOS)
    # not llama_*.npz: that pattern names the model golden files the LLaMA parity tests iterate over
    path = os.path.join(ROOT, "tests", "golden", "ziya_sft_collator.npz")
    np.savez_compressed(path, **out)
    print({k: v.shape for k, v in out.items()}, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
