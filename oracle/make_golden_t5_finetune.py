"""TEST INFRASTRUCTURE — golden batches of the UNMODIFIED reference T5 fine-tuning datasets: `LCSTSDataset.encode`
(fengshen/data/task_dataloader/task_datasets.py, the LCSTS summarisation recipe) and `TaskT5Dataset.encode`
(fengshen/data/t5_dataloader/t5_datasets.py, finetune_t5.py / qa_t5) run as written on the items below through a
deterministic tokenizer double (one id per character, eos 1 appended, pad 0), then `default_collate`d into one batch per
case. tests/test_t5_packing_cpu.py packs these batches and checks that every sample survives intact and that the loss
targets are unchanged. Cases cover a source cut at the encoder length, a summary cut at the decoder length, an empty
summary and targets of full length. Run with a checkout of the reference:
  FSB_REFERENCE_ROOT=<reference tree> python oracle/make_golden_t5_finetune.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ["FSB_REFERENCE_ROOT"]
PAD, EOS, VOCAB = 0, 1, 512


class CharTokenizer:
    """`encode`, `encode_plus` (max_length / padding='max_length' / truncation / return_tensors) and `pad_token_id`, all the
    two datasets use. Like the T5 tokenizers, an encoding ends with eos and truncation keeps that eos."""
    pad_token_id = PAD
    eos_token_id = EOS

    def encode(self, text):
        return [2 + ord(c) % (VOCAB - 2) for c in text] + [EOS]

    def encode_plus(self, text, max_length, padding, truncation, return_tensors=None):
        import torch
        assert padding == "max_length" and truncation
        ids = self.encode(text)
        if len(ids) > max_length:
            ids = ids[:max_length - 1] + [EOS]
        mask = [1] * len(ids) + [0] * (max_length - len(ids))
        ids = ids + [PAD] * (max_length - len(ids))
        if return_tensors == "pt":
            return {"input_ids": torch.tensor([ids]), "attention_mask": torch.tensor([mask])}
        return {"input_ids": ids, "attention_mask": mask}


LCSTS = {   # (max_enc_length, max_dec_length, prompt, items)
    "lcsts": (48, 16, "summary:", [
        {"text": "a short news text", "summary": "short"},
        {"text": "a source long enough that the encoder length cuts it well before its end, twice over", "summary": "cut"},
        {"text": "the summary of this one is longer than the decoder allows", "summary": "a summary past sixteen"},
        {"text": "an empty summary", "summary": ""},
        {"text": "x", "summary": "fifteen chars.."},
    ]),
}
TASK = {    # (max_seq_length, items); the target length is the dataset's fixed 16
    "task_t5": (40, [
        {"question": "which?", "choice": ["yes", "no"], "texta": "some context", "textb": "", "answer": "yes"},
        {"question": "a question", "choice": ["left", "right"], "texta": "a context long enough to be cut by the source "
         "length", "textb": "and more", "answer": "right"},
        {"question": "q", "choice": ["a"], "texta": "t", "textb": "", "answer": "an answer longer than sixteen"},
    ]),
}


def _load(name, rel):
    """The reference module at REF/rel, executed from its file (the fengshen package's __init__ imports every model)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))   # pytorch_lightning shim for the modules' imports
    sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))
    import transformers
    from torch.utils.data import default_collate
    if not hasattr(transformers, "MT5Tokenizer"):   # removed in transformers 5.x; encode never touches it
        transformers.MT5Tokenizer = type("MT5Tokenizer", (), {})
    LCSTSDataset = _load("ref_task_datasets", "fengshen/data/task_dataloader/task_datasets.py").LCSTSDataset
    TaskT5Dataset = _load("ref_t5_datasets", "fengshen/data/t5_dataloader/t5_datasets.py").TaskT5Dataset
    out = {}
    for name, (le, ld, prompt, items) in LCSTS.items():
        ds = LCSTSDataset.__new__(LCSTSDataset)          # its __init__ loads a tokenizer and a file: set what encode reads
        ds.tokenizer, ds.prompt, ds.max_enc_length, ds.max_dec_length = CharTokenizer(), prompt, le, ld
        batch = default_collate([ds.encode(it) for it in items])
        for k in ("input_ids", "attention_mask", "labels"):
            out[f"{name}/{k}"] = batch[k].numpy()
        out[f"{name}/max_source_length"], out[f"{name}/max_target_length"] = np.int64(le), np.int64(ld)
    for name, (le, items) in TASK.items():
        ds = TaskT5Dataset.__new__(TaskT5Dataset)
        ds.tokenizer, ds.max_length = CharTokenizer(), le
        encoded = [ds.encode(it) for it in items]
        for k in ("input_ids", "attention_mask", "labels"):   # force_words_ids differ in length: default_collate skipped
            out[f"{name}/{k}"] = np.stack([e[k].numpy() for e in encoded])
        out[f"{name}/max_source_length"], out[f"{name}/max_target_length"] = np.int64(le), np.int64(16)
    path = os.path.join(ROOT, "tests", "golden", "t5_finetune_batches.npz")
    np.savez_compressed(path, **out)
    print({k: v.shape for k, v in out.items()}, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
