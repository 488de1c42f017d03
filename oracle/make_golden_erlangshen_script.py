"""TEST INFRASTRUCTURE — golden batch of the UNMODIFIED reference script fengshen/examples/pretrain_erlangshen_bert/
pretrain_erlangshen.py: its module body is run as written (fsb200.launch puts the compat surface in front of sys.path, as for a
user), and ITS `ErLangShenCollator` turns the first four documents of tests/hf_fixtures.bert_corpus into a masked-LM batch with
np_rng = RandomState(5) and the vocabulary ids sorted. tests/test_hf_scripts_cpu.py checks the library collator against it, draw
for draw. Run with a checkout of the reference:  FSB_REFERENCE_ROOT=<reference tree> python oracle/make_golden_erlangshen_script.py"""
import json
import os
import runpy
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ["FSB_REFERENCE_ROOT"]
SCRIPT = os.path.join(REF, "fengshen", "examples", "pretrain_erlangshen_bert", "pretrain_erlangshen.py")
SEQ, ROWS, SEED = 64, 4, 5


def main():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))
    import hf_fixtures as F
    import fsb200.launch as launch
    launch.prepare(SCRIPT)
    ns = runpy.run_path(SCRIPT, run_name="reference_not_main")
    tmp = tempfile.mkdtemp()
    F.bert_dir(os.path.join(tmp, "m"))
    corpus = F.bert_corpus(os.path.join(tmp, "train.json"))
    rows = [json.loads(line) for line in open(corpus, encoding="utf8")][:ROWS]
    tok = ns["AutoTokenizer"].from_pretrained(os.path.join(tmp, "m"))
    coll = ns["ErLangShenCollator"](tokenizer=tok, max_seq_length=SEQ, masked_lm_prob=0.15, content_key="text")
    coll.setup()
    coll.np_rng = np.random.RandomState(SEED)
    coll.vocab_id_list = sorted(coll.vocab_id_list)
    batch = coll(rows)
    path = os.path.join(ROOT, "tests", "golden", "erlangshen_script_batch.npz")
    np.savez_compressed(path, **{k: v.numpy() for k, v in batch.items()})
    print({k: tuple(v.shape) for k, v in batch.items()}, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
