"""Throughput of the ERASER rationale evaluation on one GPU; prints one JSON line.

    python tools/bench_eraser.py [--docs 64] [--batch 16] [--methods transformer_attribution,...]

* ``docs_per_s[method]``: documents through ``eraser.eraser_eval`` (explanation + ``te_eraser_rationales`` + files and
  scores on the host) at BERT-base (12 layers, random-init weights), synthetic documents of a movie-review-like length mix
  (three quarters at the 512-piece cap, the rest 150..511 pieces), length-sorted batches of ``--batch``, after one warm-up
  pass.
* ``docs_per_s_loop[method]``: the same documents one per call, the reference pipeline's ``test_batch_size = 1`` loop, in
  the same process.
* ``eraser_rationales_ms``: ``te_eraser_rationales`` alone per batch of ``--batch`` 512-piece documents, CUDA events.
* ``gpu`` / ``power_limit_w``: the card the numbers were measured on, read in the same run.
"""
import argparse
import functools
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np                                                       # noqa: E402
import torch                                                             # noqa: E402


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def synthetic(n, seed=0):
    """n documents of one-piece words with a movie-review-like length mix; one evidence span each."""
    from transformer_explainability_b200 import eraser as te
    g = np.random.default_rng(seed)
    docs, enc, anns = {}, {}, []
    for i in range(n):
        L = 512 if g.random() < 0.75 else int(g.integers(150, 512))
        ids = [101] + [int(x) for x in g.integers(1000, 30000, L - 2)] + [102]
        d = "doc%04d" % i
        docs[d] = " ".join("w%d" % t for t in ids[1:-1])
        enc[d] = (ids, ["[CLS]"] + ["w%d" % t for t in ids[1:-1]] + ["[SEP]"])
        s = int(g.integers(0, L - 12))
        anns.append(te.Annotation(d, "", frozenset([(te.Evidence("", d, s, s + 10),)]), ("NEG", "POS")[i % 2]))
    return docs, enc, anns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=64)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--methods", default=None)
    args = ap.parse_args()
    from transformers import BertConfig
    from transformer_explainability_b200 import eraser as te, ops
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification as Ours
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
        BertForSequenceClassification as ClsLrp
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    torch.manual_seed(0)
    cfg = BertConfig(num_labels=2)                                     # BERT-base
    models = {"ours": Ours(cfg).cuda().eval(), "cls_lrp": ClsLrp(cfg).cuda().eval()}
    docs, enc, anns = synthetic(args.docs)
    classes = {"NEG": 0, "POS": 1}
    methods = args.methods.split(",") if args.methods else list(te.METHODS)
    out = {"docs": args.docs, "batch": args.batch, "gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(),
           "docs_per_s": {}, "docs_per_s_loop": {}}
    for method in methods:
        kind, fn = te.METHOD_GENERATOR[method]
        gen = getattr(Generator(models[kind]), fn)
        for key, bs in (("docs_per_s", args.batch), ("docs_per_s_loop", 1)):
            te.eraser_eval(gen, docs, anns[:bs], enc, classes, batch_size=bs)            # warm-up
            torch.cuda.synchronize()
            t = time.perf_counter()
            te.eraser_eval(gen, docs, anns, enc, classes, batch_size=bs)
            torch.cuda.synchronize()
            out[key][method] = round(args.docs / (time.perf_counter() - t), 2)
    # the op alone
    g = np.random.default_rng(1)
    B, S = args.batch, 512
    maps = torch.rand(B, S, device="cuda")
    ranges = [(p, p) for _ in range(B) for p in range(1, 511)]
    woff = list(range(0, 510 * B + 1, 510))
    spans = [(int(s), int(s) + 10) for s in g.integers(0, 500, B)]
    soff = list(range(B + 1))
    fn = functools.partial(ops.eraser_rationales, maps, ranges, woff, spans, soff, te.KS, (0.5,))
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        fn()
    b.record()
    torch.cuda.synchronize()
    out["eraser_rationales_ms"] = round(a.elapsed_time(b) / 20, 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
