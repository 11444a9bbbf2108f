"""Throughput of the ERASER tokens-to-flip search and soft-token scores on one GPU; prints one JSON line.

    python tools/bench_eraser_flip.py [--docs 16] [--batch 16] [--method transformer_attribution]

* ``docs_per_s_faith`` / ``docs_per_s_flip``: documents through ``eraser.eraser_eval`` with ``faithfulness`` and without /
  with ``tokens_to_flip`` (default ``flip_chunk``), at BERT-base (12 layers, random-init weights) on the synthetic
  documents of ``tools/bench_eraser.py`` (the model and documents of ``tools/bench_eraser_faithfulness.py``),
  length-sorted batches of ``--batch``, after a warm-up pass, in one process.  The search's worst case is W forwards
  per document; ``never_flipped`` and ``mean_tokens_to_flip`` say how close a run came to it.
* ``comp_rows_per_s``: the search's comprehensiveness rows over the time it adds (flip minus faith).
* ``padding_efficiency``: real tokens / padded tokens of the search's chunks (counted, not timed).
* ``soft_scores_ms``: ``te_eraser_soft_scores`` alone per batch of ``--batch`` documents of 510 words, CUDA events.
* ``gpu`` / ``power_limit_w``: the card the numbers were measured on, read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np                                                       # noqa: E402
import torch                                                             # noqa: E402

from bench_eraser import _power_limit, synthetic                         # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=16)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--method", default="transformer_attribution")
    args = ap.parse_args()
    from transformers import BertConfig
    from transformer_explainability_b200 import eraser as te, ops
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification as Ours
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
        BertForSequenceClassification as ClsLrp
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    torch.manual_seed(0)
    kind, fn = te.METHOD_GENERATOR[args.method]
    model = (Ours if kind == "ours" else ClsLrp)(BertConfig(num_labels=2)).cuda().eval()     # BERT-base
    gen = getattr(Generator(model), fn)
    docs, enc, anns = synthetic(args.docs)
    classes = {"NEG": 0, "POS": 1}
    out = {"method": args.method, "docs": args.docs, "batch": args.batch, "gpu": torch.cuda.get_device_name(),
           "power_limit_w": _power_limit()}
    times = {}
    for flip in (False, True):                                            # warm-up of both paths
        te.eraser_eval(gen, docs, anns[:2], enc, classes, batch_size=args.batch, faithfulness=True, tokens_to_flip=flip)
    for flip in (False, True):
        torch.cuda.synchronize()
        t = time.perf_counter()
        res = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=args.batch, faithfulness=True, tokens_to_flip=flip)
        torch.cuda.synchronize()
        times[flip] = time.perf_counter() - t
    f = res["faithfulness"]
    out["docs_per_s_faith"] = round(args.docs / times[False], 3)
    out["docs_per_s_flip"] = round(args.docs / times[True], 3)
    out["comp_rows"] = f["flip_rows"]
    out["comp_rows_per_s"] = round(f["flip_rows"] / max(times[True] - times[False], 1e-9), 1)
    out["padding_efficiency"] = round(f["flip_real_tokens"] / max(f["flip_padded_tokens"], 1), 4)
    out["never_flipped"] = f["flip_scores"]["never_flipped"]
    out["mean_tokens_to_flip"] = round(float(np.mean(f["tokens_to_flip"])), 1)
    # the soft-scores op alone
    B, W = args.batch, 510
    g = np.random.default_rng(0)
    ws = torch.from_numpy(g.random(B * W).astype(np.float32)).cuda()
    woff = list(range(0, B * W + 1, W))
    spans = [(int(s), int(s) + 10) for s in g.integers(0, W - 10, B)]
    soff = list(range(B + 1))
    tails = [(0, 50)] * B
    ops.eraser_soft_scores(ws, woff, spans, soff, tails)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        ops.eraser_soft_scores(ws, woff, spans, soff, tails)
    b.record()
    torch.cuda.synchronize()
    out["soft_scores_ms"] = round(a.elapsed_time(b) / 20, 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
