"""Throughput of the ERASER faithfulness evaluation on one GPU; prints one JSON line.

    python tools/bench_eraser_faithfulness.py [--docs 32] [--batch 16] [--method transformer_attribution]

* ``docs_per_s_off`` / ``docs_per_s_on``: documents through ``eraser.eraser_eval`` without and with ``faithfulness``
  (default k fraction and metrics.py's five AOPC bins: 12 reduced rows per document) at BERT-base (12 layers, random-init
  weights), on the synthetic documents of ``tools/bench_eraser.py``, length-sorted batches of ``--batch``, after a warm-up
  pass, in one process.
* ``reduced_rows_per_s``: the reduced rows over the time faithfulness adds (on minus off), and ``reduced_rows_per_s_loop``:
  the same rows one per engine forward with its probabilities brought to the host, as a user of the façade would write it.
* ``reduce_inputs_ms``: ``te_eraser_reduce_inputs`` alone per batch of ``--batch`` 512-piece documents of 510 words and
  six selections, CUDA events.
* ``padding_efficiency``: real tokens / padded tokens of the reduced-row chunks (counted, not timed).
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
    ap.add_argument("--docs", type=int, default=32)
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
    for faith in (False, True):                                           # warm-up of both paths
        te.eraser_eval(gen, docs, anns[:args.batch], enc, classes, batch_size=args.batch, faithfulness=faith)
    for faith in (False, True):
        torch.cuda.synchronize()
        t = time.perf_counter()
        res = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=args.batch, faithfulness=faith)
        torch.cuda.synchronize()
        times[faith] = time.perf_counter() - t
    f = res["faithfulness"]
    rows = int(f["n_select"].size * 2)
    out["docs_per_s_off"] = round(args.docs / times[False], 2)
    out["docs_per_s_on"] = round(args.docs / times[True], 2)
    out["reduced_rows"] = rows
    out["reduced_rows_per_s"] = round(rows / max(times[True] - times[False], 1e-9), 1)
    out["padding_efficiency"] = round(f["real_tokens"] / f["padded_tokens"], 4)
    # the same rows one per forward call: rebuilt from each document's batch-1 map
    eng = model.engine()
    singles = []
    for i, (a, d) in enumerate(zip(anns, res["docids"])):
        ids = torch.tensor([enc[d][0]], device="cuda")
        m = gen(input_ids=ids, attention_mask=torch.ones_like(ids), index=torch.tensor([classes[a.classification]]).cuda())
        red = ops.eraser_reduce_inputs(m.reshape(1, -1).float().contiguous(), ids, [ids.shape[1]], res["word_ranges"][i],
                                       [0, len(res["word_ranges"][i])], f["n_select"][i:i + 1])
        lens = red["lengths"][0].cpu().numpy()
        singles += [red["ids"][0, j, t, :lens[j, t]][None].clone() for j in range(lens.shape[0]) for t in range(2)]
    for x in singles[:4]:
        torch.softmax(eng.forward(x), -1).cpu()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for x in singles:
        torch.softmax(eng.forward(x), -1).cpu()
    torch.cuda.synchronize()
    out["reduced_rows_per_s_loop"] = round(len(singles) / (time.perf_counter() - t), 1)
    # the op alone
    B, S = args.batch, 512
    maps = torch.rand(B, S, device="cuda")
    ids = torch.randint(1000, 30000, (B, S), device="cuda")
    ranges = [(p, p) for _ in range(B) for p in range(1, 511)]
    woff = list(range(0, 510 * B + 1, 510))
    nsel = np.array([[204, 5, 26, 51, 102, 255]] * B)
    ops.eraser_reduce_inputs(maps, ids, [S] * B, ranges, woff, nsel)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        ops.eraser_reduce_inputs(maps, ids, [S] * B, ranges, woff, nsel)
    b.record()
    torch.cuda.synchronize()
    out["reduce_inputs_ms"] = round(a.elapsed_time(b) / 20, 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
