"""Throughput of the BERT word-importance command (``python -m transformer_explainability_b200.text_visualization``) on one
GPU; prints one JSON line.

    python tools/bench_text_visualization.py [--sentences 256] [--batches 1,16,64] [--seq 128]

BERT-base (12 layers, random-init weights) and synthetic word-piece ids of ``--seq`` tokens, as single sentences
(``[CLS] a [SEP]``, segment 0) and as pairs (``[CLS] a [SEP] b [SEP]``, segment 1 from the middle, so the token-type table
is read), per batch size after one warm-up batch: ``explain_batch`` (one engine ``explain``, ``te_class_probs``,
``te_token_importance`` and the device-to-host copy), wall clock around whole batches ending in the copy, reported as
sentences/s.  Tokenisation and file writing are host work outside the timed window.  ``token_importance_us``:
``te_token_importance`` on a [64, seq] batch, CUDA events around 1000 back-to-back calls (launch gaps included).
``gpu`` / ``power_limit_w``: the card, read in the same run.

Measured on an H100 80GB HBM3 at a 700 W power limit (S = 128): 30.0 / 206.6 / 235.3 sentences/s at batch 1 / 16 / 64
for single sentences, 30.5 / 205.3 / 235.0 for pairs; token_importance_us 27.9.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                                             # noqa: E402


def _smi(field):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=%s" % field, "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def synthetic(n, S, pairs, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1000, 29000, (n, S), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    tt = torch.zeros(n, S, dtype=torch.long)
    if pairs:
        ids[:, S // 2 - 1] = 102
        tt[:, S // 2:] = 1
    return ids, tt, torch.ones(n, S, dtype=torch.long)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sentences", type=int, default=256)
    ap.add_argument("--batches", default="1,16,64")
    ap.add_argument("--seq", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_visualization needs a CUDA device")
    from transformers import BertConfig
    from transformer_explainability_b200 import ops
    from transformer_explainability_b200 import text_visualization as tv
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    torch.manual_seed(0)
    model = BertForSequenceClassification(BertConfig(num_labels=2)).cuda().eval()
    names = ["NEGATIVE", "POSITIVE"]
    out = {"model": "bert-base (random init)", "seq": args.seq, "sentences": args.sentences,
           "gpu": torch.cuda.get_device_name(), "power_limit_w": _smi("power.limit"), "sentences_per_s": {}}
    for pairs in (False, True):
        ids, tt, mask = synthetic(args.sentences, args.seq, pairs)
        kind = "pairs" if pairs else "single"
        for b in (int(v) for v in args.batches.split(",")):
            tv.explain_batch(model, ids[:b], tt[:b], mask[:b], names)                     # warm-up of this shape
            n = (args.sentences // b) * b
            torch.cuda.synchronize()
            t = time.perf_counter()
            for s in range(0, n, b):
                tv.explain_batch(model, ids[s:s + b], tt[s:s + b], mask[s:s + b], names)
            torch.cuda.synchronize()
            out["sentences_per_s"]["%s_b%d" % (kind, b)] = round(n / (time.perf_counter() - t), 1)
    maps = torch.randn(64, args.seq, device="cuda")
    lens = torch.full((64,), args.seq, dtype=torch.int32, device="cuda")
    sign = torch.ones(64, device="cuda")
    res = torch.empty_like(maps)
    for _ in range(10):
        ops.token_importance(maps, lens, sign, out=res)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 1000
    e0.record()
    for _ in range(reps):
        ops.token_importance(maps, lens, sign, out=res)
    e1.record()
    torch.cuda.synchronize()
    out["token_importance_us"] = round(e0.elapsed_time(e1) * 1000.0 / reps, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
