"""Cost of the ERASER pipeline's LaTeX heat maps (``eraser_eval(latex=True)``, CLI ``--latex``) on one GPU; prints one JSON
line.

    python tools/bench_eraser_latex.py [--docs 48] [--batch 8] [--methods transformer_attribution,partial_lrp]

BERT-base (12 layers) at random-init weights and the synthetic documents of ``tools/bench_eraser.py`` (three quarters at
the 512-piece cap, the rest 150..511 pieces), length-sorted batches of ``--batch``, after one warm-up pass, per method:
* ``plain_ms_per_doc`` / ``latex_ms_per_doc``: ``eraser_eval`` without and with ``latex=True``, wall clock per document;
* ``cf_attribution_ms_per_doc``: the counterfactual generator calls alone (the batches of the latex run, index
  1 - target), the part of the overhead that is a second explanation; 0 for methods without a counterfactual map;
* ``rest_ms_per_doc`` = latex - plain - cf_attribution: the weight kernels, the larger device-to-host copy and building
  the documents on the host (writing them is ``write_ms_per_doc``, measured separately into a temporary directory);
* ``latex_weights_ms``: ``te_eraser_latex_weights`` alone on a [batch, 512] batch, CUDA events.
``gpu`` / ``power_limit_w`` / ``sm_clock_mhz``: the card, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch                                                             # noqa: E402


def _smi(field):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=%s" % field, "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def _timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=48)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--methods", default="transformer_attribution,partial_lrp")
    args = ap.parse_args()
    from bench_eraser import synthetic
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
    n = args.docs
    out = {"docs": n, "batch": args.batch, "gpu": torch.cuda.get_device_name(), "power_limit_w": _smi("power.limit"),
           "methods": {}}
    for method in args.methods.split(","):
        kind, fn = {**te.METHOD_GENERATOR, **te.FOLLOW_UP_GENERATOR}[method]
        gen = getattr(Generator(models[kind]), fn)
        te.eraser_eval(gen, docs, anns[:args.batch], enc, classes, batch_size=args.batch, latex=True)      # warm-up
        _, plain = _timed(lambda: te.eraser_eval(gen, docs, anns, enc, classes, batch_size=args.batch))
        res, latex = _timed(lambda: te.eraser_eval(gen, docs, anns, enc, classes, batch_size=args.batch, latex=True))
        cf = 0.0
        if method in te.LATEX_CF_METHODS:                   # the latex run's batches: length-sorted (one length for LRP)
            same = fn in ("generate_LRP", "generate_attn_gradcam")
            order = sorted(range(n), key=lambda i: len(enc[anns[i].annotation_id][0]))
            batches = []
            for i in order:
                L = len(enc[anns[i].annotation_id][0])
                if not batches or len(batches[-1]) == args.batch or \
                        (same and L != len(enc[anns[batches[-1][0]].annotation_id][0])):
                    batches.append([])
                batches[-1].append(i)
            inputs = []
            for idx in batches:
                S = max(len(enc[anns[i].annotation_id][0]) for i in idx)
                ids = torch.zeros(len(idx), S, dtype=torch.long)
                mask = torch.zeros_like(ids)
                for r, i in enumerate(idx):
                    e = enc[anns[i].annotation_id][0]
                    ids[r, :len(e)], mask[r, :len(e)] = torch.tensor(e), 1
                tgt = torch.tensor([1 - classes[anns[i].classification] for i in idx])
                inputs.append((ids.cuda(), mask.cuda(), tgt.cuda()))
            _, cf = _timed(lambda: [gen(input_ids=a, attention_mask=m, index=t) for a, m, t in inputs])
        with tempfile.TemporaryDirectory() as tmp:
            _, write = _timed(lambda: te.write_documents(
                {(j, k): v for j, d in res["latex"].items() for k, v in d.items()}, tmp))
        ms = lambda s: round(1e3 * s / n, 3)                               # noqa: E731
        out["methods"][method] = {"plain_ms_per_doc": ms(plain), "latex_ms_per_doc": ms(latex),
                                  "cf_attribution_ms_per_doc": ms(cf), "rest_ms_per_doc": ms(latex - plain - cf),
                                  "write_ms_per_doc": ms(write)}
    maps = torch.randn(args.batch, 512, device="cuda")
    lens = torch.full((args.batch,), 512, dtype=torch.int32, device="cuda")
    w = torch.empty_like(maps)
    for _ in range(3):
        ops.eraser_latex_weights(maps, lens, out=w)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(50):
        ops.eraser_latex_weights(maps, lens, out=w)
    b.record()
    torch.cuda.synchronize()
    out["latex_weights_ms"] = round(a.elapsed_time(b) / 50, 4)
    out["sm_clock_mhz"] = _smi("clocks.sm")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
