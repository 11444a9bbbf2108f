"""Time ``model.relprop(one_hot, alpha=2)`` (the LRP-alpha-beta rule: both halves of every Linear rule) against alpha = 1
(the z+ rule every generator runs); prints one JSON line.

    python tools/bench_alphabeta.py [--vit-batch 64] [--bert-batch 4] [--reps 5] [--warmup 2]

* ``vit_transformer_attribution`` / ``vit_full``: ``model.relprop(method=...)`` of the ViT-B/16 facade on the activations
  of one ``model(x)`` of ``--vit-batch`` images (the class gradient, relprop and rollout / pixel relevance: the whole call).
* ``bert_relprop``: ``model.relprop`` of the BERT-base classifier facade, S = 512, ``--bert-batch`` sequences (relevance at
  the encoder input).
* Engine flags: FLAG_BENCH_DEFAULT (7475).  alpha = 1 and alpha = 2 alternate in one process: ``--reps`` rounds, each
  timing both with CUDA events over one call after ``--warmup`` warm-up calls of each.  Reported: the median per alpha and
  their ratio.
* Weights: random init, conditioned like the test models (``oracle.conditioned``).
* ``gpu`` / ``power_limit_w``: the card the numbers were measured on, read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                                             # noqa: E402

from oracle import bert as obert                                         # noqa: E402
from oracle import conditioned                                           # noqa: E402
from oracle import vit as ovit                                           # noqa: E402
from tools.bench_lrp_rules import _power_limit, _time                    # noqa: E402
from transformer_explainability_b200 import _lib                         # noqa: E402

ALPHAS = (1.0, 2.0)


def _compare(fn, reps, warmup):
    """alternate alpha = 1 and 2; returns the median ms of each"""
    for a in ALPHAS:
        for _ in range(warmup):
            fn(a)
    torch.cuda.synchronize()
    times = ([], [])
    for _ in range(reps):
        for i, a in enumerate(ALPHAS):
            times[i].append(_time(lambda: fn(a))[0])
    return statistics.median(times[0]), statistics.median(times[1])


def _one_hot(logits):
    oh = torch.zeros_like(logits)
    oh[torch.arange(logits.shape[0]), logits.argmax(-1)] = 1
    return oh


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vit-batch", type=int, default=64)
    ap.add_argument("--bert-batch", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_alphabeta.py needs a CUDA device")
    out = {"gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "flags": _lib.FLAG_BENCH_DEFAULT,
           "reps": args.reps, "cases": {}}

    def record(name, res, batch):
        one, two = res
        out["cases"][name] = {"batch": batch, "ms_alpha1": round(one, 2), "ms_alpha2": round(two, 2),
                              "ratio": round(two / one, 3)}

    # ViT-B/16
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224
    params, _ = ovit.init_params("vit_base_patch16_224", seed=0)
    model = vit_base_patch16_224()
    model.load_state_dict(conditioned.condition_vit(params, c_qkv=1.0))
    model = model.cuda().eval()
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    x = torch.randn(args.vit_batch, 3, 224, 224, generator=torch.Generator().manual_seed(2)).cuda()
    oh = _one_hot(model(x))
    for method in ("transformer_attribution", "full"):
        record("vit_" + method, _compare(lambda a: model.relprop(oh, method=method, alpha=a), args.reps, args.warmup),
               args.vit_batch)
    del model
    torch.cuda.empty_cache()

    # BERT-base, S = 512
    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    params, _ = obert.init_params(seed=0, rand_affine=True)
    model = BertForSequenceClassification(BertConfig(num_labels=2))
    model.load_state_dict(conditioned.condition_bert(params), strict=False)
    model = model.cuda().eval()
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    g = torch.Generator().manual_seed(1)
    S, B = 512, args.bert_batch
    ids = torch.randint(1000, 30000, (B, S), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    ids, mask = ids.cuda(), torch.ones(B, S, dtype=torch.long, device="cuda")
    oh = _one_hot(model(ids, mask)[0])
    record("bert_relprop", _compare(lambda a: model.relprop(oh, alpha=a), args.reps, args.warmup), B)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
