"""Time the "LRP" baselines (the ``layers_lrp`` rule library) with and without the tensor-core Linear rule; prints one JSON
line.

    python tools/bench_lrp_rules.py [--bert-batch 4] [--vit-batch 64] [--reps 5] [--warmup 2]

* ``bert``: ``Generator.generate_full_lrp`` / ``generate_LRP_last_layer`` on the ``BERT_cls_lrp`` facade at BERT-base
  (12 layers, hidden 768, S = 512), ms per call of ``--bert-batch`` sequences.
* ``vit``: ``LRP.generate_LRP(method="full" / "last_layer")`` on ``ViT_orig_LRP`` at ViT-B/16, ms per call of
  ``--vit-batch`` images.
* Each case runs at ``FLAG_BENCH_DEFAULT`` (7475) and at 7475 | ``FLAG_RULES_LRP_TC``, alternating in one process: ``--reps``
  rounds, each timing both selections with CUDA events over one call after ``--warmup`` warm-up calls of each.  Reported:
  the median per selection, the speed-up, and the largest difference between the two selections' maps relative to the
  map maximum.
* Weights: random init, conditioned like the test models (``oracle.conditioned``), so that the maps are well defined.
* ``gpu`` / ``power_limit_w``: the card the numbers were measured on, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                                             # noqa: E402

from oracle import bert as obert                                         # noqa: E402
from oracle import conditioned                                           # noqa: E402
from oracle import vit as ovit                                           # noqa: E402
from transformer_explainability_b200 import _lib                         # noqa: E402


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def _time(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def _compare(model, fn, reps, warmup):
    """alternate the two selections; returns (median ms without, median ms with, max rel difference of the maps)"""
    sel = [_lib.FLAG_BENCH_DEFAULT, _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_RULES_LRP_TC]
    for flags in sel:
        model.engine_flags = flags
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times, maps = ([], []), [None, None]
    for _ in range(reps):
        for i, flags in enumerate(sel):
            model.engine_flags = flags
            ms, out = _time(fn)
            times[i].append(ms)
            maps[i] = out.detach().double()
    diff = ((maps[1] - maps[0]).abs().max() / maps[0].abs().max().clamp_min(1e-300)).item()
    return statistics.median(times[0]), statistics.median(times[1]), diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bert-batch", type=int, default=4)
    ap.add_argument("--vit-batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lrp_rules.py needs a CUDA device")
    out = {"gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "flags": _lib.FLAG_BENCH_DEFAULT,
           "tc_flag": _lib.FLAG_RULES_LRP_TC, "reps": args.reps, "cases": {}}

    def record(name, res, batch):
        off, on, diff = res
        out["cases"][name] = {"batch": batch, "ms": round(off, 2), "ms_tc": round(on, 2), "speedup": round(off / on, 3),
                              "max_rel_diff": float("%.2e" % diff)}

    # BERT-base on the BERT_cls_lrp facade
    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import BertForSequenceClassification
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    params, heads = obert.init_params(seed=0, rand_affine=True)
    params = conditioned.condition_bert(params)
    model = BertForSequenceClassification(BertConfig(num_labels=2))
    model.load_state_dict(params, strict=False)
    model = model.cuda().eval()
    gen = Generator(model)
    g = torch.Generator().manual_seed(1)
    S, B = 512, args.bert_batch
    ids = torch.randint(1000, 30000, (B, S), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    ids, mask = ids.cuda(), torch.ones(B, S, dtype=torch.long, device="cuda")
    record("bert_full_lrp", _compare(model, lambda: gen.generate_full_lrp(ids, mask), args.reps, args.warmup), B)
    record("bert_lrp_last_layer", _compare(model, lambda: gen.generate_LRP_last_layer(ids, mask), args.reps, args.warmup), B)
    del model, gen
    torch.cuda.empty_cache()

    # ViT-B/16 ViT_orig_LRP
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    from transformer_explainability_b200.baselines.ViT.ViT_orig_LRP import vit_base_patch16_224
    params, _ = ovit.init_params("vit_base_patch16_224", seed=0)
    model = vit_base_patch16_224()
    model.load_state_dict(conditioned.condition_vit(params, c_qkv=1.0))
    model = model.cuda().eval()
    lrp = LRP(model)
    x = torch.randn(args.vit_batch, 3, 224, 224, generator=torch.Generator().manual_seed(2)).cuda()
    for method in ("full", "last_layer"):
        record("vit_" + method, _compare(model, lambda: lrp.generate_LRP(x, method=method), args.reps, args.warmup),
               args.vit_batch)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
