"""Explanations per second of the gradient-weighted attention rollout (``attn_grad_rollout``, TE_FLAG_ATTN_GRAD_ROLLOUT)
against ``transformer_attribution`` on the same engine; prints one JSON line.

    python tools/bench_attn_grad_rollout.py [--reps 5] [--warmup 2]

* Workloads: ViT-B/16 at batch 256, DeiT-B-distilled at 256, ViT-L/16 at 64 (``engine.explain`` on 224 x 224 images),
  BERT-base at S = 512 (``--bert-batch`` sequences, default 16).  Random-init weights (``oracle.vit`` / ``oracle.bert``
  ``init_params(seed=0)``), inputs resident in HBM.
* Engine flags: FLAG_BENCH_DEFAULT (7475) for both methods, | TE_FLAG_ATTN_GRAD_ROLLOUT for the rollout.  The two methods
  alternate in one process: ``--reps`` rounds, each timing one call of each with CUDA events after ``--warmup`` warm-up
  calls of each.  Reported: the median per method, explanations / s and the speed-up.
* ``rollout_ms``: the fused rollout launch alone (``ops.attribution_rollout(fused=True)`` on the engine's own
  ``attn_grad`` / ``attn`` taps at the explained batch, the kernel the engine launches), median of the same rounds, and
  its share of the ``attn_grad_rollout`` step.
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
from oracle import vit as ovit                                           # noqa: E402
from tools.bench_lrp_rules import _power_limit, _time                    # noqa: E402
from transformer_explainability_b200 import _lib, ops                    # noqa: E402

BASE = _lib.FLAG_BENCH_DEFAULT
METHODS = (("transformer_attribution", BASE), ("attn_grad_rollout", BASE | _lib.FLAG_ATTN_GRAD_ROLLOUT))


def _layer_stack(eng, name, L):
    """[L, B, H, N, NP] copy of a per-layer workspace tensor in the engine's own layout (pad columns included)"""
    v0 = eng.tensor(name, 0)
    ls = eng.tensor(name, 1).storage_offset() - v0.storage_offset()
    B, H, N, _ = v0.shape
    NP = v0.stride(2)
    return torch.as_strided(eng._ws, (L, B, H, N, NP), (ls, v0.stride(0), v0.stride(1), NP, 1),
                            v0.storage_offset()).contiguous()


def _bench(run, eng, L, batch, reps, warmup):
    """run(flags) explains the batch; returns the case's record"""
    for _, flags in METHODS:
        for _ in range(warmup):
            run(flags)
    torch.cuda.synchronize()
    g, a = _layer_stack(eng, "attn_grad", L), _layer_stack(eng, "attn", L)      # taps of the last (rollout) call
    rollout = lambda: ops.attribution_rollout(g, a, fused=True, want_joint=False)     # noqa: E731
    for _ in range(warmup):
        rollout()
    times = {m: [] for m, _ in METHODS}
    times["rollout"] = []
    for _ in range(reps):
        for m, flags in METHODS:
            times[m].append(_time(lambda: run(flags))[0])
        times["rollout"].append(_time(rollout)[0])
    ms = {k: statistics.median(v) for k, v in times.items()}
    rec = {"batch": batch}
    for m, _ in METHODS:
        rec["ms_" + m] = round(ms[m], 2)
        rec["expl_per_s_" + m] = round(batch / ms[m] * 1e3, 1)
    rec["speedup"] = round(ms["transformer_attribution"] / ms["attn_grad_rollout"], 2)
    rec["rollout_ms"] = round(ms["rollout"], 3)
    rec["rollout_share"] = round(ms["rollout"] / ms["attn_grad_rollout"], 4)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--bert-batch", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attn_grad_rollout.py needs a CUDA device")
    out = {"gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "flags": BASE, "reps": args.reps,
           "cases": {}}

    from transformer_explainability_b200.baselines.ViT import ViT_LRP
    for name, batch in (("vit_base_patch16_224", 256), ("deit_base_distilled_patch16_224", 256),
                        ("vit_large_patch16_224", 64)):
        params, _ = ovit.init_params(name, seed=0)
        model = getattr(ViT_LRP, name)()
        model.load_state_dict(params)
        model = model.cuda().eval()
        eng = model.engine()
        x = torch.randn(batch, 3, 224, 224, generator=torch.Generator().manual_seed(2)).cuda()
        out["cases"][name] = _bench(lambda fl: eng.explain(x, flags=fl, chunk=batch), eng, len(model.blocks), batch,
                                    args.reps, args.warmup)
        del model, eng
        torch.cuda.empty_cache()

    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    params, _ = obert.init_params(seed=0)
    model = BertForSequenceClassification(BertConfig(num_labels=2))
    model.load_state_dict(params, strict=False)
    model = model.cuda().eval()
    eng = model.engine()
    S, B = 512, args.bert_batch
    ids = torch.randint(1000, 30000, (B, S), generator=torch.Generator().manual_seed(1))
    ids[:, 0], ids[:, -1] = 101, 102
    ids, mask = ids.cuda(), torch.ones(B, S, dtype=torch.long, device="cuda")
    out["cases"]["bert_base_s512"] = _bench(lambda fl: eng.explain(ids, mask, start_layer=0, flags=fl, chunk=B), eng, 12, B,
                                            args.reps, args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
