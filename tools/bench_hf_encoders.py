"""Explanations per second of BERT-base, RoBERTa-base and DistilBERT-base on the engine, on one GPU; prints a table and
one JSON line.

    python tools/bench_hf_encoders.py [--samples 256] [--batches 1,16,64] [--seq 128]

Random-init weights at the released base geometries (hidden 768, 12 heads, intermediate 3072; 12 layers for BERT and
RoBERTa, 6 for DistilBERT; RoBERTa with 514 positions, pad 1, one token type), synthetic ids of ``--seq`` tokens without
padding, ``FLAG_BENCH_DEFAULT``.  Per batch size, after one warm-up batch: ``Generator.generate_LRP_batched``
(transformer attribution, start_layer 0; one engine ``explain``), wall clock around whole batches ending in a
synchronisation, reported as explanations/s.  ``gpu`` / ``power_limit_w``: the card, read in the same run.

Measured on an H100 80GB HBM3 at a 700 W power limit (S = 128), explanations/s at batch 1 / 16 / 64:
BERT-base 82.2 / 1020.5 / 1346.3, RoBERTa-base 97.8 / 1019.5 / 1342.0, DistilBERT-base 183.5 / 2064.0 / 2795.8.
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


def models():
    import transformers
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    from transformer_explainability_b200.BERT_explainability.modules.BERT.DistilBertForSequenceClassification import \
        DistilBertForSequenceClassification
    from transformer_explainability_b200.BERT_explainability.modules.BERT.RobertaForSequenceClassification import \
        RobertaForSequenceClassification
    yield "bert-base", BertForSequenceClassification(transformers.BertConfig(num_labels=2)), 0
    yield "roberta-base", RobertaForSequenceClassification(transformers.RobertaConfig(
        vocab_size=50265, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5, pad_token_id=1,
        num_labels=2)), 1
    yield "distilbert-base", DistilBertForSequenceClassification(transformers.DistilBertConfig(num_labels=2)), 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--batches", default="1,16,64")
    ap.add_argument("--seq", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hf_encoders needs a CUDA device")
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    batches = [int(v) for v in args.batches.split(",")]
    out = {"seq": args.seq, "samples": args.samples, "flags": _lib.FLAG_BENCH_DEFAULT,
           "gpu": torch.cuda.get_device_name(), "power_limit_w": _smi("power.limit"), "explanations_per_s": {}}
    torch.manual_seed(0)
    for name, model, pad in models():
        model = model.cuda().eval()
        model.engine_flags = _lib.FLAG_BENCH_DEFAULT
        gen = Generator(model)
        g = torch.Generator().manual_seed(1)
        ids = torch.randint(5, 20000, (args.samples, args.seq), generator=g)
        ids[ids == pad] = pad + 5
        ids = ids.cuda()
        mask = torch.ones_like(ids)
        rates = {}
        for b in batches:
            gen.generate_LRP_batched(ids[:b], mask[:b], start_layer=0)                # warm-up of this shape
            n = (args.samples // b) * b
            torch.cuda.synchronize()
            t = time.perf_counter()
            for s in range(0, n, b):
                gen.generate_LRP_batched(ids[s:s + b], mask[s:s + b], start_layer=0)
            torch.cuda.synchronize()
            rates["b%d" % b] = round(n / (time.perf_counter() - t), 1)
        out["explanations_per_s"][name] = rates
        del model, gen
        torch.cuda.empty_cache()
    print("%-16s %s" % ("model", " ".join("%10s" % ("batch %d" % b) for b in batches)))
    for name, rates in out["explanations_per_s"].items():
        print("%-16s %s" % (name, " ".join("%10.1f" % rates["b%d" % b] for b in batches)))
    print("explanations/s, S = %d, %s, power limit %s W" % (args.seq, out["gpu"], out["power_limit_w"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
