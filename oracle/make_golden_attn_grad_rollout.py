"""Generate ``tests/golden/attn_grad_rollout.npz`` (TEST INFRASTRUCTURE, authoring container).

    python -m oracle.make_golden_attn_grad_rollout      # from the repo root, needs /root/reference

The gradient-weighted attention rollout (``oracle/attn_grad_rollout.py``) is not in the reference repository, so the
fixture pins what the reference does produce, its attention maps and their class gradients, plus the rule as stated
there applied to them.  The UNMODIFIED reference models run through ``oracle/ref_harness.py`` one sample at a time (the
reference is only correct at B = 1): a forward and a one-hot backward (``generate_LRP``), after which ``get_attn()`` /
``get_attn_gradients()`` are read from the reference's own hooks (``ViT_LRP.py:144-145``, ``BERT.py:347-348``).

Models (parameters regenerated from their seeds, inputs stored):

``vit``   the 3-block / 17-token tiny ``VisionTransformer`` of ``vit_tiny.npz`` (two images).
``deit``  its distilled variant (dist token, averaged heads, 18 tokens).  The reference has no distilled ViT, so its
          attention maps and gradients come from the oracle's own forward (``oracle/vit.py``, "oracle-extended").
``bert``  the 3-layer / S = 24 tiny BERT classifier of ``bert_tiny.npz``; the second sequence is padded from token 18.

Keys: ``{model}.{f32|f64}.s{sample}.attn.{l}`` / ``.grad.{l}`` [1,H,N,N], ``.index`` (the arg-max class the backward
seeded), ``.map.sl{0|1}`` (ViT / DeiT [1, N - prefix], BERT [1, S] with element 0 set to 0).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import attn_grad_rollout as agr   # noqa: E402
from oracle import bert as obert               # noqa: E402
from oracle import ref_harness as rh           # noqa: E402
from oracle import vit as ovit                 # noqa: E402
from oracle.make_golden import BERT_TINY, TINY_KW   # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "attn_grad_rollout.npz")
START_LAYERS = (0, 1)
VIT_SEED, DEIT_SEED, BERT_SEED = 1, 6, 3


def _np(t):
    return t.detach().cpu().numpy()


def vit_inputs():
    return torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(5))


def bert_inputs():
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(5, 100, (2, 24), generator=g)
    mask = torch.ones(2, 24, dtype=torch.long)
    mask[1, 18:] = 0
    return ids, mask


def _store(out, key, attns, grads, index, maps):
    for l, (a, g) in enumerate(zip(attns, grads)):
        out["%s.attn.%d" % (key, l)] = _np(a)
        out["%s.grad.%d" % (key, l)] = _np(g)
    out[key + ".index"] = np.int64(index)
    for sl, m in maps.items():
        out["%s.map.sl%d" % (key, sl)] = _np(m)


def golden():
    out = {"start_layers": np.array(START_LAYERS), "vit.param_seed": np.int64(VIT_SEED),
           "deit.param_seed": np.int64(DEIT_SEED), "bert.param_seed": np.int64(BERT_SEED)}
    xs = vit_inputs()
    ids, mask = bert_inputs()
    out["x"], out["ids"], out["mask"] = _np(xs), _np(ids), _np(mask)
    vit_p, vit_h = ovit.init_params("vit_tiny_test", seed=VIT_SEED, rand_affine=True)
    deit_p, deit_h = ovit.init_params("vit_tiny_test", seed=DEIT_SEED, rand_affine=True, distilled=True)
    bert_p, bert_h = obert.init_params(seed=BERT_SEED, vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128,
                                       rand_affine=True)
    out["vit.heads"], out["deit.heads"], out["bert.heads"] = np.int64(vit_h), np.int64(deit_h), np.int64(bert_h)
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        model = rh.build_vit("custom", state_dict=vit_p, dtype=dt, **TINY_KW)
        for s in range(xs.shape[0]):
            x = xs[s:s + 1].to(dt)
            r = rh.vit_generate_lrp(model, x, start_layer=0, taps=True)
            index = int(rh.vit_logits(model, x).argmax())
            maps = {sl: agr.vit_map(r["attn"], r["grads"], sl, prefix=1) for sl in START_LAYERS}
            _store(out, "vit.%s.s%d" % (tag, s), r["attn"], r["grads"], index, maps)
        p = {k: v.to(dt) for k, v in deit_p.items()}
        for s in range(xs.shape[0]):
            attns, grads, index = agr.vit_taps(p, xs[s:s + 1].to(dt), deit_h)
            maps = {sl: agr.vit_map(attns, grads, sl, prefix=2) for sl in START_LAYERS}
            _store(out, "deit.%s.s%d" % (tag, s), attns, grads, int(index[0]), maps)
        torch.set_default_dtype(dt)
        try:
            model = rh.build_bert(seed=BERT_SEED, dtype=dt, **BERT_TINY)
            res = model.load_state_dict({k: v.to(dt) for k, v in bert_p.items()}, strict=False)
            assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
            for s in range(ids.shape[0]):
                r = rh.bert_generate_lrp(model, ids[s:s + 1], mask[s:s + 1], start_layer=0, taps=True)
                index = int(rh.bert_logits(model, ids[s:s + 1], mask[s:s + 1]).argmax())
                maps = {sl: agr.bert_map(r["attn"], r["grads"], sl) for sl in START_LAYERS}
                _store(out, "bert.%s.s%d" % (tag, s), r["attn"], r["grads"], index, maps)
        finally:
            torch.set_default_dtype(torch.float32)
    np.savez_compressed(OUT, **out)
    print(os.path.basename(OUT), len(out), "arrays")


if __name__ == "__main__":
    golden()
