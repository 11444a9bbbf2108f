"""Generate ``tests/golden/alphabeta.npz``: the LRP-alpha-beta rule (``relprop(R, alpha)`` with alpha != 1) of the
UNMODIFIED reference (TEST INFRASTRUCTURE, authoring container).

    python -m oracle.make_golden_alphabeta          # from the repo root, needs the reference checkout

Every ``Linear.relprop`` of the reference applies the alpha-beta rule with beta = alpha - 1 (``modules/layers_ours.py:
207-230``, ``modules/layers_lrp.py:187-210`` and their BERT copies); the generators always pass alpha=1, so this fixture
calls ``model.relprop(one_hot, ..., alpha=...)`` itself.  Stored, in fp32 and fp64 (``f32.`` / ``f64.`` prefixes):

``rule.<lib>.a<alpha>``     ``Linear.relprop(r, alpha)`` of ``modules/layers_ours.py`` (lib ``ours``), ``layers_lrp.py``
                            (``lrp``) and the BERT copies (``bert_ours``, ``bert_lrp``) for alpha in ALPHAS, on the inputs
                            ``rule.x`` / ``rule.w`` / ``rule.r``.
``vit.s<k>.<method>``       ViT-tiny (the model of ``vit_tiny.npz``) ``model.relprop(alpha=2)`` for every method that reads the
                            relprop; ``vit.s<k>.cam.<l>`` the attn_cam taps of the transformer_attribution call.
``orig.s<k>.<method>``      the same for ``ViT_orig_LRP`` (its methods grad, full, rollout, last_layer).
``bert.s<k>.r`` / ``.cam.<l>``, ``cls_lrp.s<k>...``   BERT-tiny (``bert_tiny.npz``) and ``BERT_cls_lrp`` (``bert_cls_lrp.npz``)
                            ``model.relprop(alpha=2)``: relevance at the encoder input and attn_cam of every layer; sample 1
                            is the padded sequence.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import alphabeta as ab           # noqa: E402
from oracle import ref_harness as rh          # noqa: E402
from oracle import vit as ovit                # noqa: E402
from oracle import bert as obert              # noqa: E402
from oracle.make_golden import TINY_KW, BERT_TINY   # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "alphabeta.npz")
ALPHAS = (2, 0.5, 0)
MODEL_ALPHA = 2
# method name in the key -> (method, is_ablation)
VIT_METHODS = {"transformer_attribution": ("transformer_attribution", False), "full": ("full", False),
               "rollout": ("rollout", False), "last_layer": ("last_layer", False),
               "last_layer.ablation": ("last_layer", True), "second_layer": ("second_layer", False),
               "second_layer.ablation": ("second_layer", True)}
ORIG_METHODS = ("grad", "full", "rollout", "last_layer")
# the tiny BERT_cls_lrp of bert_cls_lrp.npz (tests/bert_lrp_oracle.py: TINY)
CLS_LRP_SEED = 4


def _np(t):
    return t.detach().cpu().numpy()


def rule_inputs():
    g = torch.Generator().manual_seed(4321)
    x = torch.randn(1, 7, 24, generator=g, dtype=torch.float64)
    w = torch.randn(40, 24, generator=g, dtype=torch.float64) * 0.3
    r = torch.randn(1, 7, 40, generator=g, dtype=torch.float64).abs()
    return x, w, r


def golden_rules(out):
    with rh._ref_imports():
        import modules.layers_ours as LO
        import modules.layers_lrp as LL
        import BERT_explainability.modules.layers_ours as BO
        import BERT_explainability.modules.layers_lrp as BL
    x, w, r = rule_inputs()
    out["rule.x"], out["rule.w"], out["rule.r"] = _np(x), _np(w), _np(r)
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        for lib, mod in (("ours", LO), ("lrp", LL), ("bert_ours", BO), ("bert_lrp", BL)):
            lin = mod.Linear(24, 40, bias=False).to(dt)
            with torch.no_grad():
                lin.weight.copy_(w.to(dt))
            lin(x.to(dt))
            for a in ALPHAS:
                out["%s.rule.%s.a%s" % (tag, lib, a)] = _np(lin.relprop(r.to(dt), alpha=a))


def golden_vit(out):
    params, heads = ovit.init_params("vit_tiny_test", seed=1, rand_affine=True)
    xs = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(5))
    out["vit.x"], out["vit.heads"] = _np(xs), np.int64(heads)
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        for name, build, methods in (("vit", lambda: rh.build_vit("custom", state_dict=params, dtype=dt, **TINY_KW),
                                      VIT_METHODS),
                                     ("orig", lambda: rh.build_vit_orig_lrp(state_dict=params, dtype=dt, **TINY_KW),
                                      {m: (m, False) for m in ORIG_METHODS})):
            model = build()
            for s in range(xs.shape[0]):
                x = xs[s:s + 1].to(dt)
                for key, (method, abl) in methods.items():
                    m = ab.ref_vit_relprop(model, x, method, MODEL_ALPHA, is_ablation=abl)
                    out["%s.%s.s%d.%s" % (tag, name, s, key)] = _np(m)
                    if key in ("transformer_attribution", "grad"):
                        for l, blk in enumerate(model.blocks):
                            out["%s.%s.s%d.cam.%d" % (tag, name, s, l)] = _np(blk.attn.get_attn_cam())


def _bert_cases():
    ids_t, mask_t = _tiny_ids(seed=7)
    p_tiny, _ = obert.init_params(seed=3, vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128, rand_affine=True)
    p_cls, _ = obert.init_params(seed=CLS_LRP_SEED, vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128,
                                 rand_affine=True)
    return ids_t, mask_t, (("bert", p_tiny, 3, "BertForSequenceClassification"),
                           ("cls_lrp", p_cls, CLS_LRP_SEED, "BERT_cls_lrp"))


def _tiny_ids(seed):
    g = torch.Generator().manual_seed(seed)
    S = 24
    ids = torch.randint(5, 100, (2, S), generator=g)
    mask = torch.ones(2, S, dtype=torch.long)
    mask[1, 18:] = 0                       # padded sample
    return ids, mask


def _build_bert(module, params, seed, dt):
    rh._prepare_bert_imports()
    from transformers import BertConfig
    with rh._ref_imports():
        import importlib
        cls = importlib.import_module("BERT_explainability.modules.BERT." + module).BertForSequenceClassification
        cfg = BertConfig(num_labels=2, return_dict=False, **BERT_TINY)
        torch.manual_seed(seed)
        model = cls(cfg)
        res = model.load_state_dict({k: v.to(dt) for k, v in params.items()}, strict=False)
        assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
        return model.to(dt).eval()


def golden_berts(out):
    ids, mask, cases = _bert_cases()
    out["bert.ids"], out["bert.mask"] = _np(ids), _np(mask)
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        torch.set_default_dtype(dt)
        try:
            for name, params, seed, module in cases:
                model = _build_bert(module, params, seed, dt)
                for s in range(2):
                    r, cams = ab.ref_bert_relprop(model, ids[s:s + 1], mask[s:s + 1], MODEL_ALPHA)
                    out["%s.%s.s%d.r" % (tag, name, s)] = _np(r)
                    for l, c in enumerate(cams):
                        out["%s.%s.s%d.cam.%d" % (tag, name, s, l)] = _np(c)
        finally:
            torch.set_default_dtype(torch.float32)


def main():
    torch.set_num_threads(os.cpu_count())
    out = {"alphas": np.array(ALPHAS, dtype=np.float64), "model_alpha": np.float64(MODEL_ALPHA)}
    golden_rules(out)
    golden_vit(out)
    golden_berts(out)
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), "arrays; non-finite:",
          [k for k, v in out.items() if isinstance(v, np.ndarray) and v.dtype.kind == "f" and not np.isfinite(v).all()])


if __name__ == "__main__":
    main()
