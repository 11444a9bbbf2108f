"""Perturbation-evaluation oracle (TEST INFRASTRUCTURE, CPU torch, fp32 / fp64).

Restates ``/root/reference/baselines/ViT/pertubation_eval_from_hdf5.py``:

* ``normalize``          ``:17-23`` (in-place ``sub_`` / ``div_`` on a clone)
* ``perturb``            ``:86-97``: the ``k`` most relevant pixels of ``v = -vis`` (``neg``) or ``vis`` are set to 0 in
                         every channel, then normalised.  The reference selects them with ``torch.topk``, whose choice among
                         equal values is implementation-defined; here the order is fixed by
                         ``torch.sort(descending=True, stable=True)``: NaN first, then descending value, then ascending pixel
                         index (``-0.0 == +0.0``).  Where the saliency has no tie at a step boundary both agree.
* ``logit_stats``        ``:57-68`` / ``:101-118``: arg-max, max logit, max softmax probability, log(p_target / p_second)
* ``evaluate``           the loop of ``eval`` (``:26-121``) with the documented deviation for ``wrong=True``: the model
                         arrays hold one entry per sample in loader order (the reference advances ``model_index`` by the
                         filtered count, ``:63,71-78,120``); the perturbation arrays are the reference's.
"""
import numpy as np
import torch

STEPS = {"per": (224 * 224, [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]),
         "100": (100, [5, 10, 15, 20, 25, 30, 35, 40, 45])}


def step_sizes(scale):
    """``int(base_size * step)`` in Python double, as ``:32-39, 91`` compute them."""
    if scale not in STEPS:
        raise ValueError("scale not valid")
    base_size, steps = STEPS[scale]
    return [int(base_size * s) for s in steps]


def normalize(t, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    m = torch.as_tensor(mean, dtype=t.dtype)
    s = torch.as_tensor(std, dtype=t.dtype)
    shape = (1, -1) + (1,) * (t.dim() - 2)
    return t.clone().sub_(m.reshape(shape)).div_(s.reshape(shape))


def removal_order(vis, negate):
    """vis [B,P] -> pixel indices [B,P] in removal order (NaN, descending value, ascending index)."""
    v = -vis if negate else vis
    return torch.sort(v, dim=-1, descending=True, stable=True).indices


def perturb(images, vis, ks, negate, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    """images [B,C,H,W], vis [B,P] (or any shape with P values per sample) -> [S,B,C,H,W]."""
    B, C = images.shape[:2]
    order = removal_order(vis.reshape(B, -1), negate)
    outs = []
    for k in ks:
        idx = order[:, :k].unsqueeze(1).repeat(1, C, 1)
        d = images.clone().reshape(B, C, -1).scatter_(-1, idx, 0).reshape(images.shape)
        outs.append(normalize(d, mean, std))
    return torch.stack(outs)


def logit_stats(logits, target):
    """The reference's formulas in the dtype of ``logits``: (pred, max_logit, max_prob, dissim)."""
    probs = torch.softmax(logits, dim=1)
    max_logit, pred = logits.max(1, keepdim=True)
    max_prob = probs.max(1, keepdim=True)[0].squeeze(1)
    target_probs = torch.gather(probs, 1, target.long()[:, None])[:, 0]
    second_probs = probs.topk(2, dim=1)[0][:, 1]
    return pred.squeeze(1), max_logit.squeeze(1), max_prob, torch.log(target_probs / second_probs)


def evaluate(logits_fn, loader, neg=True, scale="per", wrong=False, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    """``eval(args)`` with ``model(x)`` = ``logits_fn(x)``; returns the six arrays the reference saves (float64)."""
    ks = step_sizes(scale)
    model_hits, model_dissim = [], []
    pert = {n: [] for n in ("hits", "dissimilarities", "logit_diff", "prob_diff")}
    for data, vis, target in loader:
        data = data.to(torch.float32)
        target = target.long()
        out0 = logits_fn(normalize(data, mean, std))
        pred0, logit0, prob0, dis0 = logit_stats(out0, target)
        hit0 = (target == pred0)
        model_hits.append(hit0.double().numpy())
        model_dissim.append(dis0.double().numpy())
        if wrong:
            wid = torch.nonzero(~hit0).flatten()
            if len(wid) == 0:
                continue
            data, vis, target = data[wid], vis[wid], target[wid]
            logit0, prob0 = logit0[wid], prob0[wid]
        xs = perturb(data, vis.reshape(data.shape[0], -1), ks, neg, mean, std)
        for i in range(len(ks)):
            pred, ml, mp, dis = logit_stats(logits_fn(xs[i]), target)
            pert["hits"].append((i, (target == pred).double().numpy()))
            pert["dissimilarities"].append((i, dis.double().numpy()))
            pert["logit_diff"].append((i, (ml - logit0).double().numpy()))
            pert["prob_diff"].append((i, (mp - prob0).double().numpy()))
    res = {"model_hits": np.concatenate(model_hits) if model_hits else np.zeros(0),
           "model_dissimilarities": np.concatenate(model_dissim) if model_dissim else np.zeros(0)}
    for name, rows in pert.items():
        per_step = [[a for i, a in rows if i == s] for s in range(len(ks))]
        res["perturbations_" + name] = np.stack([np.concatenate(r) if r else np.zeros(0) for r in per_step])
    return res


def vit_logits_fn(params, num_heads, norm_eps=None, dtype=torch.float32):
    """``model(x)`` of the oracle ViT (``oracle/vit.py``) in ``dtype``, returned as fp32 like the reference's model."""
    from . import vit
    p = {k: v.to(dtype) for k, v in params.items()}

    def fn(x):
        with torch.no_grad():
            return vit.forward(p, x.to(dtype), num_heads, norm_eps=norm_eps)[0]
    return fn
