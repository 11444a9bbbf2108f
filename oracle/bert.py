"""BERT transformer-attribution oracle (TEST INFRASTRUCTURE, CPU, any float dtype).

Closed-form restatement of ``/root/reference/BERT_explainability/modules/BERT``:

* forward   ``BertEmbeddings.forward`` ``BERT.py:61-85``, ``BertSelfAttention.forward`` ``:307-365``,
            ``BertSelfOutput`` ``:420-425``, ``BertIntermediate`` ``:446-449``, ``BertOutput`` ``:467-472``,
            ``BertLayer.forward`` ``:498-519``, ``BertPooler.forward`` ``:169-179``,
            ``BertForSequenceClassification.forward`` ``BertForSequenceClassification.py:23-81``
* relprop   ``BertForSequenceClassification.relprop`` ``:83-88``, ``BertModel.relprop`` ``BERT.py:645-651``,
            ``BertPooler.relprop`` ``:181-190``, ``BertLayer.relprop`` ``:521-530``, ``BertOutput.relprop`` ``:474-487``,
            ``BertIntermediate.relprop`` ``:451-456``, ``BertAttention.relprop`` ``:240-247``,
            ``BertSelfOutput.relprop`` ``:427-434``, ``BertSelfAttention.relprop`` ``:367-409``
* generator ``Generator.generate_LRP`` ``ExplanationGenerator.py:28-59`` (normalised rollout ``:7-18``)

Third-party arithmetic that is NOT under /root/reference (transformers==3.5.1, un-vendored; installed 5.5):
``get_extended_attention_mask`` = ``(1 - mask)[:, None, None, :] * -10000.0`` and ``get_head_mask(None) = [None]*L``
are restated here from the published 3.5.1 behaviour (SURVEY.md §8c); the reference's own call sites are
``BERT.py:598`` and ``:616``.  ``params`` uses the HF state_dict key names.
"""
import math

import torch
import torch.nn.functional as F

from . import rules


class BertDims:
    def __init__(self, params, num_heads):
        self.dim = params["bert.embeddings.word_embeddings.weight"].shape[1]
        self.heads = num_heads
        self.depth = 1 + max(int(k.split(".")[3]) for k in params if k.startswith("bert.encoder.layer."))
        self.eps = 1e-12


def _heads(t, h):
    b, n, d = t.shape
    return t.reshape(b, n, h, d // h).permute(0, 2, 1, 3)


def _merge(t):
    b, h, n, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(b, n, h * d)


def layer_forward(p, dm, i, h, ext_mask):
    """``BertLayer.forward`` (``:498-519``) of layer ``i`` on its input ``h`` [B,S,D] with the additive mask ``ext_mask``:
    returns (output, the layer's cache)."""
    L = "bert.encoder.layer.%d." % i
    dh = dm.dim // dm.heads
    c = {"h": h}
    q = _heads(F.linear(h, p[L + "attention.self.query.weight"], p[L + "attention.self.query.bias"]), dm.heads)
    k = _heads(F.linear(h, p[L + "attention.self.key.weight"], p[L + "attention.self.key.bias"]), dm.heads)
    v = _heads(F.linear(h, p[L + "attention.self.value.weight"], p[L + "attention.self.value.bias"]), dm.heads)
    scores = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
    masked = scores + ext_mask
    probs = masked.softmax(dim=-1)
    ctx = _merge(probs @ v)
    d1 = F.linear(ctx, p[L + "attention.output.dense.weight"], p[L + "attention.output.dense.bias"])
    ao = F.layer_norm(d1 + h, (dm.dim,), p[L + "attention.output.LayerNorm.weight"],
                      p[L + "attention.output.LayerNorm.bias"], dm.eps)
    g = F.gelu(F.linear(ao, p[L + "intermediate.dense.weight"], p[L + "intermediate.dense.bias"]))
    d2 = F.linear(g, p[L + "output.dense.weight"], p[L + "output.dense.bias"])
    h = F.layer_norm(d2 + ao, (dm.dim,), p[L + "output.LayerNorm.weight"], p[L + "output.LayerNorm.bias"], dm.eps)
    c.update(q=q, k=k, v=v, scores=scores, probs=probs, ctx=ctx, d1=d1, ao=ao, g=g, d2=d2)
    return h, c


def forward(params, input_ids, attention_mask, num_heads, need_grad=False):
    p = params
    dm = BertDims(params, num_heads)
    dtype = p["classifier.weight"].dtype
    B, S = input_ids.shape
    E = "bert.embeddings."
    word = p[E + "word_embeddings.weight"][input_ids]
    pos = p[E + "position_embeddings.weight"][:S].unsqueeze(0).expand(B, -1, -1)
    tt = p[E + "token_type_embeddings.weight"][torch.zeros_like(input_ids)]
    emb = (tt + pos) + word                                           # add1([tt, pos]) ; add2([., word])  :80-81
    h = F.layer_norm(emb, (dm.dim,), p[E + "LayerNorm.weight"], p[E + "LayerNorm.bias"], dm.eps)
    if need_grad:
        h = h.detach().requires_grad_(True)
    ext_mask = (1.0 - attention_mask[:, None, None, :].to(dtype)) * -10000.0       # transformers 3.5.1
    cache = {"dims": dm, "layers": [], "ext_mask": ext_mask}
    for i in range(dm.depth):
        h, c = layer_forward(p, dm, i, h, ext_mask)
        cache["layers"].append(c)
    cache["h_last"] = h
    first = h[:, 0]
    pooled = torch.tanh(F.linear(first, p["bert.pooler.dense.weight"], p["bert.pooler.dense.bias"]))
    cache["pooled"] = pooled
    logits = F.linear(pooled, p["classifier.weight"], p["classifier.bias"])
    cache["logits"] = logits
    return logits, cache


def attention_gradients(cache, seed):
    loss = (seed * cache["logits"]).sum()
    return list(torch.autograd.grad(loss, [c["probs"] for c in cache["layers"]], retain_graph=True))


def relprop(params, cache, seed, lowest=0, to_input=False):
    """Returns per-layer attn_cam [B,H,S,S] (``BERT.py:380``); layers below ``lowest`` are None.
    ``to_input``: finish the lowest layer too and return ``(cams, r)``, r [B,S,D] = what ``model.relprop`` returns."""
    p = params
    dm = cache["dims"]
    r = rules.linear_relprop(cache["pooled"], p["classifier.weight"], seed)          # classifier ; dropout id
    r = rules.linear_relprop(cache["h_last"][:, 0], p["bert.pooler.dense.weight"], r)  # Tanh id ; pooler.dense
    r = rules.index_select_relprop(cache["h_last"], r.unsqueeze(1), 0)
    cams = [None] * dm.depth
    for i in reversed(range(lowest, dm.depth)):
        L = "bert.encoder.layer.%d." % i
        c = cache["layers"][i]
        # BertOutput.relprop: LN id ; add([dense_out, ao]) ; dense
        r_d2, r_ao2 = rules.add_relprop(c["d2"], c["ao"], r)
        r_g = rules.linear_relprop(c["g"], p[L + "output.dense.weight"], r_d2)
        r_ao1 = rules.linear_relprop(c["ao"], p[L + "intermediate.dense.weight"], r_g)   # GELU id
        r = rules.clone_relprop(c["ao"], (r_ao1, r_ao2))                                    # BertLayer.clone
        # BertSelfOutput.relprop
        r_d1, r_h2 = rules.add_relprop(c["d1"], c["h"], r)
        r_ctx = rules.linear_relprop(c["ctx"], p[L + "attention.output.dense.weight"], r_d1)
        # BertSelfAttention.relprop
        r_ctx = _heads(r_ctx, dm.heads)
        cam1, cam_v = rules.matmul_av_relprop(c["probs"], c["v"], r_ctx)
        cam1, cam_v = cam1 / 2, cam_v / 2
        cams[i] = cam1
        if i == lowest and not to_input:
            break
        cam1, _ = rules.add_relprop(c["scores"], cache["ext_mask"], cam1)                   # mask Add (renormalises)
        cam_q, cam_k = rules.matmul_qk_relprop(c["q"], c["k"], cam1)
        cam_q, cam_k = cam_q / 2, cam_k / 2
        r_q = rules.linear_relprop(c["h"], p[L + "attention.self.query.weight"], _merge(cam_q))
        r_k = rules.linear_relprop(c["h"], p[L + "attention.self.key.weight"], _merge(cam_k))
        r_v = rules.linear_relprop(c["h"], p[L + "attention.self.value.weight"], _merge(cam_v))
        r_a = rules.clone_relprop(c["h"], (r_q, r_k, r_v))                                  # self.clone (3-way)
        r = rules.clone_relprop(c["h"], (r_a, r_h2))                                        # attention.clone
    if to_input:
        return cams, r
    return cams


GENERATORS = ("LRP_last_layer", "full_lrp", "attn_last_layer", "rollout", "attn_gradcam")


def generate(params, input_ids, attention_mask, num_heads, which, index=None, start_layer=0):
    """The comparison generators of ``Generator`` (``ExplanationGenerator.py:61-155``), batch = independent
    sequences: ``which`` in GENERATORS -> [B,S]."""
    with torch.enable_grad():
        logits, cache = forward(params, input_ids, attention_mask, num_heads, need_grad=True)
        if index is None:
            index = logits.argmax(dim=-1)
        index = torch.as_tensor(index).reshape(-1).long()
        seed = torch.zeros_like(logits)
        seed[torch.arange(logits.shape[0]), index] = 1
        grads = attention_gradients(cache, seed)
    with torch.no_grad():
        cd = {"dims": cache["dims"], "ext_mask": cache["ext_mask"], "h_last": cache["h_last"].detach(),
              "pooled": cache["pooled"].detach(),
              "layers": [{k: v.detach() for k, v in c.items()} for c in cache["layers"]]}
        probs = [c["probs"] for c in cd["layers"]]
        if which == "LRP_last_layer":                                         # :61-83
            cams = relprop(params, cd, seed, lowest=cache["dims"].depth - 1)
            cam = cams[-1].clamp(min=0).mean(dim=1)
            cam[:, 0, 0] = 0
            return cam[:, 0]
        if which == "full_lrp":                                               # :85-105
            _, r = relprop(params, cd, seed, lowest=0, to_input=True)
            cam = r.sum(dim=2)
            cam[:, 0] = 0
            return cam
        if which == "attn_last_layer":                                        # :107-113
            cam = probs[-1].mean(dim=1)
            cam[:, 0, 0] = 0
            return cam[:, 0]
        if which == "rollout":                                                # :115-127
            joint = rules.rollout([a.mean(dim=1) for a in probs], start_layer=start_layer, normalize=True)
            joint[:, 0, 0] = 0
            return joint[:, 0]
        if which == "attn_gradcam":                                           # :129-155
            g = grads[-1].mean(dim=(2, 3), keepdim=True)
            cam = (probs[-1] * g).mean(dim=1).clamp(min=0)
            lo = cam.amin(dim=(1, 2), keepdim=True)
            hi = cam.amax(dim=(1, 2), keepdim=True)
            cam = (cam - lo) / (hi - lo)
            cam[:, 0, 0] = 0
            return cam[:, 0]
    raise ValueError("unknown generator %r" % (which,))


def explain(params, input_ids, attention_mask, num_heads, index=None, start_layer=11, return_taps=False):
    """``Generator.generate_LRP`` for a batch of independent sequences -> ([B,S] maps, [B] index)."""
    with torch.enable_grad():
        logits, cache = forward(params, input_ids, attention_mask, num_heads, need_grad=True)
        if index is None:
            index = logits.argmax(dim=-1)
        index = torch.as_tensor(index).reshape(-1).long()
        seed = torch.zeros_like(logits)
        seed[torch.arange(logits.shape[0]), index] = 1
        grads = attention_gradients(cache, seed)
    with torch.no_grad():
        cd = {"dims": cache["dims"], "ext_mask": cache["ext_mask"], "h_last": cache["h_last"].detach(),
              "pooled": cache["pooled"].detach(),
              "layers": [{k: v.detach() for k, v in c.items()} for c in cache["layers"]]}
        cams = relprop(params, cd, seed, lowest=start_layer)
        mats = [rules.aggregate(g, c) if c is not None else torch.zeros_like(g[:, 0]) for g, c in zip(grads, cams)]
        joint = rules.rollout(mats, start_layer=start_layer, normalize=True)
        row = joint[:, 0].clone()
        row[:, 0] = row.min(dim=1).values                      # rollout[:, 0, 0] = rollout[:, 0].min()  :58
    if return_taps:
        return row, index, {"logits": logits.detach(), "grads": grads, "cams": cams, "cache": cd}
    return row, index


def init_params(seed=0, vocab=30522, max_pos=512, types=2, dim=768, depth=12, heads=12, inter=3072, labels=2,
                dtype=torch.float32, rand_affine=False):
    """HF-keyed random-init parameters (N(0, 0.02) weights, zero biases, LayerNorm 1/0 — transformers init)."""
    g = torch.Generator().manual_seed(seed)

    def nrm(*s):
        return torch.randn(*s, generator=g) * 0.02

    p = {}
    E = "bert.embeddings."
    p[E + "word_embeddings.weight"] = nrm(vocab, dim)
    p[E + "position_embeddings.weight"] = nrm(max_pos, dim)
    p[E + "token_type_embeddings.weight"] = nrm(types, dim)
    p[E + "LayerNorm.weight"] = torch.ones(dim)
    p[E + "LayerNorm.bias"] = torch.zeros(dim)
    for i in range(depth):
        L = "bert.encoder.layer.%d." % i
        for name, (o, inn) in (("attention.self.query", (dim, dim)), ("attention.self.key", (dim, dim)),
                               ("attention.self.value", (dim, dim)), ("attention.output.dense", (dim, dim)),
                               ("intermediate.dense", (inter, dim)), ("output.dense", (dim, inter))):
            p[L + name + ".weight"] = nrm(o, inn)
            p[L + name + ".bias"] = torch.zeros(o)
        for name in ("attention.output.LayerNorm", "output.LayerNorm"):
            p[L + name + ".weight"] = torch.ones(dim)
            p[L + name + ".bias"] = torch.zeros(dim)
    p["bert.pooler.dense.weight"] = nrm(dim, dim)
    p["bert.pooler.dense.bias"] = torch.zeros(dim)
    p["classifier.weight"] = nrm(labels, dim)
    p["classifier.bias"] = torch.zeros(labels)
    if rand_affine:
        for k in sorted(p):
            if k.endswith("LayerNorm.weight"):
                p[k] = 1 + 0.2 * torch.randn(p[k].shape, generator=g)
            elif k.endswith(".bias"):
                p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
    return {k: v.to(dtype) for k, v in p.items()}, heads
