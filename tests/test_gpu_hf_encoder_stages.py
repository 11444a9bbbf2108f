"""GPU: the RoBERTa and DistilBERT engines stage by stage against fp64, with RoBERTa's position ids across the 32-token
embedding tiles up to 512 tokens.

The two families differ from BERT only in the embedding (``hf_embed_kernel``: RoBERTa's position ids counted from the
pad id on the device, DistilBERT's ``arange``), the head activation (RoBERTa tanh, DistilBERT ReLU, forward and
backward) and the LayerNorm eps (1e-5 / 1e-12).  Past the embedding they run BERT's encoder kernels, so the checks are
those of test_gpu_engine_stages.py, restated for each family's embedding and head.

a. The embedding stage, bit for bit (S in ``SEQ_LENGTHS``, 31 ... 512; RoBERTa at pad ids 1 and 5, DistilBERT): one
   row per padding pattern of ``test_hf_encoders_oracle.position_patterns`` (right padding from inside tile 0, from 32,
   64 and 256 and inside the last tile; left padding by 1 ... 257 pads; pad ids under mask 1; the class token followed
   only by pads).  The pre-LayerNorm sum is read from ``tmp_d0`` right after ``forward``: te_bert_forward writes
   ``tD[0]`` with the embedding kernel only (the fp16-split scratch of the forward is ``tD[1..3]``), so after the
   forward it holds the sum.  It must equal, bit for bit, the CPU fp32 sum in ``transformers``' order:
   ``(word + type) + position`` (RoBERTa), ``word + position`` (DistilBERT), at ``transformers``' position ids.
   Layer 0's ``hidden`` is held to the LayerNorm bound against the fp64 LayerNorm of that sum.  Four vocabulary rows
   cancel their token's type and position rows to a spread of 1e-3, so that the family's eps moves the LayerNorm by
   far more than the bound; the other family's eps must be rejected.
b. Every stage, teacher-forced: real width (768 / 12 / 3072, so every tensor-core predicate holds), 3 layers, S = 300,
   batch 3 (pad ids under mask 1; left-padded by 40; right-padded from 170), conditioned as the BERT stage test's
   model, under ``FLAG_SETS + LRP_SETS`` at alpha 1 and ``ALPHA_SETS`` at alpha 2 at that file's bounds: forward per
   layer, the pooled token (tanh / ReLU of the head's dense), logits, the fp64 VJP backward through the family's head,
   relprop (both rule libraries; the oracle inside ``oracle.hf_encoders.family``), rollout, forward taps unchanged.
c. RoBERTa at 512 tokens (2 layers, real width, ``max_position`` 514): a full, a right-padded and a left-padded (300
   pads) row under flags 0 and ``FLAG_BENCH_DEFAULT`` against the fp64 oracle at the bounds of
   test_gpu_engine_shapes.py; padded positions get exactly 0 relevance, padded keys exactly 0 probability, and the
   batched ``explain`` equals per-sample calls (1e-5, test_gpu_hf_encoders.py).

Measured worst cases on one H100 80GB HBM3 at a 700 W power limit (fraction of the bound): embedding sums bit-equal
in every row; embedding LayerNorm 0.02; forward stages <= 0.44 (ctx), P 0.10, pooled / logits <= 0.05; attn_grad 0.15
(fp32-grade) and 0.13 (TF32 / fp16); attn_cam / relevance_in <= 0.07; rollout 0.69; no forward tap changed.  RoBERTa at
512 tokens: logits 1.6e-6, attn 1.5e-6, attn_grad 1.2e-6 (flags 0) and 4.1e-4 (bench flags), top attn_cam 4.5e-4 (of
their maximum).  Run time 58 s.
"""
import pytest
import torch
import transformers

from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import hf_encoders as ohf
from test_gpu_engine_shapes import grad_tol, rel
from test_gpu_engine_stages import (ALPHA_SETS, BERT_LAYER_TAPS, DEV, FLAG_SETS, LN_BOUND, LRP_SETS, Log,
                                    _print_worst, bert_backward_checks, bert_head_checks, bert_layer_checks,  # noqa: F401
                                    bert_relprop_checks, bits, check_layernorm, check_rollout, check_survive, elem, ln64,
                                    snapshot)
from test_hf_encoders_oracle import CLASS_TOKEN, SEQ_LENGTHS, position_patterns
from transformer_explainability_b200 import _lib
from transformer_explainability_b200.BERT_explainability.modules.BERT.DistilBertForSequenceClassification import \
    DistilBertForSequenceClassification
from transformer_explainability_b200.BERT_explainability.modules.BERT.RobertaForSequenceClassification import \
    RobertaForSequenceClassification

pytestmark = pytest.mark.gpu

# each family's own constants, stated here and not read from the model: a wrong one in the model must fail
FAMILIES = {"roberta": dict(arch=ohf.ROBERTA, eps=1e-5, act=torch.tanh, types=1),
            "distilbert": dict(arch=ohf.DISTILBERT, eps=1e-12, act=torch.relu, types=0)}
E = "bert.embeddings."
MODEL_TAPS = ("h_last", "pooled", "logits")
_CACHE = {}


def family_model(name, pad, seed, vocab, max_pos, dim, heads, depth, inter, edit=None):
    """A random family classifier: (fp64 parameters under oracle.bert's names on the device, the facade on the GPU
    loaded with the same values under the family's own names).  edit(p): changes to the BERT-named parameters before
    both are made; its values are rounded to fp32, so that the oracle and the engine read the same numbers."""
    f = FAMILIES[name]
    fam = ohf.init_params(f["arch"], seed=seed, vocab=vocab, max_pos=max_pos, types=f["types"], dim=dim, depth=depth,
                          inter=inter, labels=2)
    back = {next(iter(ohf.to_bert_keys({k: None}, f["arch"]))): k for k in fam}
    p = ohf.to_bert_keys(fam, f["arch"])
    if edit is not None:
        p = {k: v.float().double() for k, v in edit(p).items()}
    if name == "roberta":
        cfg = transformers.RobertaConfig(vocab_size=vocab, max_position_embeddings=max_pos, type_vocab_size=1,
                                         hidden_size=dim, num_hidden_layers=depth, num_attention_heads=heads,
                                         intermediate_size=inter, num_labels=2, pad_token_id=pad, layer_norm_eps=1e-5)
        model = RobertaForSequenceClassification(cfg)
    else:
        cfg = transformers.DistilBertConfig(vocab_size=vocab, max_position_embeddings=max_pos, dim=dim, n_layers=depth,
                                            n_heads=heads, hidden_dim=inter, num_labels=2, pad_token_id=pad)
        model = DistilBertForSequenceClassification(cfg)
    res = model.load_state_dict({back[k]: v.float() for k, v in p.items()}, strict=False)
    assert not res.unexpected_keys and not res.missing_keys
    return {k: v.double().to(DEV) for k, v in p.items()}, model.cuda().eval()


def ext_mask(mask):
    return (1.0 - mask[:, None, None, :].double().to(DEV)) * -10000.0


# ---- a. the embedding stage --------------------------------------------------------------------------------------------
TINY = (96, 97, 98, 99)                   # vocabulary rows that cancel their token's type + position rows (see below)
EMBED_CASES = [("roberta", 1), ("roberta", 5), ("distilbert", 0)]


def tiny_position(name, pad, s):
    """the position of token s of the unpadded row"""
    return pad + 1 + s if name == "roberta" else s


def embed_setup(name, pad):
    key = ("embed", name, pad)
    if key not in _CACHE:
        _CACHE.clear()                                         # one model on the device at a time
        max_pos = max(SEQ_LENGTHS) + (pad + 1 if name == "roberta" else 0)     # RoBERTa at pad 1: 514; at pad 5: 518

        def edit(p):
            # token TINY[k] sits at s = 1 + k of the unpadded row: its word row is -(type + position) + 1e-3 N(0, 1),
            # so the sum there has a spread of 1e-3 (variance 1e-6) and eps 1e-5 / 1e-12 change its LayerNorm by ~3x
            g = torch.Generator().manual_seed(77)
            w = p[E + "word_embeddings.weight"].clone()
            for k, v in enumerate(TINY):
                cancel = p[E + "position_embeddings.weight"][tiny_position(name, pad, 1 + k)]
                if name == "roberta":
                    cancel = cancel + p[E + "token_type_embeddings.weight"][0]
                w[v] = (-cancel + 1e-3 * torch.randn(cancel.shape, generator=g, dtype=torch.float64)).float().double()
            return dict(p, **{E + "word_embeddings.weight": w})

        p64, model = family_model(name, pad, seed=41 + pad, vocab=100, max_pos=max_pos, dim=64, heads=4, depth=1,
                                  inter=128, edit=edit)
        _CACHE[key] = dict(p32={k: v.float().cpu() for k, v in p64.items()}, p64=p64, eng=model.engine())
    return _CACHE[key]


@pytest.mark.parametrize("S", SEQ_LENGTHS)
@pytest.mark.parametrize("name,pad", EMBED_CASES)
def test_embedding_stage(name, pad, S):
    f = FAMILIES[name]
    m = embed_setup(name, pad)
    ids, mask, rows = position_patterns(S, pad, seed=pad)
    ids[0, 1:1 + len(TINY)] = torch.tensor(TINY)                              # row 0: no padding
    assert rows[0] == "full"
    eng = m["eng"]
    eng.forward(ids, mask, flags=0)
    torch.cuda.synchronize()
    got = eng.tensor("tmp_d0").clone().cpu()
    hidden = eng.tensor("hidden", 0).clone()
    # the CPU fp32 sum in transformers' order, at transformers' position ids
    p = m["p32"]
    pos_ids = transformers.models.roberta.modeling_roberta.RobertaEmbeddings.create_position_ids_from_input_ids(
        ids, pad) if name == "roberta" else torch.arange(S).expand_as(ids)
    word, pos = p[E + "word_embeddings.weight"][ids], p[E + "position_embeddings.weight"][pos_ids]
    want = (word + p[E + "token_type_embeddings.weight"][torch.zeros_like(ids)]) + pos if name == "roberta" else word + pos
    bad = [rows[r] for r in range(len(rows)) if not torch.equal(bits(got[r]), bits(want[r]))]
    assert not bad, "%s pad %d S %d: embedding sum differs in rows %s" % (name, pad, S, bad)
    # layer 0's hidden: the fp64 LayerNorm of that sum, at the family's eps; the other family's eps is rejected
    log = Log("%s pad %d S %d" % (name, pad, S))
    x = want.double().to(DEV)
    w, b = m["p64"][E + "LayerNorm.weight"], m["p64"][E + "LayerNorm.bias"]
    check_layernorm(log, "embeddings ln", 0, x, w, b, f["eps"], hidden)
    y64, _, _, s = ln64(x, w, b, f["eps"])
    other = 1e-12 if f["eps"] == 1e-5 else 1e-5
    log.teeth("embeddings ln at eps %g" % other, 0, elem(ln64(x, w, b, other)[0], y64, s), LN_BOUND)
    log.finish()


# ---- b. every stage, teacher-forced --------------------------------------------------------------------------------------
def stage_setup(name):
    key = ("stages", name)
    if key not in _CACHE:
        _CACHE.clear()
        f = FAMILIES[name]
        pad = 1 if name == "roberta" else 0
        p64, model = family_model(name, pad, seed=52, vocab=1000, max_pos=512, dim=768, heads=12, depth=3, inter=3072,
                                  edit=lambda p: conditioned.condition_bert(p, c_qkv=3.0))
        n, S = 3, 300
        g = torch.Generator().manual_seed(53)
        ids = torch.randint(6, 1000, (n, S), generator=g)
        ids[:, 0] = CLASS_TOKEN
        mask = torch.ones(n, S, dtype=torch.long)
        ids[0, 7::23] = pad                                    # row 0: pad ids under mask 1
        ids[1, :40], mask[1, :40] = pad, 0                     # row 1: left-padded by 40 (more than one tile)
        ids[1, 40] = CLASS_TOKEN
        ids[2, 170:], mask[2, 170:] = pad, 0                   # row 2: right-padded from 170
        dm = obert.BertDims(p64, 12)
        dm.eps = f["eps"]
        _CACHE[key] = dict(eng=model.engine(), p64=p64, dm=dm, heads=12, ids=ids, mask=mask, pad=pad, name=name + "_s300")
    return _CACHE[key]


def family_forward_checks(log, m, name, flags, T, ext):
    f, p, dm = FAMILIES[name], m["p64"], m["dm"]
    ids = m["ids"].to(DEV)
    pos = p[E + "position_embeddings.weight"][ohf.position_ids(ids, f["arch"], m["pad"])]
    word = p[E + "word_embeddings.weight"][ids]
    emb = (word + p[E + "token_type_embeddings.weight"][torch.zeros_like(ids)]) + pos if name == "roberta" else word + pos
    check_layernorm(log, "embeddings + ln", 0, emb, p[E + "LayerNorm.weight"], p[E + "LayerNorm.bias"], f["eps"],
                    T[("hidden", 0)])
    bert_layer_checks(log, m, flags, T, ext)
    bert_head_checks(log, m, T, f["act"])


def run_family(name, flags, alpha):
    f = FAMILIES[name]
    m = stage_setup(name)
    eng, dm = m["eng"], m["dm"]
    log = Log("%s flags %d%s" % (m["name"], flags, " alpha %g" % alpha if alpha != 1 else ""))
    ext = ext_mask(m["mask"])
    eng.forward(m["ids"], m["mask"], flags=flags)
    before = snapshot(eng, dm.depth, BERT_LAYER_TAPS, MODEL_TAPS)
    maps, idx = eng.attribute(start_layer=0, flags=flags | _lib.FLAG_KEEP_ALL_CAMS | _lib.FLAG_RELPROP_TO_INPUT,
                              alpha=alpha)
    torch.cuda.synchronize()
    T = snapshot(eng, dm.depth, BERT_LAYER_TAPS, MODEL_TAPS)
    check_survive(log, before, T)
    G = [eng.tensor("attn_grad", l).clone() for l in range(dm.depth)]
    cams = [eng.tensor("attn_cam", l).clone() for l in range(dm.depth)]
    seed = torch.zeros(idx.shape[0], 2, dtype=torch.float64, device=DEV)
    seed[torch.arange(idx.shape[0]), idx.long()] = 1
    family_forward_checks(log, m, name, flags, T, ext)
    bert_backward_checks(log, m, flags, T, G, seed, ext, act=f["act"])
    with ohf.family(f["arch"], m["pad"], f["eps"]):
        bert_relprop_checks(log, m, flags, T, cams, eng.tensor("relevance_in").clone(), seed, ext, alpha)
    check_rollout(log, maps, G, cams, True, 0, bool(flags & _lib.FLAG_ROLLOUT_FUSED))
    log.finish()


STAGE_CASES = [(f, 1.0) for f in FLAG_SETS + LRP_SETS] + [(f, 2.0) for f in ALPHA_SETS]


@pytest.mark.parametrize("flags,alpha", STAGE_CASES, ids=lambda v: str(v) if not isinstance(v, float) else "a%g" % v)
@pytest.mark.parametrize("name", list(FAMILIES))
def test_family_stages(name, flags, alpha):
    run_family(name, flags, alpha)


# ---- c. RoBERTa at 512 tokens ----------------------------------------------------------------------------------------------
def test_roberta_512_tokens():
    _CACHE.clear()
    S, right, left = 512, 350, 300
    p64, model = family_model("roberta", 1, seed=61, vocab=1000, max_pos=514, dim=768, heads=12, depth=2, inter=3072)
    eng = model.engine()
    g = torch.Generator().manual_seed(62)
    ids = torch.randint(6, 1000, (3, S), generator=g)
    ids[:, 0] = CLASS_TOKEN
    mask = torch.ones_like(ids)
    ids[1, right:], mask[1, right:] = 1, 0                     # row 1: right-padded
    ids[2, :left], mask[2, :left] = 1, 0                       # row 2: left-padded by 300
    ids[2, left] = CLASS_TOKEN
    ocpu.set_torch_threads()
    with ohf.family(ohf.ROBERTA, 1, FAMILIES["roberta"]["eps"]):
        ref, ridx, taps = obert.explain({k: v.cpu() for k, v in p64.items()}, ids, mask, 12, start_layer=0,
                                        return_taps=True)
    lg = taps["logits"]
    assert bool(((lg[:, 0] - lg[:, 1]).abs() > 1e-3 * lg.abs().max(dim=1).values).all()), "arg-max too close to call"
    padded = (mask == 0)
    for flags in (0, _lib.FLAG_BENCH_DEFAULT):
        maps, idx, logits = eng.explain(ids.cuda(), mask.cuda(), start_layer=0, flags=flags, return_logits=True)
        torch.cuda.synchronize()
        attn = [eng.tensor("attn", l).clone() for l in range(2)]
        el = rel(logits, lg)
        ea = [rel(attn[l], taps["cache"]["layers"][l]["probs"]) for l in range(2)]
        eg = [rel(eng.tensor("attn_grad", l), taps["grads"][l]) for l in range(2)]
        ec = rel(eng.tensor("attn_cam", 1), taps["cams"][1])
        print("roberta S %d flags %d: logits %.1e | attn %s | attn_grad %s | top attn_cam %.1e" % (
            S, flags, el, ["%.1e" % e for e in ea], ["%.1e" % e for e in eg], ec))
        assert torch.equal(idx.cpu().long(), ridx)
        assert el < 1e-4 and max(ea) < 1e-5 and max(eg) < grad_tol(flags) and ec < 5e-2
        rel_pad = padded.clone()
        rel_pad[:, 0] = False                                  # element 0 is the row minimum by the generator's rule
        assert float(maps.cpu()[rel_pad].abs().max()) == 0.0, "padded positions must get exactly zero relevance"
        keys = padded.cuda()[:, None, None, :].expand_as(attn[0])
        for l in range(2):
            assert (attn[l][keys] == 0).all(), "a padded key got probability (layer %d)" % l
        for s in range(3):
            one, i1, l1 = eng.explain(ids[s:s + 1].cuda(), mask[s:s + 1].cuda(), start_layer=0, flags=flags,
                                      return_logits=True)
            assert int(i1) == int(idx[s])
            assert rel(one[0], maps[s]) < 1e-5 and rel(l1[0], logits[s]) < 1e-5, (flags, s)
