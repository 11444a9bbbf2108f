"""CPU checks of the RoBERTa / XLM-RoBERTa and DistilBERT classifiers: the fp64 oracle (``oracle/hf_encoders.py``)
reproduces ``transformers``' forward and attention gradients recorded in ``tests/golden/hf_encoders.npz``
(``oracle/make_golden_hf_encoders.py``) and the fixture's relevance maps; every family's weight table names exactly the
``transformers`` ``state_dict``; the workspace size does not depend on the family; invalid configurations are refused on
the host with a message."""
import ctypes
import os

import numpy as np
import pytest
import torch

import bert_lrp_oracle as olrp
from oracle import bert as obert
from oracle import hf_encoders as ohf
from oracle import make_golden_hf_encoders as mg

FAMILIES = tuple(mg.FAMILIES)
TE_ERR_ARG = -1


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "hf_encoders.npz"))


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def _setup(name):
    f = mg.FAMILIES[name]
    ids, mask, tt = mg.inputs(name)
    return ohf.to_bert_keys(mg.params(name), f["arch"]), ids, mask, dict(arch=f["arch"], pad=f["pad"], eps=f["eps"],
                                                                          token_type_ids=tt)


@pytest.mark.parametrize("name", FAMILIES)
def test_fixture_inputs(golden, name):
    ids, mask, tt = mg.inputs(name)
    assert np.array_equal(golden[name + ".ids"], ids.numpy()) and np.array_equal(golden[name + ".mask"], mask.numpy())
    assert mask[1, -1] == 0 and mask[1, 0] == 1, "a right-padded row"
    assert mask[2, 0] == 0 and mask[2, -1] == 1, "a left-padded row"
    pad = mg.FAMILIES[name]["pad"]
    assert bool((ids[mask == 0] == pad).all()) and bool((ids[mask == 1] != pad).all())
    if tt is not None:
        assert np.array_equal(golden[name + ".token_type_ids"], tt.numpy()) and tt[3].max() == 1


@pytest.mark.parametrize("name", FAMILIES)
def test_oracle_matches_transformers(golden, name):
    p, ids, mask, kw = _setup(name)
    with torch.enable_grad():
        logits, cache = ohf.forward(p, ids, mask, mg.HEADS, need_grad=True, **kw)
        seed = torch.zeros_like(logits)
        seed[torch.arange(4), logits.argmax(dim=-1)] = 1
        grads = obert.attention_gradients(cache, seed)
    assert rel(logits.detach(), golden[name + ".hf.logits"]) < 1e-12
    for l in range(3):
        probs = cache["layers"][l]["probs"].detach()
        assert rel(probs, golden["%s.hf.attn.%d" % (name, l)]) < 1e-12
        assert rel(grads[l], golden["%s.hf.grad.%d" % (name, l)]) < 1e-10
        # padded keys: probability exactly 0 in both (the -10000 and the dtype-minimum masks both underflow)
        hf = torch.from_numpy(golden["%s.hf.attn.%d" % (name, l)])
        keys = (mask == 0)[:, None, None, :].expand_as(hf)
        assert bool((hf[keys] == 0).all()) and bool((probs[keys] == 0).all())


def test_roberta_position_ids():
    ids = torch.tensor([[0, 5, 6, 2, 1, 1], [1, 1, 0, 7, 2, 1]])
    assert ohf.position_ids(ids, ohf.ROBERTA, 1).tolist() == [[2, 3, 4, 5, 1, 1], [1, 1, 2, 3, 4, 1]]
    assert ohf.position_ids(ids, ohf.DISTILBERT, 0).tolist() == [list(range(6))] * 2


# Sequence lengths around the engine's 32-token embedding tiles and its 256-token steps of the count of earlier tiles,
# up to RoBERTa's 512.
SEQ_LENGTHS = (31, 32, 33, 64, 65, 255, 256, 257, 300, 512)
CLASS_TOKEN = 3                                      # not a pad id of any test (1, 0, 5)


def position_patterns(S, pad, vocab=100, seed=0):
    """One row per padding pattern of length S -> (ids [R, S], mask [R, S], names): no padding; right padding from
    inside tile 0, from 32, 64 and 256 and from inside the last tile; left padding by 1, 31, 32, 40, 255, 256 and 257
    pads; pad ids scattered among the real tokens with mask 1; the class token followed only by pads.  Patterns that
    do not fit in S are left out.  Real tokens are drawn from [6, vocab), so none is a pad id of the tests."""
    g = torch.Generator().manual_seed(seed * 1000 + S)
    rows = []

    def row(name, n_left=0, right=None):
        ids = torch.randint(6, vocab, (S,), generator=g)
        mask = torch.ones(S, dtype=torch.long)
        ids[n_left] = CLASS_TOKEN
        ids[:n_left], mask[:n_left] = pad, 0
        if right is not None:
            ids[right:], mask[right:] = pad, 0
        rows.append((name, ids, mask))
        return ids

    row("full")
    last = (S - 1) // 32 * 32
    for r in sorted({5, 32, 64, 256, last + (S - last) // 2}):
        if 0 < r < S:
            row("right from %d" % r, right=r)
    for n in (1, 31, 32, 40, 255, 256, 257):
        if n < S:
            row("left by %d" % n, n_left=n)
    row("pad ids under mask 1")[2::7] = pad
    row("class token, then pads", right=1)
    return (torch.stack([r[1] for r in rows]), torch.stack([r[2] for r in rows]), [r[0] for r in rows])


@pytest.mark.parametrize("pad", [1, 0, 5])
@pytest.mark.parametrize("S", SEQ_LENGTHS)
def test_position_ids_match_transformers(S, pad):
    """The oracle's position ids are transformers' own, on every padding pattern, whatever the mask says."""
    transformers = pytest.importorskip("transformers")
    ids, mask, names = position_patterns(S, pad)
    want = transformers.models.roberta.modeling_roberta.RobertaEmbeddings.create_position_ids_from_input_ids(ids, pad)
    got = ohf.position_ids(ids, ohf.ROBERTA, pad)
    bad = [names[r] for r in range(len(names)) if not torch.equal(got[r], want[r])]
    assert not bad, bad
    assert ohf.position_ids(ids, ohf.DISTILBERT, pad).tolist() == [list(range(S))] * len(names)
    # the patterns hold what they are named for
    assert bool((ids[mask == 0] == pad).all())
    scattered = names.index("pad ids under mask 1")
    assert bool((ids[scattered] == pad).any()) and bool((mask[scattered] == 1).all())
    assert int(got.max()) == pad + S                                  # the full row reaches the last position
    if S > 257:
        left = names.index("left by 257")
        assert got[left, :257].eq(pad).all() and got[left, 257:].tolist() == list(range(pad + 1, pad + S - 256))


@pytest.mark.parametrize("name", FAMILIES)
def test_oracle_maps_reproduce_fixture(golden, name):
    p, ids, mask, kw = _setup(name)
    for sl in (0, 1):
        out = ohf.explain(p, ids, mask, mg.HEADS, start_layer=sl, **kw)[0]
        assert torch.equal(out, torch.from_numpy(golden["%s.ours.LRP.sl%d" % (name, sl)]))
        with ohf.family(**kw):
            out = olrp.explain(p, ids, mask, mg.HEADS, start_layer=sl)[0]
        assert torch.equal(out, torch.from_numpy(golden["%s.lrp.LRP.sl%d" % (name, sl)]))
    for which in obert.GENERATORS:
        out = ohf.generate(p, ids, mask, mg.HEADS, which, **kw)
        want = torch.from_numpy(golden["%s.ours.%s" % (name, which)])
        assert torch.equal(torch.nan_to_num(out), torch.nan_to_num(want)) and torch.equal(out.isnan(), want.isnan())
    assert torch.equal(ohf.explain_attn_grad_rollout(p, ids, mask, mg.HEADS, **kw)[0],
                       torch.from_numpy(golden[name + ".ours.attn_grad_rollout"]))
    with ohf.family(**kw):
        for which in olrp.GENERATORS:
            assert torch.equal(olrp.generate(p, ids, mask, mg.HEADS, which),
                               torch.from_numpy(golden["%s.lrp.%s" % (name, which)]))
    assert obert.forward.__module__ == "oracle.bert", "family() restores oracle.bert"


@pytest.mark.parametrize("name", FAMILIES)
def test_padded_rows_carry_no_relevance(golden, name):
    """Padded tokens get exactly zero relevance from the generators whose maps are attention-weighted sums."""
    mask = torch.from_numpy(golden[name + ".mask"])
    for key in ("ours.LRP.sl0", "lrp.LRP.sl0", "ours.attn_grad_rollout", "ours.attn_last_layer", "ours.rollout"):
        m = torch.from_numpy(golden["%s.%s" % (name, key)])
        pad = (mask == 0)
        pad[:, 0] = False                      # element 0 is the row minimum or 0 by the generator's rule
        assert bool((m[pad] == 0).all()), key


# ---- the C ABI on the host -----------------------------------------------------------------------------------------------
def _hf(kind):
    transformers = pytest.importorskip("transformers")
    small = dict(vocab_size=100, max_position_embeddings=40, num_labels=3)
    if kind == "distilbert":
        return (transformers.DistilBertConfig(dim=64, n_layers=2, n_heads=4, hidden_dim=128, **small),
                transformers.DistilBertForSequenceClassification)
    cfgcls, modelcls = {"bert": ("BertConfig", "BertForSequenceClassification"),
                        "roberta": ("RobertaConfig", "RobertaForSequenceClassification"),
                        "xlm-roberta": ("XLMRobertaConfig", "XLMRobertaForSequenceClassification")}[kind]
    return (getattr(transformers, cfgcls)(hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                                          intermediate_size=128, **small), getattr(transformers, modelcls))


def _facade(kind, config):
    from transformer_explainability_b200.BERT_explainability.modules.BERT import (
        BertForSequenceClassification as B, DistilBertForSequenceClassification as D, RobertaForSequenceClassification as R)
    return {"bert": B.BertForSequenceClassification, "roberta": R.RobertaForSequenceClassification,
            "xlm-roberta": R.XLMRobertaForSequenceClassification,
            "distilbert": D.DistilBertForSequenceClassification}[kind](config)


@pytest.mark.parametrize("kind", ["bert", "roberta", "xlm-roberta", "distilbert"])
def test_weight_table_matches_transformers_state_dict(kind):
    from transformer_explainability_b200 import _lib
    lib = _lib.load()
    config, hf_cls = _hf(kind)
    sd = {k: v for k, v in hf_cls(config).state_dict().items() if "position_ids" not in k}
    m = _facade(kind, config)
    assert {k: v.shape for k, v in m.state_dict().items() if "position_ids" not in k} == {k: v.shape for k, v in sd.items()}
    cfg = m._cfg
    n = lib.te_bert_num_weights(ctypes.byref(cfg))
    seen, end, names = set(), 0, []
    for i in range(n):
        name = lib.te_bert_weight_name(ctypes.byref(cfg), i).decode()
        numel = lib.te_bert_weight_numel(ctypes.byref(cfg), i)
        off = lib.te_bert_weight_offset(ctypes.byref(cfg), i)
        assert sd[name].numel() == numel, name
        assert off % 32 == 0 and off >= end
        end = off + numel
        seen.add(name)
        names.append(name)
    assert seen == set(sd)
    assert lib.te_bert_weight_total(ctypes.byref(cfg)) >= end
    # q | k | v of every layer back to back: the packed [3D, D] weight and [3D] bias
    for i, name in enumerate(names):
        if name.endswith(("query.weight", "q_lin.weight", "query.bias", "q_lin.bias")):
            offs = [lib.te_bert_weight_offset(ctypes.byref(cfg), i + j) for j in range(3)]
            assert offs[1] - offs[0] == offs[2] - offs[1] == sd[name].numel(), name
    assert len(m.attention_views()) == 2 and all(hasattr(v, "get_attn_gradients") for v in m.attention_views())


def test_arch_constants_match_header():
    from transformer_explainability_b200 import _lib
    head = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "te_b200.h")).read()
    for name in ("BERT", "ROBERTA", "DISTILBERT"):
        assert "#define TE_BERT_ARCH_%s %d" % (name, getattr(_lib, "BERT_ARCH_" + name)) in head
    assert [f[0] for f in _lib.TeBertConfig._fields_][-2:] == ["arch", "pad_token_id"]


def test_workspace_bytes_do_not_depend_on_the_family():
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.engine import bert_config
    lib = _lib.load()
    base = bert_config()
    # BERT-base, the same sizes as before the family fields existed (the workspace carve is unchanged)
    for (b, s), want in (((1, 128), 123258368), ((16, 128), 1972124160), ((3, 24), 55327488)):
        assert lib.te_bert_workspace_bytes(ctypes.byref(base), b, s) == want
        rob = bert_config(50265, 514, 1, layer_norm_eps=1e-5, arch=_lib.BERT_ARCH_ROBERTA, pad_token_id=1)
        dis = bert_config(type_vocab_size=0, arch=_lib.BERT_ARCH_DISTILBERT)
        assert lib.te_bert_workspace_bytes(ctypes.byref(rob), b, s) == want
        assert lib.te_bert_workspace_bytes(ctypes.byref(dis), b, s) == want


def test_host_validation():
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.engine import bert_config
    lib = _lib.load()
    R, D = _lib.BERT_ARCH_ROBERTA, _lib.BERT_ARCH_DISTILBERT

    def refused(cfg, s=8, needle=""):
        assert lib.te_bert_workspace_bytes(ctypes.byref(cfg), 1, s) == TE_ERR_ARG
        assert needle in lib.te_last_error().decode()

    ok = dict(vocab_size=100, max_position_embeddings=40, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
              intermediate_size=128)
    refused(bert_config(type_vocab_size=2, arch=3, **ok), needle="arch")
    refused(bert_config(type_vocab_size=0, **ok), needle="type_vocab")
    refused(bert_config(type_vocab_size=0, arch=R, pad_token_id=1, **ok), needle="type_vocab")
    refused(bert_config(type_vocab_size=2, arch=D, **ok), needle="DistilBERT")
    refused(bert_config(type_vocab_size=1, arch=R, pad_token_id=-1, **ok), needle="pad_token_id")
    refused(bert_config(type_vocab_size=1, arch=R, pad_token_id=100, **ok), needle="pad_token_id")
    # RoBERTa's usable length: seq + pad + 1 <= max_position
    rob = bert_config(type_vocab_size=1, arch=R, pad_token_id=1, **ok)
    assert lib.te_bert_workspace_bytes(ctypes.byref(rob), 1, 38) > 0
    refused(rob, s=39, needle="seq + pad_token_id + 1")
    assert lib.te_bert_num_weights(ctypes.byref(bert_config(type_vocab_size=2, arch=D, **ok))) == TE_ERR_ARG
    dis = bert_config(type_vocab_size=0, arch=D, **ok)
    assert lib.te_bert_workspace_bytes(ctypes.byref(dis), 1, 40) > 0
    refused(dis, s=41, needle="sequence length")
    # DistilBERT with token types: refused before anything touches the (here fake) device pointers
    ws = lib.te_bert_workspace_bytes(ctypes.byref(dis), 1, 8)
    fake = ctypes.c_void_p(1 << 20)
    before = lib.te_kernel_launch_count()
    assert lib.te_bert_forward(ctypes.byref(dis), fake, None, fake, fake, fake, 1, 8, 0, None, fake, ws, None) == \
        TE_ERR_ARG
    assert "token_type_ids" in lib.te_last_error().decode()
    assert lib.te_bert_explain(ctypes.byref(dis), fake, None, fake, fake, fake, 1, 8, fake, 0, 0, fake, None, fake, ws,
                               None) == TE_ERR_ARG
    assert lib.te_kernel_launch_count() == before


@pytest.mark.parametrize("kind,attr,value", [("bert", "hidden_act", "relu"), ("roberta", "hidden_act", "gelu_new"),
                                             ("distilbert", "activation", "relu")])
def test_other_activations_are_refused(kind, attr, value):
    config, _ = _hf(kind)
    setattr(config, attr, value)
    with pytest.raises(NotImplementedError):
        _facade(kind, config)
