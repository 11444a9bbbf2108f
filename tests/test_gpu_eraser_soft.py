"""GPU: the ERASER soft-token scores (``te_eraser_soft_scores``) and tokens to flip (``eraser.eraser_eval(...,
tokens_to_flip=True)``) against the CPU oracle (``oracle/eraser_soft.py``) and the reference (``tests/golden/eraser_soft.npz``).

- The soft-scores op: within 1e-12 of the oracle on seeded ragged batches (W = 1 .. 1024, all ties, +-0, long tails,
  single-class documents), a NaN document flagged; every invalid argument returns TE_ERR_ARG before anything is
  written; outputs bit-identical on poisoned memory.
- End to end on the fixture's tiny BERT for all six methods: the soft scores within 1e-6 of the reference's (the maps
  come from the engine), ``attn_gradcam``'s NaN maps raise ``ValueError``; tokens to flip equal to the reference's
  brute force with the classifier as given (nothing flips) and with FLIP_SHIFT added to class 0's bias (every document
  flips), except where a row up to the flip has a reference logit margin below MARGIN_TOL.
- The search does not depend on ``flip_chunk`` or ``batch_size``, and equals one engine forward per selection size.
Measured on an H100 80GB HBM3 at a 700 W power limit: the op 1.1e-16 from the oracle at most; the end-to-end soft scores
2.2e-16 from the reference's; tokens to flip equal to the reference's for every method, with no rounding tie.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import eraser_soft as osoft

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eraser_soft.npz")
FLIP_SHIFT = 0.0392                 # oracle/make_golden_eraser_soft.py
MARGIN_TOL = 1e-5                   # logits: the forward bound of tests/test_gpu_methods_tc.py
TE_OK, TE_ERR_ARG = 0, -1           # include/te_b200.h
CLASSES = {"NEG": 0, "POS": 1}


def _batch(B, seed, Wmax=1024):
    """A ragged batch: (word scores fp32 [words], offsets, spans, span offsets, tails [B, 2], kinds)."""
    g = np.random.default_rng(seed)
    kinds = ["random", "ties", "all_ties", "zeros", "signed_zero", "single_pos", "single_neg", "w1", "nan"]
    scores, woff, spans, soff, tails, out_kinds = [], [0], [], [0], [], []
    for b in range(B):
        kind = kinds[b % len(kinds)]
        W = 1 if kind == "w1" else (Wmax if b == 0 else int(g.integers(1, Wmax + 1)))
        if kind in ("random", "nan"):
            s = g.random(W).astype(np.float32)
        elif kind == "ties":
            s = g.integers(0, 5, W).astype(np.float32) / 4
        elif kind == "all_ties":
            s = np.full(W, 0.75, dtype=np.float32)
        elif kind == "zeros":
            s = np.zeros(W, dtype=np.float32)
        else:
            s = np.where(g.random(W) < 0.5, np.float32(-0.0), np.float32(0.0)) + \
                (g.random(W) < 0.2) * g.integers(1, 3, W).astype(np.float32)
        if kind == "nan":
            s[int(g.integers(0, W))] = np.nan
        tail = int(g.integers(0, 5000)) if b % 3 == 0 else int(g.integers(0, 3))
        n = W + tail
        if kind == "single_pos":
            sp = [(0, n)]
        elif kind == "single_neg":
            sp = []
        else:
            sp = [(int(a), int(min(n, a + g.integers(1, 30)))) for a in g.integers(0, n, int(g.integers(1, 8)))]
        scores.append(s.astype(np.float32))
        woff.append(woff[-1] + W)
        spans.extend(sp)
        soff.append(len(spans))
        tails.append(osoft.tail_counts(sp, W, n))
        out_kinds.append(kind)
    return np.concatenate(scores), woff, spans, soff, tails, out_kinds


def _oracle(ws, woff, spans, soff, tails):
    out, single = [], []
    for b in range(len(woff) - 1):
        s = ws[woff[b]:woff[b + 1]]
        W = len(s)
        n = W + sum(tails[b])
        truth = osoft.truth_vector([(a, min(e, n)) for a, e in spans[soff[b]:soff[b + 1]]], n)
        # the tail's positives are exactly tails[b][0] by construction of _batch
        single.append(len(set(truth)) < 2)
        out.append(osoft.soft_scores(osoft.soft_prediction(s, n), truth) if not np.isnan(s).any() else (math.nan,) * 3)
    return np.array(out), np.array(single)


@pytest.mark.parametrize("B,seed,Wmax", [(1, 1, 1024), (9, 2, 1024), (40, 3, 300), (64, 4, 64)])
def test_soft_scores_against_oracle(B, seed, Wmax):
    from transformer_explainability_b200 import ops
    ws, woff, spans, soff, tails, kinds = _batch(B, seed, Wmax)
    r = ops.eraser_soft_scores(torch.from_numpy(ws).cuda(), woff, spans, soff, tails)
    got, flags = r["scores"].cpu().numpy(), r["flags"].cpu().numpy()
    want, single = _oracle(ws, woff, spans, soff, tails)
    nan_doc = np.array([k == "nan" for k in kinds])
    assert np.array_equal(flags[:, 1] != 0, nan_doc)
    assert np.array_equal(flags[:, 0] != 0, single)
    assert np.isnan(got[nan_doc]).all()
    ok = ~nan_doc
    err = np.nanmax(np.abs(got[ok] - want[ok]), initial=0.0)
    assert np.array_equal(np.isnan(got[ok]), np.isnan(want[ok])), (got[ok], want[ok])
    print("MEASURED soft scores B %d: %.2e from the oracle" % (B, err))
    assert err <= 1e-12, err


def test_soft_scores_reject_bad_arguments():
    """Every invalid argument returns TE_ERR_ARG from the C entry point, and the outputs keep their sentinel."""
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200._lib import ptr
    lib = _lib.load()
    ws = torch.rand(5, device="cuda")
    ok = dict(B=2, woff=[0, 3, 5], soff=[0, 1, 2], spans=[(0, 2), (1, 4)], tails=[(0, 1), (2, 0)])
    bad = [dict(woff=[1, 3, 5]), dict(woff=[0, 3, 2]), dict(soff=[0, 2, 1]), dict(spans=[(-1, 2), (1, 4)]),
           dict(spans=[(3, 2), (1, 4)]), dict(tails=[(0, -1), (2, 0)]), dict(tails=[(0, 1), (1 << 30, 1)]),
           dict(woff=[0, 0, 5], tails=[(0, 0), (2, 0)]), dict(B=0), dict(woff=[0, 1025, 1030])]
    wsp = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")

    def call(a):
        arr = lambda v: (_lib.c_int * max(len(v), 1))(*v)                                # noqa: E731
        scores = torch.full((2, 3), -7.0, dtype=torch.float64, device="cuda")
        flags = torch.full((2, 2), -7, dtype=torch.int32, device="cuda")
        st = lib.te_eraser_soft_scores(ptr(ws), a["B"], arr(a["woff"]), arr(a["soff"]), arr([x for s in a["spans"] for x in s]),
                                       arr([x for t in a["tails"] for x in t]), ptr(scores), ptr(flags), ptr(wsp),
                                       wsp.numel(), None)
        torch.cuda.synchronize()
        return st, scores, flags
    st, scores, flags = call(ok)
    assert st == TE_OK and (flags != -7).all() and (scores != -7).all()
    for b in bad:
        st, scores, flags = call(dict(ok, **b))
        assert st == TE_ERR_ARG, b
        assert (scores == -7).all() and (flags == -7).all(), b


def test_soft_scores_on_poisoned_memory():
    from test_gpu_poison import Findings, run_case
    from transformer_explainability_b200 import ops
    found = Findings()
    for B, seed in ((3, 5), (40, 6)):
        ws, woff, spans, soff, tails, _ = _batch(B, seed, 600)
        w = torch.from_numpy(ws).cuda()
        run_case(found, "eraser_soft_scores B %d" % B, lambda p: ops.eraser_soft_scores(w, woff, spans, soff, tails))
    found.check()


# ---- end to end on the fixture's tiny BERT -----------------------------------------------------------------------------------
def _generators(shift):
    """The six bound Generator methods on the tiny BERT, with ``shift`` added to class 0's classifier bias."""
    import functools
    from test_gpu_bert import make_model, TINY
    from transformers import BertConfig
    from transformer_explainability_b200 import eraser as te
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
        BertForSequenceClassification as ClsLrp
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    z = np.load(os.path.join(HERE, "golden", "bert_tiny.npz"))
    params = {k[len("param."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("param.")}
    params["classifier.bias"] = params["classifier.bias"] + torch.tensor([shift, 0.0])
    ours = make_model(params, int(z["heads"]), **TINY)
    cls = ClsLrp(BertConfig(num_attention_heads=int(z["heads"]), num_labels=2, **TINY))
    cls.load_state_dict(params, strict=False)
    cls = cls.cuda().eval()
    out = {}
    for method, (kind, fn) in te.METHOD_GENERATOR.items():
        f = getattr(Generator(ours if kind == "ours" else cls), fn)
        out[method] = functools.partial(f, start_layer=2) if fn == "generate_LRP" else f
    return out


@pytest.fixture(scope="module")
def tiny():
    from test_gpu_eraser import _fixture
    return _fixture(), {"": _generators(0.0), "_shift": _generators(FLIP_SHIFT)}, np.load(GOLDEN)


def _check_flips(got, z, method, tag):
    """tokens to flip equal to the fixture's, except where a reference row up to the later of the two flips lies within
    MARGIN_TOL of the boundary.  Returns the number of tolerated differences."""
    want, margins = z["%s.flip%s" % (method, tag)], z["%s.margins%s" % (method, tag)]
    ties = 0
    for i, (a, b) in enumerate(zip(got, want)):
        if a != b:
            k = min(max(a, b), int(z["W"][i]))
            assert np.nanmin(np.abs(margins[i, :k])) < MARGIN_TOL, (method, tag, i, a, b)
            ties += 1
    return ties


@pytest.mark.parametrize("method", ["transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout"])
def test_end_to_end_against_the_reference(tiny, method, tmp_path):
    import json
    (g, docids, docs, anns, enc, te), gens, z = tiny
    soft = method != "attn_gradcam"
    if not soft:                                               # the reference's maps are NaN: sklearn rejects them
        with pytest.raises(ValueError, match="NaN"):
            te.eraser_eval(gens[""][method], docs, anns, enc, CLASSES, batch_size=4, soft_scores=True)
    for tag in ("", "_shift"):
        res = te.eraser_eval(gens[tag][method], docs, anns, enc, CLASSES, batch_size=4, faithfulness=True,
                             soft_scores=soft, tokens_to_flip=True)
        off = te.eraser_eval(gens[tag][method], docs, anns, enc, CLASSES, batch_size=4, faithfulness=True)
        for k in ("lines", "scores"):
            assert res[k] == off[k], k
        f, fo = res["faithfulness"], off["faithfulness"]
        assert f["scores"] == fo["scores"]
        for a, b in zip(f["lines"], fo["lines"]):
            d = json.loads(a)
            t = d.pop("tokens_to_flip")
            assert json.dumps(d) == b and isinstance(t, int)
        ties = _check_flips(f["tokens_to_flip"].tolist(), z, method, tag)
        print("MEASURED %s%s tokens to flip %s (%d rounding ties), %d rows" % (
            method, tag, f["tokens_to_flip"].tolist(), ties, f["flip_rows"]))
        assert f["flipped"].tolist() == z["%s.flipped%s" % (method, tag)].tolist() or ties
        assert f["flip_scores"]["never_flipped"] == int((~f["flipped"]).sum())
        if not ties:
            assert f["flip_scores"]["tokens_to_flip"] == float(z["%s.flip_fraction%s" % (method, tag)])
        if soft and tag == "":
            got = res["soft"]["per_document"]
            err = float(np.nanmax(np.abs(got - z["%s.soft_doc" % method]), initial=0.0))
            assert np.array_equal(np.isnan(got), np.isnan(z["%s.soft_doc" % method]))
            ref = json.loads(str(z["%s.soft_scores" % method]))
            serr = max(abs(res["soft"]["scores"][k] - ref[k]) for k in ref)
            print("MEASURED %s soft scores: per document %.2e, aggregate %.2e from the reference" % (method, err, serr))
            assert err <= 1e-6 and serr <= 1e-6, (err, serr)
            assert np.array_equal(res["soft"]["single_class"], z["%s.single" % method])
        te.write_results(res, str(tmp_path / tag))
        names = sorted(os.listdir(str(tmp_path / tag)))
        assert "tokens_to_flip.json" in names and (("soft_results.jsonl" in names) == soft)


def test_search_invariant_to_chunking_and_batching(tiny):
    (g, docids, docs, anns, enc, te), gens, z = tiny
    for method in ("transformer_attribution", "rollout"):
        gen = gens["_shift"][method]
        runs = {}
        for fc, bs in ((1, 4), (7, 4), (16, 4), (64, 4), (16, 1), (16, 8), (3, 3)):
            f = te.eraser_eval(gen, docs, anns, enc, CLASSES, batch_size=bs, faithfulness=True, tokens_to_flip=True,
                               flip_chunk=fc)["faithfulness"]
            runs[(fc, bs)] = f["tokens_to_flip"].tolist()
        print("MEASURED %s tokens to flip by (flip_chunk, batch_size): %s" % (method, runs))
        assert len(set(map(tuple, runs.values()))) == 1, runs


def test_search_matches_one_forward_per_k(tiny):
    """The batched, chunked search against a loop of one unpadded engine forward per selection size on the batch-1
    map, for every document of two methods; a difference needs an engine margin under MARGIN_TOL on the way."""
    from transformer_explainability_b200 import ops
    (g, docids, docs, anns, enc, te), gens, z = tiny
    for method in ("transformer_attribution", "lrp"):
        gen = gens["_shift"][method]
        eng = te._generator_model(gen).engine()
        res = te.eraser_eval(gen, docs, anns, enc, CLASSES, batch_size=8, faithfulness=True, tokens_to_flip=True)
        f = res["faithfulness"]
        for i, (a, d) in enumerate(zip(anns, res["docids"])):
            ids = torch.tensor([enc[d][0]]).cuda()
            m = gen(input_ids=ids, attention_mask=torch.ones_like(ids), index=torch.tensor([CLASSES[a.classification]]).cuda())
            rg = res["word_ranges"][i]
            W = len(rg)
            lg0 = eng.forward(ids, torch.ones_like(ids))[0]
            p0 = int(torch.argmax(lg0))
            red = ops.eraser_reduce_inputs(m.reshape(1, -1).float().contiguous(), ids, [ids.shape[1]], rg, [0, W],
                                           [list(range(1, W + 1))])
            lens = red["lengths"][0, :, 0].cpu().tolist()
            k_want, margins = len(docs[d].split()), []
            for k in range(1, W + 1):
                x = red["ids"][0, k - 1, 0, :lens[k - 1]][None].contiguous()
                lg = eng.forward(x, torch.ones_like(x))[0]
                margins.append(float(lg[p0] - lg[1 - p0]))
                if int(torch.argmax(lg)) != p0:
                    k_want = k
                    break
            got = int(f["tokens_to_flip"][i])
            assert got == k_want or min(abs(x) for x in margins) < MARGIN_TOL, (method, d, got, k_want, margins)
