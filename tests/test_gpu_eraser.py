"""GPU: the ERASER rationale evaluation (``te_eraser_rationales``, ``eraser.eraser_eval``) against the CPU oracle
(``oracle/eraser.py``) and the reference's own pooling, top-k lines and ``metrics.py`` run (``tests/golden/eraser.npz``).

- The op: word scores, order and counts exactly equal to the oracle's on random, quantised (tie-heavy), mostly negative
  (zero-clamped) and NaN-bearing maps, W from 0 to 510 words, k above W, B up to 64, three IoU thresholds; bad ranges are
  rejected; outputs are bit-identical on poisoned outputs and workspace.
- End to end on the fixture's tiny BERT: with the oracle fed the engine's own maps, the files and score dicts are
  identical.  Against the reference's maps the engine's differ by at most ``MAP_TOL`` of the map maximum, and the top-k
  word sets may differ only by words whose reference scores lie within twice that bound of the k-th reference score.
  Measured on an H100 80GB HBM3 at a 700 W power limit (the tiny model runs the fp32 SIMT kernels): map differences
  4.0e-5 (``transformer_attribution``), 4.0e-5 (``partial_lrp``), 1.0e-3 (``lrp``: relevance at the encoder input, summed
  over the hidden dimension), below 4e-7 for ``last_attn`` / ``rollout`` and 0 for ``attn_gradcam``; no rank swap occurred.
- Batching: on the conditioned BERT-base-width model of ``tests/test_gpu_methods_tc.py`` every method's real-token maps from
  a padded, length-sorted batch agree with per-document unpadded runs within that file's bounds (``tol(flags)`` of the map
  maximum, the forward-only and normalised bounds), and the scores of batch size 1 and 8 agree.  ``attn_gradcam`` is not
  padding-invariant (its gradient weights and min-max run over the padded [S, S] map), so its batches hold one length:
  its maps are checked on an unpadded batch of equal-length rows.  Measured on an H100 80GB HBM3 at 700 W: every method's
  batched maps equal the single-document maps bit for bit.
"""
import functools
import json
import os

import numpy as np
import pytest
import torch

from oracle import eraser as oe

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
THRESHOLDS = (0.5, 0.25, 1.0)
KS = tuple(range(5, 85, 5)) + (600,)
MAP_TOL = 2e-3


def _docs(B, seq, kind, seed):
    """Random documents: piece ranges, truth spans and maps [B, seq]."""
    g = np.random.default_rng(seed)
    ranges, woff, spans, soff, nwords = [], [0], [], [0], []
    for b in range(B):
        W = int(g.integers(0, 511)) if b else 510
        W = 1 if b == 1 else W
        p, r = 1, []
        while len(r) < W and p < seq - 1:
            n = 1 if W > (seq - 2) // 3 else int(g.integers(1, 4))     # long documents: one piece per word
            n = min(n, seq - 1 - p)
            r.append((p, p + n - 1))
            p += n
        ranges.extend(r)
        woff.append(len(ranges))
        nwords.append(len(r))
        s = []
        for _ in range(int(g.integers(0, 12))):
            a = int(g.integers(0, max(len(r), 1) + 20))
            s.append((a, a + int(g.integers(0, 6))))
        spans.extend(s)
        soff.append(len(spans))
    gen = torch.Generator().manual_seed(seed)
    m = torch.randn(B, seq, generator=gen)
    if kind == "quantised":
        m = torch.randint(-1, 3, (B, seq), generator=gen).float() / 2
    elif kind == "clamped":
        m = -m.abs()
        m[:, ::7] = m[:, ::7].abs()
    elif kind == "nan":
        m[torch.rand(B, seq, generator=gen) < 0.01] = float("nan")
        m[0, 1] = -0.0
    return m, ranges, woff, spans, soff, nwords


def _oracle(m, ranges, woff, spans, soff, ks, thr):
    m = m.numpy()
    scores, orders, counts = [], [], []
    for b in range(len(woff) - 1):
        w = []
        for a, e in ranges[woff[b]:woff[b + 1]]:
            v = m[b, a:e + 1]
            w.append(np.float32("nan") if np.isnan(v).any() else np.max(np.maximum(v, np.float32(0))))
        w = np.asarray(w, dtype=np.float32)
        o = oe.word_order(w)
        scores.append(w)
        orders.append(np.concatenate([o[:max(ks)], np.full(max(0, max(ks) - len(o)), -1)]))
        counts.append(oe.doc_counts(o, spans[soff[b]:soff[b + 1]], ks, thr))
    return np.concatenate(scores), np.stack(orders), np.stack(counts)


@pytest.mark.parametrize("kind", ["random", "quantised", "clamped", "nan"])
@pytest.mark.parametrize("B,seq", [(1, 512), (7, 300), (64, 512)])
def test_eraser_rationales_against_oracle(kind, B, seq):
    from transformer_explainability_b200 import ops
    m, ranges, woff, spans, soff, nwords = _docs(B, seq, kind, seed=B * 13 + seq + len(kind))
    r = ops.eraser_rationales(m.cuda(), ranges, woff, spans, soff, KS, THRESHOLDS)
    ws, order, counts = _oracle(m, ranges, woff, spans, soff, KS, THRESHOLDS)
    assert np.array_equal(r["word_scores"].cpu().numpy(), ws, equal_nan=True)
    assert np.array_equal(r["order"].cpu().numpy(), order)
    assert np.array_equal(r["counts"].cpu().numpy(), counts)
    assert max(nwords) == min(510, seq - 2) and (B == 1 or 1 in nwords)


def test_eraser_rationales_rejects_bad_ranges():
    from transformer_explainability_b200 import ops, _lib
    m = torch.rand(2, 16).cuda()
    ok = dict(piece_ranges=[(1, 2), (3, 3)], word_offsets=[0, 1, 2], spans=[(0, 1)], span_offsets=[0, 1, 1], ks=(5,))
    ops.eraser_rationales(m, **ok)
    bad = [dict(piece_ranges=[(1, 2), (3, 16)]), dict(piece_ranges=[(2, 1), (3, 3)]), dict(piece_ranges=[(-1, 2), (3, 3)]),
           dict(spans=[(-1, 1)]), dict(spans=[(3, 2)]), dict(ks=(10, 5)), dict(ks=(-1,)),
           dict(word_offsets=[0, 2, 1], piece_ranges=[(1, 2)])]
    for b in bad:
        with pytest.raises((_lib.TeError, ValueError)):
            ops.eraser_rationales(m, **dict(ok, **b))
    with pytest.raises(_lib.TeError):
        ops.eraser_rationales(torch.rand(1, 2000).cuda(), [(i, i) for i in range(1025)], [0, 1025], [], [0, 0], (5,))
    with pytest.raises(ValueError):
        ops.eraser_rationales(m, **ok, thresholds=[0.5] * 9)


def test_eraser_rationales_on_poisoned_memory():
    from test_gpu_poison import Findings, run_case
    from transformer_explainability_b200 import ops
    found = Findings()
    for kind, B in (("nan", 3), ("quantised", 64)):
        m, ranges, woff, spans, soff, _ = _docs(B, 512, kind, seed=5 + B)
        m = m.cuda()
        run_case(found, "eraser_rationales %s B %d" % (kind, B),
                 lambda p: ops.eraser_rationales(m, ranges, woff, spans, soff, KS, THRESHOLDS))
    found.check()


# ---- end to end on the fixture's tiny BERT -----------------------------------------------------------------------------------
def _fixture():
    import test_eraser as ce
    from transformer_explainability_b200 import eraser as te
    g, docids, docs, anns = ce.load()
    enc = {d: ([int(i) for i in g["ids." + d]], [str(p) for p in g["pieces." + d]]) for d in docids}
    return g, docids, docs, anns, enc, te


def _generators():
    from test_gpu_bert import make_model, TINY
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
        BertForSequenceClassification as ClsLrp
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    from transformers import BertConfig
    from transformer_explainability_b200 import eraser as te
    z = np.load(os.path.join(HERE, "golden", "bert_tiny.npz"))
    params = {k[len("param."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("param.")}
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
    return _fixture(), _generators()


@pytest.mark.parametrize("method", ["transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout"])
def test_end_to_end_against_oracle_and_fixture(tiny, method, tmp_path):
    (g, docids, docs, anns, enc, te), gens = tiny
    classes = {"NEG": 0, "POS": 1}
    res = te.eraser_eval(gens[method], docs, anns, enc, classes, batch_size=1, iou_thresholds=THRESHOLDS)
    # the oracle on the engine's own maps (batch size 1: the same launches as the evaluation)
    per_k, map_err, swaps = [], 0.0, 0.0
    for i, (a, d) in enumerate(zip(anns, res["docids"])):
        ids = torch.tensor([enc[d][0]]).cuda()
        m = gens[method](input_ids=ids, attention_mask=torch.ones_like(ids), index=torch.tensor([classes[a.classification]]).cuda())
        m = m[0].float().cpu().numpy()
        cam = np.where(np.isnan(m), m, np.maximum(m, np.float32(0)))
        words = oe.pool_words(docs[d].split(), enc[d][1], list(cam))
        order = oe.word_order(words)
        kmax = res["order"].shape[1]
        assert res["order"][i].tolist() == order[:kmax].tolist() + [-1] * max(0, kmax - len(order))
        per_k.append([order[:k].tolist() for k in te.KS])
        ref_map = g["%s.map.%s" % (method, d)]
        ok = ~np.isnan(ref_map)
        assert np.array_equal(np.isnan(m), ~ok), (method, d)
        scale = max(float(np.abs(ref_map[ok]).max()) if ok.any() else 0.0, 1e-30)
        map_err = max(map_err, float(np.abs(m[ok] - ref_map[ok]).max()) / scale if ok.any() else 0.0)
        ref_words = g["%s.words.%s" % (method, d)]
        for k in te.KS:                                               # rank swaps only between near-equal reference scores
            n = min(k, len(ref_words))
            ref_set = set(int(h["start_token"]) for h in json.loads(str(g["%s.lines.%d" % (method, k)][i]))["rationales"][0]
                          ["hard_rationale_predictions"][-n:])
            diff = ref_set ^ set(order[:n].tolist())
            if diff and not np.isnan(ref_words).any():
                kth = np.sort(ref_words)[::-1][n - 1]
                gap = max(abs(float(ref_words[w]) - float(kth)) for w in diff) / scale
                swaps = max(swaps, gap)
                assert gap <= 2 * MAP_TOL, (method, d, k, gap)
    lines = oe.prediction_lines(res["docids"], per_k)
    for j, k in enumerate(te.KS):
        assert res["lines"][k] == lines[j]
        assert res["scores"][k] == oe.hard_scores(anns, lines[j], THRESHOLDS)
    te.write_results(res, str(tmp_path))
    with open(os.path.join(str(tmp_path), "identifier_results_80.json")) as f:
        assert f.read().splitlines() == res["lines"][80]
    print("MEASURED %s vs fixture: map %.2e of the maximum, rank-swap score gap %.2e" % (method, map_err, swaps))
    assert map_err <= MAP_TOL, (method, map_err)


# ---- batching -----------------------------------------------------------------------------------------------------------------
def test_batching_does_not_change_results():
    """Conditioned BERT-base width (3 layers), 11 documents of 20..130 tokens: every method's real-token maps of a padded,
    length-sorted batch against per-document unpadded runs, and eraser_eval at batch size 1 and 8."""
    from test_gpu_methods_tc import tol, FWD_TOL, NORM_TOL
    from test_gpu_bert import make_model
    from oracle import bert as obert, conditioned
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
        BertForSequenceClassification as ClsLrp
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    from transformer_explainability_b200 import eraser as te
    from transformers import BertConfig
    params, heads = obert.init_params(seed=22, vocab=1000, max_pos=512, dim=768, depth=3, heads=12, inter=3072,
                                      rand_affine=True)
    params = conditioned.condition_bert(params, c_qkv=3.0)
    cfg = dict(hidden_size=768, num_hidden_layers=3, intermediate_size=3072, vocab_size=1000, max_position_embeddings=512)
    ours = make_model(params, heads, **cfg)
    cls = ClsLrp(BertConfig(num_attention_heads=heads, num_labels=2, **cfg))
    cls.load_state_dict({k: v.float() for k, v in params.items()}, strict=False)
    cls = cls.cuda().eval()
    g = np.random.default_rng(3)
    vocab = ["w%d" % i for i in range(1000)]
    docs, enc, anns = {}, {}, []
    for i, n in enumerate([20, 130, 57, 128, 90, 33, 130, 64, 101, 45, 77]):
        ids = [101] + [int(x) for x in g.integers(5, 1000, n - 2)] + [102]
        d = "d%d" % i
        docs[d] = " ".join(vocab[t] for t in ids[1:-1])
        enc[d] = (ids, ["[CLS]"] + [vocab[t] for t in ids[1:-1]] + ["[SEP]"])
        s0 = int(g.integers(0, n - 2))
        ev = (te.Evidence("", d, s0, s0 + 3),)
        anns.append(te.Annotation(d, "", frozenset([ev]), ("NEG", "POS")[i % 2]))
    classes = {"NEG": 0, "POS": 1}
    for method, (kind, fn) in te.METHOD_GENERATOR.items():
        gen = getattr(Generator(ours if kind == "ours" else cls), fn)
        gen = functools.partial(gen, start_layer=2) if fn == "generate_LRP" else gen
        order = sorted(range(len(anns)), key=lambda i: len(enc[anns[i].annotation_id][0]))
        S = max(len(e[0]) for e in enc.values())
        ids = torch.zeros(len(order), S, dtype=torch.long)
        mask = torch.zeros_like(ids)
        for r, i in enumerate(order):
            e = enc[anns[i].annotation_id][0]
            ids[r, :len(e)], mask[r, :len(e)] = torch.tensor(e), 1
        target = torch.tensor([classes[anns[i].classification] for i in order]).cuda()
        if method == "attn_gradcam":                                  # not padding-invariant: batched by equal length only
            mask[:] = 1
            ids[:, :] = ids[-1:, :]
            target[:] = target[-1]
        batched = gen(input_ids=ids.cuda(), attention_mask=mask.cuda(), index=target).float().cpu()
        worst = 0.0
        for r, i in enumerate(order):
            n = int(mask[r].sum())
            one = gen(input_ids=ids[r:r + 1, :n].cuda(), attention_mask=mask[r:r + 1, :n].cuda(), index=target[r:r + 1])
            one = one[0].float().cpu()
            a, b = batched[r, 1:n], one[1:n]                          # pooling never reads the [CLS] entry
            assert torch.equal(torch.isnan(a), torch.isnan(b)), method
            ok = ~torch.isnan(b)
            if ok.any():
                err = float((a[ok] - b[ok]).abs().max())
                worst = max(worst, err if method == "attn_gradcam" else err / max(float(b[ok].abs().max()), 1e-30))
        bound = NORM_TOL if method == "attn_gradcam" else FWD_TOL if method in ("last_attn", "rollout") else \
            tol((ours if kind == "ours" else cls).engine().flags)
        print("MEASURED batching %s: %.2e (bound %.0e)" % (method, worst, bound))
        assert worst <= bound, (method, worst, bound)
        r1 = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=1)
        r8 = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=8)
        assert r1["scores"] == r8["scores"], method
