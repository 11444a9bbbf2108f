"""GPU: the ERASER faithfulness evaluation (``te_eraser_reduce_inputs``, ``te_class_probs``, ``eraser.eraser_eval(...,
faithfulness=True)``) against the CPU oracle (``oracle/eraser_faithfulness.py``) and the reference's own forwards and
``metrics.py`` (``tests/golden/eraser_faithfulness.npz``).

- The reduce op: ids and lengths exactly equal to the oracle's on random documents with ties, NaN and -0.0 in the maps,
  shared pieces, pieces outside every range, W = 0 and 1, n = 0 and n = W, padded rows, batches of 1, 6 and 40; every
  invalid argument returns TE_ERR_ARG before anything is written; outputs bit-identical on poisoned memory.
- ``te_class_probs``: within 2 ulp of ``torch.softmax`` (a NaN row gives a NaN row, rows with +-1e30 stay finite).
- End to end on the fixture's tiny BERT for all six methods: the reduced rows equal the fixture's, the original and reduced
  probabilities lie within ``FWD_TOL`` of the reference's fp32 forward, the classification agrees wherever the reference's
  margin exceeds that bound, and the faithfulness scores within the bound that follows; the rationale results are
  bit-identical to a run without faithfulness.
- Batching: the length-sorted chunked forwards agree with one unpadded forward per row (chunks of 2 and 3 tokens occur,
  from a one-word document); at BERT-base width the probabilities agree with an fp64 oracle forward.
Measured on an H100 80GB HBM3 at a 700 W power limit: ``te_class_probs`` 0 ulp from ``torch.softmax``; every method's
probabilities 6.0e-8 from the reference's fp32 forward; chunked vs per-row forwards bit-identical; BERT-base width
2.3e-7 (flags 0) and 3.7e-7 (flags 7475) from fp64.
"""
import functools
import json
import os

import numpy as np
import pytest
import torch

from oracle import eraser_faithfulness as of

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eraser_faithfulness.npz")
FWD_TOL = 1e-5                      # the forward bound of tests/test_gpu_methods_tc.py (probabilities, absolute)
TE_OK, TE_ERR_ARG = 0, -1           # include/te_b200.h


def _docs(B, S, seed):
    """Random documents in padded rows [B, S]: (maps, ids, lengths, ranges, offsets, n_select [B, 6])."""
    g = np.random.default_rng(seed)
    lens, ranges, woff, nsel = [], [], [0], []
    for b in range(B):
        L = S if b == 0 else int(g.integers(2, S + 1))
        r, p = [], 1
        while p <= L - 2 and len(r) < 1024:
            if b % 4 == 1 and r:                                      # W = 1
                break
            if g.random() < 0.15:                                     # a piece outside every range
                p += 1
                continue
            n = int(g.integers(1, 4))
            first = p - 1 if r and p > 1 and g.random() < 0.2 else p  # a piece shared with the previous word
            last = min(L - 2, p + n - 1)
            r.append((first, last))
            p = last + 1
        ranges.extend(r)
        woff.append(len(ranges))
        lens.append(L)
        W = len(r)
        nsel.append([0, W] + [int(x) for x in g.integers(0, W + 1, 4)])
    gen = torch.Generator().manual_seed(seed)
    maps = torch.randint(-2, 4, (B, S), generator=gen).float() / 2      # tie-heavy, clamped negatives
    maps[torch.rand(B, S, generator=gen) < 0.02] = float("nan")
    maps[maps == 0] = -0.0
    ids = torch.randint(5, 30000, (B, S), generator=gen)
    for b, L in enumerate(lens):
        ids[b, L:] = 0
    return maps, ids, lens, ranges, woff, np.array(nsel)


def _pool(m, rg):
    w = []
    for a, e in rg:
        v = m[a:e + 1]
        w.append(np.float32("nan") if np.isnan(v).any() else np.max(np.maximum(v, np.float32(0))))
    return np.asarray(w, dtype=np.float32)


def _oracle(maps, ids, lens, ranges, woff, nsel):
    B, S = maps.shape
    J = nsel.shape[1]
    out_ids = np.zeros((B, J, 2, S), dtype=np.int64)
    out_len = np.zeros((B, J, 2), dtype=np.int32)
    for b in range(B):
        rg = ranges[woff[b]:woff[b + 1]]
        words = _pool(maps[b].numpy(), rg)
        row = ids[b, :lens[b]].tolist()
        for j in range(J):
            for t, r in enumerate(of.reduce_rows(row, rg, words, int(nsel[b, j]))):
                out_ids[b, j, t, :len(r)] = r
                out_len[b, j, t] = len(r)
    return out_ids, out_len


@pytest.mark.parametrize("B,S,seed", [(1, 512, 1), (6, 300, 2), (40, 512, 3), (40, 64, 4)])
def test_reduce_inputs_against_oracle(B, S, seed):
    from transformer_explainability_b200 import ops
    maps, ids, lens, ranges, woff, nsel = _docs(B, S, seed)
    r = ops.eraser_reduce_inputs(maps.cuda(), ids.cuda(), lens, ranges, woff, nsel)
    want_ids, want_len = _oracle(maps, ids, lens, ranges, woff, nsel)
    assert np.array_equal(r["lengths"].cpu().numpy(), want_len)
    assert np.array_equal(r["ids"].cpu().numpy(), want_ids)
    W = np.diff(woff)
    assert B == 1 or (1 in W.tolist() and min(lens) < S)


def test_reduce_inputs_rejects_bad_arguments():
    """Every invalid argument returns TE_ERR_ARG from the C entry point, and the outputs keep their sentinel."""
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200._lib import ptr
    lib = _lib.load()
    B, S = 2, 16
    maps = torch.rand(B, S, device="cuda")
    ids = torch.randint(5, 100, (B, S), device="cuda")
    ok = dict(lens=[16, 10], ranges=[(1, 2), (3, 14), (1, 8)], woff=[0, 2, 3], nsel=[[0, 2], [1, 1]], J=2)
    bad = [dict(ranges=[(0, 2), (3, 14), (1, 8)]), dict(ranges=[(1, 2), (3, 15), (1, 8)]),
           dict(ranges=[(1, 2), (3, 14), (1, 9)]), dict(ranges=[(2, 1), (3, 14), (1, 8)]),
           dict(lens=[16, 1]), dict(lens=[17, 10]), dict(nsel=[[0, 3], [1, 1]]), dict(nsel=[[0, -1], [1, 1]]),
           dict(nsel=[[0, 2], [2, 1]]), dict(J=0), dict(woff=[1, 2, 3])]
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")

    def call(a):
        arr = lambda v: (_lib.c_int * len(v))(*v)                                        # noqa: E731
        flat = [x for rg in a["ranges"] for x in rg]
        nflat = [x for row in a["nsel"] for x in row]
        out = torch.full((B, max(a["J"], 1), 2, S), -7, dtype=torch.int64, device="cuda")
        olen = torch.full((B, max(a["J"], 1), 2), -7, dtype=torch.int32, device="cuda")
        st = lib.te_eraser_reduce_inputs(ptr(maps), ptr(ids), B, S, arr(a["lens"]), arr(a["woff"]), arr(flat), arr(nflat),
                                         a["J"], ptr(out), ptr(olen), ptr(ws), ws.numel(), None)
        torch.cuda.synchronize()
        return st, out, olen
    st, out, _ = call(ok)
    assert st == TE_OK and (out != -7).all()
    for b in bad:
        st, out, olen = call(dict(ok, **b))
        assert st == TE_ERR_ARG, b
        assert (out == -7).all() and (olen == -7).all(), b
    # W > TE_ERASER_MAX_WORDS and seq > TE_ERASER_MAX_SEQ
    from transformer_explainability_b200 import ops
    with pytest.raises(_lib.TeError):
        ops.eraser_reduce_inputs(torch.rand(1, 2100, device="cuda"), torch.ones(1, 2100, dtype=torch.long, device="cuda"),
                                 [2100], [(i, i) for i in range(1, 1026)], [0, 1025], [[1]])
    with pytest.raises(_lib.TeError):
        ops.eraser_reduce_inputs(torch.rand(1, 8193, device="cuda"), torch.ones(1, 8193, dtype=torch.long, device="cuda"),
                                 [8193], [(1, 1)], [0, 1], [[1]])


def test_new_ops_on_poisoned_memory():
    from test_gpu_poison import Findings, run_case
    from transformer_explainability_b200 import ops
    found = Findings()
    for B, S, seed in ((3, 512, 5), (40, 300, 6)):
        maps, ids, lens, ranges, woff, nsel = _docs(B, S, seed)
        maps, ids = maps.cuda(), ids.cuda()
        run_case(found, "eraser_reduce_inputs B %d" % B,
                 lambda p: ops.eraser_reduce_inputs(maps, ids, lens, ranges, woff, nsel))
    for R, C in ((1, 2), (300, 3), (37, 1000)):
        x = torch.randn(R, C, device="cuda") * 5
        run_case(found, "class_probs %dx%d" % (R, C), lambda p: ops.class_probs(x))
    found.check()


def test_class_probs_within_2_ulp_of_torch_softmax():
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(9)
    for R, C in ((5, 2), (64, 3), (33, 47), (8, 1000)):
        x = torch.randn(R, C, generator=g) * 8
        x[0, 0] = float("nan")
        x[1, :] = 1e30
        x[2, 0] = 1e30
        x[3, 0] = -1e30
        x = x.cuda()
        got, want = ops.class_probs(x), torch.softmax(x, dim=-1)
        assert torch.isnan(got[0]).all() and torch.isnan(want[0]).all()
        assert torch.isfinite(got[1:]).all()
        ulp = (got[1:].view(torch.int32).long() - want[1:].view(torch.int32).long()).abs().max().item()
        print("MEASURED class_probs %dx%d: %d ulp" % (R, C, ulp))
        assert ulp <= 2, (R, C, ulp)


# ---- end to end on the fixture's tiny BERT -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    from test_gpu_eraser import _fixture, _generators
    return _fixture(), _generators(), np.load(GOLDEN)


@pytest.mark.parametrize("method", ["transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout"])
def test_end_to_end_against_the_reference(tiny, method, tmp_path):
    from transformer_explainability_b200 import ops
    (g, docids, docs, anns, enc, te), gens, z = tiny
    classes = {"NEG": 0, "POS": 1}
    res = te.eraser_eval(gens[method], docs, anns, enc, classes, batch_size=4, faithfulness=True)
    off = te.eraser_eval(gens[method], docs, anns, enc, classes, batch_size=4)
    for k in ("lines", "scores"):
        assert res[k] == off[k], k
    assert np.array_equal(res["order"], off["order"]) and np.array_equal(res["counts"], off["counts"])
    f = res["faithfulness"]
    assert f["fractions"] == [float(x) for x in z["fractions"]]
    assert np.array_equal(f["n_select"], z["%s.n_select" % method])
    # the reduced rows of the engine's own maps equal the fixture's (the reference's maps)
    for i, (a, d) in enumerate(zip(anns, res["docids"])):
        ids = torch.tensor([enc[d][0]]).cuda()
        m = gens[method](input_ids=ids, attention_mask=torch.ones_like(ids), index=torch.tensor([classes[a.classification]]).cuda())
        red = ops.eraser_reduce_inputs(m.reshape(1, -1).float().contiguous(), ids, [ids.shape[1]], res["word_ranges"][i],
                                       [0, len(res["word_ranges"][i])], f["n_select"][i:i + 1])
        L = ids.shape[1]
        assert np.array_equal(red["lengths"][0].cpu().numpy(), z["%s.red_len" % method][i]), (method, d)
        assert np.array_equal(red["ids"][0, :, :, :L].cpu().numpy(), z["%s.red_ids" % method][i, :, :, :L]), (method, d)
    err = max(float(np.abs(f["probs"] - z["%s.probs_f32" % method]).max()),
              float(np.abs(f["comp"] - z["%s.red_probs_f32" % method][:, :, 0]).max()),
              float(np.abs(f["suff"] - z["%s.red_probs_f32" % method][:, :, 1]).max()))
    print("MEASURED %s probabilities vs the reference fp32 forward: %.2e" % (method, err))
    assert err <= FWD_TOL, (method, err)
    ref_p = z["%s.probs_f32" % method]
    margin = np.abs(ref_p[:, 0] - ref_p[:, 1])
    ref_lines = [json.loads(str(l)) for l in z["%s.lines" % method]]
    got_lines = [json.loads(l) for l in f["lines"]]
    for r, l, mg in zip(ref_lines, got_lines, margin):
        assert l["rationales"] == r["rationales"] and l["annotation_id"] == r["annotation_id"]
        if mg > 2 * FWD_TOL:
            assert l["classification"] == r["classification"]
    ref = json.loads(str(z["%s.scores" % method]))
    for k in ("comprehensiveness", "sufficiency", "comprehensiveness_aopc", "sufficiency_aopc"):
        assert abs(f["scores"][k] - ref[k]) <= 2 * FWD_TOL, (method, k, f["scores"][k], ref[k])
    te.write_results(res, str(tmp_path))
    with open(os.path.join(str(tmp_path), "faithfulness_results.jsonl")) as fh:
        assert fh.read().splitlines() == f["lines"]


def _single_rows(gen, enc, d, target, ranges, nsel, eng):
    """Per selection and kind: the probabilities of the reduced row run alone, unpadded (batch-1 maps)."""
    from transformer_explainability_b200 import ops
    ids = torch.tensor([enc[d][0]]).cuda()
    m = gen(input_ids=ids, attention_mask=torch.ones_like(ids), index=torch.tensor([target]).cuda())
    red = ops.eraser_reduce_inputs(m.reshape(1, -1).float().contiguous(), ids, [ids.shape[1]], ranges, [0, len(ranges)],
                                   nsel[None])
    J = nsel.shape[0]
    out = np.zeros((J, 2, eng.cfg.num_labels), dtype=np.float32)
    lens = red["lengths"][0].cpu().numpy()
    for j in range(J):
        for t in range(2):
            x = red["ids"][0, j, t, :lens[j, t]][None].contiguous()
            out[j, t] = ops.class_probs(eng.forward(x, torch.ones_like(x))).cpu().numpy()[0]
    return out, lens


def test_batching_does_not_change_results(tiny):
    """Tiny BERT, the fixture's documents plus two one-word documents: chunked forwards (default and 5 rows) against one
    unpadded forward per row."""
    (g, docids, docs, anns, enc, te), gens, z = tiny
    vocab = [str(v) for v in g["vocab"]]
    docs, enc, anns = dict(docs), dict(enc), list(anns)
    for i, w in enumerate(("a", "q")):                                    # one word of one piece each
        d = "one%d.txt" % i
        docs[d] = w
        enc[d] = ([vocab.index("[CLS]"), vocab.index(w), vocab.index("[SEP]")], ["[CLS]", w, "[SEP]"])
        anns.append(te.Annotation(d, "", frozenset([(te.Evidence(w, d, 0, 1),)]), ("NEG", "POS")[i]))
    classes = {"NEG": 0, "POS": 1}
    for method in ("transformer_attribution", "rollout"):
        gen = gens[method]
        eng = te._generator_model(gen).engine()
        shapes = []
        fwd = eng.forward

        def record(x, m=None, flags=None):
            shapes.append(tuple(x.shape))
            return fwd(x, m, flags)
        for chunk in (None, 5):
            shapes.clear()
            eng.forward = record
            try:
                res = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=1, faithfulness=True, faith_chunk=chunk)
            finally:
                del eng.forward
            f = res["faithfulness"]
            # the one-word documents' rows: 3 tokens (sufficiency) and 2 ([CLS] [SEP], comprehensiveness); a chunk of
            # at most 5 rows leaves the short rows a chunk of their own
            assert any(s[1] == 3 for s in shapes) and (chunk is None or any(s[1] == 2 for s in shapes)), shapes
            worst = 0.0
            for i, (a, d) in enumerate(zip(anns, res["docids"])):
                single, _ = _single_rows(gen, enc, d, classes[a.classification], res["word_ranges"][i],
                                         f["n_select"][i], eng)
                for t, got in ((0, f["comp"][i]), (1, f["suff"][i])):
                    worst = max(worst, float(np.abs(got - single[:, t]).max()))
                    assert np.array_equal(got.argmax(-1), single[:, t].argmax(-1)) or \
                        np.abs(single[:, t, 0] - single[:, t, 1]).min() <= 2 * FWD_TOL
            print("MEASURED batching %s chunk %s: %.2e, %d forwards, real / padded tokens %d / %d" % (
                method, chunk, worst, len(shapes), f["real_tokens"], f["padded_tokens"]))
            assert worst <= FWD_TOL, (method, chunk, worst)


@pytest.mark.parametrize("flags", [0, 7475])
def test_bert_base_width_against_fp64(flags):
    """Conditioned BERT-base width (3 layers), documents of 300-510 pieces: every probability eraser_eval reports against
    the fp64 oracle forward of the same row."""
    from test_gpu_methods_tc import tol
    from test_gpu_bert import make_model
    from oracle import bert as obert, conditioned
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    from transformer_explainability_b200 import eraser as te
    params, heads = obert.init_params(seed=22, vocab=1000, max_pos=512, dim=768, depth=3, heads=12, inter=3072,
                                      rand_affine=True)
    params = conditioned.condition_bert(params, c_qkv=3.0)
    cfg = dict(hidden_size=768, num_hidden_layers=3, intermediate_size=3072, vocab_size=1000, max_position_embeddings=512)
    model = make_model(params, heads, **cfg)
    model.engine_flags = flags
    gen = functools.partial(Generator(model).generate_LRP, start_layer=2)
    g = np.random.default_rng(4)
    docs, enc, anns = {}, {}, []
    for i, n in enumerate([300, 510, 420, 512]):
        ids = [101] + [int(x) for x in g.integers(5, 1000, n - 2)] + [102]
        d = "d%d" % i
        docs[d] = " ".join("w%d" % t for t in ids[1:-1])
        enc[d] = (ids, ["[CLS]"] + ["w%d" % t for t in ids[1:-1]] + ["[SEP]"])
        s0 = int(g.integers(0, n - 40))
        anns.append(te.Annotation(d, "", frozenset([(te.Evidence("", d, s0, s0 + 30),)]), ("NEG", "POS")[i % 2]))
    classes = {"NEG": 0, "POS": 1}
    res = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=1, faithfulness=True)
    f = res["faithfulness"]
    p64 = {k: v.double().cpu() for k, v in params.items()}
    eng = model.engine()
    worst = 0.0
    for i, (a, d) in enumerate(zip(anns, res["docids"])):
        from transformer_explainability_b200 import ops
        ids = torch.tensor([enc[d][0]]).cuda()
        m = gen(input_ids=ids, attention_mask=torch.ones_like(ids), index=torch.tensor([classes[a.classification]]).cuda())
        red = ops.eraser_reduce_inputs(m.reshape(1, -1).float().contiguous(), ids, [ids.shape[1]], res["word_ranges"][i],
                                       [0, len(res["word_ranges"][i])], f["n_select"][i:i + 1])
        lens = red["lengths"][0].cpu().numpy()
        rows = [(None, enc[d][0], f["probs"][i])]
        for j in range(lens.shape[0]):
            for t, key in ((0, "comp"), (1, "suff")):
                rows.append((j, red["ids"][0, j, t, :lens[j, t]].cpu().tolist(), f[key][i, j]))
        for _, row, got in rows:
            x = torch.tensor([row])
            want = torch.softmax(obert.forward(p64, x, torch.ones_like(x), heads)[0], -1)[0].numpy()
            worst = max(worst, float(np.abs(got - want).max()))
    bound = FWD_TOL if flags == 0 else tol(flags)
    print("MEASURED BERT-base width flags %d: probabilities vs fp64 %.2e (bound %.0e), real / padded tokens %d / %d" % (
        flags, worst, bound, f["real_tokens"], f["padded_tokens"]))
    assert worst <= bound, (flags, worst)
    assert eng is model.engine()
