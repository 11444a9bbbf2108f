"""GPU: sentence-pair BERT inputs (``token_type_ids``) on the engine, and the word-importance command.

- ``model(**encoding)`` logits and every layer's ``get_attn`` / ``get_attn_gradients`` against the unmodified reference's
  fixture ``tests/golden/bert_pairs.npz`` at the bounds of ``test_gpu_bert.py``.
- Every generator with ``token_type_ids``, for both rule libraries (``BertForSequenceClassification``, ``BERT_cls_lrp``),
  under ``engine_flags`` 0 and ``FLAG_BENCH_DEFAULT``, against the fixture's fp64 results (NaN pattern included).
- A batched ``explain`` of the padded pairs against per-sample calls; no token types, all-zero token types and the call
  without the argument bit for bit; an out-of-range type id: NaN logits from a device tensor, ``ValueError`` from a host one.
- Poisoned workspace and outputs give bit-identical results (the scheme of ``test_gpu_poison.py``).
- ``te_token_importance`` bit for bit against ``oracle/text_visualization.py``, argument checks before any launch.
- The command end to end on a tiny model directory, and its F + A + 2 launches per batch.
"""
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import bert as obert
from oracle import make_golden_bert_pairs as mgp
from oracle import text_visualization as otv
from transformer_explainability_b200 import _lib, engine, ops
from transformer_explainability_b200 import text_visualization as tv

pytestmark = pytest.mark.gpu

FLAGS = [0, _lib.FLAG_BENCH_DEFAULT]
LIBS = ("ours", "lrp")


def T(a):
    return torch.from_numpy(np.asarray(a))


def rel(a, b):
    b = torch.as_tensor(b).double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "bert_pairs.npz"))


def make_model(lib, flags=0):
    from transformers import BertConfig
    if lib == "ours":
        from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
            BertForSequenceClassification
    else:
        from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
            BertForSequenceClassification
    params, _ = obert.init_params(**mgp.PARAMS)
    m = BertForSequenceClassification(BertConfig(num_labels=2, **mgp.CFG))
    res = m.load_state_dict(params, strict=False)
    assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
    m.engine_flags = flags
    return m.cuda().eval()


def inputs(golden):
    return T(golden["ids"]).cuda(), T(golden["mask"]).cuda(), T(golden["token_type_ids"]).cuda()


def test_model_call_with_encoding_vs_reference(golden):
    model = make_model("ours")
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    gen = Generator(model)
    ids, mask, tt = inputs(golden)
    for s in range(ids.shape[0]):
        enc = {"input_ids": ids[s:s + 1], "attention_mask": mask[s:s + 1], "token_type_ids": tt[s:s + 1]}
        logits = model(**enc)[0]
        key = "ours.f64.s%d" % s
        assert rel(logits, golden[key + ".logits"]) < 1e-5, s
        assert int(logits.argmax()) == int(np.argmax(golden["ours.f32.s%d.logits" % s]))
        gen.generate_LRP(start_layer=0, **enc)
        for l, layer in enumerate(model.bert.encoder.layer):
            assert rel(layer.attention.self.get_attn(), golden["%s.attn.%d" % (key, l)]) < 1e-5, (s, l)
            assert rel(layer.attention.self.get_attn_gradients(), golden["%s.grad.%d" % (key, l)]) < 1e-4, (s, l)
    with pytest.raises(NotImplementedError):
        model(ids[:1], mask[:1], position_ids=torch.arange(ids.shape[1], device="cuda")[None])


TOL = {"LRP": 2e-2, "LRP_last_layer": 2e-2, "full_lrp": 2e-2, "attn_last_layer": 1e-5, "rollout": 1e-5,
       "attn_gradcam": 2e-3, "attn_grad_rollout": 2e-4}


def tol(which, flags):
    return TOL[which] if flags == 0 else max(TOL[which], 5e-3)


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("lib", LIBS)
def test_every_generator_with_token_types_vs_reference(golden, lib, flags):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model = make_model(lib, flags)
    gen = Generator(model)
    ids, mask, tt = inputs(golden)
    cases = [("LRP", "sl%d" % sl, dict(start_layer=sl)) for sl in (0, 1)]
    cases += [(w, vt, kw) for w in obert.GENERATORS for vt, kw in mgp.variants(w)]
    for s in range(ids.shape[0]):
        x, m, t = ids[s:s + 1], mask[s:s + 1], tt[s:s + 1]
        for which, vt, kw in cases:
            key = "%s.%%s.s%d.%s.%s" % (lib, s, which, vt)
            out = getattr(gen, "generate_" + which)(x, m, token_type_ids=t, **kw)
            ref32, ref = T(golden[key % "f32"]), T(golden[key % "f64"])
            assert out.shape == ref.shape == (1, mask.shape[1]), key
            if torch.isnan(ref32).any():
                if flags == 0:
                    assert torch.equal(torch.isnan(out.cpu()), torch.isnan(ref32)), key
                continue
            assert not torch.isnan(out).any(), key
            e = rel(out, ref)
            assert e < tol(which, flags), "%s flags %d: rel %g" % (key % "gpu", flags, e)
            if s == 1 and which == "LRP" and flags == 0:
                assert float(out[0, 19:].abs().max()) == 0.0, "padded tokens get exactly zero"
        if lib == "ours":
            for sl in (0, 1):
                out = gen.generate_attn_grad_rollout(x, m, start_layer=sl, token_type_ids=t)
                ref = golden["oracle.s%d.attn_grad_rollout.sl%d" % (s, sl)]
                assert rel(out, ref) < tol("attn_grad_rollout", flags), (s, sl, rel(out, ref))


@pytest.mark.parametrize("flags", FLAGS)
def test_batched_pairs_equal_per_sample(golden, flags):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model = make_model("ours", flags)
    gen = Generator(model)
    ids, mask, tt = inputs(golden)
    eng = model.engine()
    maps, idx, logits = eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=tt)
    for s in range(ids.shape[0]):
        one, i1, l1 = eng.explain(ids[s:s + 1], mask[s:s + 1], start_layer=0, return_logits=True,
                                  token_type_ids=tt[s:s + 1])
        assert int(i1[0]) == int(idx[s])
        assert torch.allclose(one[0], maps[s], rtol=1e-5, atol=1e-6 * float(maps[s].abs().max()))
        assert torch.allclose(l1[0], logits[s], rtol=1e-5, atol=1e-6)
    # chunked: token types are sliced with the ids
    chunked, cidx = eng.explain(ids, mask, start_layer=0, chunk=2, token_type_ids=tt)
    assert torch.equal(cidx, idx)
    assert torch.allclose(chunked[2], maps[2], rtol=1e-5, atol=1e-6 * float(maps[2].abs().max()))
    batched = gen.generate_LRP_batched(ids, mask, start_layer=0, token_type_ids=tt)
    assert torch.equal(batched, maps)


@pytest.mark.parametrize("flags", FLAGS)
def test_no_token_types_is_bit_identical_to_segment_zero(golden, flags):
    model = make_model("ours", flags)
    eng = model.engine()
    ids, mask, tt = inputs(golden)
    zeros = torch.zeros_like(tt)
    runs = [eng.explain(ids, mask, start_layer=0, return_logits=True),
            eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=None),
            eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=zeros),
            eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=zeros.cpu().to(torch.int32))]
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)
    assert torch.equal(model(ids, mask)[0], model(ids, mask, token_type_ids=zeros)[0])
    with_pairs = eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=tt)
    assert not torch.equal(with_pairs[2], runs[0][2]), "segment 1 must change the logits"


def test_out_of_range_token_types(golden):
    model = make_model("ours")
    eng = model.engine()
    ids, mask, tt = inputs(golden)
    bad = tt.clone()
    bad[1, 3] = 2
    bad[2, 0] = -1
    logits = eng.forward(ids, mask, token_type_ids=bad)
    torch.cuda.synchronize()
    assert torch.isnan(logits[1]).all() and torch.isnan(logits[2]).all() and not torch.isnan(logits[0]).any()
    for host in (bad.cpu(), tt.cpu() * 2):
        with pytest.raises(ValueError):
            eng.forward(ids, mask, token_type_ids=host)
        with pytest.raises(ValueError):
            eng.explain(ids, mask, start_layer=0, token_type_ids=host)
    with pytest.raises(ValueError):
        eng.explain(ids, mask, start_layer=0, token_type_ids=tt[:, :-1])


# ---- poisoned allocations (the scheme of test_gpu_poison.py) -----------------------------------------------------------------
GUARD = 2 << 20
PATTERNS = (0xFF, 0x5A)


class _PoisonTorch(types.SimpleNamespace):
    """``torch`` for the package modules, with ``empty`` / ``empty_like`` handing out a pattern-filled allocation followed by
    a guard of the same pattern."""
    def __init__(self, pattern):
        super().__init__(pattern=pattern, guards=[])

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *size, dtype=None, device=None, **kw):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        dtype = dtype or torch.get_default_dtype()
        dev = torch.device(device) if device is not None else torch.device("cpu")
        if dev.type != "cuda":
            return torch.empty(*size, dtype=dtype, device=device, **kw)
        n = int(np.prod(size)) if size else 1
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        raw = torch.full((nbytes + GUARD,), self.pattern, dtype=torch.uint8, device=dev)
        self.guards.append(raw[nbytes:])
        return raw[:nbytes].view(dtype).view(size)

    def empty_like(self, t, dtype=None, device=None, memory_format=None, **kw):
        return self.empty(tuple(t.shape), dtype=dtype or t.dtype, device=device or t.device)


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int64) if t.element_size() == 8 else t


@pytest.mark.parametrize("flags", FLAGS)
def test_poisoned_allocations_give_identical_results(golden, flags, monkeypatch):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model = make_model("ours", flags)
    gen = Generator(model)
    ids, mask, tt = inputs(golden)
    names = ["NEGATIVE", "POSITIVE"]

    def run():
        eng = model.engine()
        eng._ws, eng.derived = None, None
        eng._derived(eng.flags)
        maps, idx, logits = eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=tt)
        out = {"maps": maps, "idx": idx, "logits": logits}
        for l, layer in enumerate(model.bert.encoder.layer):
            out["attn%d" % l] = layer.attention.self.get_attn().clone()
            out["grad%d" % l] = layer.attention.self.get_attn_gradients().clone()
        out["full_lrp"] = gen.generate_full_lrp(ids, mask, token_type_ids=tt)
        scores, probs, explained, _ = tv.explain_batch(model, ids.cpu(), tt.cpu(), mask.cpu(), names)
        out["scores"], out["probs"], out["explained"] = T(scores), T(probs), T(explained)
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in out.items()}

    ref = run()
    assert torch.equal(_bits(run()["maps"]), _bits(ref["maps"])), "two normal runs differ"
    for pattern in PATTERNS:
        pt = _PoisonTorch(pattern)
        with monkeypatch.context() as mp:
            for mod in (engine, ops, tv):
                mp.setattr(mod, "torch", pt)
            got = run()
        for k in ref:
            assert torch.equal(_bits(got[k]), _bits(ref[k])), "%s differs under pattern 0x%02X" % (k, pattern)
        for g in pt.guards:
            assert bool((g == pattern).all()), "a guard was overwritten (pattern 0x%02X)" % pattern


# ---- te_token_importance -------------------------------------------------------------------------------------------------
def _oracle(maps, lengths, sign):
    return np.stack([otv.normalize(maps[b], int(lengths[b]), float(sign[b])) for b in range(maps.shape[0])])


def _same(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.int32), want[~nan].view(np.int32))


def test_token_importance_bit_identical_to_oracle():
    g = np.random.default_rng(5)
    for B, S in ((1, 1), (3, 17), (9, 128), (4, 700)):
        maps = (g.standard_normal((B, S)) * 10.0 ** g.integers(-9, 3, (B, 1))).astype(np.float32)
        lengths = g.integers(1, S + 1, B)
        lengths[0] = S
        sign = np.where(g.random(B) < 0.5, -1.0, 1.0).astype(np.float32)
        if B > 2:
            maps[1, :] = 0.25                                   # a constant row
            maps[2, int(lengths[2]) // 2] = np.nan              # a NaN row
            maps[0, S - 1] = np.inf                             # inf / inf: NaN at the maximum, 0 elsewhere
        maps_d = T(maps).cuda()
        got = ops.token_importance(maps_d, lengths.tolist(), sign.tolist())
        _same(got.cpu().numpy(), _oracle(maps, lengths, sign))
        # device lengths and sign, into a view of a larger buffer; the padding is never read
        poisoned = maps_d.clone()
        for b in range(B):
            poisoned[b, int(lengths[b]):] = float("nan")
        buf = torch.full((B * S + 7,), 3.0, device="cuda")
        out = ops.token_importance(poisoned, T(lengths.astype(np.int32)).cuda(), T(sign).cuda(), out=buf[:B * S].view(B, S))
        _same(out.cpu().numpy(), _oracle(maps, lengths, sign))
        assert (buf[B * S:] == 3.0).all()


def test_token_importance_rejects_bad_arguments_before_launching():
    lib = _lib.load()
    maps = torch.zeros(2, 4, device="cuda")
    lens = torch.full((2,), 4, dtype=torch.int32, device="cuda")
    sign = torch.ones(2, device="cuda")
    out = torch.empty_like(maps)
    p = _lib.ptr
    before = lib.te_kernel_launch_count()
    for args in ((None, p(lens), p(sign), 2, 4, p(out)), (p(maps), None, p(sign), 2, 4, p(out)),
                 (p(maps), p(lens), None, 2, 4, p(out)), (p(maps), p(lens), p(sign), 2, 4, None),
                 (p(maps), p(lens), p(sign), 0, 4, p(out)), (p(maps), p(lens), p(sign), 65536, 4, p(out)),
                 (p(maps), p(lens), p(sign), 2, 0, p(out)), (p(maps), p(lens), p(sign), -1, 4, p(out))):
        assert lib.te_token_importance(*args, None) == -1
    assert lib.te_kernel_launch_count() == before
    for bad in (dict(lengths=[0, 4]), dict(lengths=[4, 5]), dict(lengths=[4]), dict(sign=[1.0])):
        kw = dict(lengths=[4, 4], sign=[1.0, -1.0])
        kw.update(bad)
        with pytest.raises(ValueError):
            ops.token_importance(maps, **kw)
    with pytest.raises(ValueError):
        ops.token_importance(maps, [4, 4], torch.ones(2, device="cuda", dtype=torch.float64))
    assert lib.te_kernel_launch_count() == before


# ---- the command ---------------------------------------------------------------------------------------------------------
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + ["w%d" % i for i in range(90)] + ["##s", "a", "b", "c", "d", "."]


def save_model_dir(path, names=("NEGATIVE", "POSITIVE")):
    from safetensors.torch import save_file
    from transformers import BertConfig
    params, _ = obert.init_params(**mgp.PARAMS)
    cfg = BertConfig(num_labels=2, id2label={i: n for i, n in enumerate(names)}, label2id={n: i for i, n in enumerate(names)},
                     **mgp.CFG)
    os.makedirs(path, exist_ok=True)
    cfg.to_json_file(os.path.join(path, "config.json"))
    with open(os.path.join(path, "vocab.txt"), "w") as f:
        f.write("\n".join(VOCAB) + "\n")
    save_file({k: v.contiguous() for k, v in params.items()}, os.path.join(path, "model.safetensors"))
    return str(path)


TEXTS = ["a b w3 w7 .", "w10 w11 w12 w13 w14 w15 w16", "c d"]
PAIRS = ["c d w5", "a", "w20 w21 w22 w23 b"]


def _oracle_records(model_dir, texts, pairs, batch, labels, start_layer=0):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model = tv.load_model(model_dir)
    tok = tv.load_tokenizer(model_dir)
    gen = Generator(model)
    recs = []
    for s in range(0, len(texts), batch):
        tx, px = texts[s:s + batch], pairs[s:s + batch] if pairs else None
        ids, tt, mask = tv.tokenize(tok, tx, px)
        maps, idx = gen.generate_LRP_batched(ids.cuda(), mask.cuda(), start_layer=start_layer, return_index=True,
                                             token_type_ids=tt.cuda())
        probs = ops.class_probs(model(ids.cuda(), mask.cuda(), token_type_ids=tt.cuda())[0]).cpu().numpy()
        idx = idx.cpu().numpy()
        lens = mask.sum(1).numpy()
        scores = np.stack([otv.normalize(maps[b].cpu().numpy(), int(lens[b]), otv.sign_of(labels[idx[b]]))
                           for b in range(len(tx))])
        toks = [tok.convert_ids_to_tokens(ids[b, :lens[b]].tolist()) for b in range(len(tx))]
        r = otv.records(toks, [tt[b, :lens[b]].tolist() for b in range(len(tx))], scores, probs, labels, idx)
        for b, rec in enumerate(r):
            rec.update(text=tx[b], text_pair=px[b] if px else None)
        recs += r
    return recs


@pytest.mark.parametrize("pairs", [PAIRS, None])
def test_command_end_to_end(tmp_path, pairs):
    model_dir = save_model_dir(tmp_path / "model")
    out_dir = str(tmp_path / "out")
    argv = ["--model-dir", model_dir, "--output-dir", out_dir, "--batch-size", "2"]
    for i, t in enumerate(TEXTS):
        argv += ["--text", t] + (["--text-pair", pairs[i]] if pairs else [])
    tv.main(argv)
    got = json.load(open(os.path.join(out_dir, "word_importance.json")))
    want = _oracle_records(model_dir, TEXTS, pairs, 2, ["NEGATIVE", "POSITIVE"])
    assert got == json.loads(json.dumps(want))
    if pairs:
        assert all(1 in r["token_type_ids"] for r in got)
    page = open(os.path.join(out_dir, "word_importance.html")).read()
    assert page == otv.table(got)
    pos = 0
    for r in got:
        for t, a in zip(r["tokens"], r["scores"]):
            m = otv.mark(t, a)
            i = page.find(m, pos)
            assert i >= 0, (t, a)
            pos = i + len(m)
    # the explained class named NEGATIVE flips the sign
    for r in got:
        assert (max(r["scores"]) <= 0) if r["explained_label"] == "NEGATIVE" else (min(r["scores"]) >= 0)


def test_command_class_index_and_labels(tmp_path):
    model_dir = save_model_dir(tmp_path / "model", names=("LABEL_0", "LABEL_1"))
    out_dir = str(tmp_path / "out")
    for method in ("transformer_attribution", "attn_grad_rollout"):
        tv.main(["--model-dir", model_dir, "--output-dir", out_dir, "--text", TEXTS[0], "--text-pair", PAIRS[0],
                 "--class-index", "0", "--labels", "NEGATIVE", "POSITIVE", "--method", method])
        got = json.load(open(os.path.join(out_dir, "word_importance.json")))
        assert got[0]["explained_class"] == 0 and got[0]["explained_label"] == "NEGATIVE", method
        assert max(got[0]["scores"]) <= 0, method


def test_command_launches_per_batch(tmp_path):
    lib = _lib.load()
    model_dir = save_model_dir(tmp_path / "model")
    model = tv.load_model(model_dir)
    tok = tv.load_tokenizer(model_dir)
    ids, tt, mask = tv.tokenize(tok, TEXTS, PAIRS)
    eng = model.engine()
    c0 = lib.te_kernel_launch_count()
    eng.forward(ids.cuda(), mask.cuda(), token_type_ids=tt.cuda())
    c1 = lib.te_kernel_launch_count()
    eng.attribute(start_layer=0)
    c2 = lib.te_kernel_launch_count()
    f, a = c1 - c0, c2 - c1
    for method in ("transformer_attribution", "attn_grad_rollout"):
        before = lib.te_kernel_launch_count()
        tv.explain_batch(model, ids, tt, mask, ["NEGATIVE", "POSITIVE"], method=method)
        n = lib.te_kernel_launch_count() - before
        if method == "transformer_attribution":
            assert n == f + a + 2, (n, f, a)
        else:
            assert f + 2 < n < f + a + 2
