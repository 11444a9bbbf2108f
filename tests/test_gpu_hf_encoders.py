"""GPU: RoBERTa / XLM-RoBERTa and DistilBERT sequence classifiers on the engine.

- Logits, ``get_attn`` and ``get_attn_gradients`` of a right-padded, a left-padded and a pair row against
  ``transformers`` in fp64 (``tests/golden/hf_encoders.npz``) at ``test_gpu_bert.py``'s bounds, under engine flags 0 and
  ``FLAG_BENCH_DEFAULT``.
- All seven ``Generator`` methods for both rule libraries against the fp64 oracle's maps (``oracle/hf_encoders.py``).
- One full-width case per family (hidden 768, 12 heads, intermediate 3072, 2 layers, S = 128) against the fp64 oracle
  under ``FLAG_BENCH_DEFAULT``: the tiny widths run SIMT, this one reaches the tensor cores.
- Padded rows in a batch equal per-sample calls; RoBERTa's usable length; the forward launch count equals BERT's;
  poisoned workspace and outputs give bit-identical results; the word-importance command end to end on tiny local
  RoBERTa and DistilBERT directories, with F + A + 2 launches per batch.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import bert as obert
from oracle import hf_encoders as ohf
from oracle import make_golden_hf_encoders as mg
from transformer_explainability_b200 import _lib
from transformer_explainability_b200 import text_visualization as tv
from transformer_explainability_b200.BERT_explainability.modules.BERT.DistilBertForSequenceClassification import \
    DistilBertForSequenceClassification
from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
from transformer_explainability_b200.BERT_explainability.modules.BERT.RobertaForSequenceClassification import \
    RobertaForSequenceClassification

pytestmark = pytest.mark.gpu

FAMILIES = tuple(mg.FAMILIES)
FLAGS = [0, _lib.FLAG_BENCH_DEFAULT]
TOL = {"LRP": 2e-2, "LRP_last_layer": 2e-2, "full_lrp": 2e-2, "attn_last_layer": 1e-5, "rollout": 1e-5,
       "attn_gradcam": 2e-3, "attn_grad_rollout": 2e-4}


def tol(which, flags):
    return TOL[which] if flags == 0 else max(TOL[which], 5e-3)


def T(a):
    return torch.from_numpy(np.asarray(a))


def rel(a, b):
    b = torch.as_tensor(b).double().cpu()
    return ((torch.as_tensor(a).double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "hf_encoders.npz"))


def facade(name, config):
    return (RobertaForSequenceClassification if name == "roberta" else DistilBertForSequenceClassification)(config)


def make_model(name, lib="ours", flags=0, config=None, params=None):
    m = facade(name, config or mg.hf_config(name))
    res = m.load_state_dict(params if params is not None else mg.params(name), strict=False)
    assert not res.unexpected_keys and not res.missing_keys
    m.engine_flags = flags | (_lib.FLAG_RULES_LRP if lib == "lrp" else 0)
    return m.cuda().eval()


def inputs(golden, name):
    tt = T(golden[name + ".token_type_ids"]).cuda() if name == "roberta" else None
    return T(golden[name + ".ids"]).cuda(), T(golden[name + ".mask"]).cuda(), tt


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("name", FAMILIES)
def test_forward_and_gradients_vs_transformers(golden, name, flags):
    model = make_model(name, flags=flags)
    gen = Generator(model)
    ids, mask, tt = inputs(golden, name)
    kw = {"token_type_ids": tt} if tt is not None else {}
    logits = model(ids, mask, **kw)[0]
    assert rel(logits, golden[name + ".hf.logits"]) < 1e-5
    assert torch.equal(logits.argmax(-1).cpu(), T(golden[name + ".hf.logits"]).argmax(-1))
    gen.generate_LRP(ids, mask, start_layer=0, **kw)
    for l, v in enumerate(model.attention_views()):
        assert rel(v.get_attn(), golden["%s.hf.attn.%d" % (name, l)]) < 1e-5, l
        assert rel(v.get_attn_gradients(), golden["%s.hf.grad.%d" % (name, l)]) < 1e-4, l


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("lib", ["ours", "lrp"])
@pytest.mark.parametrize("name", FAMILIES)
def test_every_generator_vs_oracle(golden, name, lib, flags):
    model = make_model(name, lib, flags)
    gen = Generator(model)
    ids, mask, tt = inputs(golden, name)
    cases = [("LRP", "LRP.sl%d" % sl, dict(start_layer=sl)) for sl in (0, 1)]
    cases += [(w, w, {}) for w in obert.GENERATORS] + [("attn_grad_rollout", "attn_grad_rollout", {})]
    for which, key, kw in cases:
        # the rule libraries differ in relprop only: the other generators read the "ours" entries
        src = lib if which in ("LRP", "LRP_last_layer", "full_lrp") else "ours"
        ref = T(golden["%s.%s.%s" % (name, src, key)])
        out = getattr(gen, "generate_" + which)(ids, mask, token_type_ids=tt, **kw)
        assert out.shape == ref.shape, key
        nan = torch.isnan(ref).any(dim=1)
        if flags == 0:
            assert torch.equal(torch.isnan(out.cpu()).any(dim=1), nan), key
        ok = ~nan
        e = rel(out.cpu()[ok], ref[ok])
        assert e < tol(which, flags), "%s %s %s flags %d: rel %g" % (name, lib, key, flags, e)
        if which in ("LRP", "attn_grad_rollout", "rollout", "attn_last_layer"):
            pad = (mask == 0).cpu()
            pad[:, 0] = False
            assert float(out.cpu()[pad].abs().max()) == 0.0, "padded tokens get exactly zero"


def _full_width(name):
    import transformers
    w = dict(vocab_size=1000, max_position_embeddings=160, num_labels=3)
    if name == "roberta":
        cfg = transformers.RobertaConfig(hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                                         intermediate_size=3072, type_vocab_size=1, pad_token_id=1, layer_norm_eps=1e-5, **w)
    else:
        cfg = transformers.DistilBertConfig(dim=768, n_layers=2, n_heads=12, hidden_dim=3072, pad_token_id=0, **w)
    f = mg.FAMILIES[name]
    params = ohf.init_params(f["arch"], seed=5, vocab=1000, max_pos=160, types=1 if name == "roberta" else 0, dim=768,
                             depth=2, inter=3072, labels=3)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(5, 1000, (2, 128), generator=g)
    ids[:, 0] = 3
    mask = torch.ones_like(ids)
    mask[1, 100:] = 0
    ids[1, 100:] = f["pad"]
    return cfg, params, ids, mask, f


@pytest.mark.parametrize("name", FAMILIES)
def test_full_width_vs_fp64(name):
    cfg, params, ids, mask, f = _full_width(name)
    model = make_model(name, flags=_lib.FLAG_BENCH_DEFAULT, config=cfg, params=params)
    gen = Generator(model)
    p64 = ohf.to_bert_keys(params, f["arch"])
    kw = dict(arch=f["arch"], pad=f["pad"], eps=f["eps"])
    logits = model(ids.cuda(), mask.cuda())[0]
    want_logits, _ = ohf.forward(p64, ids, mask, 12, **kw)
    assert rel(logits, want_logits) < 1e-3
    maps = gen.generate_LRP(ids.cuda(), mask.cuda(), start_layer=0)
    want, idx = ohf.explain(p64, ids, mask, 12, start_layer=0, **kw)
    assert torch.equal(model.engine().explain(ids.cuda(), mask.cuda(), start_layer=0)[1].cpu().long(), idx)
    assert rel(maps, want) < 2e-2, rel(maps, want)
    agr = gen.generate_attn_grad_rollout(ids.cuda(), mask.cuda())
    assert rel(agr, ohf.explain_attn_grad_rollout(p64, ids, mask, 12, **kw)[0]) < 5e-3
    assert float(maps[1, 100:].abs().max()) == 0.0


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("name", FAMILIES)
def test_batched_equals_per_sample(golden, name, flags):
    model = make_model(name, flags=flags)
    eng = model.engine()
    ids, mask, tt = inputs(golden, name)
    maps, idx, logits = eng.explain(ids, mask, start_layer=0, return_logits=True, token_type_ids=tt)
    for s in range(ids.shape[0]):
        one, i1, l1 = eng.explain(ids[s:s + 1], mask[s:s + 1], start_layer=0, return_logits=True,
                                  token_type_ids=tt[s:s + 1] if tt is not None else None)
        assert int(i1) == int(idx[s])
        assert rel(one[0], maps[s]) < 1e-5 and rel(l1[0], logits[s]) < 1e-5, s


def test_roberta_length_limit():
    """S = max_position - pad - 1 runs; one more token is refused before any launch."""
    model = make_model("roberta")
    S = model.max_length()
    assert S == 32 - 1 - 1
    ids = torch.randint(5, 100, (1, S + 1), device="cuda")
    logits = model(ids[:, :S], torch.ones_like(ids[:, :S]))[0]
    assert torch.isfinite(logits).all()
    lib = _lib.load()
    before = lib.te_kernel_launch_count()
    with pytest.raises(_lib.TeError, match="seq \\+ pad_token_id \\+ 1"):
        model(ids, torch.ones_like(ids))
    assert lib.te_kernel_launch_count() == before


def test_distilbert_refuses_token_types(golden):
    model = make_model("distilbert")
    ids, mask, _ = inputs(golden, "distilbert")
    with pytest.raises(ValueError, match="token_type_ids"):
        model(ids, mask, token_type_ids=torch.zeros_like(ids))


@pytest.mark.parametrize("name", FAMILIES)
def test_forward_launch_count_equals_bert(golden, name):
    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    lib = _lib.load()
    ids, mask, tt = inputs(golden, name)
    bert = BertForSequenceClassification(BertConfig(hidden_size=64, num_hidden_layers=3, num_attention_heads=4,
                                                    intermediate_size=128, vocab_size=100, max_position_embeddings=32,
                                                    num_labels=2)).cuda().eval()
    model = make_model(name)
    counts = []
    for m in (bert, model):
        for flags in FLAGS:
            m.engine_flags = flags
            m(ids, mask)
            c0 = lib.te_kernel_launch_count()
            m(ids, mask)
            counts.append(lib.te_kernel_launch_count() - c0)
    assert counts[:2] == counts[2:], counts


@pytest.mark.parametrize("name", FAMILIES)
def test_poisoned_workspace_and_outputs_bit_identical(golden, name):
    model = make_model(name, flags=_lib.FLAG_BENCH_DEFAULT)
    eng = model.engine()
    lib = _lib.load()
    ids, mask, tt = inputs(golden, name)
    B, S = ids.shape
    ws = eng._workspace(B, S)
    derived = eng._derived(eng.flags)
    results = []
    for pattern in (0x00, 0xFF, 0x7F, 0xA5):
        ws.view(torch.uint8).fill_(pattern)
        maps = torch.empty(B, S, device="cuda")
        logits = torch.empty(B, 2, device="cuda")
        maps.view(torch.uint8).fill_(pattern)
        logits.view(torch.uint8).fill_(pattern)
        idx = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        _lib.check(lib.te_bert_explain(ctypes.byref(eng.cfg), _lib.ptr(eng.weights), _lib.ptr(derived), _lib.ptr(ids),
                                       _lib.ptr(mask), _lib.ptr(tt) if tt is not None else None, B, S, _lib.ptr(idx), 0,
                                       eng.flags, _lib.ptr(maps), _lib.ptr(logits), _lib.ptr(ws), ws.numel() * 4,
                                       eng._stream()), "te_bert_explain")
        torch.cuda.synchronize()
        results.append((maps.cpu(), logits.cpu(), idx.cpu()))
    for r in results[1:]:
        for a, b in zip(results[0], r):
            assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a,
                               b.view(torch.uint8) if b.is_floating_point() else b)


# ---- the command on local RoBERTa / DistilBERT directories (tokenizers built offline) ------------------------------------
WORDS = ["a", "b", "c", "d", "movie", "good", "bad", "the", "."] + ["w%d" % i for i in range(20)]
TEXTS = ["a movie good .", "w3 w4 w5 w6 w7 w8", "the bad"]
PAIRS = ["the bad", "c", "w10 w11 d"]


def _roberta_tokenizer_files(path):
    vocab = {"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3, "<mask>": 4}
    for c in sorted(set("".join(WORDS)) | {"Ġ"}):
        vocab.setdefault(c, len(vocab))
    merges = []
    for w in WORDS:
        for cur in (list(w), ["Ġ"] + list(w)):
            while len(cur) > 1:
                if (cur[0], cur[1]) not in merges:
                    merges.append((cur[0], cur[1]))
                cur = [cur[0] + cur[1]] + cur[2:]
                vocab.setdefault(cur[0], len(vocab))
    with open(os.path.join(path, "vocab.json"), "w") as f:
        json.dump(vocab, f)
    with open(os.path.join(path, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n" + "".join("%s %s\n" % m for m in merges))
    return len(vocab)


def save_model_dir(path, name):
    import transformers
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    names = {0: "NEGATIVE", 1: "POSITIVE"}
    f = mg.FAMILIES[name]
    if name == "roberta":
        n = _roberta_tokenizer_files(path)
        cfg = transformers.RobertaConfig(vocab_size=n, max_position_embeddings=40, type_vocab_size=1, hidden_size=64,
                                         num_hidden_layers=3, num_attention_heads=4, intermediate_size=128,
                                         pad_token_id=1, bos_token_id=0, eos_token_id=2, id2label=names)
    else:
        vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
        with open(os.path.join(path, "vocab.txt"), "w") as fh:
            fh.write("\n".join(vocab) + "\n")
        n = len(vocab)
        cfg = transformers.DistilBertConfig(vocab_size=n, max_position_embeddings=40, dim=64, n_layers=3, n_heads=4,
                                            hidden_dim=128, pad_token_id=0, id2label=names)
    cfg.to_json_file(os.path.join(path, "config.json"))
    params = ohf.init_params(f["arch"], seed=3, vocab=n, max_pos=40, types=1 if name == "roberta" else 0, dim=64,
                             depth=3, inter=128, labels=2)
    save_file({k: v.float().contiguous() for k, v in params.items()}, os.path.join(path, "model.safetensors"))
    return str(path)


@pytest.mark.parametrize("pairs", [None, PAIRS])
@pytest.mark.parametrize("name", FAMILIES)
def test_command_end_to_end(tmp_path, name, pairs):
    model_dir = save_model_dir(tmp_path / "model", name)
    out_dir = str(tmp_path / "out")
    argv = ["--model-dir", model_dir, "--output-dir", out_dir, "--batch-size", "2"]
    for i, t in enumerate(TEXTS):
        argv += ["--text", t] + (["--text-pair", pairs[i]] if pairs else [])
    tv.main(argv)
    got = json.load(open(os.path.join(out_dir, "word_importance.json")))
    assert os.path.exists(os.path.join(out_dir, "word_importance.html"))
    model = tv.load_model(model_dir)
    assert type(model).__name__ == {"roberta": "RobertaForSequenceClassification",
                                    "distilbert": "DistilBertForSequenceClassification"}[name]
    tok = tv.load_tokenizer(model_dir)
    gen = Generator(model)
    for s in range(0, len(TEXTS), 2):
        tx, px = TEXTS[s:s + 2], pairs[s:s + 2] if pairs else None
        ids, tt, mask = tv.tokenize(tok, tx, px, model.max_length())
        kw = {"token_type_ids": tt.cuda()} if name == "roberta" else {}
        maps, idx = gen.generate_LRP_batched(ids.cuda(), mask.cuda(), start_layer=0, return_index=True, **kw)
        for b in range(len(tx)):
            r = got[s + b]
            n = int(mask[b].sum())
            assert r["tokens"] == tok.convert_ids_to_tokens(ids[b, :n].tolist())
            assert set(r) >= {"text", "text_pair", "tokens", "token_type_ids", "scores", "predicted_class",
                              "explained_class", "explained_label", "predicted_probability"}
            m = maps[b, :n].double().cpu()
            want = (m - m.min()) / (m.max() - m.min()) * (-1 if r["explained_label"] == "NEGATIVE" else 1)
            assert int(idx[b]) == r["explained_class"]
            assert np.allclose(r["scores"], want.numpy(), atol=1e-6)


@pytest.mark.parametrize("name", FAMILIES)
def test_command_launches_per_batch(tmp_path, name):
    lib = _lib.load()
    model_dir = save_model_dir(tmp_path / "model", name)
    model = tv.load_model(model_dir)
    tok = tv.load_tokenizer(model_dir)
    ids, tt, mask = tv.tokenize(tok, TEXTS, PAIRS, model.max_length())
    eng = model.engine()
    kw = {"token_type_ids": tt.cuda()} if name == "roberta" else {}
    c0 = lib.te_kernel_launch_count()
    eng.forward(ids.cuda(), mask.cuda(), **kw)
    c1 = lib.te_kernel_launch_count()
    eng.attribute(start_layer=0)
    c2 = lib.te_kernel_launch_count()
    before = lib.te_kernel_launch_count()
    tv.explain_batch(model, ids, tt, mask, ["NEGATIVE", "POSITIVE"])
    assert lib.te_kernel_launch_count() - before == (c1 - c0) + (c2 - c1) + 2
