"""CPU: a façade model is freed as soon as its last reference goes, without waiting for Python's cyclic garbage collector.

The model owns its engine (flat weights, derived tensor-core copies, activation workspace: ~12 GB for ViT-B/16 at batch 32),
so a reference cycle through the attention views' back-reference would hold that device memory until a collection happened
to run, and a test session or a service that builds several models in turn runs out of GPU memory."""
import copy
import gc
import pickle
import weakref

import pytest


def _vit_models():
    from transformer_explainability_b200.baselines.ViT import ViT_LRP, ViT_new, ViT_orig_LRP
    kw = dict(img_size=32, patch_size=8, embed_dim=64, depth=2, num_heads=4, num_classes=10)
    return [ViT_LRP.VisionTransformer(**kw), ViT_new.VisionTransformer(**kw), ViT_orig_LRP.VisionTransformer(**kw)]


def _bert_model():
    transformers = pytest.importorskip("transformers")
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    return BertForSequenceClassification(transformers.BertConfig(hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                                                                 intermediate_size=128, vocab_size=100,
                                                                 max_position_embeddings=32, num_labels=2))


def _views(m):
    if hasattr(m, "blocks"):
        return [blk.attn for blk in m.blocks]
    return [l.attention.self for l in m.bert.encoder.layer]


def test_models_are_freed_without_the_cyclic_collector():
    enabled = gc.isenabled()
    gc.disable()
    try:
        refs = []
        for m in _vit_models():
            refs.append(weakref.ref(m))
            del m
        m = _bert_model()
        refs.append(weakref.ref(m))
        del m
        assert all(r() is None for r in refs), "a façade model outlived its last reference (reference cycle)"
    finally:
        if enabled:
            gc.enable()


def test_attention_views_follow_copies_and_report_a_dropped_model():
    models = _vit_models() + [_bert_model()]
    while models:
        m = models.pop()
        for c in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
            assert all(v._owner() is c for v in _views(c))
        assert all(v._owner() is m for v in _views(m))
        view = _views(m)[0]
        del m, c
        with pytest.raises(RuntimeError, match="no longer exists"):
            view.get_attn()
