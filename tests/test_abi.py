"""CPU: the C-ABI library loads and exports exactly what include/te_b200.h declares; host-side tables agree."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "te_b200.h")).read()
    return sorted(set(re.findall(r"TE_API[^;(]*?\b(te_\w+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from transformer_explainability_b200 import _lib
    lib = _lib.load()
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), "library does not export %s" % s
    assert set(syms) == set(_lib.PROTOTYPES), "ctypes prototypes out of sync with the header"
    assert lib.te_version() >= 100


def test_weight_table_matches_facade_state_dict():
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import VisionTransformer
    lib = _lib.load()
    for distilled in (False, True):
        m = VisionTransformer(img_size=32, patch_size=8, embed_dim=64, depth=2, num_heads=4, num_classes=10,
                              qkv_bias=True, distilled=distilled)
        cfg = m._cfg
        n = lib.te_vit_num_weights(ctypes.byref(cfg))
        sd = m.state_dict()
        seen, end = set(), 0
        for i in range(n):
            name = lib.te_vit_weight_name(ctypes.byref(cfg), i).decode()
            numel = lib.te_vit_weight_numel(ctypes.byref(cfg), i)
            off = lib.te_vit_weight_offset(ctypes.byref(cfg), i)
            assert sd[name].numel() == numel
            assert off % 32 == 0 and off >= end
            end = off + numel
            seen.add(name)
        assert seen == set(sd.keys())
        assert lib.te_vit_weight_total(ctypes.byref(cfg)) >= end


def test_workspace_query_and_errors_without_gpu():
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.engine import vit_config
    lib = _lib.load()
    cfg = vit_config()
    b1 = lib.te_vit_workspace_bytes(ctypes.byref(cfg), 1)
    b2 = lib.te_vit_workspace_bytes(ctypes.byref(cfg), 2)
    assert 0 < b1 < b2 and b1 % 256 == 0
    assert lib.te_vit_workspace_bytes(ctypes.byref(cfg), 0) < 0
    bad = vit_config(embed_dim=770)
    assert lib.te_vit_workspace_bytes(ctypes.byref(bad), 1) < 0
    assert b"invalid" in lib.te_last_error()
    assert lib.te_rollout_workspace_bytes(12, 2, 197) > 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the loud failure on a GPU-less host")
def test_no_cpu_fallback():
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import VisionTransformer
    from transformer_explainability_b200 import ops
    m = VisionTransformer(img_size=32, patch_size=8, embed_dim=64, depth=1, num_heads=4, num_classes=10)
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 32, 32))
    with pytest.raises(ValueError):
        ops.linear_relprop(torch.zeros(2, 4), torch.zeros(3, 4), torch.zeros(2, 3))


def test_reference_import_paths_resolve():
    import transformer_explainability_b200 as te
    te.install_aliases()
    from baselines.ViT.ViT_LRP import vit_base_patch16_224, compute_rollout_attention   # noqa: F401
    from baselines.ViT.ViT_explanation_generator import LRP                             # noqa: F401
    from modules.layers_ours import Linear, Add, Clone, einsum, IndexSelect, safe_divide  # noqa: F401
    import inspect
    sig = inspect.signature(LRP.generate_LRP)
    assert list(sig.parameters) == ["self", "input", "index", "method", "is_ablation", "start_layer"]


def test_bert_weight_table_matches_facade_state_dict():
    transformers = pytest.importorskip("transformers")
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    lib = _lib.load()
    m = BertForSequenceClassification(transformers.BertConfig(hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                                                              intermediate_size=128, vocab_size=100,
                                                              max_position_embeddings=32, num_labels=2))
    cfg = m._cfg
    sd = m.state_dict()
    n = lib.te_bert_num_weights(ctypes.byref(cfg))
    seen, end = set(), 0
    for i in range(n):
        name = lib.te_bert_weight_name(ctypes.byref(cfg), i).decode()
        numel = lib.te_bert_weight_numel(ctypes.byref(cfg), i)
        off = lib.te_bert_weight_offset(ctypes.byref(cfg), i)
        assert sd[name].numel() == numel, name
        assert off % 32 == 0 and off >= end
        end = off + numel
        seen.add(name)
    assert seen == {k for k in sd if "position_ids" not in k}
    assert lib.te_bert_weight_total(ctypes.byref(cfg)) >= end


def test_host_only_queries_and_option_errors():
    """Entry points that need no device: workspace sizes grow with the batch, bad arguments and unknown options are
    reported through the status code + te_last_error (never an exception, never a crash)."""
    from transformer_explainability_b200 import _lib
    lib = _lib.load()
    assert lib.te_rollout_workspace_bytes(12, 2, 197) < lib.te_rollout_workspace_bytes(12, 4, 197)
    assert lib.te_rollout_workspace_bytes(0, 2, 197) < 0
    a = lib.te_patch_embed_relprop_workspace_bytes(1, 3, 224, 16, 768)
    b = lib.te_patch_embed_relprop_workspace_bytes(2, 3, 224, 16, 768)
    assert 0 < a < b
    assert lib.te_patch_embed_relprop_workspace_bytes(1, 3, 225, 16, 768) < 0          # patch does not divide the image
    assert lib.te_set_option(b"no_such_option", 1) < 0
    assert b"unknown option" in lib.te_last_error()
    assert lib.te_set_option(b"cls_row_top_block", 1) == 0 and lib.te_set_option(b"gelu_split_fused", 1) == 0


def test_baseline_and_generator_surfaces_resolve():
    """The comparison classes keep the reference's names and signatures (ViT_explanation_generator.py:45-83,
    ExplanationGenerator.py:61-155)."""
    import inspect
    import transformer_explainability_b200 as te
    te.install_aliases()
    from baselines.ViT.ViT_new import vit_base_patch16_224                              # noqa: F401
    from baselines.ViT.ViT_explanation_generator import Baselines
    from BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    from BERT_explainability.modules.BERT.BERT import BertModel, BertSelfAttention, BertLayer, compute_rollout_attention  # noqa: F401
    assert all(hasattr(BertSelfAttention, a) for a in ("get_attn", "get_attn_cam", "get_attn_gradients"))      # BERT.py:281-297
    assert list(inspect.signature(Baselines.generate_cam_attn).parameters) == ["self", "input", "index"]
    assert list(inspect.signature(Baselines.generate_rollout).parameters) == ["self", "input", "start_layer"]
    for name in ("generate_LRP", "generate_LRP_last_layer", "generate_full_lrp", "generate_attn_last_layer",
                 "generate_rollout", "generate_attn_gradcam"):
        params = list(inspect.signature(getattr(Generator, name)).parameters)
        assert params[:3] == ["self", "input_ids", "attention_mask"], name


def test_flag_constants_match_the_header():
    """Every TE_FLAG_* of include/te_b200.h has the same value in the Python binding, and the bench default is a union of them."""
    from transformer_explainability_b200 import _lib
    src = open(os.path.join(ROOT, "include", "te_b200.h")).read()
    flags = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+TE_FLAG_(\w+)\s+(\d+)u", src)}
    assert len(flags) >= 12
    for name, value in flags.items():
        assert getattr(_lib, "FLAG_" + name) == value, "FLAG_%s differs from the header" % name
        assert value & (value - 1) == 0, "TE_FLAG_%s is not a single bit" % name
    assert len(set(flags.values())) == len(flags), "two flags share a bit"
    known = 0
    for v in flags.values():
        known |= v
    assert _lib.FLAG_BENCH_DEFAULT & ~known == 0
    assert _lib.FLAG_BENCH_DEFAULT == 7475           # what DESIGN.md documents as the benched selection
