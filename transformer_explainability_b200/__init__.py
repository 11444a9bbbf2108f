"""transformer_explainability_b200 — transformer-attribution engine for the H100.

Drop-in for the ``transformer_attribution`` hot path of hila-chefer/Transformer-Explainability:
``LRP(model).generate_LRP`` / ``model.relprop`` / ``compute_rollout_attention`` /
``generate_visualization`` keep the reference API; the work is done by hand-written sm_90a CUDA
kernels behind the C ABI of ``include/te_b200.h``.  There is no CPU fallback.

``install_aliases()`` registers the reference's top-level module names (``modules.layers_ours``,
``baselines.ViT.ViT_LRP``, ``baselines.ViT.ViT_explanation_generator``, ``dataset.expl_hdf5``,
``BERT_explainability.modules.BERT.ExplanationGenerator`` ...) so that the reference's notebooks and
eval scripts import this engine unchanged.
"""
import importlib
import sys

__version__ = "0.1.0"

_ALIASES = {
    "modules": "transformer_explainability_b200.modules",
    "modules.layers_ours": "transformer_explainability_b200.modules.layers_ours",
    "modules.layers_lrp": "transformer_explainability_b200.modules.layers_lrp",
    "baselines": "transformer_explainability_b200.baselines",
    "baselines.ViT": "transformer_explainability_b200.baselines.ViT",
    "baselines.ViT.ViT_LRP": "transformer_explainability_b200.baselines.ViT.ViT_LRP",
    "baselines.ViT.ViT_new": "transformer_explainability_b200.baselines.ViT.ViT_new",
    "baselines.ViT.ViT_orig_LRP": "transformer_explainability_b200.baselines.ViT.ViT_orig_LRP",
    "baselines.ViT.ViT_explanation_generator": "transformer_explainability_b200.baselines.ViT.ViT_explanation_generator",
    "dataset": "transformer_explainability_b200.dataset",
    "dataset.expl_hdf5": "transformer_explainability_b200.dataset.expl_hdf5",
}


def install_aliases(extra=True):
    """Make ``from baselines.ViT.ViT_LRP import vit_base_patch16_224 as vit_LRP`` (example.ipynb) resolve here."""
    names = dict(_ALIASES)
    if extra:
        try:
            importlib.import_module("transformer_explainability_b200.BERT_explainability")
            names.update({
                "BERT_explainability": "transformer_explainability_b200.BERT_explainability",
                "BERT_explainability.modules": "transformer_explainability_b200.BERT_explainability.modules",
                "BERT_explainability.modules.layers_ours":
                    "transformer_explainability_b200.BERT_explainability.modules.layers_ours",
                "BERT_explainability.modules.BERT": "transformer_explainability_b200.BERT_explainability.modules.BERT",
                "BERT_explainability.modules.BERT.BERT": "transformer_explainability_b200.BERT_explainability.modules.BERT.BERT",
                "BERT_explainability.modules.BERT.ExplanationGenerator":
                    "transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator",
                "BERT_explainability.modules.BERT.BertForSequenceClassification":
                    "transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification",
            })
        except ImportError:
            pass
    for alias, target in names.items():
        sys.modules[alias] = importlib.import_module(target)


def library_path():
    from . import _lib
    return _lib.LIB_PATH
