"""Import-path drop-in for ``BERT_explainability/modules/BERT/BERT.py``.

The reference builds its BERT encoder out of relprop-capable layer classes in this module (``BertModel`` ``:533``,
``BertSelfAttention`` ``:249``, ``BertLayer`` ``:490`` ...).  Here the encoder runs as one engine call
(``engine.BertEngine``), so these names are the parameter containers of the facade — same constructor argument
(``config``), same ``state_dict`` keys, same accessors on ``BertSelfAttention`` (``get_attn`` / ``get_attn_cam`` /
``get_attn_gradients``, ``:281-297``) — exported under the reference's names so that
``from BERT_explainability.modules.BERT.BERT import BertModel`` keeps resolving after ``install_aliases()``.
A ``BertModel`` on its own cannot run forward / relprop: the classifier head picks the class the gradient and the
relevance start from; use ``BertForSequenceClassification`` (what every caller of the reference does).
"""
import torch

from transformer_explainability_b200 import ops
from .BertForSequenceClassification import (_Attention, _BertModel, _Dense, _DenseLN, _Embeddings, _Encoder, _Layer,
                                            _SelfAttention)

BertEmbeddings = _Embeddings
BertEncoder = _Encoder
BertLayer = _Layer
BertAttention = _Attention
BertSelfAttention = _SelfAttention
BertSelfOutput = _DenseLN
BertOutput = _DenseLN
BertIntermediate = _Dense
BertPooler = _Dense


class BertModel(_BertModel):
    def __init__(self, config):
        super().__init__(config)
        self.config = config

    def forward(self, *args, **kwargs):
        raise NotImplementedError("the CUDA engine runs encoder + pooler + classifier as one call: wrap the weights in "
                                  "BertForSequenceClassification (BERT_explainability.modules.BERT."
                                  "BertForSequenceClassification) and call that")

    relprop = forward


def get_activation(activation_string):
    """``BERT.py:22-26``."""
    acts = {"gelu": torch.nn.functional.gelu, "relu": torch.nn.functional.relu, "tanh": torch.tanh}
    if activation_string not in acts:
        raise KeyError("function {} not found in ACT2FN mapping {}".format(activation_string, list(acts)))
    return acts[activation_string]


def compute_rollout_attention(all_layer_matrices, start_layer=0):
    """``BERT.py:28-39``: identity added, rows normalised, chained product — on the rollout kernels."""
    return ops.compute_rollout_attention(all_layer_matrices, start_layer=start_layer, normalize=True)
