"""The DistilBERT sequence classifier on the CUDA engine (``transformers.DistilBertForSequenceClassification``).

Parameter container with the ``transformers`` ``state_dict`` keys: ``distilbert.embeddings.{word,position}_embeddings``
and ``LayerNorm`` (no token-type table), ``distilbert.transformer.layer.{i}.attention.{q,k,v,out}_lin.*``,
``sa_layer_norm``, ``ffn.lin1`` / ``ffn.lin2``, ``output_layer_norm``, and the head ``pre_classifier.*`` /
``classifier.*``.  The layer is BERT's post-LN layer under other names; the engine runs it as
``te_bert_config.arch = TE_BERT_ARCH_DISTILBERT``: embeddings ``word + position`` with ``arange`` positions, LayerNorm
eps 1e-12, head ``classifier(relu(pre_classifier(h[:, 0])))``.  The relevance rules take ReLU as the identity, as they
take BERT's tanh, so every generator carries over.  ``engine_flags |= FLAG_RULES_LRP`` selects the layers_lrp rules.
"""
import torch.nn as nn

from transformer_explainability_b200 import _lib
from transformer_explainability_b200.engine import bert_config
from .BertForSequenceClassification import _AttentionView, _EngineClassifier

EPS = 1e-12                                   # DistilBERT's LayerNorms use a fixed eps


class MultiHeadSelfAttention(_AttentionView, nn.Module):
    def __init__(self, d):
        super().__init__()
        self.q_lin = nn.Linear(d, d)
        self.k_lin = nn.Linear(d, d)
        self.v_lin = nn.Linear(d, d)
        self.out_lin = nn.Linear(d, d)
        self._owner = None
        self._layer = -1


class _FFN(nn.Module):
    def __init__(self, d, f):
        super().__init__()
        self.lin1 = nn.Linear(d, f)
        self.lin2 = nn.Linear(f, d)


class TransformerBlock(nn.Module):
    def __init__(self, d, f):
        super().__init__()
        self.attention = MultiHeadSelfAttention(d)
        self.sa_layer_norm = nn.LayerNorm(d, eps=EPS)
        self.ffn = _FFN(d, f)
        self.output_layer_norm = nn.LayerNorm(d, eps=EPS)


class _Transformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.layer = nn.ModuleList([TransformerBlock(cfg.dim, cfg.hidden_dim) for _ in range(cfg.n_layers)])


class _Embeddings(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.word_embeddings = nn.Embedding(cfg.vocab_size, cfg.dim)
        self.position_embeddings = nn.Embedding(cfg.max_position_embeddings, cfg.dim)
        self.LayerNorm = nn.LayerNorm(cfg.dim, eps=EPS)


class _DistilBertModel(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = _Embeddings(cfg)
        self.transformer = _Transformer(cfg)


class DistilBertForSequenceClassification(_EngineClassifier):
    def __init__(self, config):
        super().__init__()
        if getattr(config, "activation", "gelu") != "gelu":
            raise NotImplementedError("only activation='gelu' (the DistilBertConfig default) is implemented")
        self.distilbert = _DistilBertModel(config)
        self.pre_classifier = nn.Linear(config.dim, config.dim)
        self.classifier = nn.Linear(config.dim, config.num_labels)
        self._setup(config, bert_config(config.vocab_size, config.max_position_embeddings, 0, config.dim,
                                        config.n_layers, config.n_heads, config.hidden_dim, config.num_labels, EPS,
                                        arch=_lib.BERT_ARCH_DISTILBERT))

    def attention_views(self):
        return [l.attention for l in self.distilbert.transformer.layer]

    def forward(self, input_ids=None, attention_mask=None, head_mask=None, inputs_embeds=None, labels=None,
                output_attentions=None, output_hidden_states=None, return_dict=None, token_type_ids=None,
                position_ids=None):
        """``DistilBertForSequenceClassification.forward`` with return_dict=False: returns ``(logits,)``.  The model has
        no token-type table: ``token_type_ids`` other than None raises ``ValueError``."""
        if position_ids is not None or head_mask is not None or inputs_embeds is not None:
            raise NotImplementedError("position_ids, head_mask and inputs_embeds are not used on the attribution path")
        return (self.engine().forward(input_ids, attention_mask, token_type_ids=token_type_ids),)
