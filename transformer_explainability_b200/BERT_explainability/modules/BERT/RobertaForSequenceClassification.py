"""The RoBERTa / XLM-RoBERTa sequence classifier on the CUDA engine (``transformers.RobertaForSequenceClassification``,
``XLMRobertaForSequenceClassification``).

Parameter container with the ``transformers`` ``state_dict`` keys: ``roberta.embeddings.*``, ``roberta.encoder.layer.{i}.*``
(the BERT layer's names), no pooler, and the head ``classifier.dense.*`` / ``classifier.out_proj.*``.  The engine runs
it as ``te_bert_config.arch = TE_BERT_ARCH_ROBERTA``: position ids ``pad + cumsum(ids != pad)`` for non-pad tokens and
``pad`` for pad tokens, embeddings ``(word + type) + position``, head ``out_proj(tanh(dense(h[:, 0])))``.  The usable
length is ``max_position_embeddings - pad_token_id - 1`` (512 tokens for roberta-base).  Relevance rules, generators and
views are those of ``BertForSequenceClassification``; ``engine_flags |= FLAG_RULES_LRP`` selects the layers_lrp rules.
The attention mask is BERT's additive ``(1 - mask) * -10000``: padded keys get zero probability either way.
"""
import torch.nn as nn

from transformer_explainability_b200 import _lib
from transformer_explainability_b200.engine import bert_config
from .BertForSequenceClassification import _EngineClassifier, _Embeddings, _Encoder


class _RobertaModel(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = _Embeddings(cfg, position_ids=False)
        self.encoder = _Encoder(cfg)


class _ClassificationHead(nn.Module):
    """``RobertaClassificationHead``: dense -> tanh -> out_proj on the first token."""

    def __init__(self, d, c):
        super().__init__()
        self.dense = nn.Linear(d, d)
        self.out_proj = nn.Linear(d, c)


class RobertaForSequenceClassification(_EngineClassifier):
    def __init__(self, config):
        super().__init__()
        if getattr(config, "hidden_act", "gelu") != "gelu":
            raise NotImplementedError("only hidden_act='gelu' (the RobertaConfig default) is implemented")
        self.roberta = _RobertaModel(config)
        self.classifier = _ClassificationHead(config.hidden_size, config.num_labels)
        self._setup(config, bert_config(config.vocab_size, config.max_position_embeddings, config.type_vocab_size,
                                        config.hidden_size, config.num_hidden_layers, config.num_attention_heads,
                                        config.intermediate_size, config.num_labels, config.layer_norm_eps,
                                        arch=_lib.BERT_ARCH_ROBERTA, pad_token_id=config.pad_token_id))

    def attention_views(self):
        return [l.attention.self for l in self.roberta.encoder.layer]

    def _head_weight(self):
        return self.classifier.out_proj.weight

    def forward(self, input_ids=None, attention_mask=None, token_type_ids=None, position_ids=None, head_mask=None,
                inputs_embeds=None, labels=None, output_attentions=None, output_hidden_states=None, return_dict=None):
        """``RobertaForSequenceClassification.forward`` with return_dict=False: returns ``(logits,)``.  The position ids
        are computed from ``input_ids`` on the device; ``token_type_ids`` None is segment 0."""
        if position_ids is not None or head_mask is not None or inputs_embeds is not None:
            raise NotImplementedError("position_ids, head_mask and inputs_embeds are not used on the attribution path")
        return (self.engine().forward(input_ids, attention_mask, token_type_ids=token_type_ids),)


XLMRobertaForSequenceClassification = RobertaForSequenceClassification
