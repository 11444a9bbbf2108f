"""Drop-in for ``BERT_explainability/modules/BERT/BertForSequenceClassification.py``.

``BertForSequenceClassification(config)`` is a parameter container with the HF ``state_dict`` keys
(``bert.embeddings.*``, ``bert.encoder.layer.{i}.attention.self.{query,key,value}.*`` ...,
``bert.pooler.dense.*``, ``classifier.*``); ``forward`` and ``relprop`` run on the CUDA engine
(``engine.BertEngine``) for a batch of independent sequences.  ``config`` is a ``transformers.BertConfig`` or any
object with the same attribute names.  No ``param.grad`` side effect, no autograd graph.

``_EngineClassifier`` is what this classifier shares with the RoBERTa and DistilBERT façades next to it: the engine and
its weight version, ``relprop``, and the per-layer attention views (``attention_views()``).
"""
import weakref

import torch
import torch.nn as nn

from transformer_explainability_b200 import _lib
from transformer_explainability_b200.engine import BertEngine, bert_config


class _AttentionView:
    """``get_attn`` / ``get_attn_cam`` / ``get_attn_gradients`` of one encoder layer, served from the owning model's
    engine workspace.  ``_owner`` (a weak reference) and ``_layer`` are set by ``_EngineClassifier._link_views``."""
    _owner = None
    _layer = -1

    # accessors of BERT.py:281-297, served from the engine workspace
    def _t(self, name):
        owner = self._owner() if self._owner is not None else None
        if owner is None:
            raise RuntimeError("this attention view's model no longer exists")
        return owner._engine_tensor(name, self._layer)

    def get_attn(self):
        return self._t("attn")

    def get_attn_cam(self):
        return self._t("attn_cam")

    def get_attn_gradients(self):
        return self._t("attn_grad")

    def __getstate__(self):                    # the back-reference is re-made by the owning model's __setstate__
        state = self.__dict__.copy()
        state["_owner"] = None
        return state


class _SelfAttention(_AttentionView, nn.Module):
    def __init__(self, d):
        super().__init__()
        self.query = nn.Linear(d, d)
        self.key = nn.Linear(d, d)
        self.value = nn.Linear(d, d)
        self._owner = None
        self._layer = -1


class _DenseLN(nn.Module):
    def __init__(self, i, o, eps):
        super().__init__()
        self.dense = nn.Linear(i, o)
        self.LayerNorm = nn.LayerNorm(o, eps=eps)


class _Dense(nn.Module):
    def __init__(self, i, o):
        super().__init__()
        self.dense = nn.Linear(i, o)


class _Attention(nn.Module):
    def __init__(self, d, eps):
        super().__init__()
        self.self = _SelfAttention(d)
        self.output = _DenseLN(d, d, eps)


class _Layer(nn.Module):
    def __init__(self, d, f, eps):
        super().__init__()
        self.attention = _Attention(d, eps)
        self.intermediate = _Dense(d, f)
        self.output = _DenseLN(f, d, eps)


class _Embeddings(nn.Module):
    def __init__(self, cfg, position_ids=True):
        super().__init__()
        self.word_embeddings = nn.Embedding(cfg.vocab_size, cfg.hidden_size)
        self.position_embeddings = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size)
        self.token_type_embeddings = nn.Embedding(cfg.type_vocab_size, cfg.hidden_size)
        self.LayerNorm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)
        if position_ids:                       # transformers 3.5.1 kept it in the state_dict; later versions do not
            self.register_buffer("position_ids", torch.arange(cfg.max_position_embeddings).expand((1, -1)))


class _Encoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.layer = nn.ModuleList([_Layer(cfg.hidden_size, cfg.intermediate_size, cfg.layer_norm_eps)
                                    for _ in range(cfg.num_hidden_layers)])


class _BertModel(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = _Embeddings(cfg)
        self.encoder = _Encoder(cfg)
        self.pooler = _Dense(cfg.hidden_size, cfg.hidden_size)


class _EngineClassifier(nn.Module):
    """The engine side of an encoder sequence classifier: subclasses build their parameter modules, then call
    ``_setup`` with the ``te_bert_config`` of their family, and name their attention modules in ``attention_views``."""

    def _setup(self, config, cfg):
        self.config = config
        self.num_labels = config.num_labels
        self._link_views()
        self._cfg = cfg
        self._engine = None
        self._weights_version = None
        self.engine_flags = 0
        self._rule_flags = 0                   # BERT_cls_lrp sets TE_FLAG_RULES_LRP (the modules/layers_lrp.py rule library)
        std = getattr(config, "initializer_range", 0.02)
        for m in self.modules():                                   # transformers' _init_weights
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, mean=0.0, std=std)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def attention_views(self):
        """The attention module of every encoder layer, bottom to top: each has ``get_attn`` / ``get_attn_gradients`` /
        ``get_attn_cam`` (``BERT.py:281-297``), views of the engine's last call."""
        raise NotImplementedError

    def max_length(self):
        """The longest input the position table holds: ``max_position_embeddings``, less ``pad_token_id + 1`` for
        RoBERTa, whose positions start after the pad id."""
        c = self._cfg
        return c.max_position - (c.pad_token_id + 1 if c.arch == _lib.BERT_ARCH_ROBERTA else 0)

    def _head_weight(self):                    # the classifier's output weight: the device the model lives on
        return self.classifier.weight

    def _link_views(self):
        # a weak back-reference: a strong one would make model <-> view a reference cycle, so a dropped model and its
        # engine's device memory would live on until Python's cyclic garbage collector happened to run
        for i, v in enumerate(self.attention_views()):
            v._owner = weakref.ref(self)
            v._layer = i

    def __setstate__(self, state):             # pickle / copy.deepcopy: the views answer for the new model
        super().__setstate__(state)
        self._link_views()

    def _version(self):
        return tuple(p._version for p in self.parameters()) + (str(self._head_weight().device),)

    def engine(self):
        dev = self._head_weight().device
        if dev.type != "cuda":
            raise RuntimeError("the CUDA engine has no CPU path: move the model to a CUDA device (model.cuda())")
        v = self._version()
        flags = self.engine_flags | getattr(self, "_rule_flags", 0)
        if self._engine is None or self._engine.device != dev:
            self._engine = BertEngine(self._cfg, device=dev, flags=flags)
            self._weights_version = None
        if self._weights_version != v:
            self._engine.load_state_dict(self.state_dict())
            self._weights_version = v
        self._engine.flags = flags
        return self._engine

    def _engine_tensor(self, name, layer):
        if self._engine is None or self._engine.last[0] <= 0:
            raise RuntimeError("no saved activations: call model(input_ids, attention_mask) first")
        return self._engine.tensor(name, layer)

    def relprop(self, cam=None, **kwargs):
        """``relprop`` (:83-88): relevance at the encoder input [B,S,D]; leaves attn_cam / attn_gradients of every
        layer readable through ``layer.attention.self.get_attn_cam()`` ... like the reference.  ``alpha`` (default 1)
        selects the LRP-alpha-beta rule, beta = alpha - 1, in every Linear.relprop."""
        eng = self.engine()
        index = cam.argmax(dim=-1).to(torch.int32) if cam is not None else None
        eng.attribute(index=index, start_layer=0, flags=eng.flags | _lib.FLAG_RELPROP_TO_INPUT, alpha=kwargs.get("alpha", 1))
        return eng.tensor("relevance_in")


class BertForSequenceClassification(_EngineClassifier):
    def __init__(self, config):
        super().__init__()
        if getattr(config, "hidden_act", "gelu") != "gelu":
            raise NotImplementedError("only hidden_act='gelu' (the BertConfig default) is implemented")
        self.bert = _BertModel(config)
        self.classifier = nn.Linear(config.hidden_size, config.num_labels)
        self._setup(config, bert_config(config.vocab_size, config.max_position_embeddings, config.type_vocab_size,
                                        config.hidden_size, config.num_hidden_layers, config.num_attention_heads,
                                        config.intermediate_size, config.num_labels, config.layer_norm_eps))

    def attention_views(self):
        return [l.attention.self for l in self.bert.encoder.layer]

    def forward(self, input_ids=None, attention_mask=None, token_type_ids=None, position_ids=None, head_mask=None,
                inputs_embeds=None, labels=None, output_attentions=None, output_hidden_states=None, return_dict=None):
        """``BertForSequenceClassification.forward`` (:23-81) with return_dict=False: returns ``(logits,)``.
        ``token_type_ids`` (the segments of a sentence pair, what a tokenizer returns) enter the embeddings as in
        ``BertEmbeddings.forward`` (``BERT.py:61-85``); None puts every token in segment 0, so ``model(**encoding)``
        explains what the model was given."""
        if position_ids is not None or head_mask is not None or inputs_embeds is not None:
            raise NotImplementedError("position_ids, head_mask and inputs_embeds are not used on the attribution path "
                                      "(bert_pipeline.py:443,551)")
        return (self.engine().forward(input_ids, attention_mask, token_type_ids=token_type_ids),)
