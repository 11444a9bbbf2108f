"""Drop-in for ``BERT_explainability/modules/BERT/BERT_cls_lrp.py``: the BERT sequence classifier on the rule library of
``modules/layers_lrp.py`` (through ``BERT_orig_lrp.py``) — the model the reference's ERASER pipeline explains for
``partial_lrp``, ``lrp``, ``last_attn``, ``attn_gradcam`` and ``rollout`` (``bert_pipeline.py:422-448``).  Linear divides
its two halves by their own denominators (``layers_lrp.py:199-200``) and every Add, the attention-mask Add included, is
a plain ``RelPropSimple`` (``:98-100``).  Same parameters, ``state_dict`` keys and accessors as
``BertForSequenceClassification``; the same engine with ``TE_FLAG_RULES_LRP``.  ``engine_flags`` selects kernels as for
the other classifier; ``FLAG_RULES_LRP_TC`` runs the Linear rule on the tensor cores."""
from transformer_explainability_b200 import _lib
from .BertForSequenceClassification import BertForSequenceClassification as _Base
from .BERT_orig_lrp import BertModel                                      # noqa: F401  (the reference's module-level name)


class BertForSequenceClassification(_Base):
    def __init__(self, config):
        super().__init__(config)
        self._rule_flags = _lib.FLAG_RULES_LRP
