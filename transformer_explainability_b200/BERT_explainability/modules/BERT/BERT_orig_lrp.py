"""Import-path drop-in for ``BERT_explainability/modules/BERT/BERT_orig_lrp.py``: the reference's ``BERT.py`` on the rule
library of ``modules/layers_lrp.py``.  The encoder's parameter containers do not depend on the rule library (the engine
applies it, ``BERT_cls_lrp.BertForSequenceClassification``), so these are the names of the facade's ``BERT.py``."""
from .BERT import (BertAttention, BertEmbeddings, BertEncoder, BertIntermediate, BertLayer, BertModel,  # noqa: F401
                   BertOutput, BertPooler, BertSelfAttention, BertSelfOutput, compute_rollout_attention, get_activation)
