"""Drop-in for ``BERT_explainability/modules/BERT/ExplanationGenerator.py`` (class ``Generator``).

``generate_LRP`` is the transformer-attribution hot path; the comparison generators of the same class
(``generate_LRP_last_layer``, ``generate_full_lrp``, ``generate_attn_last_layer``, ``generate_rollout``,
``generate_attn_gradcam``, reference ``:61-155``) are served from the same engine passes and the same kernels.
Every generator accepts a batch of independent sequences of one length ([B,S] -> [B,S]); B = 1 is the reference call.
Every generator also takes ``token_type_ids`` (the segments of sentence pairs, [B,S]); None puts every token in segment 0.
``model`` is any of the engine's encoder classifiers (BERT, RoBERTa / XLM-RoBERTa, DistilBERT): the generators read its
layers through ``model.attention_views()``."""
import torch

from transformer_explainability_b200 import _lib, ops


def compute_rollout_attention(all_layer_matrices, start_layer=0):
    """``ExplanationGenerator.py:7-18``: (M + I) / rowsum, chained from ``start_layer``."""
    return ops.compute_rollout_attention(all_layer_matrices, start_layer=start_layer, normalize=True)


class Generator:
    def __init__(self, model):
        self.model = model
        self.model.eval()

    def forward(self, input_ids, attention_mask, token_type_ids=None):
        return self.model(input_ids, attention_mask, token_type_ids=token_type_ids)

    def generate_LRP(self, input_ids, attention_mask, index=None, start_layer=11, token_type_ids=None):
        """``:28-59``: [1,S] ids -> [1,S] token relevance (row 0 of the normalised rollout, element 0 = row minimum)."""
        maps, _ = self.model.engine().explain(input_ids, attention_mask, index=index, start_layer=start_layer,
                                              token_type_ids=token_type_ids)
        return maps

    # ---- comparison generators (reference :61-155) ---------------------------------------------------------------
    def _last(self):
        return self.model.attention_views()[-1]

    def _forward(self, input_ids, attention_mask, token_type_ids):
        # without token types this stays the engine's two-argument call, which callers may wrap (e.g. to record shapes)
        eng = self.model.engine()
        if token_type_ids is None:
            eng.forward(input_ids, attention_mask)
        else:
            eng.forward(input_ids, attention_mask, token_type_ids=token_type_ids)
        return eng

    def _run(self, input_ids, attention_mask, index, start_layer, extra_flags, token_type_ids):
        eng = self._forward(input_ids, attention_mask, token_type_ids)
        eng.attribute(index=index, start_layer=start_layer, flags=eng.flags | extra_flags)
        return eng

    def generate_LRP_last_layer(self, input_ids, attention_mask, index=None, token_type_ids=None):
        """``:61-83``: head-mean of the clamped attention relevance (attn_cam) of the last layer, row 0, [0] = 0."""
        eng = self._run(input_ids, attention_mask, index, self.model._cfg.layers - 1, 0, token_type_ids)
        cam = ops.head_reduce(self._last().get_attn_cam(), mode="relu_mean")
        cam[:, 0, 0] = 0
        return cam[:, 0]

    def generate_full_lrp(self, input_ids, attention_mask, index=None, token_type_ids=None):
        """``:85-105``: LRP carried to the encoder input, summed over the hidden dimension, [0] = 0."""
        eng = self._run(input_ids, attention_mask, index, 0, _lib.FLAG_RELPROP_TO_INPUT, token_type_ids)
        cam = eng.tensor("relevance_in").sum(dim=2)
        cam[:, 0] = 0
        return cam

    def generate_attn_last_layer(self, input_ids, attention_mask, index=None, token_type_ids=None):
        """``:107-113``: head-mean of the last layer's raw attention, row 0, [0] = 0."""
        self._forward(input_ids, attention_mask, token_type_ids)
        cam = ops.head_reduce(self._last().get_attn(), mode="mean")
        cam[:, 0, 0] = 0
        return cam[:, 0]

    def generate_rollout(self, input_ids, attention_mask, start_layer=0, index=None, token_type_ids=None):
        """``:115-127``: rollout of the head-averaged raw attention, row 0, [0] = 0."""
        self._forward(input_ids, attention_mask, token_type_ids)
        mats = [ops.head_reduce(v.get_attn(), mode="mean") for v in self.model.attention_views()]
        rollout = compute_rollout_attention(mats, start_layer=start_layer)
        rollout[:, 0, 0] = 0
        return rollout[:, 0]

    def generate_attn_gradcam(self, input_ids, attention_mask, index=None, token_type_ids=None):
        """``:129-155``: last-layer attention weighted per head by its mean gradient, relu(mean over heads), min-max
        normalised over the [S,S] map, row 0, [0] = 0."""
        eng = self._run(input_ids, attention_mask, index, self.model._cfg.layers - 1, _lib.FLAG_GRADIENTS_ONLY,
                        token_type_ids)
        att = self._last()
        w = ops.head_region_mean(att.get_attn_gradients())
        cam = ops.head_reduce(att.get_attn(), head_weight=w, mode="mean_relu")
        lo = cam.amin(dim=(1, 2), keepdim=True)
        hi = cam.amax(dim=(1, 2), keepdim=True)
        cam = (cam - lo) / (hi - lo)
        cam[:, 0, 0] = 0
        return cam[:, 0]

    def generate_attn_grad_rollout(self, input_ids, attention_mask, index=None, start_layer=0, token_type_ids=None):
        """The LRP-free gradient-weighted attention rollout of Chefer, Gur, Wolf (ICCV 2021): for l = start_layer .. L-1,
        R <- R + mean_h relu(dy_c/dA_l * A_l) R from R = I, row 0 with [0] = 0 as the comparison generators above.
        [B,S] -> [B,S]; padded positions come out exactly 0."""
        eng = self.model.engine()
        maps, _ = eng.explain(input_ids, attention_mask, index=index, start_layer=start_layer,
                              flags=eng.flags | _lib.FLAG_ATTN_GRAD_ROLLOUT, token_type_ids=token_type_ids)
        return maps

    def generate_LRP_batched(self, input_ids, attention_mask=None, index=None, start_layer=11, chunk=None,
                             return_index=False, token_type_ids=None):
        """B independent sequences of equal length in one engine call: [B,S] -> [B,S]."""
        maps, idx = self.model.engine().explain(input_ids, attention_mask, index=index, start_layer=start_layer,
                                                chunk=chunk, token_type_ids=token_type_ids)
        return (maps, idx) if return_index else maps
