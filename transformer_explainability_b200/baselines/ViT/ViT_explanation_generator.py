"""Drop-in for ``baselines/ViT/ViT_explanation_generator.py`` (class ``LRP``).

``generate_LRP`` keeps the reference signature and return shape ([1, 196]); ``generate_LRP_batched`` is the
batched addition: B independent explanations per call, device-resident in and out.
``Baselines`` (raw-attention rollout / attention GradCAM, reference ``:45-83``) runs on the same engine: it needs
the forward pass (+ the class-gradient of the last block's attention) only.
"""
import torch

from transformer_explainability_b200 import _lib, ops


def compute_rollout_attention(all_layer_matrices, start_layer=0):
    """``ViT_explanation_generator.py:7-18`` — this file's own rollout ROW-NORMALISES (M + I) / rowsum before chaining
    (unlike ``ViT_LRP.compute_rollout_attention``); list of [B,N,N] -> [B,N,N]."""
    return ops.compute_rollout_attention(all_layer_matrices, start_layer=start_layer, normalize=True)


class LRP:
    def __init__(self, model):
        self.model = model
        self.model.eval()

    def generate_LRP(self, input, index=None, method="transformer_attribution", is_ablation=False, start_layer=0):
        """``ViT_explanation_generator.py:25-41``: forward, class pick, one-hot seed, relprop."""
        output = self.model(input)
        if index is None:
            index = output.argmax(dim=-1)
        index = torch.as_tensor(index, device=output.device).reshape(-1).long()
        one_hot = torch.zeros_like(output)
        one_hot[torch.arange(output.shape[0], device=output.device), index] = 1
        return self.model.relprop(one_hot, method=method, is_ablation=is_ablation, start_layer=start_layer, alpha=1)

    def generate_LRP_batched(self, input, index=None, start_layer=0, chunk=None, return_index=False):
        """B independent ``transformer_attribution`` explanations in one engine call: [B,3,H,W] -> [B,196]."""
        maps, idx = self.model.engine().explain(input, index=index, start_layer=start_layer, chunk=chunk)
        return (maps, idx) if return_index else maps

    def generate_attn_grad_rollout(self, input, index=None, start_layer=0):
        """The LRP-free gradient-weighted attention rollout of Chefer, Gur, Wolf (ICCV 2021): for l = start_layer .. L-1,
        R <- R + mean_h relu(dy_c/dA_l * A_l) R from R = I, row 0 without the prefix token(s).  [B,3,H,W] -> [B,N-prefix];
        ``index`` as for ``generate_LRP`` (arg-max when None).  The model's rule-library and relprop precision flags are
        accepted and change nothing: no relprop runs."""
        eng = self.model.engine()
        maps, _ = eng.explain(input, index=index, start_layer=start_layer, flags=eng.flags | _lib.FLAG_ATTN_GRAD_ROLLOUT)
        return maps


class Baselines:
    """``ViT_explanation_generator.py:45-83`` for a ``baselines.ViT.ViT_new`` (or ``ViT_LRP``) model."""

    def __init__(self, model):
        self.model = model
        self.model.eval()

    def generate_cam_attn(self, input, index=None):
        """``:50-71``: CLS-row attention of the last block, weighted per head by the mean of its gradient over the
        patch positions, relu(mean over heads), min-max normalised -> [g,g] (B = 1) or [B,g,g]."""
        eng = self.model.engine()
        eng.forward(input)
        eng.attribute(index=index, start_layer=self.model._cfg.depth - 1, flags=eng.flags | _lib.FLAG_GRADIENTS_ONLY)
        attn = self.model.blocks[-1].attn
        n = eng.tokens
        first = eng.prefix
        w = ops.head_region_mean(attn.get_attn_gradients(), rows=(0, 1), cols=(first, n))
        cam = ops.head_reduce(attn.get_attn(), head_weight=w, mode="mean_relu")[:, 0, first:]
        lo = cam.amin(dim=1, keepdim=True)
        hi = cam.amax(dim=1, keepdim=True)
        cam = (cam - lo) / (hi - lo)
        g = int(round((n - first) ** 0.5))
        cam = cam.reshape(-1, g, g)
        return cam[0] if cam.shape[0] == 1 else cam

    def generate_rollout(self, input, start_layer=0):
        """``:73-83``: rollout of the head-averaged raw attention maps, CLS row -> [B,N-1]."""
        eng = self.model.engine()
        eng.forward(input)
        mats = [ops.head_reduce(blk.attn.get_attn(), mode="mean") for blk in self.model.blocks]
        return compute_rollout_attention(mats, start_layer=start_layer)[:, 0, eng.prefix:]
