"""``generate_visualization`` of the reference notebooks (``example.ipynb:55-66``), batched on the GPU.

relevance [B,196] -> reshape 14x14 -> bilinear x16 (align_corners=False) -> per-sample min-max -> [B,224,224];
the JET overlay (cv2) stays on the host exactly like the notebook.
"""
import numpy as np
import torch


def relevance_to_heatmap(maps, grid=14, scale=16):
    """[B, grid*grid] -> min-max normalised [B, grid*scale, grid*scale] (device tensor) through the engine's kernel
    (``te_relevance_heatmap``, one block per sample).  CUDA tensors only: there is no host path."""
    if not maps.is_cuda:
        raise ValueError("relevance_to_heatmap needs a CUDA tensor (no CPU fallback)")
    if maps.dim() != 2 or maps.shape[1] != grid * grid:
        raise ValueError("relevance_to_heatmap: maps %s, expected [B, grid*grid] = [B, %d]" % (tuple(maps.shape), grid * grid))
    b = maps.shape[0]
    from . import _lib
    m = maps.detach().to(torch.float32).contiguous()
    out = torch.empty(b, grid * scale, grid * scale, device=m.device, dtype=torch.float32)
    with torch.cuda.device(m.device):
        _lib.check(_lib.load().te_relevance_heatmap(_lib.ptr(m), b, grid, scale, _lib.ptr(out),
                                                    _lib.ctypes.c_void_p(torch.cuda.current_stream(m.device).cuda_stream)),
                   "te_relevance_heatmap")
    return out


def show_cam_on_image(img, mask):
    """``example.ipynb:48-53``: JET heat-map overlay (host, needs cv2)."""
    import cv2
    heatmap = cv2.applyColorMap(np.uint8(255 * mask), cv2.COLORMAP_JET)
    heatmap = np.float32(heatmap) / 255
    cam = heatmap + np.float32(img)
    return cam / np.max(cam)


def generate_visualization(attribution_generator, original_image, class_index=None, start_layer=0):
    """``example.ipynb:55-66``: original_image [3,224,224] -> uint8 RGB overlay [224,224,3]."""
    import cv2
    dev = next(attribution_generator.model.parameters()).device
    maps = attribution_generator.generate_LRP(original_image.unsqueeze(0).to(dev), method="transformer_attribution",
                                              index=class_index, start_layer=start_layer).detach()
    heat = relevance_to_heatmap(maps)[0].cpu().numpy()
    img = original_image.permute(1, 2, 0).cpu().numpy()
    img = (img - img.min()) / (img.max() - img.min())
    vis = show_cam_on_image(img, heat)
    vis = np.uint8(255 * vis)
    return cv2.cvtColor(np.array(vis), cv2.COLOR_RGB2BGR)
