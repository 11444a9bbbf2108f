"""CPU restatement of the colour weights of ``bert_pipeline.py``'s ``generate()`` (``:50-56``) in numpy fp32, the oracle of
``te_eraser_latex_weights`` (TEST INFRASTRUCTURE).  ``tests/golden/eraser_latex.npz`` pins it to the reference's files."""
import re

import numpy as np


def latex_weights(cam, n, clamp=True):
    """The weights of the first n entries of cam: optionally clamp(min=0); NaN anywhere makes min and max NaN (torch.min /
    torch.max); a constant row gives zeros, else (100 * (a - min)) / (max - min) in fp32, one rounding per operation;
    values below 1 become 0."""
    a = np.array(cam, dtype=np.float32)[:n]
    if clamp:
        a = np.where(a < 0, np.float32(0), a)
    if np.isnan(a).any():
        mn = mx = np.float32("nan")
    else:
        mn, mx = a.min(), a.max()
    if mx == mn:
        return np.zeros_like(a)
    with np.errstate(all="ignore"):
        w = (np.float32(100) * (a - mn)) / (mx - mn)
        w[w < 1] = 0
    return w.astype(np.float32)


_BOX = re.compile(r"\\colorbox\{[a-z]+!([^}]*)\}\{\\strut ")          # a token's box, not the page's white one


def file_weights(text):
    """The weights printed in a ``generate()`` file, in token order, as fp32 (each was printed as the Python float of an
    fp32 value, so the round trip is exact)."""
    return np.array([float(v) for v in _BOX.findall(text)], dtype=np.float32)
