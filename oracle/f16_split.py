"""CPU restatement (numpy) of the block-scaled fp16 (hi, lo) operand format of the fp16-split forward Linear
(transformer_explainability_b200/csrc/te_common.cuh: te_f16_block_scale / te_f16_split4; te_tc_wgmma.cu).

Test infrastructure only (tests/test_f16_split_format.py): it pins the NUMBER FORMAT the kernels use — exact power-of-two
scaling, 22 significant bits down to 2^-17 of the block maximum, no overflow for any finite input — independently of a GPU.
Not part of the product path.
"""
import numpy as np


def block_scale(m):
    """(s, si) = (2^e, 2^-e) with 2^e * m in [2^14, 2^15); (1, 1) for m == 0 or non-finite m."""
    m = np.asarray(m, dtype=np.float32)
    s = np.ones_like(m)
    si = np.ones_like(m)
    ok = np.isfinite(m) & (m > 0)
    _, e = np.frexp(m[ok])                    # m = f * 2^e, f in [0.5, 1)
    e = np.maximum(e, -100)
    s[ok] = np.ldexp(np.float32(1), 15 - e).astype(np.float32)
    si[ok] = np.ldexp(np.float32(1), e - 15).astype(np.float32)
    return s, si


def split_rows(x, block=128):
    """x [rows, cols] fp32 -> hi, lo fp16 [rows, cols] and si [rows, ceil(cols / block)] (block = cols: one scale per row)."""
    x = np.asarray(x, dtype=np.float32)
    rows, cols = x.shape
    nblk = (cols + block - 1) // block
    hi = np.zeros((rows, cols), np.float16)
    lo = np.zeros((rows, cols), np.float16)
    si = np.ones((rows, nblk), np.float32)
    for b in range(nblk):
        sl = slice(b * block, min(cols, (b + 1) * block))
        s, si[:, b] = block_scale(np.abs(x[:, sl]).max(axis=1))
        a = x[:, sl] * s[:, None]             # exact: power of two (fp32)
        h = a.astype(np.float16)
        hi[:, sl] = h
        lo[:, sl] = (a - h.astype(np.float32)).astype(np.float16)
    return hi, lo, si


def reconstruct(hi, lo, si, block=128):
    rows, cols = hi.shape
    out = np.zeros((rows, cols), np.float64)
    for b in range(si.shape[1]):
        sl = slice(b * block, min(cols, (b + 1) * block))
        out[:, sl] = (hi[:, sl].astype(np.float64) + lo[:, sl].astype(np.float64)) * si[:, b:b + 1].astype(np.float64)
    return out


def linear_f16_split(x, w, block=128):
    """y = x W^T as the kernel forms it: x_hi W_hi + x_lo W_hi + x_hi W_lo per 128-element chunk (exact products, here summed in
    fp64), chunk scaled by the activation block's 2^-e, columns by the weight row's 2^-f."""
    xh, xl, xs = split_rows(x, block)
    wh, wl, ws = split_rows(w, block=w.shape[1])
    rows, K = x.shape
    y = np.zeros((rows, w.shape[0]), np.float64)
    for b in range(xs.shape[1]):
        sl = slice(b * block, min(K, (b + 1) * block))
        a_h, a_l = xh[:, sl].astype(np.float64), xl[:, sl].astype(np.float64)
        b_h, b_l = wh[:, sl].astype(np.float64), wl[:, sl].astype(np.float64)
        y += (a_h @ b_h.T + a_l @ b_h.T + a_h @ b_l.T) * xs[:, b:b + 1].astype(np.float64)
    return y * ws[:, 0].astype(np.float64)[None, :]
