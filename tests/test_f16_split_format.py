"""The block-scaled fp16 (hi, lo) operand format of the fp16-split forward Linear, pinned on CPU (oracle/f16_split.py restates
te_f16_block_scale / te_f16_split4 of csrc/te_common.cuh and the three-term product of te_tc_wgmma.cu)."""
import numpy as np

from oracle import f16_split as F


def test_block_scale_is_an_exact_power_of_two_in_range():
    m = np.array([0.0, 1e-30, 3e-5, 0.5, 1.0, 1.5, 300.0, 6.5e4, 1e30, np.inf, np.nan], np.float32)
    s, si = F.block_scale(m)
    ok = np.isfinite(m) & (m > 0)
    assert (s[~ok] == 1).all() and (si[~ok] == 1).all()
    assert (np.frexp(s[ok])[0] == 0.5).all()                          # powers of two
    assert (s[ok].astype(np.float64) * si[ok].astype(np.float64) == 1.0).all()
    sm = m[ok].astype(np.float64) * s[ok].astype(np.float64)
    assert ((sm >= 2.0 ** 14) & (sm < 2.0 ** 15)).all()               # the block maximum lands in [2^14, 2^15): below 65504


def test_split_keeps_22_bits_and_never_overflows():
    g = np.random.default_rng(0)
    x = g.standard_normal((64, 384)).astype(np.float32)
    x *= np.logspace(-30, 30, 64, dtype=np.float64)[:, None].astype(np.float32)      # rows spanning 60 decades
    x[:, ::7] *= 1e-4                                                                 # four decades inside a block
    x[5] = 0.0
    hi, lo, si = F.split_rows(x)
    assert np.isfinite(hi.astype(np.float32)).all() and np.isfinite(lo.astype(np.float32)).all()
    r = F.reconstruct(hi, lo, si)
    bmax = np.abs(x.astype(np.float64)).reshape(64, 3, 128).max(axis=2).repeat(128, axis=1)
    err = np.abs(r - x.astype(np.float64))
    big = np.abs(x) >= bmax * 2.0 ** -17
    assert (err[big] <= np.abs(x.astype(np.float64))[big] * 2.0 ** -21).all()          # 22 significant bits (half-ulp: 2^-22, slack 2x)
    assert (err <= bmax * 2.0 ** -38 + np.abs(x.astype(np.float64)) * 2.0 ** -21).all()   # graceful below: absolute floor of the block
    assert (r[5] == 0).all()


def test_three_term_product_is_fp32_grade():
    g = np.random.default_rng(1)
    x = (g.standard_normal((96, 768)) * np.logspace(-3, 1, 768)).astype(np.float32)
    x *= np.logspace(-6, 6, 96)[:, None].astype(np.float32)
    w = (g.standard_normal((256, 768)) * 0.05 * np.logspace(-4, 2, 256)[:, None]).astype(np.float32)
    y = F.linear_f16_split(x, w)
    ref = x.astype(np.float64) @ w.astype(np.float64).T
    scale = (np.abs(x.astype(np.float64)) @ np.abs(w.astype(np.float64)).T) / np.sqrt(768)
    assert (np.abs(y - ref) / scale).max() < 2e-6                     # the dropped lo*lo term and the lo roundings: ~2^-22 each
