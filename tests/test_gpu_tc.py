"""GPU: the tensor-core (TF32 tensor-core) z+ Linear rule against the fp32 SIMT path and the fp64 oracle.

Tolerance: TF32 operands carry a 10-bit mantissa (rna), accumulation is fp32, Z is a sum of non-negative
products -> relative error of a few 1e-4 on Z/S and on the output (stated: 2e-3 of the tensor maximum)."""
import pytest
import torch

from oracle import rules

pytestmark = pytest.mark.gpu


def rel(a, b):
    b = b.double()
    return ((a.double().cpu() - b.cpu()).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304),
                                           (256, 1024, 1024)])
def test_tc_linear_relprop_matches_simt_and_oracle(rows, inf, outf):
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    r = torch.rand(rows, outf, generator=g)
    xd, wd, rd = x.cuda(), w.cuda(), r.cuda()
    simt = ops.linear_relprop(xd, wd, rd, tensor_cores=False)
    tc = ops.linear_relprop(xd, wd, rd, tensor_cores=True)
    torch.cuda.synchronize()
    ref = rules.linear_relprop(x.double(), w.double(), r.double())
    assert rel(simt, ref) < 2e-5
    assert rel(tc, ref) < 2e-3, "tensor-core path: rel err %g" % rel(tc, ref)
    # conservation of relevance survives the reduced-precision operands
    assert abs(tc.double().sum().item() - r.double().sum().item()) < 2e-3 * r.sum().item()
    # single-pass variant fed with the saved forward output: Z = ((y - b) + |x||W|^T)/2 (what the engines run)
    b = torch.randn(outf, generator=g)
    y = ops.linear_forward(xd, wd, b.cuda())
    tc1 = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=b.cuda())
    assert rel(tc1, ref) < 3e-3, "single-pass tensor-core path: rel err %g" % rel(tc1, ref)


def test_tc_engine_vit_base_vs_simt_and_oracle():
    """ViT-B/16: engine with the tensor-core z+ path vs the fp32 SIMT engine and the fp64 oracle; medians over
    1e-7-perturbed copies (see tests/test_gpu_vit.py::_noise_trials for why)."""
    from oracle import cpu as ocpu
    from oracle import vit as ovit
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224
    from test_gpu_vit import _noise_trials, check_parity
    trials = 16
    params, heads = ovit.init_params("vit_base_patch16_224", seed=0)
    xs = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(100))
    m = vit_base_patch16_224()
    m.load_state_dict(params)
    m = m.cuda().eval()
    eng = m.engine()
    xb = torch.cat([_noise_trials(xs[s:s + 1], trials) for s in range(2)]).cuda()
    simt, idx0 = eng.explain(xb, flags=0)
    tc, idx1 = eng.explain(xb, flags=_lib.FLAG_ZPLUS_TENSOR_CORES)
    torch.cuda.synchronize()
    assert torch.equal(idx0, idx1)
    ocpu.set_torch_threads()
    for s in range(2):
        ref, ridx = ovit.explain({k: v.double() for k, v in params.items()}, xs[s:s + 1].double(), heads)
        check_parity(simt[s * trials:(s + 1) * trials], ref[0], "sample %d fp32 SIMT" % s)
        check_parity(tc[s * trials:(s + 1) * trials], ref[0], "sample %d tensor-core z+" % s)


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304)])
def test_tc_3xtf32_linear_is_fp32_grade(rows, inf, outf):
    """Forward / backward Linear GEMMs on tensor-core with the error-compensated 3xTF32 split.  The split removes the
    TF32 operand rounding (1e-3 -> 1e-6); what remains is the tensor core's own fp32 accumulation, which truncates
    (round-toward-zero) at every MMA, so the error grows linearly with the reduction length: measured 7e-9 * K
    (K = 3072: 2e-5) against 5e-7 for the fp32 SIMT kernel.  Stated bound: 1.5e-8 * K + 2e-6."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 1)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    b = torch.randn(outf, generator=g)
    dy = torch.randn(rows, outf, generator=g)
    ref_y = torch.nn.functional.linear(x.double(), w.double(), b.double())
    ref_dx = dy.double() @ w.double()
    for tc in (False, True):
        y = ops.linear_forward(x.cuda(), w.cuda(), b.cuda(), tensor_cores=tc)
        dx = ops.linear_backward(dy.cuda(), w.cuda(), tensor_cores=tc)
        torch.cuda.synchronize()
        ey, edx = rel(y, ref_y), rel(dx, ref_dx)
        print("rows %d in %d out %d tc=%s: fwd %.2e bwd %.2e" % (rows, inf, outf, tc, ey, edx))
        if tc:
            assert ey < 1.5e-8 * inf + 2e-6 and edx < 1.5e-8 * outf + 2e-6
        else:
            assert ey < 3e-6 and edx < 3e-6


def test_tc_linear_engine_vit_base():
    """ViT-B/16 with every Linear GEMM (forward, backward, z+ rule) on tensor cores vs the fp32 SIMT engine and the
    fp64 oracle: class index bit-exact, logits at fp32 accuracy, maps in the same noise class (medians)."""
    from oracle import cpu as ocpu
    from oracle import vit as ovit
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224
    from test_gpu_vit import _noise_trials, check_parity
    trials = 16
    params, heads = ovit.init_params("vit_base_patch16_224", seed=0)
    xs = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(100))
    m = vit_base_patch16_224()
    m.load_state_dict(params)
    m = m.cuda().eval()
    eng = m.engine()
    xb = torch.cat([_noise_trials(xs[s:s + 1], trials) for s in range(2)]).cuda()
    simt, idx0, lg0 = eng.explain(xb, flags=0, return_logits=True)
    full = _lib.FLAG_TENSOR_CORES | _lib.FLAG_ROLLOUT_FUSED
    tc, idx1, lg1 = eng.explain(xb, flags=full, return_logits=True)
    torch.cuda.synchronize()
    assert torch.equal(idx0, idx1)
    ocpu.set_torch_threads()
    for s in range(2):
        ref, ridx, taps = ovit.explain({k: v.double() for k, v in params.items()}, xs[s:s + 1].double(), heads,
                                       return_taps=True)
        assert int(idx1[s * trials]) == int(ridx)
        assert rel(lg1[s * trials], taps["logits"][0]) < 1e-5
        check_parity(tc[s * trials:(s + 1) * trials], ref[0], "sample %d all-tensor-core" % s)


def test_tc_attention_contractions_engine():
    """Every attention-shaped contraction on tensor-core (3xTF32): the N x N ones (QK^T, dctx V^T, attn_cam, S1; K-major
    operands) and the N x d ones reduced over tokens (attn v, attn^T dctx, dS k, dS^T q, S1 k, S1^T q, attn^T S2; MN-major
    tf32 operands in the SWIZZLE_128B_BASE32B layout).  Attention probabilities and attention gradients of every layer
    stay at fp32 accuracy (they chain through all of these kernels); maps in the same noise class."""
    from oracle import cpu as ocpu
    from oracle import vit as ovit
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224
    from test_gpu_vit import _noise_trials, check_parity
    trials = 16
    params, heads = ovit.init_params("vit_base_patch16_224", seed=0)
    xs = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(100))
    m = vit_base_patch16_224()
    m.load_state_dict(params)
    m = m.cuda().eval()
    eng = m.engine()
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    ref, ridx, taps = ovit.explain(p64, xs[0:1].double(), heads, return_taps=True)
    maps, idx = eng.explain(xs[0:1].cuda(), flags=_lib.FLAG_ALL_FAST)
    assert int(idx[0]) == int(ridx)
    for l in (0, 6, 11):
        assert rel(m.blocks[l].attn.get_attn()[0], taps["cache"]["blocks"][l]["attn"][0]) < 1e-5
        assert rel(m.blocks[l].attn.get_attn_gradients()[0], taps["grads"][l][0]) < 1e-4
    assert rel(m.blocks[11].attn.get_attn_cam()[0], taps["cams"][11][0]) < 5e-2      # TF32 z+ rules feed this one
    xb = torch.cat([_noise_trials(xs[s:s + 1], trials) for s in range(2)]).cuda()
    fast, idx1 = eng.explain(xb, flags=_lib.FLAG_ALL_FAST)
    for s in range(2):
        r, _ = ovit.explain(p64, xs[s:s + 1].double(), heads)
        check_parity(fast[s * trials:(s + 1) * trials], r[0], "sample %d all-fast" % s)


@pytest.mark.parametrize("rows,inf,outf", [(394, 768, 3072), (1000, 3072, 768), (128, 256, 256)])
def test_tc_bf16_second_contraction(rows, inf, outf):
    """TE_FLAG_ZPLUS_BF16: S stored as bf16 and R_in = x+ (S W+) + x- (S W-) on fp16 / bf16 tensor-core MMAs with bf16 operands
    (8-bit mantissa, fp32 accumulate).  Stated tolerance 1.5e-2 of the tensor maximum; relevance is conserved to 1e-2."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 7)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    b = torch.randn(outf, generator=g)
    r = torch.rand(rows, outf, generator=g)
    xd, wd, rd, bd = x.cuda(), w.cuda(), r.cuda(), b.cuda()
    y = ops.linear_forward(xd, wd, bd)
    out = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=bd, bf16=True)
    torch.cuda.synchronize()
    ref = rules.linear_relprop(x.double(), w.double(), r.double())
    e = rel(out, ref)
    print("bf16 R kernel rows %d in %d out %d: rel %.2e" % (rows, inf, outf, e))
    assert e < 1.5e-2
    assert abs(out.double().sum().item() - r.double().sum().item()) < 1e-2 * r.sum().item()


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304),
                                           (50432, 768, 768)])
def test_tc_persistent_pair_kernels(rows, inf, outf):
    """The z+ kernels the engines run by default — single-pass S kernel with the |x| transform + R kernel whose two products
    share one A tile — against the fp64 oracle; the single-pass TF32 backward Linear against fp64 (TF32 operand error,
    stated 2e-3 of the tensor maximum).  Every shape is also compared element by element with the fp32 SIMT path.  Shapes include
    partial row tiles and many more tiles than SMs."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 3)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    r = torch.rand(rows, outf, generator=g)
    b = torch.randn(outf, generator=g)
    dy = torch.randn(rows, outf, generator=g)
    xd, wd, rd, bd = x.cuda(), w.cuda(), r.cuda(), b.cuda()
    y = ops.linear_forward(xd, wd, bd)
    new = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=bd)
    simt = ops.linear_relprop(xd, wd, rd, tensor_cores=False)        # fp32 SIMT path: every element, every tile, all shapes
    torch.cuda.synchronize()
    assert rel(new, simt) < 3e-3, "z+ kernels vs fp32 SIMT: rel err %g" % rel(new, simt)
    if rows <= 4096:
        ref = rules.linear_relprop(x.double(), w.double(), r.double())
        assert rel(new, ref) < 3e-3, "z+ kernels: rel err %g" % rel(new, ref)
    assert abs(new.double().sum().item() - r.double().sum().item()) < 2e-3 * r.sum().item()
    dx = ops.linear_backward_tf32(dy.cuda(), wd)
    torch.cuda.synchronize()
    ref_dx = (dy.double().cuda() @ w.double().cuda()).cpu()
    e = rel(dx, ref_dx)
    print("tf32 backward rows %d in %d out %d: rel %.2e" % (rows, inf, outf, e))
    assert e < 2e-3


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304)])
def test_tc_bf16_single_pass_denominator(rows, inf, outf):
    """TE_FLAG_ZPLUS_S1_BF16: the |x||W|^T term of the single-pass z+ denominator with bf16 operands (bf16 wgmma
    S kernel).  A sum of K non-negative products: the 2^-9 operand roundings average out; stated tolerance = the TF32 path's."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 5)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    b = torch.randn(outf, generator=g)
    r = torch.rand(rows, outf, generator=g)
    xd, wd, rd, bd = x.cuda(), w.cuda(), r.cuda(), b.cuda()
    y = ops.linear_forward(xd, wd, bd)
    tf = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=bd)
    bf = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=bd, bf16="s1")
    torch.cuda.synchronize()
    ref = rules.linear_relprop(x.double(), w.double(), r.double())
    e_tf, e_bf = rel(tf, ref), rel(bf, ref)
    print("bf16 S1 rows %d in %d out %d: TF32 %.2e  bf16 denominator %.2e" % (rows, inf, outf, e_tf, e_bf))
    assert e_bf < 3e-3
    assert abs(bf.double().sum().item() - r.double().sum().item()) < 2e-3 * r.sum().item()


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304),
                                           (20000, 768, 768), (300, 64, 256)])
def test_tc_f16_split_linear_is_fp32_grade(rows, inf, outf):
    """TE_FLAG_LINEAR_F16_SPLIT: forward Linear on fp16 / bf16 tensor-core MMAs with the row-scaled fp16 (hi, lo) split of both operands
    (te_tc_wgmma.cu).  fp16 carries the same 11-bit significand as TF32, so the bound is the 3xTF32 one; the per-row power-of-two
    scaling has to cope with rows and weight rows whose magnitudes span 12 decades, zero rows, and activations spanning four
    decades inside a row."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 23)
    x = torch.randn(rows, inf, generator=g) * torch.logspace(-3, 1, inf)
    x = x * torch.logspace(-6, 6, rows)[:, None]                   # row magnitudes 1e-6 .. 1e6 (fp16 alone would over/underflow)
    x[rows // 2] = 0.0
    w = torch.randn(outf, inf, generator=g) * 0.05 * torch.logspace(-4, 2, outf)[:, None]
    w[3] = 0.0
    b = torch.randn(outf, generator=g)
    ref = torch.nn.functional.linear(x.double(), w.double())
    # without a bias: at row magnitudes of 1e-6 a bias of O(1) would swamp the product and hide the kernel's error
    y3 = ops.linear_forward(x.cuda(), w.cuda(), None, tensor_cores=True)
    yh = ops.linear_forward(x.cuda(), w.cuda(), None, tensor_cores=True, f16_split=True)
    yb = ops.linear_forward(x.cuda(), w.cuda(), b.cuda(), tensor_cores=True, f16_split=True)
    torch.cuda.synchronize()
    # error of every element relative to the scale of its own row and column
    scale = (x.double().abs() @ w.double().abs().T).clamp_min(1e-300) / inf ** 0.5
    e3 = ((y3.double().cpu() - ref).abs() / scale).max().item()
    eh = ((yh.double().cpu() - ref).abs() / scale).max().item()
    print("rows %d in %d out %d: 3xTF32 %.2e  fp16 split %.2e (per-element, relative to |x||W|^T / sqrt(K))" % (rows, inf, outf, e3, eh))
    assert torch.isfinite(yh).all()
    assert eh < 2e-5 and eh < 2 * e3 + 1e-6          # fp32 grade, and no worse than the 3xTF32 kernel on the same data
    assert (yh[rows // 2] == 0).all() and (yh[:, 3] == 0).all()                       # zero row / zero weight row: exactly zero
    assert torch.equal(yb.cpu(), (yh.cpu() + b))                                      # the bias is added last, in fp32


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304), (20000, 768, 768)])
def test_tc_fp16_second_contraction(rows, inf, outf):
    """TE_FLAG_ZPLUS_R_F16: R_in = x+ (S W+) + x- (S W-) on fp16 / bf16 tensor-core MMAs — S as hi-only block-scaled fp16 (one power of two
    per row and 128 columns), W+^T / W-^T as row-scaled fp16 (te_tc_wgmma.cu).  Same 11 significant bits as the TF32 form
    (rounded to nearest): the rule error must not exceed the TF32 path's bound.  The relevance rows span 12 decades (S = R / Z
    inherits them): fp16 without the block scaling would over- / underflow."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 31)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    b = torch.randn(outf, generator=g)
    r = torch.rand(rows, outf, generator=g) * torch.logspace(-6, 6, rows)[:, None]
    r[rows // 3] = 0.0
    xd, wd, rd, bd = x.cuda(), w.cuda(), r.cuda(), b.cuda()
    y = ops.linear_forward(xd, wd, bd)
    tf = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=bd, bf16="s1")
    hf = ops.linear_relprop(xd, wd, rd, tensor_cores=True, y=y, bias=bd, bf16="s1", r_f16=True)
    torch.cuda.synchronize()
    ref = rules.linear_relprop(x.double(), w.double(), r.double())
    rowmax = ref.abs().amax(dim=1, keepdim=True).clamp_min(1e-300)
    e_tf = ((tf.double().cpu() - ref).abs() / rowmax).max().item()        # per row: the rows differ by 12 decades
    e_hf = ((hf.double().cpu() - ref).abs() / rowmax).max().item()
    print("fp16 R rows %d in %d out %d: TF32 R %.2e  fp16 R %.2e (per row, relative to the row maximum)" % (rows, inf, outf, e_tf, e_hf))
    assert torch.isfinite(hf).all() and (hf[rows // 3] == 0).all()
    assert e_hf < 3e-3 and e_hf < 1.5 * e_tf + 1e-4
    rs, hs = r.double().sum(dim=1), hf.double().cpu().sum(dim=1)          # conservation per row (Z > 0 almost surely)
    assert ((hs - rs).abs() <= 3e-3 * rs.abs() + 1e-30).all()


@pytest.mark.parametrize("rows,inf,outf", [(128, 256, 256), (394, 768, 3072), (1000, 3072, 768), (77, 768, 2304), (20000, 768, 768)])
def test_tc_fp16_single_pass_backward(rows, inf, outf):
    """TE_FLAG_BACKWARD_F16: dx = dy W as ONE fp16 MMA per k-step (te_tc_wgmma.cu): block-scaled fp16 gradient rows that
    span 12 decades, row-scaled fp16 weights.  The operands keep TF32's 11 significant bits, rounded to nearest: the error
    stays below the single-pass TF32 kernel's bound, per row."""
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(rows + 41)
    dy = torch.randn(rows, outf, generator=g) * torch.logspace(-9, 3, rows)[:, None]
    dy[rows // 3] = 0.0
    w = torch.randn(outf, inf, generator=g) * 0.05
    ref = dy.double() @ w.double()
    tf = ops.linear_backward_tf32(dy.cuda(), w.cuda())
    hf = ops.linear_backward_f16(dy.cuda(), w.cuda())
    torch.cuda.synchronize()
    rowmax = ref.abs().amax(dim=1, keepdim=True).clamp_min(1e-300)
    e_tf = ((tf.double().cpu() - ref).abs() / rowmax).max().item()
    e_hf = ((hf.double().cpu() - ref).abs() / rowmax).max().item()
    print("fp16 backward rows %d in %d out %d: TF32 %.2e  fp16 %.2e (per row, relative to the row maximum)" % (rows, inf, outf, e_tf, e_hf))
    assert torch.isfinite(hf).all() and (hf[rows // 3] == 0).all()
    assert e_hf < 2e-3 and e_hf < 1.5 * e_tf + 1e-4


def test_f16_block_split_format_bit_exact():
    """The operand format of the fp16-split forward Linear, GPU pre-pass against its CPU restatement (oracle/f16_split.py): hi, lo and
    the block scales are BIT-EXACT (integer / byte work: exact power-of-two scaling, round-to-nearest-even fp16 conversions)."""
    import numpy as np
    from oracle import f16_split as F
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(77)
    x = torch.randn(300, 768, generator=g) * torch.logspace(-3, 1, 768)
    x = x * torch.logspace(-30, 30, 300)[:, None]                # rows spanning 60 decades
    x[7] = 0.0
    x[9, 5] = float("inf")                                       # a non-finite block keeps scale 1 and propagates
    hi, lo, si = ops.f16_block_split(x.cuda())
    torch.cuda.synchronize()
    with np.errstate(invalid="ignore", over="ignore"):
        rh, rl, rs = F.split_rows(x.numpy())
    assert np.array_equal(si.cpu().numpy(), rs)
    assert np.array_equal(hi.cpu().numpy().view(np.uint16), rh.view(np.uint16))
    ok = np.ones_like(rh, dtype=bool)
    ok[9, :128] = False                                          # lo of the non-finite block is inf - inf = NaN (payload unspecified)
    assert np.array_equal(lo.cpu().numpy().view(np.uint16)[ok], rl.view(np.uint16)[ok])


# ---- fused Linear epilogues of every kernel family (te_linear_forward / te_linear_backward: no fall-back) -------------------
# Bounds per element, relative to the element's own scale |x||W|^T (+ |bias|): fp32 SIMT 3e-6 (test_tc_3xtf32_linear_is_fp32_grade),
# 3xTF32 and the fp16 split 1.5e-8 * K + 2e-6 (same test; the fp16 split keeps the 3xTF32 operand precision), single-pass
# TF32 / fp16 2e-3 (test_tc_persistent_pair_kernels).
LIN_BOUND = {"simt": lambda K: 3e-6, "3xtf32": lambda K: 1.5e-8 * K + 2e-6, "f16_split": lambda K: 1.5e-8 * K + 2e-6,
             "tf32": lambda K: 2e-3, "f16": lambda K: 2e-3}
# GELU'(x) = Phi(x) + x phi(x) in the epilogue, absolute error: the erff / expf form (every family but single-pass TF32) to a
# few fp32 ulp of values <= 1.13; te_gelu_grad_fast (single-pass TF32 backward) has erf by Abramowitz-Stegun 7.1.26 (1.5e-7
# absolute, so 7.5e-8 on Phi) with ex2.approx / rcp.approx operands.  Measured maxima over e0 in [-12, 12] on one H100 80GB HBM3
# at a 400 W power limit: 1.9e-7 (SIMT, 3xTF32, single-pass fp16), 3.2e-7 (te_gelu_grad_fast).  Measured per-element GEMM errors:
# forward y 4.3e-7 (SIMT), 6.1e-7 (3xTF32), 4.7e-7 (fp16 split); GELU_BWD at most 0.19 of its bound in every family.
GELU_GRAD_EXACT = 3e-7
GELU_GRAD_FAST = 6e-7


def elem_err(out, ref, scale):
    """largest |out - ref| over the element's own scale (fp64 ref and scale): the measure LIN_BOUND bounds"""
    return ((out.double() - ref).abs() / scale).max().item()


def _gelu64(y):
    return 0.5 * y * (1 + torch.erf(y / 2 ** 0.5))


def _gelu_grad64(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def _e0_grid(rows, cols, g):
    """GELU inputs over [-12, 12]: uniform, plus 0, +-1e-6, +-1 and the tails, where the erf approximation is weakest"""
    e0 = torch.rand(rows, cols, generator=g, device="cuda") * 24 - 12
    special = torch.tensor([0.0, 1e-6, -1e-6, 1.0, -1.0, 0.5, -0.5, 3.0, -3.0, 6.0, -6.0, 12.0, -12.0], device="cuda")
    flat = e0.view(-1)
    flat[:special.numel() * (flat.numel() // (4 * special.numel()))] = special.repeat(flat.numel() // (4 * special.numel()))
    return e0


@pytest.mark.parametrize("K", [64, 768, 3072])
@pytest.mark.parametrize("rows", [1, 77, 591, 20000])
def test_linear_forward_epilogues(rows, K):
    """BIAS_GELU (y, y2 = erf-GELU(y)) and BIAS_ADD (y, y2 = e0 + y) on fp32 SIMT, 3xTF32 and the fp16 split against fp64.
    Rows span six decades of magnitude (the fp16 split scales every 128-column block on its own)."""
    from transformer_explainability_b200 import ops
    N = 256
    g = torch.Generator(device="cuda").manual_seed(rows * 3 + K)
    x = torch.randn(rows, K, generator=g, device="cuda") * torch.logspace(-3, 3, rows, device="cuda")[:, None]
    w = torch.randn(N, K, generator=g, device="cuda") * 0.05
    b = torch.randn(N, generator=g, device="cuda") * 0.1
    e0 = torch.randn(rows, N, generator=g, device="cuda")
    y64 = x.double() @ w.double().T + b.double()
    scale = x.double().abs() @ w.double().abs().T + b.double().abs()
    for family in ("simt", "3xtf32", "f16_split"):
        bound = LIN_BOUND[family](K)
        for epi in ("bias_gelu", "bias_add"):
            y, y2 = ops.linear_forward_epi(x, w, b, e0 if epi == "bias_add" else None, epi=epi, family=family)
            torch.cuda.synchronize()
            ey = elem_err(y, y64, scale)
            if epi == "bias_gelu":      # |GELU'| <= 1.13, plus the fp32 GELU itself
                e2 = ((y2.double() - _gelu64(y64)).abs() / (1.13 * scale)).max().item()
                b2 = bound + 5e-7
            else:                       # e0 + y in fp32: one rounding of |e0| + |y|
                e2 = ((y2.double() - (e0.double() + y64)).abs() / (scale + e0.double().abs())).max().item()
                b2 = bound + 1.2e-7
            print("linear fwd %s %s rows %d K %d: y %.2e y2 %.2e (per element; bound %.1e)" % (family, epi, rows, K, ey, e2, bound))
            assert ey < bound and e2 < b2, (family, epi)


@pytest.mark.parametrize("K", [64, 768, 3072])
@pytest.mark.parametrize("rows", [1, 77, 591, 20000])
def test_linear_backward_gelu_epilogue(rows, K):
    """GELU_BWD, dx = (dy W) * GELU'(e0), on fp32 SIMT, 3xTF32, single-pass TF32 (te_gelu_grad_fast) and single-pass fp16
    against fp64, e0 over [-12, 12] with 0, +-1e-6 and the tails.  The GEMM part keeps the family's bound per element; the
    gradient itself is isolated by dividing by the same family's STORE result (the same accumulation, so the quotient is
    GELU'(e0) up to one fp32 rounding) and held to GELU_GRAD_FAST / GELU_GRAD_EXACT absolute — the exact families no worse
    than SIMT."""
    from transformer_explainability_b200 import ops
    N = 256
    g = torch.Generator(device="cuda").manual_seed(rows * 5 + K)
    dy = torch.randn(rows, K, generator=g, device="cuda")
    w = torch.randn(K, N, generator=g, device="cuda") * 0.05
    e0 = _e0_grid(rows, N, g)
    gp = _gelu_grad64(e0.double())
    v64 = dy.double() @ w.double()
    scale = dy.double().abs() @ w.double().abs()
    grad_err = {}
    for family in ("simt", "3xtf32", "tf32", "f16"):
        bound = LIN_BOUND[family](K)
        gb = GELU_GRAD_FAST if family == "tf32" else GELU_GRAD_EXACT
        dx = ops.linear_backward_epi(dy, w, e0, epi="gelu_bwd", family=family)
        v = ops.linear_backward_epi(dy, w, None, epi="store", family=family)
        torch.cuda.synchronize()
        e_full = ((dx.double() - v64 * gp).abs() / (scale * ((bound + 1.2e-7) * gp.abs() + gb))).max().item()
        live = v != 0
        ratio = dx.double()[live] / v.double()[live]
        grad_err[family] = (ratio - gp[live]).abs().max().item()
        print("linear bwd GELU_BWD %s rows %d K %d: %.2f of the bound (per element), GELU' abs err %.2e" % (
            family, rows, K, e_full, grad_err[family]))
        assert e_full < 1, family
        assert grad_err[family] < gb + 6e-8 * 1.13, family
    for family in ("3xtf32", "f16"):
        assert grad_err[family] <= grad_err["simt"] + 1.2e-7, "%s: GELU' worse than the SIMT epilogue" % family


def test_linear_epilogue_entry_points_do_not_fall_back():
    """A family that does not take the shape / epilogue is TE_ERR_UNSUPPORTED, never a silent fall-back: width 64 (BERT-tiny)
    for every tensor-core family, K % 64 != 0 for the fp16 ones."""
    from transformer_explainability_b200 import _lib, ops
    x = torch.randn(10, 96, device="cuda")
    for fam in ("3xtf32", "f16_split"):
        with pytest.raises(_lib.TeError) as ex:
            ops.linear_forward_epi(x, torch.randn(64, 96, device="cuda"), None, epi="store", family=fam)
        assert ex.value.status == _lib.TE_ERR_UNSUPPORTED
    with pytest.raises(_lib.TeError) as ex:
        ops.linear_forward_epi(x, torch.randn(128, 96, device="cuda"), None, epi="store", family="f16_split")   # K = 96
    assert ex.value.status == _lib.TE_ERR_UNSUPPORTED
    dy = torch.randn(10, 96, device="cuda")
    for fam in ("3xtf32", "tf32", "f16"):
        with pytest.raises(_lib.TeError) as ex:
            ops.linear_backward_epi(dy, torch.randn(96, 64, device="cuda"), None, epi="store", family=fam)
        assert ex.value.status == _lib.TE_ERR_UNSUPPORTED
    with pytest.raises(_lib.TeError) as ex:
        ops.linear_backward_epi(dy, torch.randn(96, 128, device="cuda"), None, epi="store", family="f16")      # K = 96
    assert ex.value.status == _lib.TE_ERR_UNSUPPORTED
    y, _ = ops.linear_forward_epi(x, torch.randn(64, 96, device="cuda"), None, epi="store", family="simt")
    assert torch.isfinite(y).all()


def test_linear_convenience_functions_fall_back_family_by_family():
    """linear_forward / linear_backward / _f16 / _tf32 fall back where the family they ask for does not take the shape:
    forward fp16 split -> 3xTF32 -> SIMT, backward fp16 or single-pass TF32 -> 3xTF32 -> SIMT.  Each result is bit-identical
    to the strict entry point run on the family it should land on: width 64 (BERT-tiny) for every tensor-core family,
    K = 96 (3xTF32 takes it, the fp16 kernels do not) and K = 128 (every family takes it)."""
    from transformer_explainability_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(7)
    rows = 77
    for K, N, f16_lands, tc_lands in ((96, 64, "simt", "simt"), (96, 128, "3xtf32", "3xtf32"),
                                      (128, 128, "f16_split", "3xtf32")):
        x = torch.randn(rows, K, generator=g, device="cuda")
        w = torch.randn(N, K, generator=g, device="cuda") * 0.05
        b = torch.randn(N, generator=g, device="cuda")
        for got, family in ((ops.linear_forward(x, w, b, tensor_cores=True), tc_lands),
                            (ops.linear_forward(x, w, b, tensor_cores=True, f16_split=True), f16_lands)):
            want, _ = ops.linear_forward_epi(x, w, b, epi="bias", family=family)
            assert torch.equal(got, want), ("forward", K, N, family)
    for K, N, f16_lands, tf32_lands, tc_lands in ((96, 64, "simt", "simt", "simt"), (96, 128, "3xtf32", "tf32", "3xtf32"),
                                                  (128, 128, "f16", "tf32", "3xtf32")):
        dy = torch.randn(rows, K, generator=g, device="cuda")
        w = torch.randn(K, N, generator=g, device="cuda") * 0.05
        for got, family in ((ops.linear_backward(dy, w, tensor_cores=True), tc_lands),
                            (ops.linear_backward_f16(dy, w), f16_lands), (ops.linear_backward_tf32(dy, w), tf32_lands)):
            assert torch.equal(got, ops.linear_backward_epi(dy, w, epi="store", family=family)), ("backward", K, N, family)


# ---- the other producers of the fp16-split operand format ----------------------------------------------------------------
@pytest.mark.parametrize("D", [768, 1024, 64])
def test_layernorm_split_format_bit_exact(D):
    """te_launch_layernorm_split (feeds every qkv / fc1 GEMM under TE_FLAG_LINEAR_F16_SPLIT): y against fp64 LayerNorm,
    mean / rstd against fp64, and hi, lo and the block scales BIT-identical to oracle/f16_split.split_rows applied to the
    kernel's own y.  Stress data as in test_f16_block_split_format_bit_exact: y spans 60 decades (through the LayerNorm
    weight), one row of x is constant (y = bias = 0: a zero row).  The y error is measured against (|x| + |mean|) rstd |w|,
    the scale the fp32 subtraction x - mean works at."""
    import numpy as np
    from oracle import f16_split as F
    from transformer_explainability_b200 import ops
    g = torch.Generator().manual_seed(D)
    rows, eps = 300, 1e-6
    x = torch.randn(rows, D, generator=g) * torch.logspace(-3, 1, D) + torch.randn(rows, 1, generator=g)
    x[7] = 0.0                                                              # constant row: y == bias
    w = (torch.randn(D, generator=g) * torch.logspace(-30, 30, D)).float()  # y spans 60 decades inside every row
    b = torch.zeros(D)
    y, mean, rstd, hi, lo, si = ops.layernorm_split(x.cuda(), w.cuda(), b.cuda(), eps)
    torch.cuda.synchronize()
    xd = x.double()
    m64 = xd.mean(1, keepdim=True)
    r64 = 1 / torch.sqrt(((xd - m64) ** 2).mean(1, keepdim=True) + eps)
    y64 = (xd - m64) * r64 * w.double() + b.double()
    ey = ((y.double().cpu() - y64).abs() / ((xd.abs() + m64.abs()) * r64 * w.double().abs() + 1e-300)).max().item()
    print("layernorm split D %d: y per element %.2e" % (D, ey))
    assert ey < 1e-5
    assert (y[7] == 0).all()
    rh, rl, rs = F.split_rows(y.cpu().numpy())
    assert np.array_equal(si.cpu().numpy(), rs)
    assert np.array_equal(hi.cpu().numpy().view(np.uint16), rh.view(np.uint16))
    assert np.array_equal(lo.cpu().numpy().view(np.uint16), rl.view(np.uint16))
    assert (si.cpu()[7] == 1).all() and (hi.cpu()[7] == 0).all()


@pytest.mark.parametrize("rows,inf,outf", [(77, 768, 2304), (591, 768, 768), (300, 3072, 768)])
def test_zplus_s1_f16_output(rows, inf, outf):
    """te_tc_zplus_s1 with S leaving as hi-only block-scaled fp16 (ZO_F16S, the A operand of te_tc_zplus_r16), against the fp32
    form of the same kernel on the same inputs.  The fp32 form is tf32(S) while the fp16 form scales the unrounded S, so they
    are not compared bit for bit.  Instead: every block scale equals the one oracle/f16_split picks from the fp32 form's block
    maximum, except where tf32 rounding lifted that maximum onto a power of two (counted: rare); hi decodes, per element, to the
    fp32 form within half an fp16 ulp plus the 2^-11 of its tf32 rounding; the fp32 form is the z+ rule's S to the TF32 bound
    (3e-3) against fp64; a zero row of R gives zero hi and the neutral scale; the scale array holds N / 128 columns per row,
    the row stride te_tc_zplus_r16 reads it with."""
    import numpy as np
    from oracle import f16_split as F
    from transformer_explainability_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(rows + inf)
    x = torch.randn(rows, inf, generator=g, device="cuda")
    w = torch.randn(outf, inf, generator=g, device="cuda") * 0.05
    b = torch.randn(outf, generator=g, device="cuda") * 0.1
    r = torch.rand(rows, outf, generator=g, device="cuda") * torch.logspace(-6, 6, rows, device="cuda")[:, None]
    r[rows // 3] = 0.0
    y = ops.linear_forward(x, w, b)
    s32 = ops.tc_zplus_s(x, w, r, y, bias=b)
    s16, sc = ops.tc_zplus_s(x, w, r, y, bias=b, f16=True)
    torch.cuda.synchronize()
    assert sc.shape == (rows, outf // 128) and torch.isfinite(sc).all(), "a block scale was not written"
    z64 = x.double().clamp(min=0) @ w.double().clamp(min=0).T + x.double().clamp(max=0) @ w.double().clamp(max=0).T
    s64 = rules.safe_divide(r.double(), z64)
    es = ((s32.double() - s64).abs() / s64.abs().clamp_min(1e-300)).max().item()
    m = s32.abs().view(rows, outf // 128, 128).amax(-1).cpu().numpy()
    _, want = F.block_scale(m)
    got = sc.cpu().numpy()
    on_pow2 = (m > 0) & (np.frexp(m)[0] == 0.5)
    mismatch = got != want
    print("zplus S fp16 rows %d in %d out %d: fp32 S vs fp64 %.1e, %d of %d block maxima on a power of two, %d scale mismatches" % (
        rows, inf, outf, es, on_pow2.sum(), m.size, mismatch.sum()))
    assert es < 3e-3
    assert not (mismatch & ~on_pow2).any(), "a block scale differs from the one the format prescribes"
    assert (got[mismatch] == 0.5 * want[mismatch]).all()                # the unrounded maximum sat just below 2^k
    assert on_pow2.sum() <= max(2, m.size // 100), "the exemption must stay rare"
    sc64 = sc.double()[..., None]
    hi = s16.double().view(rows, outf // 128, 128) * sc64
    s32b = s32.double().view(rows, outf // 128, 128)
    # fp16 spacing in [2^14, 2^15) is 16: half an ulp of the block maximum is 8 * 2^-e
    assert ((hi - s32b).abs() <= 8 * sc64 + 2.0 ** -11 * s32b.abs()).all(), "decoded hi off by more than half an fp16 ulp"
    assert (s16[rows // 3] == 0).all() and (sc[rows // 3] == 1).all()
