"""Stand-alone LRP rules and rollout on CUDA tensors (thin wrappers over the C ABI).

Each function is the CUDA counterpart of one ``relprop`` of the reference's
``modules/layers_ours.py``; see ``include/te_b200.h`` for the citations.  Only the Linear rule depends on alpha.
All inputs must be contiguous fp32 CUDA tensors; there is no CPU path.
"""
import torch

from . import _lib
from ._lib import check, ptr


import functools


def _stream():
    return _lib.ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_device(fn):
    """Run the op with the device of its first CUDA tensor argument current: the C library launches on the current
    device and the stream handed to it must belong to that device (a model on a non-current GPU otherwise fails with
    an invalid resource handle)."""
    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        dev = None
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (list, tuple)) and a and torch.is_tensor(a[0]):
                a = a[0]
            if torch.is_tensor(a) and a.is_cuda:
                dev = a.device
                break
        if dev is None:
            raise ValueError("te_b200 ops need CUDA tensors (no CPU fallback)")
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    return wrapped


def _req(*ts):
    dev = None
    for t in ts:
        if t is None:
            continue
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise ValueError("te_b200 ops need contiguous fp32 CUDA tensors (no CPU fallback)")
        if dev is not None and t.device != dev:
            raise ValueError("te_b200 ops: all tensors of one call must live on the same device")
        dev = t.device


def _same_shape(what, *ts):
    ts = [t for t in ts if t is not None]
    for t in ts[1:]:
        if t.shape != ts[0].shape:
            raise ValueError("%s: shape mismatch %s vs %s" % (what, tuple(ts[0].shape), tuple(t.shape)))


def _workspace(nbytes, device):
    return torch.empty((nbytes + 255) // 256 * 64, dtype=torch.float32, device=device)   # 256-byte multiple


def _up64(n):
    return (n + 63) // 64 * 64


def _tc_scratch(w, device, s=0, operand=0, split=None):
    """The scratch of the tensor-core stand-alone entry points for the weight w [out, in], laid out as include/te_b200.h
    documents it: [s floats of S, rounded up to 64 | 16 * in * out derived weight copies | operand floats], or with
    split = (rows, cols, hi_only) the fp16 split of a [rows, cols] operand, rounded up to 64, and its rows * ceil(cols / 128)
    block scales in place of the operand."""
    n = _up64(s) + 16 * w.numel() + operand
    if split is not None:
        rows, cols, hi_only = split
        n += _up64(rows * cols // 2 if hi_only else rows * cols) + rows * ((cols + 127) // 128)
    return torch.empty(n, device=device, dtype=torch.float32)


# ---- Linear GEMMs: te_linear_forward / te_linear_backward run the kernel family named or return TE_ERR_UNSUPPORTED ----------
LINEAR_FAMILIES = {
    "simt": 0,
    "3xtf32": _lib.FLAG_LINEAR_TENSOR_CORES,
    "f16_split": _lib.FLAG_LINEAR_TENSOR_CORES | _lib.FLAG_LINEAR_F16_SPLIT,          # forward only
    "tf32": _lib.FLAG_LINEAR_TENSOR_CORES | _lib.FLAG_BACKWARD_TF32,                  # backward only
    "f16": _lib.FLAG_LINEAR_TENSOR_CORES | _lib.FLAG_BACKWARD_F16,                    # backward only
}
LINEAR_EPI = {"store": 0, "bias": 1, "bias_gelu": 2, "bias_add": 3, "gelu_bwd": 4}
ATTN_EPI = {"store": 0, "mul": 1, "sd": 2, "softmax": 3}
# where the convenience functions fall back to when a family does not take the shape (every shape the fp16 kernels take,
# 3xTF32 takes as well)
_STEP_DOWN = {"f16_split": "3xtf32", "f16": "3xtf32", "tf32": "3xtf32", "3xtf32": "simt"}


def _linear_call(fn, args, epi, family, fall_back):
    """fn(*args, epi, the family's flags, stream); with fall_back a family that returns TE_ERR_UNSUPPORTED steps down."""
    while True:
        status = fn(*args, LINEAR_EPI[epi], LINEAR_FAMILIES[family], _stream())
        if not (fall_back and status == _lib.TE_ERR_UNSUPPORTED):
            return check(status, fn.__name__)
        family = _STEP_DOWN[family]


def _linear_forward(x, w, bias, e0, epi, family, fall_back):
    """x [rows,in] -> (y [rows,out], y2 or None), see linear_forward_epi."""
    rows, K, N = x.shape[0], x.shape[1], w.shape[0]
    y = torch.empty(rows, N, device=x.device, dtype=torch.float32)
    y2 = torch.empty_like(y) if epi in ("bias_gelu", "bias_add") else None
    scratch = _tc_scratch(w, x.device, split=(rows, K, False) if family == "f16_split" else None) if family != "simt" else None
    _linear_call(_lib.load().te_linear_forward, (ptr(x), ptr(w), ptr(bias), ptr(e0), ptr(y), ptr(y2), ptr(scratch), rows, K, N),
                 epi, family, fall_back)
    return y, y2


def _linear_backward(dy, w, e0, epi, family, fall_back):
    """dy [rows,out] -> dx [rows,in], see linear_backward_epi."""
    rows, K, N = dy.shape[0], w.shape[0], w.shape[1]
    dx = torch.empty(rows, N, device=dy.device, dtype=torch.float32)
    scratch = _tc_scratch(w, dy.device, split=(rows, K, True) if family == "f16" else None) if family != "simt" else None
    _linear_call(_lib.load().te_linear_backward, (ptr(dy), ptr(w), ptr(e0), ptr(dx), ptr(scratch), rows, N, K), epi, family,
                 fall_back)
    return dx


def _linear_backward_any(what, dy, w, family):
    """dy [...,out] -> dx [...,in] on the family, falling back where it does not take the shape."""
    _req(dy, w)
    if w.dim() != 2 or dy.shape[-1] != w.shape[0]:
        raise ValueError("%s: dy [...,out], w [out,in] expected" % what)
    dx = _linear_backward(dy.reshape(-1, dy.shape[-1]), w, None, "store", family, True)
    return dx.view(*dy.shape[:-1], w.shape[1])


@_on_device
def linear_forward(x, w, bias=None, tensor_cores=False, f16_split=False):
    """y = x W^T + b.  tensor_cores: fp32-grade 3xTF32 split on the tensor cores (shapes that do not qualify fall back);
    f16_split (with tensor_cores): the row-scaled fp16 (hi, lo) split on fp16 tensor-core MMAs (TE_FLAG_LINEAR_F16_SPLIT)."""
    _req(x, w, bias)
    if w.dim() != 2 or x.shape[-1] != w.shape[1] or (bias is not None and bias.numel() != w.shape[0]):
        raise ValueError("linear_forward: x [...,in], w [out,in], bias [out] expected")
    family = ("f16_split" if f16_split else "3xtf32") if tensor_cores else "simt"
    y, _ = _linear_forward(x.reshape(-1, x.shape[-1]), w, bias, None, "bias", family, True)
    return y.view(*x.shape[:-1], w.shape[0])


@_on_device
def f16_block_split(x):
    """The block-scaled fp16 (hi, lo) operand format of the fp16-split forward Linear: x [rows, cols] fp32 ->
    (hi, lo) fp16 [rows, cols], scale_inv fp32 [rows, ceil(cols / 128)]  (see include/te_b200.h: te_f16_block_split)."""
    _req(x)
    if x.dim() != 2 or x.shape[1] % 4 != 0:
        raise ValueError("f16_block_split: x [rows, cols] with cols % 4 == 0 expected")
    rows, cols = x.shape
    buf = torch.empty(2, rows, cols, device=x.device, dtype=torch.float16)
    scale = torch.empty(rows, (cols + 127) // 128, device=x.device, dtype=torch.float32)
    check(_lib.load().te_f16_block_split(ptr(x), rows, cols, ptr(buf[0]), ptr(buf[1]), ptr(scale), _stream()), "te_f16_block_split")
    return buf[0], buf[1], scale


@_on_device
def linear_backward(dy, w, tensor_cores=False):
    """dx = dy W  (activation gradient of a Linear; no dW on this path)."""
    return _linear_backward_any("linear_backward", dy, w, "3xtf32" if tensor_cores else "simt")


@_on_device
def linear_backward_f16(dy, w):
    """dx = dy W as a single-pass fp16 GEMM (block-scaled fp16 gradient, row-scaled fp16 weights; TE_FLAG_BACKWARD_F16)."""
    return _linear_backward_any("linear_backward_f16", dy, w, "f16")


@_on_device
def linear_backward_tf32(dy, w):
    """dx = dy W as a single-pass TF32 wgmma GEMM (what TE_FLAG_BACKWARD_TF32 selects)."""
    return _linear_backward_any("linear_backward_tf32", dy, w, "tf32")


# ---- diagnostic wrappers of the kernels (include/te_b200.h: "Diagnostic entry points"): no fall-back, a shape the requested
# kernel does not take raises TeError with status TE_ERR_UNSUPPORTED -------------------------------------------------------
@_on_device
def linear_forward_epi(x, w, bias=None, e0=None, epi="bias", family="simt"):
    """y = x W^T (+ bias) with a fused epilogue on the kernel family named (LINEAR_FAMILIES) -> (y, y2); y2 is None unless
    epi is "bias_gelu" (erf GELU of y) or "bias_add" (e0 + y)."""
    _req(x, w, bias, e0)
    if x.dim() != 2 or w.dim() != 2 or w.shape[1] != x.shape[1] or (e0 is not None and e0.shape != (x.shape[0], w.shape[0])):
        raise ValueError("linear_forward_epi: x [rows,in], w [out,in], e0 [rows,out] expected")
    return _linear_forward(x, w, bias, e0, epi, family, False)


@_on_device
def linear_backward_epi(dy, w, e0=None, epi="store", family="simt"):
    """dx = dy W, times GELU'(e0) with epi="gelu_bwd", on the kernel family named (LINEAR_FAMILIES)."""
    _req(dy, w, e0)
    if dy.dim() != 2 or w.dim() != 2 or dy.shape[1] != w.shape[0] or (e0 is not None and e0.shape != (dy.shape[0], w.shape[1])):
        raise ValueError("linear_backward_epi: dy [rows,out], w [out,in], e0 [rows,in] expected")
    return _linear_backward(dy, w, e0, epi, family, False)


@_on_device
def layernorm_split(x, w, b, eps):
    """LayerNorm of x [rows, D] that also emits the fp16-split operand of y -> (y, mean, rstd, hi, lo, scale_inv)
    (see include/te_b200.h: te_layernorm_split)."""
    _req(x, w, b)
    rows, D = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(rows, device=x.device, dtype=torch.float32)
    rstd = torch.empty_like(mean)
    buf = torch.empty(2, rows, D, device=x.device, dtype=torch.float16)
    scale = torch.empty(rows, (D + 127) // 128, device=x.device, dtype=torch.float32)
    check(_lib.load().te_layernorm_split(ptr(x), ptr(w), ptr(b), ptr(y), ptr(mean), ptr(rstd), ptr(buf[0]), ptr(buf[1]),
                                         ptr(scale), rows, D, eps, _stream()), "te_layernorm_split")
    return y, mean, rstd, buf[0], buf[1], scale


@_on_device
def tc_zplus_s(x, w, r, y, bias=None, f16=False, bf16=False):
    """S = safe_divide(r, Z) of the z+ rule on the single-pass tensor-core S kernel (Z from the saved forward output y).
    f16=False: S fp32 (TF32-rounded) [rows, out]; f16=True: (s16 fp16 [rows, out], scale_inv [rows, out / 128])."""
    _req(x, w, r, y, bias)
    if x.dim() != 2 or w.dim() != 2 or w.shape[1] != x.shape[1] or r.shape != y.shape or r.shape != (x.shape[0], w.shape[0]):
        raise ValueError("tc_zplus_s: x [rows,in], w [out,in], r / y [rows,out] expected")
    rows, K, N = x.shape[0], x.shape[1], w.shape[0]
    scratch = _tc_scratch(w, x.device, operand=rows * K)
    s = None if f16 else torch.empty(rows, N, device=x.device, dtype=torch.float32)
    s16 = torch.empty(rows, N, device=x.device, dtype=torch.float16) if f16 else None
    sc = torch.full((rows, N // 128), float("nan"), device=x.device, dtype=torch.float32) if f16 else None
    check(_lib.load().te_tc_zplus_s(ptr(x), ptr(w), ptr(bias), ptr(y), ptr(r), ptr(s), ptr(s16), ptr(sc), ptr(scratch), rows,
                                    K, N, _lib.FLAG_ZPLUS_S1_BF16 if bf16 else 0, _stream()), "te_tc_zplus_s")
    return (s16, sc) if f16 else s


def _span(t, n, what):
    """t must be an fp32 CUDA tensor (a view is fine) whose storage holds n floats from its first element."""
    if not (t.is_cuda and t.dtype == torch.float32):
        raise ValueError("%s: fp32 CUDA tensor expected" % what)
    if t.untyped_storage().nbytes() // 4 - t.storage_offset() < n:
        raise ValueError("%s: the kernel would address %d floats, the tensor's storage holds fewer" % (what, n))


@_on_device
def tc_attention_nn(a, lda, b, ldb, batch, heads, n, dh, out, ld_out, e=None, alpha=1.0, epi="store", single_pass=False):
    """out[b,h,i,j] = epi(alpha * sum_d a[b*n+i, h*dh+d] b[b*n+j, h*dh+d]) on the tensor-core N x N kernel, in place into out
    ([batch, heads, n, ld_out] storage).  a / b: the first element of head 0 of packed rows (views into [rows, 3D] allowed)."""
    _span(a, (batch * n - 1) * lda + heads * dh, "a")
    _span(b, (batch * n - 1) * ldb + heads * dh, "b")
    for t, nm in ((out, "out"), (e, "e")):
        if t is not None:
            _span(t, (batch * heads * n - 1) * ld_out + ((n + 3) & ~3), nm)
    check(_lib.load().te_tc_attention_nn(ptr(a), lda, ptr(b), ldb, batch, heads, n, dh, ptr(out), ld_out, ptr(e), alpha,
                                         ATTN_EPI[epi], int(single_pass), _stream()), "te_tc_attention_nn")
    return out


@_on_device
def tc_attention_nk(amap, np_, amn, x, ldx, batch, heads, n, out, ld_out, e=None, alpha=1.0, epi="store", single_pass=False):
    """out[b*n+m, h*64+d] = epi(alpha * sum_k M_h[m,k] x[b*n+k, h*64+d]), M_h = amap[b,h] ([n, np]) or its transpose (amn=1), on
    the tensor-core token-reduction kernel, in place into out (packed rows of stride ld_out)."""
    _span(amap, batch * heads * n * np_, "map")
    _span(x, (batch * n - 1) * ldx + heads * 64, "x")
    for t, nm in ((out, "out"), (e, "e")):
        if t is not None:
            _span(t, (batch * n - 1) * ld_out + heads * 64, nm)
    check(_lib.load().te_tc_attention_nk(ptr(amap), np_, amn, ptr(x), ldx, batch, heads, n, ptr(out), ld_out, ptr(e), alpha,
                                         ATTN_EPI[epi], int(single_pass), _stream()), "te_tc_attention_nk")
    return out


@_on_device
def linear_relprop(x, w, r, tensor_cores=False, y=None, bias=None, bf16=False, variant="ours", r_f16=False, alpha=1.0):
    """``Linear.relprop(R, alpha)`` (layers_ours.py:207-230): x [...,in], w [out,in], r [...,out] -> [...,in].
    y / bias: the layer's saved forward output (and bias) — lets the tensor-core path form the denominator in one pass.
    variant="lrp": the rule of ``modules/layers_lrp.py:187-210`` (separate denominators; fp32 SIMT); variant="lrp_tc": the
    same rule on single-pass TF32 tensor cores (TE_FLAG_RULES_LRP_TC; in / out multiples of 128, other shapes run the SIMT
    rule; tensor_cores, y, bias, bf16 and r_f16 do not apply to either).
    alpha: the LRP-alpha-beta rule, beta = alpha - 1: alpha * activator - beta * inhibitor relevance (the inhibitor is the
    same rule with the weight signs swapped); alpha=1 is the z+ rule.  A non-finite alpha raises."""
    _req(x, w, r, y, bias)
    if (w.dim() != 2 or x.shape[-1] != w.shape[1] or r.shape[-1] != w.shape[0] or r.shape[:-1] != x.shape[:-1]
            or (y is not None and y.shape != r.shape) or (bias is not None and bias.numel() != w.shape[0])):
        raise ValueError("linear_relprop: x [...,in], w [out,in], r / y [...,out], bias [out] expected")
    rows = x.numel() // x.shape[-1]
    out = torch.empty_like(x)
    if variant == "lrp_tc":
        scratch = _tc_scratch(w, x.device, s=rows * w.shape[0])
        check(_lib.load().te_linear_relprop(ptr(x), ptr(w), None, None, ptr(r), ptr(out), ptr(scratch), rows, x.shape[-1],
                                            w.shape[0], float(alpha), _lib.FLAG_RULES_LRP | _lib.FLAG_RULES_LRP_TC, _stream()),
              "te_linear_relprop")
        return out
    if tensor_cores:
        scratch = _tc_scratch(w, x.device, s=rows * w.shape[0], operand=x.numel())
    else:
        scratch = torch.empty(rows * w.shape[0], device=x.device, dtype=torch.float32)
    flags = _lib.FLAG_ZPLUS_TENSOR_CORES if tensor_cores else 0
    if r_f16:
        flags |= _lib.FLAG_ZPLUS_R_F16
    if bf16 == "s1":
        flags |= _lib.FLAG_ZPLUS_S1_BF16              # bf16 operands for the |x||W|^T term of the single-pass denominator
    elif bf16:
        flags |= _lib.FLAG_ZPLUS_BF16
    if variant == "lrp":
        flags, y = _lib.FLAG_RULES_LRP, None
    elif variant != "ours":
        raise ValueError("variant: 'ours', 'lrp' or 'lrp_tc'")
    # y None: the two-pass rule; y given: the single-pass form
    check(_lib.load().te_linear_relprop(ptr(x), ptr(w), ptr(bias) if y is not None else None, ptr(y), ptr(r), ptr(out),
                                        ptr(scratch), rows, x.shape[-1], w.shape[0], float(alpha), flags, _stream()),
          "te_linear_relprop")
    return out


@_on_device
def add_relprop(x1, x2, r, variant="ours"):
    """``Add.relprop`` (layers_ours.py:97-120), sums per sample (dim 0).  variant="lrp": ``modules/layers_lrp.py:98-100``
    (x1*S, x2*S with S = sd(r, x1+x2); no ratio normalisation)."""
    _req(x1, x2, r)
    _same_shape("add_relprop", x1, x2, r)           # a broadcast operand (pos_embed [1,N,D]) must be expanded by the caller
    if (x1.numel() // max(x1.shape[0], 1)) % 4 != 0:
        raise ValueError("add_relprop: elements per sample must be a multiple of 4")
    b = x1.shape[0]
    r1, r2 = torch.empty_like(x1), torch.empty_like(x1)
    scratch = None if variant == "lrp" else torch.empty(b * 48, device=x1.device, dtype=torch.float64)
    check(_lib.load().te_add_relprop(ptr(x1), ptr(x2), ptr(r), ptr(r1), ptr(r2), ptr(scratch), b, x1.numel() // b,
                                     _stream()), "te_add_relprop")
    return r1, r2


@_on_device
def clone_relprop(x, rs):
    """``Clone.relprop`` (layers_ours.py:151-169) for 2 or 3 branches."""
    rs = list(rs)
    _req(x, *rs)
    if len(rs) not in (2, 3):
        raise ValueError("clone_relprop: 2 or 3 branches")
    _same_shape("clone_relprop", x, *rs)
    out = torch.empty_like(x)
    r3 = rs[2] if len(rs) > 2 else None
    check(_lib.load().te_clone_relprop(ptr(x), ptr(rs[0]), ptr(rs[1]), ptr(r3), ptr(out), x.numel(), _stream()),
          "te_clone_relprop")
    return out


@_on_device
def index_select_relprop(x, r):
    """``IndexSelect.relprop`` (layers_ours.py:129-147), dim=1, index 0: x [B,N,D], r [B,1,D]|[B,D]."""
    if x.dim() != 3 or r.numel() != x.shape[0] * x.shape[2]:
        raise ValueError("index_select_relprop: x [B,N,D], r [B,1,D] expected")
    r = r.reshape(x.shape[0], x.shape[2]).contiguous()
    _req(x, r)
    out = torch.empty_like(x)
    check(_lib.load().te_index_select_relprop(ptr(x), ptr(r), ptr(out), x.shape[0], x.shape[1], x.shape[2], _stream()),
          "te_index_select_relprop")
    return out


@_on_device
def matmul_av_relprop(p, v, r):
    """``einsum('bhij,bhjd->bhid').relprop``: returns UN-halved (R_attn, R_v)."""
    _req(p, v, r)
    if v.dim() != 4 or p.shape != v.shape[:2] + (v.shape[2], v.shape[2]):
        raise ValueError("matmul_av_relprop: p [B,H,N,N], v [B,H,N,d], r [B,H,N,d] expected")
    _same_shape("matmul_av_relprop", v, r)
    b, h, n, d = v.shape
    rp, rv = torch.empty_like(p), torch.empty_like(v)
    scratch = torch.empty(b * h * n * d, device=p.device, dtype=torch.float32)
    check(_lib.load().te_matmul_av_relprop(ptr(p), ptr(v), ptr(r), ptr(rp), ptr(rv), ptr(scratch), b * h, n, d,
                                           _stream()), "te_matmul_av_relprop")
    return rp, rv


@_on_device
def matmul_qk_relprop(q, k, r):
    """``einsum('bhid,bhjd->bhij').relprop``: returns UN-halved (R_q, R_k)."""
    _req(q, k, r)
    if q.dim() != 4 or r.shape != q.shape[:2] + (q.shape[2], q.shape[2]):
        raise ValueError("matmul_qk_relprop: q, k [B,H,N,d], r [B,H,N,N] expected")
    _same_shape("matmul_qk_relprop", q, k)
    b, h, n, d = q.shape
    rq, rk = torch.empty_like(q), torch.empty_like(k)
    scratch = torch.empty(b * h * n * n, device=q.device, dtype=torch.float32)
    check(_lib.load().te_matmul_qk_relprop(ptr(q), ptr(k), ptr(r), ptr(rq), ptr(rk), ptr(scratch), b * h, n, d,
                                           _stream()), "te_matmul_qk_relprop")
    return rq, rk


def _attn_layout(t):
    """[B,H,N,N] view (row stride ld >= N, as handed out by the engine accessors) -> (tensor, ld)."""
    if t.dim() != 4 or t.shape[-1] != t.shape[-2] or t.dtype != torch.float32 or not t.is_cuda:
        raise ValueError("expected an fp32 CUDA tensor [B,H,N,N]")
    B, H, N, _ = t.shape
    ld = t.stride(2)
    if t.stride(3) != 1 or ld < N or t.stride(1) != N * ld or t.stride(0) != H * N * ld:
        t = t.contiguous()
        ld = N
    return t, ld


@_on_device
def head_reduce(a, g=None, head_weight=None, mode="mean"):
    """Reduce an attention-shaped tensor over its heads: a [B,H,N,N] (optionally * g, * head_weight[B,H]) -> [B,N,N].
    mode: "mean" | "relu_mean" (``clamp(min=0).mean(heads)``) | "mean_relu" (``mean(heads).clamp(min=0)``)."""
    a, ld = _attn_layout(a)
    if g is not None:
        g, ldg = _attn_layout(g)
        if ldg != ld:
            a, g, ld = a.contiguous(), g.contiguous(), a.shape[-1]
    B, H, N, _ = a.shape
    if head_weight is not None:
        _req(head_weight)
    out = torch.empty(B, N, N, device=a.device, dtype=torch.float32)
    m = {"mean": 0, "relu_mean": 1, "mean_relu": 2}[mode]
    check(_lib.load().te_head_reduce(ptr(a), ptr(g), ptr(head_weight), B, H, N, ld, m, ptr(out), _stream()),
          "te_head_reduce")
    return out


@_on_device
def head_region_mean(g, rows=None, cols=None):
    """``g[b,h, rows, cols].mean()`` per (b,h): [B,H,N,N] -> [B,H] (``grad.mean(dim=[1,2])`` of the GradCAM baselines)."""
    g, ld = _attn_layout(g)
    B, H, N, _ = g.shape
    r0, r1 = rows if rows is not None else (0, N)
    c0, c1 = cols if cols is not None else (0, N)
    out = torch.empty(B, H, device=g.device, dtype=torch.float32)
    check(_lib.load().te_head_region_mean(ptr(g), B, H, N, ld, r0, r1, c0, c1, ptr(out), _stream()), "te_head_region_mean")
    return out


@_on_device
def patch_embed_relprop(images, weight, r, per_channel=True):
    """``PatchEmbed.relprop`` -> ``Conv2d.relprop`` z^B branch (ViT_LRP.py:238-242, layers_ours.py:242-259).
    images [B,C,S,S]; weight [D,C,P,P] (or flattened [D,C*P*P]); r [B,(S/P)^2,D] -> [B,C,S,S] (or [B,S,S] channel sum)."""
    _req(images, weight, r)
    B, C, S, _ = images.shape
    D = weight.shape[0]
    P = int(round((weight.numel() // (D * C)) ** 0.5))
    lib = _lib.load()
    nbytes = check(lib.te_patch_embed_relprop_workspace_bytes(B, C, S, P, D), "te_patch_embed_relprop_workspace_bytes")
    ws = _workspace(nbytes, images.device)
    out = torch.empty((B, C, S, S) if per_channel else (B, S, S), device=images.device, dtype=torch.float32)
    check(lib.te_patch_embed_relprop(ptr(images), ptr(weight), ptr(r), B, C, S, P, D, ptr(out) if per_channel else None,
                                     None if per_channel else ptr(out), ptr(ws), ws.numel() * 4, _stream()),
          "te_patch_embed_relprop")
    return out


@_on_device
def attribution_rollout(grad, cam, start_layer=0, normalize=False, fused=False, want_joint=True):
    """grad, cam [L,B,H,N,N] -> (joint [B,N,N] or None, row0 [B,N]).
    ``ViT_LRP.py:357-368`` (normalize=False) / ``ExplanationGenerator.py:47-57`` (normalize=True)."""
    _req(grad, cam)
    _same_shape("attribution_rollout", grad, cam)
    if grad.dim() != 5 or grad.shape[4] < grad.shape[3]:
        raise ValueError("attribution_rollout: grad, cam [L,B,H,N,ld] with ld >= N expected")
    L, B, H, N, ld = grad.shape
    lib = _lib.load()
    nbytes = check(lib.te_rollout_workspace_bytes(L, B, N), "te_rollout_workspace_bytes")
    ws = _workspace(nbytes, grad.device)
    joint = torch.empty(B, N, N, device=grad.device, dtype=torch.float32) if want_joint else None
    row0 = torch.empty(B, N, device=grad.device, dtype=torch.float32)
    flags = _lib.FLAG_ROLLOUT_FUSED if fused else 0
    check(lib.te_attribution_rollout(ptr(grad), ptr(cam), L, B, H, N, ld, start_layer, int(normalize), flags, ptr(joint),
                                     ptr(row0), ptr(ws), ws.numel() * 4, _stream()), "te_attribution_rollout")
    return joint, row0


@_on_device
def compute_rollout_attention(all_layer_matrices, start_layer=0, normalize=False):
    """``compute_rollout_attention`` (ViT_LRP.py:38-49; BERT variant with normalize=True,
    ExplanationGenerator.py:7-18): list of [B,N,N] -> [B,N,N]."""
    mats = torch.stack([m.to(torch.float32) for m in all_layer_matrices]).contiguous()
    _req(mats)
    L, B, N, _ = mats.shape
    lib = _lib.load()
    nbytes = check(lib.te_rollout_workspace_bytes(L, B, N), "te_rollout_workspace_bytes")
    ws = _workspace(nbytes, mats.device)
    joint = torch.empty(B, N, N, device=mats.device, dtype=torch.float32)
    check(lib.te_compute_rollout_attention(ptr(mats), L, B, N, start_layer, int(normalize), ptr(joint), ptr(ws),
                                           ws.numel() * 4, _stream()), "te_compute_rollout_attention")
    return joint


# ---- perturbation evaluation (baselines/ViT/pertubation_eval_from_hdf5.py) ------------------------------------------------
@_on_device
def perturb_images(images, saliency, ks, negate=False, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    """Every perturbed, normalised input of a batch: images [B,C,H,W] (or [B,C,P]) in [0, 1], saliency [B,H,W] / [B,1,H,W] /
    [B,P], ks non-decreasing pixel counts -> out [S,B,C,H,W] (or [S,B,C,P]).  Step i removes the ks[i] pixels that come first
    in the order NaN, descending (negate ? -s : s), ascending pixel index, and normalises ((x - mean) / std, fp32)
    (see include/te_b200.h: te_perturb_images)."""
    _req(images, saliency)
    if images.dim() < 3:
        raise ValueError("perturb_images: images [B,C,H,W] or [B,C,P] expected")
    B, C = images.shape[0], images.shape[1]
    P = images[0, 0].numel()
    if saliency.shape[0] != B or saliency.numel() != B * P:
        raise ValueError("perturb_images: saliency must hold one value per pixel of each sample, got %s for images %s"
                         % (tuple(saliency.shape), tuple(images.shape)))
    ks = [int(k) for k in ks]
    if len(mean) != C or len(std) != C:
        raise ValueError("perturb_images: mean / std need one value per channel")
    lib = _lib.load()
    nbytes = check(lib.te_perturb_workspace_bytes(B, P), "te_perturb_workspace_bytes")
    ws = _workspace(nbytes, images.device)
    out = torch.empty((len(ks),) + tuple(images.shape), device=images.device, dtype=torch.float32)
    ks_c = (_lib.c_int * max(len(ks), 1))(*ks)
    mean_c = (_lib.c_float * C)(*[float(m) for m in mean])
    std_c = (_lib.c_float * C)(*[float(s) for s in std])
    check(lib.te_perturb_images(ptr(images), ptr(saliency), B, C, P, ks_c, len(ks), int(bool(negate)), mean_c, std_c, ptr(out),
                                ptr(ws), ws.numel() * 4, _stream()), "te_perturb_images")
    return out


@_on_device
def logit_stats(logits, target):
    """Per row of logits [R,K] and target [R]: (pred int32, max_logit, max_prob, dissim) with dissim =
    log(p_target / p_second) in fp32 (see include/te_b200.h: te_logit_stats)."""
    _req(logits)
    if logits.dim() != 2 or target.dim() != 1 or target.shape[0] != logits.shape[0] or not target.is_cuda:
        raise ValueError("logit_stats: logits [R,K] and a CUDA target [R] expected")
    if target.device != logits.device:
        raise ValueError("te_b200 ops: all tensors of one call must live on the same device")
    R, K = logits.shape
    t = target.to(torch.int32).contiguous()
    pred = torch.empty(R, device=logits.device, dtype=torch.int32)
    max_logit, max_prob, dissim = (torch.empty(R, device=logits.device, dtype=torch.float32) for _ in range(3))
    check(_lib.load().te_logit_stats(ptr(logits), ptr(t), R, K, ptr(pred), ptr(max_logit), ptr(max_prob), ptr(dissim),
                                     _stream()), "te_logit_stats")
    return pred, max_logit, max_prob, dissim


@_on_device
def class_probs(logits, out=None):
    """The fp32 softmax of each row of logits [R, K] (see include/te_b200.h: te_class_probs); ``out`` [R, K] fp32 may be
    given (a view into a larger buffer, contiguous)."""
    _req(logits)
    if logits.dim() != 2 or logits.shape[0] == 0:
        raise ValueError("class_probs: logits [R, K] with R > 0 expected")
    out = torch.empty_like(logits) if out is None else out
    _req(out)
    if out.shape != logits.shape or out.device != logits.device:
        raise ValueError("class_probs: out must be [R, K] on the logits' device")
    R, K = logits.shape
    check(_lib.load().te_class_probs(ptr(logits), R, K, ptr(out), _stream()), "te_class_probs")
    return out


# ---- segmentation evaluation (baselines/ViT/imagenet_seg_eval.py) ----------------------------------------------------------
def _req_u32(t, what):
    if not (t.is_cuda and t.dtype in (torch.int32, torch.uint32) and t.is_contiguous()):
        raise ValueError("%s: a contiguous int32 / uint32 CUDA tensor expected" % what)


@_on_device
def seg_metrics(maps, labels, grid=14, scale=16, thr=0.0, pr_keys=False):
    """Per sample of maps [B, grid*grid] (any shape with B leading) and labels [B, P] (0 / 1, any integer dtype),
    P = (grid*scale)^2: the mean threshold of the min-max normalised, up-sampled map, the confusion counts of Res > mean,
    the average precision of the two score channels and, with ``pr_keys``, the PR-curve keys of the sample
    (see include/te_b200.h: te_seg_metrics).  Returns a dict of CUDA tensors: ``mean`` fp32 [B], ``counts`` int64 [B,4]
    (TP, FP, FN, TN), ``row_counts`` int32 [B, grid*scale, 3] (TP, FP, FN per image row), ``ap`` fp64 [B], ``degenerate`` int32 [B], ``invalid`` int64 [B], ``pr_keys`` int32 [B,P] (bit
    patterns of uint32 keys) or None."""
    B = maps.shape[0]
    m = maps.reshape(B, -1)
    _req(m)
    if m.shape[1] != grid * grid:
        raise ValueError("seg_metrics: maps must hold grid*grid = %d values per sample, got %d" % (grid * grid, m.shape[1]))
    P = (grid * scale) ** 2
    if not labels.is_cuda or labels.device != m.device or labels.shape[0] != B or labels.numel() != B * P:
        raise ValueError("seg_metrics: labels [B, %d] on the maps' device expected" % P)
    lab = labels.reshape(B, P).to(torch.int32).contiguous()
    lib = _lib.load()
    ws = _workspace(check(lib.te_seg_workspace_bytes(B, grid, scale), "te_seg_workspace_bytes"), m.device)
    dev = m.device
    out = {"mean": torch.empty(B, device=dev, dtype=torch.float32),
           "counts": torch.empty(B, 4, device=dev, dtype=torch.int64),
           "row_counts": torch.empty(B, grid * scale, 3, device=dev, dtype=torch.int32),
           "ap": torch.empty(B, device=dev, dtype=torch.float64),
           "degenerate": torch.empty(B, device=dev, dtype=torch.int32),
           "invalid": torch.empty(B, device=dev, dtype=torch.int64),
           "pr_keys": torch.empty(B, P, device=dev, dtype=torch.int32) if pr_keys else None}
    check(lib.te_seg_metrics(ptr(m), ptr(lab), B, grid, scale, float(thr), ptr(out["mean"]), ptr(out["counts"]), ptr(out["row_counts"]),
                             ptr(out["ap"]),
                             ptr(out["degenerate"]), ptr(out["invalid"]), ptr(out["pr_keys"]), ptr(ws), ws.numel() * 4,
                             _stream()), "te_seg_metrics")
    return out


@_on_device
def sort_keys(keys, segments=1, out=None):
    """Stable ascending sort of uint32 keys (int32 / uint32 tensor holding the bit patterns), each of ``segments`` equal
    segments on its own (see include/te_b200.h: te_sort_keys_u32).  ``out`` may be ``keys`` (in place)."""
    _req_u32(keys, "sort_keys")
    n = keys.numel()
    out = torch.empty_like(keys) if out is None else out
    _req_u32(out, "sort_keys")
    if out.numel() != n:
        raise ValueError("sort_keys: out must hold as many keys as the input")
    lib = _lib.load()
    ws = _workspace(check(lib.te_sort_workspace_bytes(n, segments), "te_sort_workspace_bytes"), keys.device)
    check(lib.te_sort_keys_u32(ptr(keys), ptr(out), n, segments, ptr(ws), ws.numel() * 4, _stream()), "te_sort_keys_u32")
    return out


@_on_device
def pr_curve(sorted_keys):
    """sklearn's ``_binary_clf_curve`` over ascending-sorted keys (``sort_keys``): (thresholds fp32, tps int64, fps int64),
    one entry per distinct score in descending score order (see include/te_b200.h: te_pr_curve)."""
    _req_u32(sorted_keys, "pr_curve")
    n = sorted_keys.numel()
    dev = sorted_keys.device
    if n == 0:
        return (torch.empty(0, device=dev), torch.empty(0, device=dev, dtype=torch.int64),
                torch.empty(0, device=dev, dtype=torch.int64))
    lib = _lib.load()
    ws = _workspace(check(lib.te_pr_curve_workspace_bytes(n), "te_pr_curve_workspace_bytes"), dev)
    thr = torch.empty(n, device=dev, dtype=torch.float32)
    tps = torch.empty(n, device=dev, dtype=torch.int64)
    fps = torch.empty(n, device=dev, dtype=torch.int64)
    count = torch.empty(1, device=dev, dtype=torch.int64)
    check(lib.te_pr_curve(ptr(sorted_keys), n, ptr(thr), ptr(tps), ptr(fps), ptr(count), ptr(ws), ws.numel() * 4, _stream()),
          "te_pr_curve")
    k = int(count.item())
    return thr[:k], tps[:k], fps[:k]


# ---- ERASER rationale evaluation (BERT_rationale_benchmark/models/pipeline/bert_pipeline.py, metrics.py) ---------------------
def _host_i32(a, what, cols=None, op="eraser_rationales"):
    import numpy as np
    a = np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1, cols) if cols else np.asarray(a, dtype=np.int64))
    if a.size and (a.min() < -2 ** 31 or a.max() >= 2 ** 31):
        raise ValueError("%s: %s outside the int32 range" % (op, what))
    return np.ascontiguousarray(a.astype(np.int32))


@_on_device
def eraser_rationales(maps, piece_ranges, word_offsets, spans, span_offsets, ks, thresholds=(0.5,)):
    """Per document b of maps [B, S] (padded rows, fp32 CUDA): the word scores (max of the clamped map over each word's
    inclusive piece range ``piece_ranges[word_offsets[b]:word_offsets[b+1]]``), the top-kmax word order (NaN first, then
    descending score, then ascending word index) and per k the counts (n_pred, tok_hits, span_hits, iou_hits per
    threshold) against the truth spans ``spans[span_offsets[b]:span_offsets[b+1]]`` of (start, end) word indices
    (see include/te_b200.h: te_eraser_rationales).  The ranges, spans, offsets, ks and thresholds are host sequences.
    Returns a dict of CUDA tensors: ``word_scores`` fp32 [words], ``order`` int32 [B, max(ks)] (-1 past the last word),
    ``counts`` int32 [B, len(ks), 3 + len(thresholds)]."""
    import numpy as np
    _req(maps)
    if maps.dim() != 2:
        raise ValueError("eraser_rationales: maps [B, S] expected")
    B, S = maps.shape
    woff = _host_i32(word_offsets, "word_offsets")
    soff = _host_i32(span_offsets, "span_offsets")
    if woff.shape != (B + 1,) or soff.shape != (B + 1,):
        raise ValueError("eraser_rationales: word_offsets and span_offsets need B + 1 = %d entries" % (B + 1))
    ranges = _host_i32(piece_ranges, "piece_ranges", 2)
    sp = _host_i32(spans, "spans", 2)
    if len(ranges) != int(woff[-1]) or len(sp) != int(soff[-1]):
        raise ValueError("eraser_rationales: %d piece ranges / %d spans, the offsets end at %d / %d"
                         % (len(ranges), len(sp), woff[-1], soff[-1]))
    ks = [int(k) for k in ks]
    thr = np.ascontiguousarray(np.asarray([float(t) for t in thresholds], dtype=np.float64))
    if not 0 < len(ks) <= _lib.ERASER_MAX_KS or len(thr) > _lib.ERASER_MAX_THRESHOLDS:
        raise ValueError("eraser_rationales: 1..%d ks and at most %d thresholds expected"
                         % (_lib.ERASER_MAX_KS, _lib.ERASER_MAX_THRESHOLDS))
    lib = _lib.load()
    ws = _workspace(check(lib.te_eraser_workspace_bytes(B, len(ranges), len(sp)), "te_eraser_workspace_bytes"), maps.device)
    dev = maps.device
    out = {"word_scores": torch.empty(len(ranges), device=dev, dtype=torch.float32),
           "order": torch.empty(B, max(max(ks), 0), device=dev, dtype=torch.int32),
           "counts": torch.empty(B, len(ks), 3 + len(thr), device=dev, dtype=torch.int32)}
    ks_c = (_lib.c_int * len(ks))(*ks)
    host = lambda a: a.ctypes.data_as(_lib.c_void_p) if a.size else None      # noqa: E731
    check(lib.te_eraser_rationales(ptr(maps), B, S, host(woff), host(ranges), host(soff), host(sp), ks_c, len(ks), host(thr),
                                   len(thr), ptr(out["word_scores"]) if len(ranges) else None,
                                   ptr(out["order"]) if max(ks) > 0 else None, ptr(out["counts"]), ptr(ws), ws.numel() * 4,
                                   _stream()), "te_eraser_rationales")
    return out


@_on_device
def eraser_reduce_inputs(maps, input_ids, lengths, piece_ranges, word_offsets, n_select):
    """The comprehensiveness and sufficiency rows of each document b of maps [B, S] (fp32 CUDA) and input_ids [B, S]
    (int64 CUDA) for each selection size ``n_select[b][j]`` (host [B, J], 0 <= n <= W): the words are ranked as
    ``eraser_rationales`` ranks them; the sufficiency row is [CLS], the inner pieces held by a word of the first n ranks,
    [SEP]; the comprehensiveness row is [CLS], the other inner pieces, [SEP] (see include/te_b200.h:
    te_eraser_reduce_inputs).  lengths [B], the ranges and offsets are host sequences.  Returns a dict of CUDA tensors:
    ``ids`` int64 [B, J, 2, S] (comprehensiveness, sufficiency; zero past each length), ``lengths`` int32 [B, J, 2]."""
    _req(maps)
    if maps.dim() != 2:
        raise ValueError("eraser_reduce_inputs: maps [B, S] expected")
    B, S = maps.shape
    if not (input_ids.is_cuda and input_ids.dtype == torch.int64 and input_ids.is_contiguous()) or \
            input_ids.shape != maps.shape or input_ids.device != maps.device:
        raise ValueError("eraser_reduce_inputs: input_ids int64 [B, S] contiguous on the maps' device expected")
    op = "eraser_reduce_inputs"
    lens = _host_i32(lengths, "lengths", op=op)
    woff = _host_i32(word_offsets, "word_offsets", op=op)
    nsel = _host_i32(n_select, "n_select", op=op)
    if lens.shape != (B,) or woff.shape != (B + 1,):
        raise ValueError("eraser_reduce_inputs: lengths need B = %d and word_offsets B + 1 entries" % B)
    if nsel.ndim != 2 or nsel.shape[0] != B or not 0 < nsel.shape[1] <= _lib.ERASER_MAX_SELECTIONS:
        raise ValueError("eraser_reduce_inputs: n_select [B, J] with 1 <= J <= %d expected" % _lib.ERASER_MAX_SELECTIONS)
    ranges = _host_i32(piece_ranges, "piece_ranges", 2, op=op)
    if len(ranges) != int(woff[-1]):
        raise ValueError("eraser_reduce_inputs: %d piece ranges, the offsets end at %d" % (len(ranges), woff[-1]))
    J = nsel.shape[1]
    lib = _lib.load()
    ws = _workspace(check(lib.te_eraser_reduce_workspace_bytes(B, len(ranges), J), "te_eraser_reduce_workspace_bytes"),
                    maps.device)
    out = {"ids": torch.empty(B, J, 2, S, device=maps.device, dtype=torch.int64),
           "lengths": torch.empty(B, J, 2, device=maps.device, dtype=torch.int32)}
    host = lambda a: a.ctypes.data_as(_lib.c_void_p) if a.size else None      # noqa: E731
    check(lib.te_eraser_reduce_inputs(ptr(maps), ptr(input_ids), B, S, host(lens), host(woff), host(ranges), host(nsel), J,
                                      ptr(out["ids"]), ptr(out["lengths"]), ptr(ws), ws.numel() * 4, _stream()),
          "te_eraser_reduce_inputs")
    return out


# ---- input preparation (baselines/ViT/generate_visualizations.py: Resize((224, 224)) + ToTensor()) ---------------------------
@_on_device
def prepare_images(packed_u8, sizes, offsets, out_hw=(224, 224), mean=None, std=None):
    """A ragged batch of decoded RGB images, HWC uint8 each, packed into the 1-D uint8 CUDA tensor ``packed_u8`` at byte
    ``offsets[b]`` with ``sizes[b] = (h, w)`` (host sequences), resized to ``out_hw`` exactly as
    ``PIL.Image.resize((w, h), BILINEAR)`` does (see include/te_b200.h: te_prepare_images).  Returns ``(out01, out_norm)``:
    fp32 CUDA [B, 3, h, w], out01 = ``ToTensor()`` of the resized image and out_norm = (out01 - mean) / std, None unless
    ``mean`` and ``std`` (three values each) are given."""
    import numpy as np
    if not (packed_u8.is_cuda and packed_u8.dtype == torch.uint8 and packed_u8.dim() == 1 and packed_u8.is_contiguous()):
        raise ValueError("prepare_images: packed_u8 must be a contiguous 1-D uint8 CUDA tensor")
    sz = _host_i32(sizes, "sizes", 2, op="prepare_images")
    off = np.ascontiguousarray(np.asarray(offsets, dtype=np.int64).reshape(-1))
    B = len(sz)
    if B == 0 or off.shape != (B,):
        raise ValueError("prepare_images: sizes [B, 2] and offsets [B] with B >= 1 expected")
    if (mean is None) != (std is None) or (mean is not None and (len(mean) != 3 or len(std) != 3)):
        raise ValueError("prepare_images: mean and std are given together, three values each")
    oh, ow = (int(v) for v in out_hw)
    lib = _lib.load()
    nbytes = check(lib.te_prepare_images_workspace_bytes(B, int(sz[:, 0].max()), int(sz[:, 1].max()), oh, ow),
                   "te_prepare_images_workspace_bytes")
    dev = packed_u8.device
    ws = _workspace(nbytes, dev)
    out01 = torch.empty(B, 3, oh, ow, device=dev, dtype=torch.float32)
    out_norm = None if mean is None else torch.empty_like(out01)
    mean_c = None if mean is None else (_lib.c_float * 3)(*[float(m) for m in mean])
    std_c = None if std is None else (_lib.c_float * 3)(*[float(s) for s in std])
    host = lambda a: a.ctypes.data_as(_lib.c_void_p)      # noqa: E731
    check(lib.te_prepare_images(ptr(packed_u8), packed_u8.numel(), B, host(sz), host(off), oh, ow, mean_c, std_c, ptr(out01),
                                ptr(out_norm), ptr(ws), ws.numel() * 4, _stream()), "te_prepare_images")
    return out01, out_norm
