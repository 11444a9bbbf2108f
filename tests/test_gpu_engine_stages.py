"""GPU: every forward, backward and relprop stage of the ViT and BERT engines against fp64 evaluated on the engine's own
saved tensors (teacher forcing).

The façade tests (test_gpu_parity_full.py, test_gpu_methods_tc.py) compare against an fp64 oracle that runs its own
forward, and the relprop chain amplifies any difference between the two forwards, so their bounds are loose (5e-3 of the
tensor maximum at tensor-core flags).  Here the engine is driven directly (``forward``, then ``attribute``) and every
stage is recomputed in fp64 from the engine's own fp32 input to that stage, read through ``te_*_tensor``:

a. forward, per layer: the token assembly (ViT: im2col, patch GEMM, cls / dist / pos; BERT: embeddings + LayerNorm),
   every LayerNorm (output, mean, rstd), qkv, P (softmax, the BERT key mask, pad columns +0.0), ctx = P V, the proj /
   dense output and its residual sum, fc1 and its GELU, fc2 and its residual sum, the final LayerNorm / pooler, logits.
   Per element, over the scale models of the ops tests: ``LIN_BOUND[family](K)`` over |x||W|^T + |b| (+ |residual|),
   the GELU epilogue bound of test_gpu_reduction_tails.py, the LayerNorm bound of test_gpu_tc.py, ``bound_3x`` and the
   softmax bound of test_gpu_tma_attention.py.  The family of each launch follows from the flags (te_engine_util.h).
b. class-gradient backward: from ``x_last`` / ``h_last`` and the engine's arg-max seed, the fp64 VJP block by block,
   each block recomputed in fp64 from the engine's own input to it; ``attn_grad`` of every layer, relative to the
   layer's maximum.
c. relprop: ``oracle.vit.relprop`` / ``oracle.bert.relprop`` (``layers_lrp``: ``variant="lrp"`` /
   tests/bert_lrp_oracle.py; alpha = 2: oracle/alphabeta.py) in fp64 on a cache built from the taps (q / k / v split
   from qkv, BERT scores recomputed from qkv), to the encoder input: ``attn_cam`` of every layer and ``relevance_in``.
d. aggregation and rollout: fp64 ``rules.rollout(rules.aggregate(G, cam))`` of the engine's own ``attn_grad`` /
   ``attn_cam`` (BERT: row-normalised, ``[0, 0] = min``) against the engine's map (fused row kernel or composed path,
   by flag) and the dense joint of ``ops.attribution_rollout`` (fused and composed).
e. every forward tap is bit-equal before and after ``attribute`` (no forward tap is reused as scratch).

Teeth: each bound class rejects, inside the test, its own near-miss: the stage recomputed from the engine's inputs with
operands one class lower (TF32 for an fp32-grade stage, bf16 for a TF32 stage; for the rollout the head mean taken
before the ReLU).  A bound that accepts both fails the test.

Chained bounds (relative to the layer maximum): attn_grad 2e-5 (fp32-grade backward), 3e-3 (single-pass TF32 / fp16
backward); attn_cam / relevance_in 2e-5 with fp32-grade relevance rules, 5e-3 with tensor-core rules, 2e-2 with bf16 z+
operands (the bounds of test_gpu_parity_full.py / test_gpu_methods_tc.py); rollout 5e-6.

Where a bound differs from the ops tests' model, and why:
- fp32-grade forward Linears are held to the fp32 SIMT class bound (3e-6) whatever their family.  ``LIN_BOUND`` of
  3xTF32 / the fp16 split grows with K (4.8e-5 at K = 3072) to cover the ops tests' stress data (six decades of row
  magnitude, a 2^20-scaled tail block); at K = 3072 it accepts TF32-rounded operands, so on engine data it has no teeth.
  Every family meets 3e-6 here (worst 1.0e-6, qkv).
- LayerNorm: the scale adds mean|x| to the ops tests' (|x| + |mean|): the fp32 mean carries an error of the order of the
  scale it is summed at, and on random-init rows, where |mean| << mean|x|, an output near the mean was 2.0e-5 of the
  narrower scale.
- layers_lrp rules in fp32 (flags 512): their denominators x+W+ / x-W- are not bounded away from zero by the
  conditioning.  The fp32 oracle run on the same taps is 3.9e-4 off fp64 at ViT-B (the engine: the same 3.9e-4), so the
  engine is held to 10x the fp32 oracle's own error there, as test_gpu_parity_full.py does for the matmul1 rule.
- rollout 5e-6, not 2e-6: the map leaves out the cls column that carries most of the row, and the composed fp32 chain of
  12 N x N products reached 3.9e-6 of the map maximum (flags 512).
- The teeth of the chained TF32-class bounds are reported, not asserted: a bf16 near-miss of the tap's last contraction
  alone lands at 0.14 ... 0.5 of those bounds, because the engine's own single-pass chain error is already of that size
  (attn_grad 1.5e-3 at 3e-3).  The fp32-grade chained bounds reject their TF32 near-miss in every case.

Measured worst cases on one H100 80GB HBM3 at a 700 W power limit (fraction of the bound): forward stages <= 0.61 (ctx);
attn_grad 1.6e-5 (fp32-grade, BERT flags 51) and 1.5e-3 (TF32 / fp16); attn_cam / relevance_in 1.2e-6 (fp32-grade
layers_ours), 7.7e-4 (tensor-core z+), 4.9e-4 (bf16 z+); rollout 3.9e-6; no forward tap changed.  Run time 26 s.
"""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import alphabeta
from oracle import bert as obert
from oracle import conditioned
from oracle import rules
from oracle import vit as ovit
from test_gpu_tc import LIN_BOUND, _gelu64
from transformer_explainability_b200 import _lib, ops
from transformer_explainability_b200.engine import BertEngine, ViTEngine, bert_config, vit_config

pytestmark = pytest.mark.gpu

DEV = "cuda"
LN_BOUND = 1e-5                    # test_gpu_tc.py::test_layernorm_split: per element over (|x| + |mean|) rstd |w|
ROLLOUT_BOUND = 5e-6
FP32_CHAIN = 2e-5                  # chained bound of the fp32-grade classes
FLAG_SETS = [0, 51, 4147, 307, 1331, 3379, 15667, 7475, 115, 32051]
LRP_SETS = [_lib.FLAG_RULES_LRP, _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_RULES_LRP | _lib.FLAG_RULES_LRP_TC]
ALPHA_SETS = [0, _lib.FLAG_BENCH_DEFAULT]


def bound_3x(K):                   # test_gpu_tma_attention.py
    return 1.5e-8 * K + 2e-6


def tf32(t):
    """round to nearest (ties to even) onto the TF32 grid: 10 explicit mantissa bits"""
    i = t.float().contiguous().view(torch.int32)
    i = (i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF
    return i.view(torch.float32).to(t.dtype)


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def alpha_ctx(alpha):
    """the alpha-beta Linear rule of oracle/alphabeta.py for alpha != 1, else the z+ / layers_lrp rule itself"""
    return alphabeta.alpha_rules(alpha) if alpha != 1 else contextlib.nullcontext()


def bits(t):
    return t.contiguous().view(torch.int32)


# ---- bound classes of one flag set (te_engine_util.h: decode_flags and the kernel selection) --------------------------
def lin_family(flags):
    return "3xtf32" if flags & _lib.FLAG_LINEAR_TENSOR_CORES else "simt"     # the fp16 split has the 3xTF32 bound


def fp32_backward(flags):
    return not flags & (_lib.FLAG_BACKWARD_TF32 | _lib.FLAG_BACKWARD_F16)


def relprop_bound(flags):
    if flags & _lib.FLAG_RULES_LRP:
        tc = flags & _lib.FLAG_RULES_LRP_TC
    else:
        tc = flags & _lib.FLAG_ZPLUS_TENSOR_CORES
    if not tc and not flags & _lib.FLAG_RELPROP_TF32:
        return 2e-5
    return 2e-2 if flags & _lib.FLAG_ZPLUS_BF16 else 5e-3


# ---- bookkeeping: every number is collected, printed per stage and layer as a fraction of its bound, then asserted -----
WORST = {}


class Log:
    def __init__(self, tag):
        self.tag, self.rows, self.bad = tag, {}, []

    def check(self, stage, layer, err, bound):
        self.rows.setdefault(stage, []).append((layer, err, bound))
        key = (stage.split(" ")[0], bound)
        WORST[key] = max(WORST.get(key, 0.0), err)
        if not err < bound:
            self.bad.append("%s L%s: %.3g >= %.3g" % (stage, layer, err, bound))

    def teeth(self, stage, layer, err, bound, required=True):
        """the near-miss copy must fail the check (required=False: reported only, see the module docstring)"""
        if not required:
            self.rows.setdefault(stage + " near-miss", []).append((layer, err, bound))
        elif not err >= bound:
            self.bad.append("teeth %s L%s: near-miss %.3g accepted by %.3g" % (stage, layer, err, bound))

    def finish(self):
        for stage, rows in self.rows.items():
            worst = max(rows, key=lambda r: r[1] / r[2])
            print("%s | %-22s worst %.2f of %.1e (L%s) | %s" % (
                self.tag, stage, worst[1] / worst[2], worst[2], worst[0],
                " ".join("%s:%.2f" % (l, e / b) for l, e, b in rows)))
        assert not self.bad, "%s:\n  %s" % (self.tag, "\n  ".join(self.bad))


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for (stage, bound), err in sorted(WORST.items()):
        print("worst %-14s bound %.1e: %.2e (%.2f of the bound)" % (stage, bound, err, err / bound))


# ---- per-element measures --------------------------------------------------------------------------------------------
def elem(out, ref, scale):
    return ((out.double() - ref).abs() / scale.clamp_min(1e-300)).max().item()


def of_max(out, ref):
    return ((out.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def lin64(x, w, b=None):
    """fp64 y = x W^T + b and its scale |x||W|^T + |b|"""
    y, s = x @ w.T, x.abs() @ w.abs().T
    if b is not None:
        y, s = y + b, s + b.abs()
    return y, s


def check_linear(log, stage, l, fam, x, w, b, y, y2=None, e0=None, gelu=False):
    """a forward Linear with its epilogue: y (and y2 = e0 + y or gelu(y)) against fp64 of the engine's own x"""
    K = x.shape[-1]
    bound = min(LIN_BOUND[fam](K), LIN_BOUND["simt"](K))       # see the module docstring: fp32-grade families
    y64, s = lin64(x, w, b)
    log.check(stage, l, elem(y, y64, s), bound)
    if y2 is not None and gelu:
        log.check(stage + " gelu", l, elem(y2, _gelu64(y64), 1.13 * s), bound + 5e-7)
    elif y2 is not None:
        log.check(stage + " +res", l, elem(y2, e0 + y64, s + e0.abs()), bound + 1.2e-7)
    near = lin64(tf32(x), tf32(w), b)[0]                   # TF32 operands: one class below every forward family
    log.teeth(stage, l, elem(near, y64, s), bound)


def ln64(x, w, b, eps):
    m = x.mean(-1, keepdim=True)
    r = 1 / torch.sqrt(((x - m) ** 2).mean(-1, keepdim=True) + eps)
    xa = x.abs()
    return (x - m) * r * w + b, m, r, (xa + m.abs() + xa.mean(-1, keepdim=True)) * r * w.abs() + b.abs()


def check_layernorm(log, stage, l, x, w, b, eps, y, mean=None, rstd=None):
    y64, m64, r64, s = ln64(x, w, b, eps)
    log.check(stage, l, elem(y, y64, s), LN_BOUND)
    if mean is not None:
        log.check(stage + " mean", l, elem(mean, m64[..., 0], x.abs().mean(-1)), LN_BOUND)
        log.check(stage + " rstd", l, elem(rstd, r64[..., 0], r64[..., 0]), LN_BOUND)
    log.teeth(stage, l, elem(ln64(tf32(x), w, b, eps)[0], y64, s), LN_BOUND)


def heads(t, H):
    return obert._heads(t, H)


def check_attention(log, l, P_tap, P_pad, ctx, qkv, H, flags, maskadd=None):
    """P = softmax(alpha q k^T [+ mask]) and ctx = P v from the engine's own qkv / P"""
    B, N, D3 = qkv.shape
    D = D3 // 3
    dh = D // H
    alpha = float(torch.tensor(1.0 / math.sqrt(dh)))
    q, k, v = [heads(u, H) for u in qkv.chunk(3, dim=-1)]
    s64, a64 = alpha * (q @ k.transpose(-1, -2)), alpha * (q.abs() @ k.abs().transpose(-1, -2))
    if maskadd is not None:
        s64 = s64 + maskadd
    ref = torch.softmax(s64, dim=-1)
    live = ref > 1e-30
    eb = 2 * a64.amax(dim=-1, keepdim=True) * bound_3x(dh) + 1e-5            # relative, per element
    P = P_tap.double()
    assert (P[~live].abs() <= 1e-30).all(), "L%d: P non-zero where the reference underflows (masked keys)" % l
    assert (bits(P_pad) == 0).all(), "L%d: pad columns of P are not +0.0" % l
    rel_frac = lambda p: (((p - ref).abs() / ref.clamp_min(1e-300))[live] / eb.expand_as(ref)[live]).max().item()  # noqa
    log.check("P", l, rel_frac(P), 1.0)
    s_near = alpha * (tf32(q) @ tf32(k).transpose(-1, -2)) + (maskadd if maskadd is not None else 0)
    log.teeth("P", l, rel_frac(torch.softmax(s_near, dim=-1)), 1.0)
    # ctx = P v (3xTF32 with the attention tensor-core flag, else fp32 SIMT), reduction over the N keys
    bound = bound_3x(N) if flags & _lib.FLAG_ATTN_TENSOR_CORES else LIN_BOUND["simt"](N)
    c64, cs = obert._merge(P @ v), obert._merge(P.abs() @ v.abs())
    log.check("ctx", l, elem(ctx, c64, cs), bound)
    log.teeth("ctx", l, elem(obert._merge(tf32(P) @ tf32(v)), c64, cs), bound)


# ---- engine runs ------------------------------------------------------------------------------------------------------
VIT_LAYER_TAPS = ("x_in", "xn1", "mean1", "rstd1", "qkv", "attn", "ctx", "attn_out", "x_mid", "xn2", "mean2", "rstd2", "h",
                  "g", "mlp_out")
BERT_LAYER_TAPS = ("hidden", "qkv", "attn", "ctx", "d1", "s1", "ao", "mean1", "rstd1", "hpre", "g", "d2", "s2", "mean2",
                   "rstd2")


def pad_view(eng, layer):
    """the pad columns N .. NP-1 of P [B, H, N, NP - N]"""
    t = eng.tensor("attn", layer)
    B, H, N, _ = t.shape
    NP = t.stride(2)
    return torch.as_strided(t, (B, H, N, NP - N), t.stride(), t.storage_offset() + N)


def snapshot(eng, depth, layer_taps, model_taps):
    out = {(n, l): eng.tensor(n, l).clone() for l in range(depth) for n in layer_taps}
    out.update({(n, 0): eng.tensor(n).clone() for n in model_taps})
    out.update({("attn_pad", l): pad_view(eng, l).clone() for l in range(depth)})
    return out


def check_survive(log, before, after):
    changed = [n for n in before if not torch.equal(bits(before[n]), bits(after[n]))]
    log.check("taps unchanged by attribute", "-", float(len(changed)), 0.5)
    assert not changed, "forward taps rewritten by attribute: %s" % changed


def check_rollout(log, maps, G, cam, normalize, prefix, fused):
    """d: fp64 rollout of the engine's own attn_grad / attn_cam against its map and the dense joint"""
    g64 = [t.double().cpu() for t in G]
    c64 = [t.double().cpu() for t in cam]
    joint = rules.rollout([rules.aggregate(a, b) for a, b in zip(g64, c64)], normalize=normalize)

    def row(j):
        r = j[:, 0].clone()
        if normalize:
            r[:, 0] = r.min(dim=1).values                     # ExplanationGenerator.py:58
            return r
        return r[:, prefix:]
    ref = row(joint)
    log.check("rollout map (%s)" % ("fused" if fused else "composed"), "-", of_max(maps.cpu(), ref), ROLLOUT_BOUND)
    near = rules.rollout([(a * b).mean(dim=1).clamp(min=0) for a, b in zip(g64, c64)], normalize=normalize)
    log.teeth("rollout map", "-", of_max(row(near), ref), ROLLOUT_BOUND)
    gs, cs = torch.stack([t.contiguous() for t in G]), torch.stack([t.contiguous() for t in cam])
    for f in (True, False):
        j, _ = ops.attribution_rollout(gs, cs, normalize=normalize, fused=f, want_joint=True)
        log.check("rollout joint (%s)" % ("fused" if f else "composed"), "-", of_max(j.cpu(), joint), ROLLOUT_BOUND)


def check_chain(log, stage, l, got, ref, bound, near=None):
    log.check(stage, l, of_max(got, ref), bound)
    if near is not None:
        log.teeth(stage, l, of_max(near, ref), bound, required=bound <= FP32_CHAIN)


# ---- ViT ---------------------------------------------------------------------------------------------------------------
def vit_model(name, seed, xseed, conditioned_=True, n=2, **over):
    params, heads_ = ovit.init_params(name, seed=seed, rand_affine=conditioned_, **over)
    if conditioned_:
        params = conditioned.condition_vit(params, c_qkv=1.0)
    p64 = {k: v.double().to(DEV) for k, v in params.items()}
    cfg = ovit.ViTConfig(p64, heads_)
    ecfg = vit_config(img_size=224, patch_size=cfg.patch, num_classes=cfg.num_classes, embed_dim=cfg.dim,
                      depth=cfg.depth, num_heads=heads_, mlp_ratio=cfg.mlp_dim / cfg.dim, distilled=cfg.distilled)
    eng = ViTEngine(ecfg, params)
    x = torch.randn(n, 3, 224, 224, generator=torch.Generator().manual_seed(xseed))
    return dict(eng=eng, p64=p64, cfg=cfg, x=x, heads=heads_, conditioned=conditioned_)


def vit_forward_checks(log, m, flags, T):
    p, cfg, H = m["p64"], m["cfg"], m["heads"]
    fam = lin_family(flags)
    D64 = lambda name, l=0: T[(name, l)].double()          # noqa: E731
    # x_in[0]: im2col, patch GEMM (fp32 SIMT), tokens + pos
    img = m["x"].double().to(DEV)
    P_ = cfg.patch
    patches = F.unfold(img, P_, stride=P_).transpose(1, 2)                         # [B, np, C P P]
    y64, s = lin64(patches, p["patch_embed.proj.weight"].reshape(cfg.dim, -1), p["patch_embed.proj.bias"])
    B = img.shape[0]
    toks = [p["cls_token"].expand(B, -1, -1)] + ([p["dist_token"].expand(B, -1, -1)] if cfg.distilled else [])
    pos = p["pos_embed"]
    ref = torch.cat(toks + [y64], 1) + pos
    scale = torch.cat([t.abs() for t in toks] + [s], 1) + pos.abs()
    log.check("x_in[0] tokens", 0, elem(T[("x_in", 0)], ref, scale), LIN_BOUND["simt"](patches.shape[-1]) + 1.2e-7)
    near = torch.cat(toks + [lin64(tf32(patches), tf32(p["patch_embed.proj.weight"].reshape(cfg.dim, -1)),
                                   p["patch_embed.proj.bias"])[0]], 1) + pos
    log.teeth("x_in[0] tokens", 0, elem(near, ref, scale), LIN_BOUND["simt"](patches.shape[-1]) + 1.2e-7)
    for l in range(cfg.depth):
        pre = "blocks.%d." % l
        x_next = T[("x_in", l + 1)] if l + 1 < cfg.depth else T[("x_last", 0)]
        check_layernorm(log, "ln1", l, D64("x_in", l), p[pre + "norm1.weight"], p[pre + "norm1.bias"], cfg.eps_block,
                        T[("xn1", l)], T[("mean1", l)], T[("rstd1", l)])
        check_linear(log, "qkv", l, fam, D64("xn1", l), p[pre + "attn.qkv.weight"], p[pre + "attn.qkv.bias"], T[("qkv", l)])
        check_attention(log, l, T[("attn", l)], T[("attn_pad", l)], T[("ctx", l)], D64("qkv", l), H, flags)
        check_linear(log, "proj", l, fam, D64("ctx", l), p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"],
                     T[("attn_out", l)], T[("x_mid", l)], D64("x_in", l))
        check_layernorm(log, "ln2", l, D64("x_mid", l), p[pre + "norm2.weight"], p[pre + "norm2.bias"], cfg.eps_block,
                        T[("xn2", l)], T[("mean2", l)], T[("rstd2", l)])
        check_linear(log, "fc1", l, fam, D64("xn2", l), p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"], T[("h", l)],
                     T[("g", l)], gelu=True)
        check_linear(log, "fc2", l, fam, D64("g", l), p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"], T[("mlp_out", l)],
                     x_next, D64("x_mid", l))
    check_layernorm(log, "final norm", "-", D64("x_last"), p["norm.weight"], p["norm.bias"], cfg.eps_final,
                    T[("x_final_norm", 0)])
    xf = D64("x_final_norm")
    y, s = lin64(xf[:, 0], p["head.weight"], p["head.bias"])
    if cfg.distilled:
        y2, s2 = lin64(xf[:, 1], p["head_dist.weight"], p["head_dist.bias"])
        y, s = (y + y2) / 2, (s + s2) / 2
    log.check("logits", "-", elem(T[("logits", 0)], y, s + y.abs()), LIN_BOUND["simt"](cfg.dim))


def vit_seed(m, idx):
    seed = torch.zeros(idx.shape[0], m["cfg"].num_classes, dtype=torch.float64, device=DEV)
    seed[torch.arange(idx.shape[0]), idx.long()] = 1
    return seed


def vit_backward_checks(log, m, flags, T, G, seed):
    """b: the fp64 VJP from x_last, block by block at the engine's own x_in[l]"""
    p, cfg, H = m["p64"], m["cfg"], m["heads"]
    bound = 2e-5 if fp32_backward(flags) else 3e-3
    rnd = tf32 if fp32_backward(flags) else bf16
    with torch.enable_grad():
        xl = T[("x_last", 0)].double().requires_grad_(True)
        xf = F.layer_norm(xl, (cfg.dim,), p["norm.weight"], p["norm.bias"], cfg.eps_final)
        logits = F.linear(xf[:, 0], p["head.weight"], p["head.bias"])
        if cfg.distilled:
            logits = (logits + F.linear(xf[:, 1], p["head_dist.weight"], p["head_dist.bias"])) / 2
        dx, = torch.autograd.grad((seed * logits).sum(), xl)
        for l in reversed(range(cfg.depth)):
            t = T[("x_in", l)].double().requires_grad_(True)
            out, c = ovit.block_forward(p, cfg, l, t)
            dx, g64, dctx = torch.autograd.grad(out, [t, c["attn"], c["ctx"]], grad_outputs=dx)
            near = heads(rnd(dctx), H) @ rnd(c["v"].detach()).transpose(-1, -2)
            check_chain(log, "attn_grad", l, G[l], g64, bound, near)


def vit_cache(m, T, dtype=torch.float64):
    cfg, H = m["cfg"], m["heads"]
    blocks = []
    for l in range(cfg.depth):
        d = lambda n: T[(n, l)].to(dtype)                  # noqa: E731
        q, k, v = [heads(u, H) for u in d("qkv").chunk(3, dim=-1)]
        blocks.append(dict(x_in=d("x_in"), xn1=d("xn1"), q=q, k=k, v=v, attn=d("attn"), ctx=d("ctx"),
                           attn_out=d("attn_out"), x_mid=d("x_mid"), xn2=d("xn2"), g=d("g"), mlp_out=d("mlp_out")))
    return {"cfg": cfg, "x_final_norm": T[("x_final_norm", 0)].to(dtype), "blocks": blocks}


def lrp_gate(log, got32, ref):
    """layers_lrp rules in fp32: their denominators x+W+ / x-W- are not bounded away from zero by the conditioning, so the
    fp32 oracle on the same cache is itself off fp64; the engine is held to 10x that, or to the fp32 class bound"""
    e32 = max(of_max(a, b) for a, b in zip(got32, ref))
    log.check("fp32 oracle on the taps", "-", e32, 1.0)
    return max(FP32_CHAIN, 10 * e32)


def vit_relprop_checks(log, m, flags, T, cams, rin, seed, alpha):
    variant = "lrp" if flags & _lib.FLAG_RULES_LRP else "ours"
    cache = vit_cache(m, T)
    taps = {}
    with torch.no_grad(), alpha_ctx(alpha):
        ref_cams, r = ovit.relprop(m["p64"], cache, seed, 0, taps=taps, to_input=True, variant=variant)
    bound = relprop_bound(flags)
    rnd = tf32 if bound == FP32_CHAIN else bf16
    if variant == "lrp" and bound == FP32_CHAIN:
        p32 = {k: v.float() for k, v in m["p64"].items()}
        with torch.no_grad(), alpha_ctx(alpha):
            c32, r32 = ovit.relprop(p32, vit_cache(m, T, torch.float32), seed.float(), 0, to_input=True, variant=variant)
        bound = lrp_gate(log, [c32[l] for l in range(m["cfg"].depth)] + [r32], ref_cams + [r])
    for l in range(m["cfg"].depth):
        c = cache["blocks"][l]
        rctx = heads(taps[l]["proj"], m["heads"])
        near = rules.matmul_av_relprop(rnd(c["attn"]), rnd(c["v"]), rnd(rctx))[0] / 2
        check_chain(log, "attn_cam", l, cams[l], ref_cams[l], bound, near)
    check_chain(log, "relevance_in", "-", rin, r, bound)


def run_vit(m, flags, alpha=1.0, cls_rows=1, relprop=True):
    eng = m["eng"]
    tag = "%s flags %d%s%s" % (m["name"], flags, " alpha %g" % alpha if alpha != 1 else "",
                               " cls_row_top_block 0" if not cls_rows else "")
    log = Log(tag)
    model_taps = ("x_last", "x_final_norm", "logits")
    depth = m["cfg"].depth
    _lib.check(_lib.load().te_set_option(b"cls_row_top_block", cls_rows), "te_set_option")
    try:
        eng.forward(m["x"].to(DEV), flags=flags)
        before = snapshot(eng, depth, VIT_LAYER_TAPS, model_taps)
        maps, idx = eng.attribute(start_layer=0, flags=flags | _lib.FLAG_KEEP_ALL_CAMS | _lib.FLAG_RELPROP_TO_INPUT,
                                  alpha=alpha)
        torch.cuda.synchronize()
        T = snapshot(eng, depth, VIT_LAYER_TAPS, model_taps)
    finally:
        _lib.check(_lib.load().te_set_option(b"cls_row_top_block", 1), "te_set_option")
    check_survive(log, before, T)
    G = [eng.tensor("attn_grad", l).clone() for l in range(depth)]
    seed = vit_seed(m, idx)
    vit_forward_checks(log, m, flags, T)
    vit_backward_checks(log, m, flags, T, G, seed)
    cams = [eng.tensor("attn_cam", l).clone() for l in range(depth)]
    if relprop:                # random init: the relprop is ill-conditioned even teacher-forced, so only its rollout is judged
        vit_relprop_checks(log, m, flags, T, cams, eng.tensor("relevance_in").clone(), seed, alpha)
    check_rollout(log, maps, G, cams, False, 2 if m["cfg"].distilled else 1, bool(flags & _lib.FLAG_ROLLOUT_FUSED))
    log.finish()


VIT_MODELS = {
    "vit_b": dict(name="vit_base_patch16_224", seed=11, xseed=12),
    "deit_distilled": dict(name="deit_base_distilled_patch16_224", seed=4, xseed=9),
    "d256_mlp128": dict(name="vit_base_patch16_224", seed=31, xseed=32, dim=256, heads=4, mlp=128, depth=3, classes=100),
}
_CACHE = {}


def vit_setup(key, conditioned_=True):
    k = (key, conditioned_)
    if k not in _CACHE:
        _CACHE.clear()                                     # one model on the device at a time
        kw = dict(VIT_MODELS[key])
        name = kw.pop("name")
        m = vit_model(name, conditioned_=conditioned_, **kw)
        m["name"] = key if conditioned_ else key + " random-init"
        _CACHE[k] = m
    return _CACHE[k]


VIT_CASES = [(key, f, 1.0, 1) for key in VIT_MODELS for f in FLAG_SETS + LRP_SETS] + \
            [(key, f, 2.0, 1) for key in ("vit_b", "deit_distilled") for f in ALPHA_SETS] + \
            [("vit_b", _lib.FLAG_BENCH_DEFAULT, 1.0, 0)]


@pytest.mark.parametrize("key,flags,alpha,cls_rows", VIT_CASES,
                         ids=lambda v: str(v) if not isinstance(v, float) else "a%g" % v)
def test_vit_stages(key, flags, alpha, cls_rows):
    run_vit(vit_setup(key), flags, alpha=alpha, cls_rows=cls_rows)


@pytest.mark.parametrize("flags", [0, 51, _lib.FLAG_BENCH_DEFAULT])
def test_vit_b_random_init_stages(flags):
    """the bench regime: forward, backward and rollout (the relprop is ill-conditioned there even teacher-forced)"""
    run_vit(vit_setup("vit_b", conditioned_=False), flags, relprop=False)


# ---- BERT --------------------------------------------------------------------------------------------------------------
def bert_model():
    if "bert" not in _CACHE:
        _CACHE.clear()
        params, H = obert.init_params(seed=22, vocab=1000, max_pos=512, dim=768, depth=12, heads=12, inter=3072,
                                      rand_affine=True)
        params = conditioned.condition_bert(params, c_qkv=3.0)
        n, seq = 3, 130
        g = torch.Generator().manual_seed(23)
        ids = torch.randint(5, 1000, (n, seq), generator=g)
        ids[:, 0], ids[:, -1] = 101, 102
        mask = torch.ones(n, seq, dtype=torch.long)
        mask[1, seq // 2:] = 0                                   # sample 1 is padded from the middle on
        p64 = {k: v.double().to(DEV) for k, v in params.items()}
        eng = BertEngine(bert_config(vocab_size=1000), params)
        _CACHE["bert"] = dict(eng=eng, p64=p64, dm=obert.BertDims(p64, H), heads=H, ids=ids, mask=mask, name="bert_s130")
    return _CACHE["bert"]


def bert_forward_checks(log, m, flags, T, ext):
    p, dm = m["p64"], m["dm"]
    E = "bert.embeddings."
    ids = m["ids"].to(DEV)
    S = ids.shape[1]
    emb = (p[E + "token_type_embeddings.weight"][torch.zeros_like(ids)] + p[E + "position_embeddings.weight"][:S]) + \
        p[E + "word_embeddings.weight"][ids]
    check_layernorm(log, "embeddings + ln", 0, emb, p[E + "LayerNorm.weight"], p[E + "LayerNorm.bias"], dm.eps,
                    T[("hidden", 0)])
    bert_layer_checks(log, m, flags, T, ext)
    bert_head_checks(log, m, T, torch.tanh)


def bert_layer_checks(log, m, flags, T, ext):
    """every encoder layer, each stage from the engine's own input to it"""
    p, dm, H = m["p64"], m["dm"], m["heads"]
    fam = lin_family(flags)
    D64 = lambda name, l=0: T[(name, l)].double()          # noqa: E731
    for l in range(dm.depth):
        L = "bert.encoder.layer.%d." % l
        h_next = T[("hidden", l + 1)] if l + 1 < dm.depth else T[("h_last", 0)]
        qkv_w = torch.cat([p[L + "attention.self.%s.weight" % n] for n in ("query", "key", "value")])
        qkv_b = torch.cat([p[L + "attention.self.%s.bias" % n] for n in ("query", "key", "value")])
        check_linear(log, "qkv", l, fam, D64("hidden", l), qkv_w, qkv_b, T[("qkv", l)])
        check_attention(log, l, T[("attn", l)], T[("attn_pad", l)], T[("ctx", l)], D64("qkv", l), H, flags, ext)
        check_linear(log, "dense1", l, fam, D64("ctx", l), p[L + "attention.output.dense.weight"],
                     p[L + "attention.output.dense.bias"], T[("d1", l)], T[("s1", l)], D64("hidden", l))
        check_layernorm(log, "ln1", l, D64("s1", l), p[L + "attention.output.LayerNorm.weight"],
                        p[L + "attention.output.LayerNorm.bias"], dm.eps, T[("ao", l)], T[("mean1", l)], T[("rstd1", l)])
        check_linear(log, "fc1", l, fam, D64("ao", l), p[L + "intermediate.dense.weight"], p[L + "intermediate.dense.bias"],
                     T[("hpre", l)], T[("g", l)], gelu=True)
        check_linear(log, "dense2", l, fam, D64("g", l), p[L + "output.dense.weight"], p[L + "output.dense.bias"],
                     T[("d2", l)], T[("s2", l)], D64("ao", l))
        check_layernorm(log, "ln2", l, D64("s2", l), p[L + "output.LayerNorm.weight"], p[L + "output.LayerNorm.bias"],
                        dm.eps, h_next, T[("mean2", l)], T[("rstd2", l)])


def bert_head_checks(log, m, T, act):
    """pooled = act(dense(h_last[:, 0])) (BERT's pooler: tanh) and the logits; act is 1-Lipschitz, so the dense's scale
    bounds it"""
    p, dm = m["p64"], m["dm"]
    y, s = lin64(T[("h_last", 0)].double()[:, 0], p["bert.pooler.dense.weight"], p["bert.pooler.dense.bias"])
    log.check("pooled", "-", elem(T[("pooled", 0)], act(y), s + act(y).abs()), LIN_BOUND["simt"](dm.dim))
    y, s = lin64(T[("pooled", 0)].double(), p["classifier.weight"], p["classifier.bias"])
    log.check("logits", "-", elem(T[("logits", 0)], y, s), LIN_BOUND["simt"](dm.dim))


def bert_backward_checks(log, m, flags, T, G, seed, ext, act=torch.tanh):
    """b: the fp64 VJP from h_last through the head (act: its activation, BERT's pooler tanh)"""
    p, dm, H = m["p64"], m["dm"], m["heads"]
    bound = 2e-5 if fp32_backward(flags) else 3e-3
    rnd = tf32 if fp32_backward(flags) else bf16
    with torch.enable_grad():
        hl = T[("h_last", 0)].double().requires_grad_(True)
        pooled = act(F.linear(hl[:, 0], p["bert.pooler.dense.weight"], p["bert.pooler.dense.bias"]))
        logits = F.linear(pooled, p["classifier.weight"], p["classifier.bias"])
        dx, = torch.autograd.grad((seed * logits).sum(), hl)
        for l in reversed(range(dm.depth)):
            h = T[("hidden", l)].double().requires_grad_(True)
            out, c = obert.layer_forward(p, dm, l, h, ext)
            dx, g64, dctx = torch.autograd.grad(out, [h, c["probs"], c["ctx"]], grad_outputs=dx)
            near = heads(rnd(dctx), H) @ rnd(c["v"].detach()).transpose(-1, -2)
            check_chain(log, "attn_grad", l, G[l], g64, bound, near)


def bert_cache(m, T, ext, dtype=torch.float64):
    dm, H = m["dm"], m["heads"]
    layers = []
    for l in range(dm.depth):
        d = lambda n: T[(n, l)].to(dtype)                  # noqa: E731
        q, k, v = [heads(u, H) for u in d("qkv").chunk(3, dim=-1)]
        layers.append(dict(h=d("hidden"), q=q, k=k, v=v, scores=(q @ k.transpose(-1, -2)) / math.sqrt(dm.dim // H),
                           probs=d("attn"), ctx=d("ctx"), d1=d("d1"), ao=d("ao"), g=d("g"), d2=d("d2")))
    return {"dims": dm, "ext_mask": ext.to(dtype), "h_last": T[("h_last", 0)].to(dtype),
            "pooled": T[("pooled", 0)].to(dtype), "layers": layers}


def bert_relprop_checks(log, m, flags, T, cams, rin, seed, ext, alpha):
    import bert_lrp_oracle as olrp
    dm = m["dm"]
    lrp = flags & _lib.FLAG_RULES_LRP
    relprop = olrp.relprop if lrp else obert.relprop
    with torch.no_grad(), alpha_ctx(alpha):
        ref_cams, r = relprop(m["p64"], bert_cache(m, T, ext), seed, lowest=0, to_input=True)
    bound = relprop_bound(flags)
    if lrp and bound == FP32_CHAIN:
        p32 = {k: v.float() for k, v in m["p64"].items()}
        with torch.no_grad(), alpha_ctx(alpha):
            c32, r32 = relprop(p32, bert_cache(m, T, ext, torch.float32), seed.float(), lowest=0, to_input=True)
        bound = lrp_gate(log, list(c32) + [r32], list(ref_cams) + [r])
    for l in range(dm.depth):
        check_chain(log, "attn_cam", l, cams[l], ref_cams[l], bound)
    check_chain(log, "relevance_in", "-", rin, r, bound)


def run_bert(flags, alpha=1.0, cls_rows=1):
    m = bert_model()
    eng, dm = m["eng"], m["dm"]
    tag = "%s flags %d%s%s" % (m["name"], flags, " alpha %g" % alpha if alpha != 1 else "",
                               " cls_row_top_block 0" if not cls_rows else "")
    log = Log(tag)
    ext = (1.0 - m["mask"][:, None, None, :].double().to(DEV)) * -10000.0
    model_taps = ("h_last", "pooled", "logits")
    _lib.check(_lib.load().te_set_option(b"cls_row_top_block", cls_rows), "te_set_option")
    try:
        eng.forward(m["ids"], m["mask"], flags=flags)
        before = snapshot(eng, dm.depth, BERT_LAYER_TAPS, model_taps)
        maps, idx = eng.attribute(start_layer=0, flags=flags | _lib.FLAG_KEEP_ALL_CAMS | _lib.FLAG_RELPROP_TO_INPUT,
                                  alpha=alpha)
        torch.cuda.synchronize()
        T = snapshot(eng, dm.depth, BERT_LAYER_TAPS, model_taps)
    finally:
        _lib.check(_lib.load().te_set_option(b"cls_row_top_block", 1), "te_set_option")
    check_survive(log, before, T)
    G = [eng.tensor("attn_grad", l).clone() for l in range(dm.depth)]
    cams = [eng.tensor("attn_cam", l).clone() for l in range(dm.depth)]
    seed = torch.zeros(idx.shape[0], 2, dtype=torch.float64, device=DEV)
    seed[torch.arange(idx.shape[0]), idx.long()] = 1
    bert_forward_checks(log, m, flags, T, ext)
    bert_backward_checks(log, m, flags, T, G, seed, ext)
    bert_relprop_checks(log, m, flags, T, cams, eng.tensor("relevance_in").clone(), seed, ext, alpha)
    check_rollout(log, maps, G, cams, True, 0, bool(flags & _lib.FLAG_ROLLOUT_FUSED))
    log.finish()


BERT_CASES = [(f, 1.0, 1) for f in FLAG_SETS + LRP_SETS] + [(f, 2.0, 1) for f in ALPHA_SETS] + \
             [(_lib.FLAG_BENCH_DEFAULT, 1.0, 0)]


@pytest.mark.parametrize("flags,alpha,cls_rows", BERT_CASES, ids=lambda v: str(v) if not isinstance(v, float) else "a%g" % v)
def test_bert_stages(flags, alpha, cls_rows):
    run_bert(flags, alpha=alpha, cls_rows=cls_rows)
