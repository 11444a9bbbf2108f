"""GPU: the engines and their batch-dependent kernel choices at the benchmark's batch sizes, against fp64 and against
per-sample runs.

bench.py times ViT-B/16 and DeiT at batch 256, ViT-L and BERT-base at 64.  Several launch choices depend on the batch, so
at those sizes other code runs than at the batch 2 / 3 of the fp64 engine tests:

- the cluster size K of the fused row rollout (``te_rollout_fused.cu:169``): 8 for B <= 65, 4 for 66-131, 2 for
  132-263, 1 from 264 (the benchmark's batch 256 runs K = 2);
- the SIMT GEMM tile (64 x 64 or 128 x 128 by the CTA count), the grid-stride passes of the element-wise and z^B kernels,
  the tiles per persistent TMA CTA, and the position of a sample's rows in a 128-row tile.

Apart from the fused rollout, every kernel's arithmetic order is independent of the batch (one fmaf chain over k in the
SIMT GEMM, a fixed k order and per-row scales in the wgmma tiles, per-row LayerNorm / softmax, a per-sample split of the
Add rule).  So a sample's result is asserted bit-identical whether it runs alone or at any row of a batch; the fused
rollout only reorders sums of non-negative terms when K changes, and is held to that reordering bound.

1. ``ops.attribution_rollout(fused=True, want_joint=False)`` at B in {65, 66, 131, 132, 263, 264} (both sides of every
   K boundary; the file asserts that all four K occur), (N, ld) in {(17, 20), (129, 132), (197, 200), (300, 300),
   (512, 512)} (all three NCHUNK instantiations), L = 3, start_layer 0 / 2, normalize off / on, H = 12 and 3 (H = 3 only
   at N = 300, H = 2 at N = 512, which keeps each operand under ~2 GB), NaN in the pad columns.  Against the fp64 row
   recurrence v <- v (mean_h relu(G cam) + I) (row-normalised with normalize) from v = e_0: 1e-5 of the row maximum (the
   bound of test_aggregation_rollout).  Same K: bit-identical whatever the sample's position and the batch size.
   Across K: |d| <= (L - start) N 2^-24 |v| per element.  That bound rejects, by at least 10x, the near-miss that drops
   one rank's partial of a K = 2 cluster for one layer (rows i = 1 mod 2).
2. One launch of 140 * 197 = 27580 rows at the ViT-B Linear shapes (768 -> 2304, 768 -> 3072, 3072 -> 768) against
   launches of single samples' 197 rows at offsets b * 197 that are not multiples of 128: ``linear_forward_epi``
   (simt, 3xtf32, f16_split; every epilogue), ``linear_backward_epi`` (simt, 3xtf32, tf32, f16; store and gelu_bwd) and
   ``linear_relprop`` (SIMT, TF32 with y, with the fp16 R operand, with the bf16 S1 operands), bit for bit.
3. Conditioned 2-block models (``oracle/conditioned.py``) at batch 140 (K = 2) and 70 (K = 4), under flags 0 and
   FLAG_BENCH_DEFAULT: ViT-B width (transformer_attribution at start_layer 0 / 1, full, rollout, the gradient-weighted
   attention rollout), DeiT-B-distilled width (N = 198, the fused kernel's first = 2), BERT-base width at S = 130,
   right-padded to lengths 2 ... 130 (the engine call of Generator.generate_LRP at start_layer 0: normalize and
   bert_fix at K != 8; the gradient-weighted rollout).  ``explain`` runs with an explicit chunk = B, as bench.py does, so the free memory of a
   shared card cannot change K.  Checks:
   - fp64: four samples (first, middle, last two) through the oracle alone, behind the regime gate of
     test_gpu_methods_tc.py (fp32 oracle within 1e-4 of fp64); class index bit-exact, maps 2e-4 (SIMT) / 5e-3
     (tensor-core sets) of the sample's own maximum;
   - 8 samples, first and last included, against the sample run alone (BERT: padded to the same S with the same mask):
     logits, class index and every written layer's attn / attn_grad / attn_cam bit-identical; maps bit-identical under
     flags 0 (composed rollout), within the reordering bound of 1. under the bench flags (fused rollout, another K);
   - a rolled batch of the same size (same K, every sample at another row offset): maps, logits and taps bit-identical;
   - chunk = 70 on the batch of 140 equals two calls of 70 bit for bit, and chunk = 140 within the reordering bound;
   - ViTEngine.explain_graphed equals the launch-by-launch maps bit for bit (batch 140, bench flags);
   - the profiler's kernel list contains rollout_row_kernel under the bench flags (no fall-back to the dense path).

Every bitwise check above holds as stated, the wgmma Linear launches of 2. included: none needed the per-element
fallback bound.  Measured worst cases on one H100 80GB HBM3 at a 700 W power limit:
  fused rollout vs fp64 1.0e-6 | across K 0.20 of the reordering bound | the near-miss 1.1e4 ... 3.3e5 times the bound
  engines vs fp64       ViT-B SIMT 5.3e-6, tensor cores 6.0e-4 | DeiT 3.2e-6, 1.0e-3 | BERT 1.3e-5, 4.4e-4
  engine maps across K  0.03 of the reordering bound (per-sample runs, chunk 140 vs 70)
Peak device memory (torch.cuda.max_memory_allocated) 8.0 GiB (ViT-B width, batch 140, bench flags), 5.0 GiB for BERT;
part 1 at most ~4 GB (N = 512).  Wall time: about 70 s for this file.
"""
import pytest
import torch

from oracle import attn_grad_rollout as agr
from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import vit as ovit
from test_gpu_methods_tc import GATE, VIT_C_QKV, rel, tol
from transformer_explainability_b200 import _lib

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
AGR = _lib.FLAG_ATTN_GRAD_ROLLOUT
BENCH = _lib.FLAG_BENCH_DEFAULT
WORST = {}


def record(what, err, bound):
    WORST[what] = max(WORST.get(what, 0.0), err)
    assert err <= bound, "%s: %g > %g" % (what, err, bound)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for what, err in sorted(WORST.items()):
        print("worst %s: %.2e" % (what, err))


# ---- 1. fused row rollout at every cluster size -------------------------------------------------------------------------
def cluster_size(B):
    """the cluster size of the fused row rollout, te_rollout_fused.cu:169: the smallest K in {1, 2, 4, 8} with B K >= 264
    (about two CTAs per SM on 132 SMs), at most 8"""
    K = 1
    while K < 8 and B * K < 264:
        K *= 2
    return K


BATCHES = (65, 66, 131, 132, 263, 264)
assert sorted({cluster_size(b) for b in BATCHES}) == [1, 2, 4, 8], "the batches must reach every cluster size"
L_ROLL = 3
# (N, ld, H): every NCHUNK instantiation (ld <= 128, <= 256, <= 512); H = 3 at N = 300 and H = 2 at N = 512 keep each
# operand [L, 264, H, N, ld] under ~2 GB
ROLL_SHAPES = [(17, 20, 3), (17, 20, 12), (129, 132, 3), (129, 132, 12), (197, 200, 3), (197, 200, 12), (300, 300, 3),
               (512, 512, 2)]


def _operands(N, ld, H, o, B):
    """[L, B, H, N, ld] G and cam of samples o .. o+B-1: each sample's values depend on its index only, NaN in the pad
    columns (the kernel must select them away)"""
    G = torch.empty(L_ROLL, B, H, N, ld, device="cuda")
    C = torch.empty_like(G)
    g = torch.Generator(device="cuda")
    for j in range(B):
        g.manual_seed(1000003 * N + 7919 * H + o + j)
        G[:, j] = torch.randn(L_ROLL, H, N, ld, generator=g, device="cuda") * 0.05
        C[:, j] = torch.randn(L_ROLL, H, N, ld, generator=g, device="cuda") * 0.05
    if ld > N:
        G[..., N:] = float("nan")
        C[..., N:] = float("nan")
    return G, C


def _mats64(G, C, N):
    """mean_h relu(G cam) in fp64, [L, B, N, N] (the product of two fp32 values is exact in fp64)"""
    return torch.stack([(G[l, ..., :N].double() * C[l, ..., :N].double()).clamp(min=0).mean(dim=1)
                        for l in range(G.shape[0])])


def _row64(M, start, normalize, drop_odd_rows_at=None):
    """row 0 of rules.rollout from the row recurrence v <- v M^_l, l = L-1 .. start, M^ = M + I (/ row sums)"""
    L, B, N, _ = M.shape
    eye = torch.eye(N, dtype=torch.float64, device=M.device)
    v = torch.zeros(B, N, dtype=torch.float64, device=M.device)
    v[:, 0] = 1
    for l in range(L - 1, start - 1, -1):
        Mh = M[l] + eye
        if normalize:
            Mh = Mh / Mh.sum(dim=-1, keepdim=True)
        w = v
        if l == drop_odd_rows_at:                    # the near-miss: one rank of a K = 2 cluster loses its partial
            w = v.clone()
            w[:, 1::2] = 0
        v = torch.bmm(w.unsqueeze(1), Mh).squeeze(1)
    return v


def _launch(G, C, start, normalize):
    from transformer_explainability_b200 import ops
    _, row = ops.attribution_rollout(G, C, start_layer=start, normalize=normalize, fused=True, want_joint=False)
    torch.cuda.synchronize()
    return row


def _reorder_bound(start, N, v):
    return (L_ROLL - start) * N * U32 * v.abs()


def _of_bound(d, bound):
    """max |d| / bound per element; an exact zero of both (an entry every head's ReLU zeroed) counts as 0"""
    d = d.abs()
    return torch.where(d == 0, torch.zeros_like(d), d / bound).max().item()


@pytest.mark.parametrize("N,ld,H", ROLL_SHAPES)
def test_fused_rollout_every_cluster_size(N, ld, H):
    combos = [(start, normalize) for start in (0, L_ROLL - 1) for normalize in (False, True)]
    rows, refs = {}, {}
    # the batch of B samples from sample 0, and the same K one row over (samples 1 .. B): B - 1 samples at new offsets
    for B in BATCHES:
        for o in (0, 1):
            G, C = _operands(N, ld, H, o, B)
            for sc in combos:
                rows[(o, B) + sc] = _launch(G, C, *sc)
            if o == 0:
                for b0 in range(0, B, 33):
                    M = _mats64(G[:, b0:b0 + 33], C[:, b0:b0 + 33], N)
                    for sc in combos:
                        refs.setdefault((B,) + sc, []).append(_row64(M, *sc))
                    if B == BATCHES[0] and b0 == 0:
                        near = {n: _row64(M, 0, n, drop_odd_rows_at=0) for n in (False, True)}
                        base = {n: refs[(B, 0, n)][0] for n in (False, True)}
            del G, C
    # the same K at other batch sizes and offsets: samples 65 .. 130 of B = 131 against B = 66 from sample 65,
    # samples 131 .. 262 of B = 263 against B = 132 from sample 131
    for o, B, big in ((65, 66, 131), (131, 132, 263)):
        assert cluster_size(B) == cluster_size(big)
        G, C = _operands(N, ld, H, o, B)
        for sc in combos:
            rows[(o, B) + sc] = _launch(G, C, *sc)
            assert torch.equal(rows[(o, B) + sc], rows[(0, big) + sc][o:o + B]), (N, H, o, B, big, sc)
        del G, C
    for sc in combos:
        start = sc[0]
        for B in BATCHES:
            ref = torch.cat(refs[(B,) + sc])
            out = rows[(0, B) + sc]
            assert torch.isfinite(out).all()
            record("rollout vs fp64 (1e-5)", rel(out, ref), 1e-5)
            assert torch.equal(out[1:], rows[(1, B) + sc][:-1]), ("same K, one row over", N, H, B, sc)
        # across K: 8 -> 4, 4 -> 2, 2 -> 1 on the samples both launches hold
        for b1, b2 in ((65, 66), (131, 132), (132, 264)):
            assert cluster_size(b1) != cluster_size(b2)
            a, b = rows[(0, b1) + sc], rows[(0, b2) + sc][:b1]
            v = torch.cat(refs[(b1,) + sc])
            ratio = _of_bound(a.double() - b.double(), _reorder_bound(start, N, v))
            record("rollout across K (of the reordering bound)", ratio, 1.0)
    # the near-miss is rejected by the cross-K bound with a margin of 10
    for n in (False, True):
        miss = _of_bound(near[n] - base[n], _reorder_bound(0, N, base[n]))
        print("N %d H %d normalize %s: near-miss at %.1e of the reordering bound" % (N, H, n, miss))
        assert miss >= 10, (N, H, n, miss)


# ---- 2. row position and tile size do not change a row's result -----------------------------------------------------------
ROWS_PER_SAMPLE, SAMPLES = 197, 140
PICKS = (1, 37, 70, 139)                        # offsets b * 197 = 69, 121, 94, 119 mod 128
assert all(b * ROWS_PER_SAMPLE % 128 for b in PICKS)
LIN_SHAPES = [(768, 2304), (768, 3072), (3072, 768)]


def _rows(t, b):
    return t[b * ROWS_PER_SAMPLE:(b + 1) * ROWS_PER_SAMPLE].contiguous()


def _same_rows(name, big, small_fn):
    for b in PICKS:
        small = small_fn(b)
        for i, (x, y) in enumerate(zip(big, small)):
            if x is None:
                continue
            assert torch.equal(_rows(x, b), y), "%s output %d: sample %d (row offset %d) differs alone" % (
                name, i, b, b * ROWS_PER_SAMPLE)


@pytest.mark.parametrize("K,Nout", LIN_SHAPES)
def test_linear_rows_independent_of_position_and_batch(K, Nout):
    from transformer_explainability_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(K + Nout)
    R = ROWS_PER_SAMPLE * SAMPLES
    x = torch.randn(R, K, generator=g, device="cuda")
    w = torch.randn(Nout, K, generator=g, device="cuda") * K ** -0.5
    bias = torch.randn(Nout, generator=g, device="cuda")
    e0 = torch.randn(R, Nout, generator=g, device="cuda")
    dy = torch.randn(R, Nout, generator=g, device="cuda")
    e0b = torch.randn(R, K, generator=g, device="cuda")
    for fam in ("simt", "3xtf32", "f16_split"):
        for epi in ("store", "bias", "bias_gelu", "bias_add"):
            bb = None if epi == "store" else bias
            e = e0 if epi == "bias_add" else None
            big = ops.linear_forward_epi(x, w, bb, e, epi=epi, family=fam)
            _same_rows("forward %s %s" % (fam, epi), big, lambda b: ops.linear_forward_epi(
                _rows(x, b), w, bb, None if e is None else _rows(e, b), epi=epi, family=fam))
    for fam in ("simt", "3xtf32", "tf32", "f16"):
        for epi in ("store", "gelu_bwd"):
            e = e0b if epi == "gelu_bwd" else None
            big = ops.linear_backward_epi(dy, w, e, epi=epi, family=fam)
            _same_rows("backward %s %s" % (fam, epi), (big,), lambda b: (ops.linear_backward_epi(
                _rows(dy, b), w, None if e is None else _rows(e, b), epi=epi, family=fam),))
    # z+ rule on positive-denominator data: y = x W^T + b of the layer, R > 0
    y, _ = ops.linear_forward_epi(x, w, bias, epi="bias", family="simt")
    r = torch.rand(R, Nout, generator=g, device="cuda") * y.abs()
    for name, kw in (("simt", {}), ("tf32 y", dict(tensor_cores=True, y=y, bias=bias)),
                     ("tf32 y r_f16", dict(tensor_cores=True, y=y, bias=bias, r_f16=True)),
                     ("tf32 y bf16 s1", dict(tensor_cores=True, y=y, bias=bias, bf16="s1"))):
        big = ops.linear_relprop(x, w, r, **kw)

        def small(b, kw=kw):
            k2 = dict(kw)
            if "y" in k2:
                k2["y"] = _rows(y, b)
            return (ops.linear_relprop(_rows(x, b), w, _rows(r, b), **k2),)
        _same_rows("relprop %s" % name, (big,), small)
    torch.cuda.synchronize()


# ---- 3. the engines at the benchmark's cluster sizes ------------------------------------------------------------------------
BIG, SMALL = 140, 70                            # K = 2 and K = 4
assert cluster_size(BIG) == 2 and cluster_size(SMALL) == 4
DEPTH = 2
REF_SAMPLES = (0, 70, 138, 139)                 # the batch of 70 is every other sample of the batch of 140


def _sel(B):
    return sorted({0, 1, B // 3, B // 2, (2 * B) // 3, 101 % B, B - 2, B - 1})


def _vit_params(name, seed):
    params, heads = ovit.init_params(name, seed=seed, rand_affine=True, depth=DEPTH, classes=100)
    return conditioned.condition_vit(params, c_qkv=VIT_C_QKV), heads


def _bert_batch(seed):
    g = torch.Generator().manual_seed(seed)
    S = 130
    ids = torch.randint(5, 1000, (BIG, S), generator=g)
    mask = torch.ones(BIG, S, dtype=torch.long)
    for s in range(BIG):
        n = 2 + (128 * s) // (BIG - 1)            # lengths 2 (the shortest ERASER reduced row) ... 130
        ids[s, 0], ids[s, n - 1] = 101, 102
        ids[s, n:] = 0
        mask[s, n:] = 0
    return ids, mask


def _refs(explain32, explain64):
    """fp64 maps and class indices of REF_SAMPLES, each sample through the oracle alone, behind the regime gate"""
    out = {}
    for s in REF_SAMPLES:
        r64, i64 = explain64(s)
        r32, _ = explain32(s)
        gate = rel(r32, r64)
        assert gate < GATE, "regime is not conditioned for sample %d: fp32 oracle vs fp64 oracle %g" % (s, gate)
        out[s] = (r64[0], int(i64[0]))
    return out


VIT_METHODS = [("transformer_attribution", 0), ("transformer_attribution", 1), ("full", 0), ("rollout", 0),
               ("attn_grad_rollout", 0)]


@pytest.fixture(scope="module")
def vit_case():
    params, heads = _vit_params("vit_base_patch16_224", 51)
    x = torch.randn(BIG, 3, 224, 224, generator=torch.Generator().manual_seed(52))
    return _vit_refs(params, heads, x, VIT_METHODS)


@pytest.fixture(scope="module")
def deit_case():
    params, heads = _vit_params("deit_base_distilled_patch16_224", 53)
    x = torch.randn(BIG, 3, 224, 224, generator=torch.Generator().manual_seed(54))
    return _vit_refs(params, heads, x, [("transformer_attribution", 0), ("attn_grad_rollout", 0)])


def _vit_refs(params, heads, x, methods):
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs = {}
    for method, sl in methods:
        def run(p, s, dt):
            xs = x[s:s + 1].to(dt)
            if method == "attn_grad_rollout":
                return agr.explain_vit(p, xs, heads, start_layer=sl)
            return ovit.explain_method(p, xs, heads, method, start_layer=sl)
        refs[(method, sl)] = _refs(lambda s: run(params, s, torch.float32), lambda s: run(p64, s, torch.float64))
    return dict(params=params, heads=heads, x=x, refs=refs, methods=methods)


def _taps(eng, layers, names, samples):
    out = {"logits": eng.tensor("logits")[samples].clone()}
    for l in layers:
        for name in names:
            out["%s%d" % (name, l)] = eng.tensor(name, l)[samples].clone()
    return out


def _tap_names(method, sl):
    """the per-layer taps a method writes: attn_cam only where the relprop ran, attn_grad from start_layer on"""
    if method == "attn_grad_rollout":
        return [(range(DEPTH), ("attn",)), (range(sl, DEPTH), ("attn_grad",))]
    if method in ("full", "rollout"):
        return [(range(DEPTH), ("attn", "attn_grad", "attn_cam"))]
    return [(range(DEPTH), ("attn",)), (range(sl, DEPTH), ("attn_grad", "attn_cam"))]


def _all_taps(eng, method, sl, samples):
    out = {}
    for layers, names in _tap_names(method, sl):
        out.update(_taps(eng, layers, names, samples))
    return out


def _equal_taps(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), "%s: tap %s differs" % (what, k)


def _within_reorder(a, b, span, n, what):
    """maps of the fused rollout at two cluster sizes: per element within (L - start) N 2^-24 |v|"""
    v = torch.maximum(a.abs(), b.abs()).double()
    ratio = _of_bound(a.double() - b.double(), span * n * U32 * v)
    record("engine maps across K (of the reordering bound)", ratio, 1.0)
    assert ratio <= 1.0, what


def _peak(tag):
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print("%s: peak device memory %.2f GiB" % (tag, peak))
    WORST["peak GiB"] = max(WORST.get("peak GiB", 0.0), peak)
    assert peak < 10.5, "%s needs %.1f GiB" % (tag, peak)


def _release(model):
    model._engine = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _vit_model(case):
    from test_gpu_attn_grad_rollout import _vit_facade
    return _vit_facade(case["params"], case["heads"], 224, 16, DEPTH, 100)


def _vit_run(model, method, sl, x, flags, chunk=None):
    """-> (maps, class index) of one batch, explain with chunk = B where the method goes through explain"""
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    eng = model.engine()
    if method in ("transformer_attribution", "attn_grad_rollout"):
        fl = flags | (AGR if method == "attn_grad_rollout" else 0)
        maps, idx = eng.explain(x, start_layer=sl, flags=fl, chunk=chunk or x.shape[0])
    else:
        model.engine_flags = flags
        maps = LRP(model).generate_LRP(x, method=method, start_layer=sl)
        idx = eng.tensor("logits").argmax(-1).int()
    torch.cuda.synchronize()
    return maps.clone(), idx.clone()


def _engine_case(tag, run, eng_of, x_all, refs, method, sl, n_tok, fused_span, explain_based, graphed=None,
                 xs=lambda x, s: x[s:s + 1] if isinstance(s, int) else x[s]):
    """every check of part 3 for one method of one model; run(x, flags[, chunk]) -> (maps, idx)"""
    from test_gpu_model_geometries import census
    for flags in (0, BENCH):
        fused = bool(flags & _lib.FLAG_ROLLOUT_FUSED) and fused_span is not None
        for B in (BIG, SMALL):
            x = x_all if B == BIG else x_all[::2]
            orig = list(range(BIG)) if B == BIG else list(range(0, BIG, 2))
            torch.cuda.reset_peak_memory_stats()
            maps, idx = run(x, flags)
            _peak("%s %s sl %d flags %d B %d" % (tag, method, sl, flags, B))
            sel = _sel(B)
            taps = _all_taps(eng_of(), method, sl, sel)
            # fp64
            for i, s in enumerate(orig):
                if s in refs:
                    ref, ridx = refs[s]
                    assert int(idx[i]) == ridx, "%s %s flags %d B %d sample %d: class index" % (tag, method, flags, B, s)
                    record("%s vs fp64, each sample's maximum (bound %.0e)" % (tag, tol(flags)), rel(maps[i], ref), tol(flags))
            # per sample alone
            for j, s in enumerate(sel):
                one, oidx = run(xs(x, s), flags)
                _equal_taps({k: v[j:j + 1] for k, v in taps.items()}, _all_taps(eng_of(), method, sl, [0]),
                            "%s %s flags %d B %d sample %d alone" % (tag, method, flags, B, s))
                assert int(oidx[0]) == int(idx[s])
                if fused:
                    _within_reorder(maps[s], one[0], fused_span, n_tok, (tag, method, flags, B, s))
                else:
                    assert torch.equal(maps[s], one[0]), "%s %s flags %d B %d sample %d alone" % (tag, method, flags, B, s)
            # a rolled batch: the same K, every sample at another row offset
            perm = (torch.arange(B) + 53) % B
            pmaps, pidx = run(xs(x, perm), flags)
            assert torch.equal(pmaps, maps[perm]) and torch.equal(pidx, idx[perm]), "%s %s flags %d B %d rolled" % (
                tag, method, flags, B)
            inv = torch.argsort(perm)
            _equal_taps({k: v for k, v in taps.items()}, _all_taps(eng_of(), method, sl, inv[sel]),
                        "%s %s flags %d B %d rolled taps" % (tag, method, flags, B))
            if B != BIG or not explain_based:
                continue
            # chunk = 70 is two calls of 70; chunk = 140 is within the reordering bound of it
            c70, i70 = run(x, flags, SMALL)
            halves = [run(x[:SMALL], flags), run(x[SMALL:], flags)]
            assert torch.equal(c70, torch.cat([h[0] for h in halves])) and torch.equal(i70, idx)
            if fused:
                _within_reorder(maps, c70, fused_span, n_tok, (tag, method, "chunk"))
            else:
                assert torch.equal(maps, c70)
            if flags == BENCH:
                fams = census(lambda: run(x, flags))
                assert any(f.startswith("rollout_row_kernel") for f in fams), "%s %s: no fused row rollout ran: %s" % (
                    tag, method, sorted(fams))
                if graphed is not None:
                    gmaps, gidx = graphed(x, flags)
                    assert torch.equal(gmaps, maps) and torch.equal(gidx, idx), "%s %s: graph replay" % (tag, method)
                    eng_of()._graphs.clear()          # the captured graph pins the batch-140 workspace
            torch.cuda.synchronize()
            torch.cuda.empty_cache()


@pytest.mark.parametrize("method,sl", VIT_METHODS)
def test_vit_b_at_bench_cluster_sizes(vit_case, method, sl):
    model = _vit_model(vit_case)
    _run_vit_case("vit-b2", model, vit_case, method, sl, 197)


@pytest.mark.parametrize("method", ["transformer_attribution", "attn_grad_rollout"])
def test_deit_distilled_at_bench_cluster_sizes(deit_case, method):
    model = _vit_model(deit_case)
    _run_vit_case("deit-b2", model, deit_case, method, 0, 198)


def _run_vit_case(tag, model, case, method, sl, n_tok):
    x = case["x"].cuda()
    explain_based = method in ("transformer_attribution", "attn_grad_rollout")
    # fused rollout spans L - start layers; "rollout" composes (ops.compute_rollout_attention) and "full" has none
    span = DEPTH - sl if explain_based else None

    def graphed(xx, flags):
        fl = flags | (AGR if method == "attn_grad_rollout" else 0)
        m, i = model.engine().explain_graphed(xx, start_layer=sl, flags=fl)
        torch.cuda.synchronize()
        return m.clone(), i.clone()
    try:
        _engine_case(tag, lambda xx, flags, chunk=None: _vit_run(model, method, sl, xx, flags, chunk), model.engine, x,
                     case["refs"][(method, sl)], method, sl, n_tok, span, explain_based,
                     graphed=graphed if explain_based else None)
    finally:
        _release(model)


BERT_CFG = dict(hidden_size=768, num_hidden_layers=DEPTH, intermediate_size=3072, vocab_size=1000,
                max_position_embeddings=512)


@pytest.fixture(scope="module")
def bert_case():
    params, heads = obert.init_params(seed=61, vocab=1000, max_pos=512, dim=768, depth=DEPTH, heads=12, inter=3072,
                                      rand_affine=True)
    params = conditioned.condition_bert(params, c_qkv=3.0)
    ids, mask = _bert_batch(62)
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs = {}
    for which in ("LRP", "attn_grad_rollout"):
        def run(p, s, which=which):
            if which == "LRP":
                return obert.explain(p, ids[s:s + 1], mask[s:s + 1], heads, start_layer=0)
            return agr.explain_bert(p, ids[s:s + 1], mask[s:s + 1], heads)
        refs[which] = _refs(lambda s: run(params, s), lambda s: run(p64, s))
    return dict(params=params, heads=heads, ids=ids, mask=mask, refs=refs)


@pytest.mark.parametrize("which", ["LRP", "attn_grad_rollout"])
def test_bert_at_bench_cluster_sizes(bert_case, which):
    from test_gpu_bert import make_model
    model = make_model(bert_case["params"], bert_case["heads"], **BERT_CFG)
    ids, mask = bert_case["ids"].cuda(), bert_case["mask"].cuda()
    both = torch.stack([ids, mask])                # one batch tensor: rows of ids and mask move together

    def run(b, flags, chunk=None):
        fl = flags | (AGR if which == "attn_grad_rollout" else 0)
        maps, idx = model.engine().explain(b[0], b[1], start_layer=0, flags=fl, chunk=chunk or b.shape[1])
        torch.cuda.synchronize()
        return maps.clone(), idx.clone()

    class Rows:                                     # x[s:s+1], x[::2], x[perm], x[:70] of the stacked batch
        def __init__(self, t):
            self.t = t
            self.shape = (t.shape[1],)

        def __getitem__(self, k):
            return Rows(self.t[:, k])
    run_rows = lambda r, flags, chunk=None: run(r.t, flags, chunk)
    try:
        _engine_case("bert-b2", run_rows, model.engine, Rows(both), bert_case["refs"][which], which, 0, 130, DEPTH, True,
                     )
        pad = ~bert_case["mask"].bool()
        maps, _ = run(both, BENCH)
        assert (maps.cpu()[pad] == 0).all(), "padded tokens must get exactly zero"
    finally:
        _release(model)
