"""GPU: the perturbation evaluation (``te_perturb_images``, ``te_logit_stats``, ``perturbation.perturbation_eval``) against
the CPU oracle (``oracle/perturbation.py``) and the reference's own ``eval(args)`` (``tests/golden/perturbation.npz``).

Measured on an H100 80GB HBM3 at a 700 W power limit:
 * ``te_perturb_images``: bit-equal (``torch.equal``) to the oracle in every case below.
 * ``te_logit_stats`` against an fp64 restatement on the same fp32 logits: pred / max_logit exact; max_prob relative error
   at most 2.5e-7 (bound 2e-6); finite dissim absolute error at most 6.0e-7 (bound 1e-5); every +-inf row equal to the
   reference's fp32 formula.
 * end to end on the tiny model of the fixture (flags 0): hits exact, every other array within 4.8e-6 of the reference's
   (bound 2e-4 absolute + 1e-4 relative).  Conditioned ViT-B/16, 8 samples: every one of the 80 forwards has a top-two
   logit margin above 1e-3 in the fp64 oracle and its hit is exact; the other arrays are within 5.5e-6 of the fp64 oracle
   at flags 0 and 5.6e-6 at the bench flags 7475 (bound 2e-3 + 1e-3 relative).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_perturbation as mg
from oracle import perturbation as opert

pytestmark = pytest.mark.gpu

NAMES = mg.NAMES


def _rand_images(B, side, seed):
    return torch.rand(B, 3, side, side, generator=torch.Generator().manual_seed(seed))


def _saliency(kind, B, side, seed):
    g = torch.Generator().manual_seed(seed)
    P = side * side
    if kind == "random":
        return torch.randn(B, P, generator=g)
    if kind == "heatmap":                       # writer-style maps: bilinear x16 + min-max, ties everywhere
        from transformer_explainability_b200 import visualization
        grid = side // 16
        maps = torch.rand(B, grid * grid, generator=g).cuda()
        return visualization.relevance_to_heatmap(maps, grid=grid, scale=16).reshape(B, P).cpu()
    if kind == "quantised":
        return torch.randint(0, 4, (B, P), generator=g).to(torch.float32) / 4
    if kind == "constant":                      # a constant map min-max normalises to a NaN row; plus scattered NaN
        s = torch.randn(B, P, generator=g)
        s[0] = float("nan")
        s[:, torch.randint(0, P, (P // 7,), generator=g)] = float("nan")
        return s
    if kind == "zeros":
        vals = torch.tensor([0.0, -0.0, 0.5, -0.5])
        return vals[torch.randint(0, 4, (B, P), generator=g)]
    raise ValueError(kind)


def _ks(side, which):
    P = side * side
    if which == "per" and side == 224:
        return [0] + opert.step_sizes("per")
    if which == "100" and side == 224:
        return [0] + opert.step_sizes("100")
    if which == "edges":
        return [0, 0, 1, P // 2, P - 1, P, P]
    return [0] + [int(P * f) for f in (0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9)]


CASES = [  # (side, B, saliency, step set)
    (224, 7, "random", "per"), (224, 7, "random", "100"), (224, 1, "heatmap", "per"), (224, 33, "heatmap", "per"),
    (224, 7, "heatmap", "100"), (224, 7, "constant", "per"), (224, 7, "zeros", "edges"), (224, 1, "random", "edges"),
    (17, 7, "random", "frac"), (17, 33, "quantised", "frac"), (17, 1, "zeros", "edges"), (17, 7, "constant", "edges"),
    (384, 1, "heatmap", "frac"), (384, 7, "random", "edges"), (384, 7, "quantised", "frac"),
]


@pytest.mark.parametrize("negate", [False, True])
@pytest.mark.parametrize("side,B,kind,steps", CASES)
def test_perturb_images_bit_exact(side, B, kind, steps, negate):
    from transformer_explainability_b200 import ops
    x = _rand_images(B, side, seed=side + B)
    s = _saliency(kind, B, side, seed=2 * side + B)
    ks = _ks(side, steps)
    got = ops.perturb_images(x.cuda(), s.cuda(), ks, negate=negate)
    torch.cuda.synchronize()
    want = opert.perturb(x, s, ks, negate)
    assert got.shape == want.shape
    for i in range(len(ks)):
        assert torch.equal(got[i].cpu(), want[i]), "step %d (k = %d) differs" % (i, ks[i])


@pytest.mark.parametrize("side,offset", [(224, 0), (224, 1), (17, 3)])
def test_perturb_images_writes_nothing_outside_out(side, offset):
    """A NaN canary margin on both sides of out survives; offset 1 also runs the scalar path on a 224 x 224 image."""
    from transformer_explainability_b200 import _lib, ops
    B, C = 5, 3
    x = _rand_images(B, side, seed=9).cuda()
    s = _saliency("heatmap" if side == 224 else "quantised", B, side, seed=10).cuda()
    ks = _ks(side, "per" if side == 224 else "frac")
    n = len(ks) * B * C * side * side
    margin = 4096
    buf = torch.full((offset + n + margin,), float("nan"), device="cuda")
    buf_pre = torch.full((margin,), float("nan"), device="cuda")
    buf = torch.cat([buf_pre, buf])
    lib = _lib.load()
    ws = torch.empty(lib.te_perturb_workspace_bytes(B, side * side) // 4, device="cuda")
    out = buf[margin + offset:margin + offset + n]
    kc = (_lib.c_int * len(ks))(*ks)
    m = (_lib.c_float * 3)(0.5, 0.5, 0.5)
    _lib.check(lib.te_perturb_images(_lib.ptr(x), _lib.ptr(s), B, C, side * side, kc, len(ks), 1, m, m, _lib.ptr(out),
                                     _lib.ptr(ws), ws.numel() * 4, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "te_perturb_images")
    torch.cuda.synchronize()
    assert torch.isnan(buf[:margin + offset]).all() and torch.isnan(buf[margin + offset + n:]).all()
    want = opert.perturb(x.cpu(), s.cpu(), ks, True)
    assert torch.equal(out.cpu().reshape(want.shape), want)
    assert torch.equal(ops.perturb_images(x, s, ks, negate=True).cpu(), want)


def _logit_cases():
    g = torch.Generator().manual_seed(21)
    rows = []
    for K in (10, 1000):
        l = torch.randn(64, K, generator=g) * 3
        l[1, 3] = l[1, 5] = l[1].max() + 1                  # tie at the maximum: first index, p_second = p_max
        l[2, :] = 0.25                                       # all equal
        l[3, 7] = l[3].max() + 200                           # p_second underflows, target on top: +inf
        l[4, 0] = l[4].max() - 200                           # p_target underflows: -inf
        l[5, 2] = l[5, 9] = l[5].max() + 300                 # duplicated runaway maximum
        t = torch.randint(0, K, (64,), generator=g)
        t[3], t[4], t[5] = 7, 0, 9
        rows.append((l, t))
    return rows


def test_logit_stats_against_fp64():
    from transformer_explainability_b200 import ops
    worst_p, worst_d = 0.0, 0.0
    for l, t in _logit_cases():
        pred, ml, mp, dis = (u.cpu() for u in ops.logit_stats(l.cuda(), t.cuda()))
        assert torch.equal(pred.long(), torch.from_numpy(np.argmax(l.numpy(), axis=1)))   # first index of the maximum
        assert torch.equal(ml, l.max(1)[0])
        l64 = l.double()
        p64 = torch.softmax(l64, dim=1)
        mp64 = p64.max(1)[0]
        rel = ((mp.double() - mp64).abs() / mp64).max().item()
        assert rel <= 2e-6, rel
        worst_p = max(worst_p, rel)
        _, _, _, d32 = opert.logit_stats(l, t)               # the reference's fp32 formula
        inf = torch.isinf(d32)
        assert inf[3] and inf[4] and d32[3] > 0 and d32[4] < 0
        assert torch.equal(dis[inf], d32[inf])
        d64 = torch.log(torch.gather(p64, 1, t[:, None])[:, 0] / p64.topk(2, dim=1)[0][:, 1])
        fin = ~inf
        assert torch.isfinite(dis[fin]).all()
        err = (dis[fin].double() - d64[fin]).abs().max().item()
        assert err <= 1e-5, err
        worst_d = max(worst_d, err)
        assert dis[1].item() == pytest.approx(float(d64[1]), abs=1e-5) and pred[1] == 3
    print("MEASURED logit_stats max_prob rel %.3g dissim abs %.3g" % (worst_p, worst_d))


def _tiny_model(flags=0):
    import functools
    import torch.nn as nn
    from transformer_explainability_b200.baselines.ViT.ViT_new import VisionTransformer
    p, heads = mg.params()
    m = VisionTransformer(norm_layer=functools.partial(nn.LayerNorm, eps=mg.EPS), **mg.KW)
    m.load_state_dict(p)
    m = m.cuda().eval()
    m.engine_flags = flags
    return m


def _close(got, want, atol, rtol):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    if got.size == 0:
        return 0.0
    assert np.array_equal(np.isinf(got), np.isinf(want)) and np.array_equal(got[np.isinf(got)], want[np.isinf(want)])
    fin = np.isfinite(want)
    err = np.abs(got[fin] - want[fin])
    assert (err <= atol + rtol * np.abs(want[fin])).all(), err.max()
    return float(err.max()) if err.size else 0.0


@pytest.fixture(scope="module")
def tiny():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "perturbation.npz"))
    images, vis, target = mg.samples()
    assert np.array_equal(target.numpy(), g["target"])
    loader = torch.utils.data.DataLoader(mg._Samples(images, vis, target), batch_size=int(g["batch"]), shuffle=False)
    return g, loader


@pytest.mark.parametrize("neg", [True, False])
@pytest.mark.parametrize("scale", ["per", "100"])
def test_end_to_end_against_reference_fixture(tiny, neg, scale):
    from transformer_explainability_b200.perturbation import perturbation_eval
    g, loader = tiny
    res = perturbation_eval(_tiny_model(), loader, neg=neg, scale=scale)
    tag = "%s.%s." % ("neg" if neg else "pos", scale)
    worst = 0.0
    for n in NAMES:
        want = g[tag + n]
        assert res[n].dtype == np.float64 and res[n].shape == want.shape, n
        if n.endswith("hits"):
            assert np.array_equal(res[n], want), n
        else:
            worst = max(worst, _close(res[n], want, 2e-4, 1e-4))
    print("MEASURED tiny end-to-end %s max abs %.3g" % (tag, worst))


def test_end_to_end_wrong_mode_against_reference_fixture(tiny):
    from transformer_explainability_b200.perturbation import perturbation_eval
    g, loader = tiny
    res = perturbation_eval(_tiny_model(), loader, neg=True, scale="per", wrong=True)
    assert np.array_equal(res["model_hits"], g["neg.per.model_hits"])
    assert np.array_equal(res["perturbations_hits"], g["wrong.neg.per.perturbations_hits"])
    for n in NAMES[3:]:
        _close(res[n], g["wrong.neg.per." + n], 2e-4, 1e-4)


@pytest.fixture(scope="module")
def vitb():
    """Conditioned ViT-B/16 (``oracle/conditioned.py``), 8 samples, writer-style heatmaps (ties at every step boundary), and
    the fp64 CPU oracle's six arrays on the same masks (computed once for both flag selections)."""
    from oracle import conditioned, vit as ovit
    from transformer_explainability_b200 import visualization
    p, heads = ovit.init_params("vit_base_patch16_224", seed=0)
    p = conditioned.condition_vit(p)
    N = 8
    images = _rand_images(N, 224, seed=77)
    maps = torch.rand(N, 196, generator=torch.Generator().manual_seed(78)).cuda()
    vis = visualization.relevance_to_heatmap(maps).reshape(N, 1, 224, 224).cpu()
    fn64 = opert.vit_logits_fn(p, heads, norm_eps=1e-6, dtype=torch.float64)
    xs = opert.perturb(images, vis.reshape(N, -1), [0] + opert.step_sizes("per"), True)
    logits = torch.stack([fn64(xs[i]) for i in range(xs.shape[0])])                  # [10, N, 1000]
    target = logits[0].argmax(1)
    target[::2] = (target[::2] + 1) % 1000
    top2 = logits.topk(2, dim=2)[0]
    margin_ok = ((top2[..., 0] - top2[..., 1]) > 1e-3).numpy()       # where an arg-max comparison is meaningful
    st = [opert.logit_stats(logits[i], target) for i in range(10)]
    hits = torch.stack([(s[0] == target).double() for s in st])
    want = {"model_hits": hits[0], "model_dissimilarities": st[0][3], "perturbations_hits": hits[1:],
            "perturbations_dissimilarities": torch.stack([s[3] for s in st[1:]]),
            "perturbations_logit_diff": torch.stack([s[1] - st[0][1] for s in st[1:]]),
            "perturbations_prob_diff": torch.stack([s[2] - st[0][2] for s in st[1:]])}
    return p, images, vis, target, {k: v.numpy() for k, v in want.items()}, margin_ok


@pytest.mark.parametrize("flags", ["0", "bench"])
def test_conditioned_vit_base_against_oracle(vitb, flags):
    from transformer_explainability_b200 import _lib
    from transformer_explainability_b200.baselines.ViT.ViT_new import vit_base_patch16_224
    from transformer_explainability_b200.perturbation import perturbation_eval
    p, images, vis, target, want, margin_ok = vitb
    m = vit_base_patch16_224()
    m.load_state_dict(p)
    m = m.cuda().eval()
    m.engine_flags = 0 if flags == "0" else _lib.FLAG_BENCH_DEFAULT
    loader = torch.utils.data.DataLoader(mg._Samples(images, vis, target), batch_size=3, shuffle=False)
    res = perturbation_eval(m, loader, neg=True, scale="per")
    assert margin_ok.sum() >= 0.8 * margin_ok.size
    assert (res["model_hits"] == want["model_hits"])[margin_ok[0]].all()
    assert (res["perturbations_hits"] == want["perturbations_hits"])[margin_ok[1:]].all()
    worst = 0.0
    for n in NAMES:
        if not n.endswith("hits"):
            worst = max(worst, _close(res[n], want[n], 2e-3, 1e-3))
    print("MEASURED conditioned ViT-B flags %s max abs %.3g; arg-max margins > 1e-3: %d / %d"
          % (flags, worst, int(margin_ok.sum()), margin_ok.size))


def test_results_file_round_trip(tmp_path):
    """compute_saliency_and_save(backend="builtin") -> ImagenetResults -> perturbation_eval equals the evaluation of the
    same tensors in memory."""
    from transformer_explainability_b200 import hdf5_writer
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    from transformer_explainability_b200.perturbation import ImagenetResults, perturbation_eval
    model = _tiny_model()
    images, _, target = mg.samples()
    src = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(images, target), batch_size=4, shuffle=False)
    d = str(tmp_path / "transformer_attribution")
    hdf5_writer.compute_saliency_and_save(src, d, "transformer_attribution", lrp=LRP(model), backend="builtin")
    ds = ImagenetResults(d)
    assert len(ds) == images.shape[0]
    raw = hdf5_writer.read_minimal_hdf5(os.path.join(d, "results.hdf5"))
    assert np.array_equal(raw["image"], images.numpy()) and np.array_equal(raw["target"], target.numpy())
    mem = torch.utils.data.TensorDataset(torch.from_numpy(raw["image"]), torch.from_numpy(raw["vis"]),
                                         torch.from_numpy(raw["target"]).long())
    for scale, neg in (("per", True), ("100", False)):
        a = perturbation_eval(model, torch.utils.data.DataLoader(ds, batch_size=5, shuffle=False), neg=neg, scale=scale)
        b = perturbation_eval(model, torch.utils.data.DataLoader(mem, batch_size=5, shuffle=False), neg=neg, scale=scale)
        for n in NAMES:
            assert np.array_equal(a[n], b[n], equal_nan=True), n
