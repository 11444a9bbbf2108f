"""CPU: the perturbation-evaluation oracle against the reference's own ``eval(args)`` (``tests/golden/perturbation.npz``),
its removal order on hand-written cases, the results-file reader and the command line."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_perturbation as mg
from oracle import perturbation as opert

NAMES = mg.NAMES


def _equal(a, b):
    """torch.equal that also matches NaN positions (a dissimilarity is NaN when both probabilities underflow)."""
    a, b = torch.from_numpy(np.asarray(a)), torch.from_numpy(np.asarray(b))
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(torch.isnan(a), torch.isnan(b)) and \
        torch.equal(a.nan_to_num(nan=0.), b.nan_to_num(nan=0.))


@pytest.fixture(scope="module")
def fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "perturbation.npz"))
    p, heads = mg.params()
    images, vis, target = mg.samples(p, heads)
    assert np.array_equal(images.double().sum(dim=(1, 2, 3)).numpy(), g["image_checksum"])
    assert np.array_equal(vis.double().sum(dim=(1, 2, 3)).numpy(), g["vis_checksum"])
    assert np.array_equal(target.numpy(), g["target"])
    loader = torch.utils.data.DataLoader(mg._Samples(images, vis, target), batch_size=int(g["batch"]), shuffle=False)
    return g, opert.vit_logits_fn(p, heads, norm_eps=mg.EPS), loader


@pytest.mark.parametrize("neg", [True, False])
@pytest.mark.parametrize("scale", ["per", "100"])
def test_oracle_matches_reference_eval(fixture, neg, scale):
    g, fn, loader = fixture
    res = opert.evaluate(fn, loader, neg=neg, scale=scale)
    for n in NAMES:
        assert _equal(res[n], g["%s.%s.%s" % ("neg" if neg else "pos", scale, n)]), n
    assert res["perturbations_hits"].shape == (9, int(g["n"]))


def test_oracle_wrong_mode_perturbation_arrays_match_reference(fixture):
    """``--wrong``: the perturbation arrays are the reference's; the model arrays hold one entry per sample (the
    reference's are overwritten out of place, a documented deviation)."""
    g, fn, loader = fixture
    res = opert.evaluate(fn, loader, neg=True, scale="per", wrong=True)
    for n in NAMES[2:]:
        assert _equal(res[n], g["wrong.neg.per." + n]), n
    assert res["model_hits"].shape == (int(g["n"]),)
    assert _equal(res["model_hits"], g["neg.per.model_hits"])


def test_step_sizes_follow_python_double():
    assert opert.step_sizes("per") == [int(224 * 224 * s) for s in (0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9)]
    assert opert.step_sizes("per")[2] == 15052 and opert.step_sizes("100") == list(range(500, 4501, 500))
    from transformer_explainability_b200 import perturbation as tp
    for scale in ("per", "100"):
        assert tp.perturbation_steps(scale)[1] == opert.step_sizes(scale)
    with pytest.raises(ValueError):
        opert.step_sizes("10")


def test_removal_order_hand_written_cases():
    """NaN first, then descending value, then ascending index; -0.0 == +0.0."""
    v = torch.tensor([[0.5, float("nan"), -0.0, 0.0, 0.5, 1.0]])
    assert opert.removal_order(v, negate=False).tolist() == [[1, 5, 0, 4, 2, 3]]
    assert opert.removal_order(v, negate=True).tolist() == [[1, 2, 3, 0, 4, 5]]
    v = torch.tensor([[0.0, -0.0, 0.0, -0.0]])
    assert opert.removal_order(v, negate=False).tolist() == [[0, 1, 2, 3]]
    assert opert.removal_order(v, negate=True).tolist() == [[0, 1, 2, 3]]
    v = torch.tensor([[float("nan")] * 3 + [float("-inf"), float("inf")]])
    assert opert.removal_order(v, negate=False).tolist() == [[0, 1, 2, 4, 3]]
    assert opert.removal_order(v, negate=True).tolist() == [[0, 1, 2, 3, 4]]


def test_perturb_is_scatter_then_normalize():
    g = torch.Generator().manual_seed(3)
    x = torch.rand(2, 3, 4, 4, generator=g)
    vis = torch.randn(2, 16, generator=g)
    out = opert.perturb(x, vis, [0, 5, 16], negate=False)
    assert torch.equal(out[0], (x - 0.5) / 0.5)
    assert torch.equal(out[2], torch.full_like(x, -1.0))
    order = vis.argsort(dim=1, descending=True)[:, :5]
    want = x.clone().reshape(2, 3, 16)
    for b in range(2):
        want[b][:, order[b]] = 0
    assert torch.equal(out[1], (want.reshape(x.shape) - 0.5) / 0.5)


def test_imagenet_results_reads_builtin_file_lazily(tmp_path):
    from transformer_explainability_b200 import hdf5_writer
    from transformer_explainability_b200.perturbation import ImagenetResults
    g = torch.Generator().manual_seed(1)
    with hdf5_writer.ResultsWriter(str(tmp_path), size=16, backend="builtin") as w:
        for _ in range(2):
            w.append(torch.rand(3, 3, 16, 16, generator=g).numpy(), torch.rand(3, 1, 16, 16, generator=g).numpy(),
                     torch.randint(0, 1000, (3,), generator=g).numpy())
    want = hdf5_writer.read_minimal_hdf5(os.path.join(str(tmp_path), "results.hdf5"))
    try:
        import h5py      # noqa: F401
        pytest.skip("h5py present: ImagenetResults reads through h5py")
    except ImportError:
        pass
    ds = ImagenetResults(str(tmp_path))
    assert len(ds) == 6
    assert ds.data is None                                     # nothing is read before the first item
    for i in range(len(ds)):
        image, vis, target = ds[i]
        assert isinstance(ds.data["image"], np.memmap)
        assert torch.equal(image, torch.from_numpy(want["image"][i]))
        assert torch.equal(vis, torch.from_numpy(want["vis"][i]))
        assert target.dtype == torch.int64 and int(target) == int(want["target"][i])
    import pickle
    copy = pickle.loads(pickle.dumps(ds))                      # what a DataLoader worker receives: it re-opens the file
    assert copy.data is None and torch.equal(copy[5][0], torch.from_numpy(want["image"][5]))


def test_dataset_alias_resolves():
    import transformer_explainability_b200 as te
    te.install_aliases()
    from dataset.expl_hdf5 import ImagenetResults
    from transformer_explainability_b200.perturbation import ImagenetResults as ours
    assert ImagenetResults is ours


def test_cli_parses_real_booleans_and_names_experiments(tmp_path):
    from transformer_explainability_b200 import perturbation as tp
    p = tp.build_parser()
    a = p.parse_args([])
    assert a.neg is True and a.is_ablation is False and a.scale == "per" and a.method == "grad_rollout"
    assert a.batch_size == 16 and a.vis_class == "top" and not a.wrong and a.state_dict is None
    a = p.parse_args(["--neg", "False", "--is-ablation", "true", "--method", "transformer_attribution", "--state-dict", "w.pth"])
    assert a.neg is False and a.is_ablation is True and a.state_dict == "w.pth"
    with pytest.raises(SystemExit):
        p.parse_args(["--neg", "maybe"])
    root = str(tmp_path)
    a = p.parse_args(["--method", "rollout", "--neg", "0"])
    assert tp.runs_dir(a, root) == os.path.join(root, "experiments/perturbations/rollout_pos/top/not_ablation")
    assert tp.vis_method_dir(a, root) == os.path.join(root, "visualizations/rollout/top/not_ablation")
    a = p.parse_args(["--method", "lrp", "--is-ablation", "1", "--wrong"])
    assert tp.runs_dir(a, root) == os.path.join(root, "experiments/perturbations/lrp_neg/top/ablation_wrong")
    a = p.parse_args(["--method", "lrp", "--vis-class", "index", "--class-id", "7"])
    assert tp.runs_dir(a, root) == os.path.join(root, "experiments/perturbations/lrp_neg/index_7")
    runs = tp.runs_dir(a, root)
    assert tp.next_experiment_dir(runs) == os.path.join(runs, "experiment_0")
    os.makedirs(os.path.join(runs, "experiment_0"))
    os.makedirs(os.path.join(runs, "experiment_1"))
    assert tp.next_experiment_dir(runs) == os.path.join(runs, "experiment_2")


def test_save_and_hits_auc(tmp_path):
    from transformer_explainability_b200 import perturbation as tp
    res = {"model_hits": np.ones(4), "model_dissimilarities": np.zeros(4),
           "perturbations_hits": np.tile(np.linspace(0.9, 0.1, 9)[:, None], (1, 4)),
           "perturbations_dissimilarities": np.zeros((9, 4)), "perturbations_logit_diff": np.zeros((9, 4)),
           "perturbations_prob_diff": np.zeros((9, 4))}
    tp.save(res, str(tmp_path / "experiment_0"))
    for n in NAMES:
        assert np.array_equal(np.load(str(tmp_path / "experiment_0" / (n + ".npy"))), res[n])
    xs = [0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]
    ys = [1.0] + list(np.linspace(0.9, 0.1, 9))
    assert tp.hits_auc(res, "per") == pytest.approx(np.trapezoid(ys, xs))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the loud failure on a GPU-less host")
def test_perturbation_ops_have_no_cpu_fallback():
    from transformer_explainability_b200 import ops
    with pytest.raises(ValueError):
        ops.perturb_images(torch.zeros(1, 3, 4, 4), torch.zeros(1, 16), [0, 1])
    with pytest.raises(ValueError):
        ops.logit_stats(torch.zeros(2, 10), torch.zeros(2, dtype=torch.long))


def test_perturb_entry_points_validate_arguments_without_gpu():
    """Bad shapes are reported through the status code before anything is launched."""
    import ctypes
    from transformer_explainability_b200 import _lib
    lib = _lib.load()
    assert lib.te_perturb_workspace_bytes(2, 50176) > 0 and lib.te_perturb_workspace_bytes(2, 50176) % 256 == 0
    assert lib.te_perturb_workspace_bytes(0, 50176) < 0 and lib.te_perturb_workspace_bytes(1, 0) < 0
    fake = ctypes.c_void_p(256)
    mean = (_lib.c_float * 3)(0.5, 0.5, 0.5)

    def call(ks, steps=None, channels=3, pixels=16):
        k = (_lib.c_int * len(ks))(*ks)
        return lib.te_perturb_images(fake, fake, 1, channels, pixels, k, len(ks) if steps is None else steps, 0, mean, mean,
                                     fake, fake, 1 << 20, None)
    assert call([0, 17]) == -1 and b"[0, pixels]" in lib.te_last_error()
    assert call([5, 4]) == -1 and b"non-decreasing" in lib.te_last_error()
    assert call([0] * 65) == -1 and call([0], channels=17) == -1
    assert lib.te_logit_stats(fake, fake, 4, 1, fake, fake, fake, fake, None) == -1
