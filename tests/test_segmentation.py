"""CPU: the segmentation-evaluation oracle against the reference's own ``imagenet_seg_eval.py`` run
(``tests/golden/segmentation.npz``), its sklearn restatement against sklearn, and the command line / output layout."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_segmentation as mgs
from oracle import segmentation as oseg

METHODS = mgs.METHODS


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "segmentation.npz"))


@pytest.mark.parametrize("method", METHODS)
def test_oracle_matches_reference_script(golden, method):
    g = golden
    maps = torch.from_numpy(g[method + ".maps"])
    labels = torch.from_numpy(g["labels"].astype(np.int64))[g[method + ".samples"]]
    assert np.array_equal(g[method + ".samples"], mgs.method_samples(method))
    per, tot, precision, recall = oseg.evaluate(maps, labels, scale=1 if method == "full_lrp" else 16)
    pre = method + "."
    assert np.array_equal([p["correct"] for p in per], g[pre + "correct"])
    assert np.array_equal([p["labeled"] for p in per], g[pre + "labeled"])
    assert np.array_equal(np.stack([p["inter"] for p in per]), g[pre + "inter"])
    assert np.array_equal(np.stack([p["union"] for p in per]), g[pre + "union"])
    assert np.array_equal([p["ap"] for p in per], g[pre + "ap"])
    assert np.array_equal(np.stack([p["f1"] for p in per]), g[pre + "f1"])
    for k in ("pixAcc", "mIoU", "mF1"):
        assert tot[k] == g[pre + k], k
    assert tot["mAP"] == g[pre + "mAp"]
    assert np.array_equal(tot["IoU"], g[pre + "IoU"])
    for k, v in oseg.pr_summary(precision, recall).items():
        assert np.array_equal(v, g[pre + k]), k
    from transformer_explainability_b200 import segmentation as ts
    res = {"mIoU": tot["mIoU"], "pixAcc": tot["pixAcc"], "mAP": tot["mAP"], "mF1": tot["mF1"]}
    assert "".join(ts.report_lines(res)) == str(g[pre + "txt"])
    assert "result_mIoU_%.4f.txt" % tot["mIoU"] == str(g[pre + "txt_name"])


def test_fixture_covers_empty_and_full_masks(golden):
    lab = golden["labels"]
    assert lab[int(golden["empty_mask"])].max() == 0 and lab[int(golden["full_mask"])].min() == 1
    images, labels = mgs.samples()
    assert np.array_equal(labels.numpy(), lab.astype(np.int64))
    assert np.array_equal(images.double().sum(dim=(1, 2, 3)).numpy(), golden["image_checksum"])


def _tie_heavy(seed, n):
    g = np.random.default_rng(seed)
    scores = (g.integers(0, 7, n) / 6).astype(np.float32)
    scores[g.random(n) < 0.1] = -0.0 if seed % 2 else 0.0
    return g.integers(0, 2, n), scores


@pytest.mark.parametrize("seed", range(6))
def test_restatement_equals_sklearn(seed):
    sk = pytest.importorskip("sklearn.metrics")
    for n in (1, 2, 17, 5000):
        y, s = _tie_heavy(seed, n)
        if seed == 0:
            y[:] = 1
        p1, r1, t1 = oseg.precision_recall_curve(y, s)
        with np.errstate(all="ignore"):
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                p2, r2, t2 = sk.precision_recall_curve(y, s)
                ap2 = np.nan_to_num(sk.average_precision_score(y, s)) if 0 < y.sum() < n or y.sum() == n else None
                f2 = sk.f1_score(y, (s > 0.5).astype(np.float32))
        assert np.array_equal(p1, p2) and np.array_equal(r1, r2) and np.array_equal(t1, t2)
        if ap2 is not None:
            assert oseg.average_precision(y, s) == ap2
        pred = s > 0.5
        tp, fp, fn = int((pred & (y == 1)).sum()), int((pred & (y == 0)).sum()), int((~pred & (y == 1)).sum())
        assert oseg.f1(tp, fp, fn) == f2


def test_cli_arguments_and_validation():
    from transformer_explainability_b200 import segmentation as ts
    a = ts.parse_args(["--method", "rollout", "--imagenet-seg-path", "x.mat"])
    assert a.thr == 0. and a.is_ablation is False and a.batch_size == 32 and a.arc == "vgg" and a.state_dict is None
    a = ts.parse_args(["--method", "lrp_last_layer", "--imagenet-seg-path", "x.mat", "--is-ablation", "False",
                       "--batch-size", "7", "--arc", "vit", "--no-ia", "--K", "3"])
    assert a.is_ablation is False and a.batch_size == 7 and a.arc == "vit"
    assert ts.parse_args(["--method", "full_lrp", "--imagenet-seg-path", "x", "--is-ablation", "1"]).is_ablation is True
    for bad in (["--method", "lrp", "--imagenet-seg-path", "x"], ["--method", "blur", "--imagenet-seg-path", "x"],
                ["--method", "rollout"], ["--imagenet-seg-path", "x"],
                ["--method", "rollout", "--imagenet-seg-path", "x", "--save-img"],
                ["--method", "rollout", "--imagenet-seg-path", "x", "--is-ablation", "maybe"],
                ["--method", "rollout", "--imagenet-seg-path", "x", "--batch-size", "0"]):
        with pytest.raises(SystemExit):
            ts.parse_args(bad)
    with pytest.raises(ValueError):
        ts.check_method("lrp")
    with pytest.raises(ValueError):
        ts.explain("rollout", torch.zeros(1, 3, 224, 224))                # no generator for the method


def test_experiment_layout_and_outputs(tmp_path, capsys):
    from transformer_explainability_b200 import segmentation as ts
    a = ts.parse_args(["--method", "attn_gradcam", "--imagenet-seg-path", "x", "--arc", "vit"])
    runs = ts.runs_dir(a, str(tmp_path))
    assert runs == os.path.join(str(tmp_path), "run", "imagenet", "attn_gradcam_vit")
    d0 = ts.make_experiment_dir(runs)
    assert d0 == os.path.join(runs, "experiment_0")
    for sub in ("input", "explain/img", "explain/np"):
        assert os.path.isdir(os.path.join(d0, "results", sub)) and not os.listdir(os.path.join(d0, "results", sub))
    assert ts.make_experiment_dir(runs) == os.path.join(runs, "experiment_1")
    res = {"correct": np.array([3, 4]), "labeled": np.array([4, 4]), "inter": np.array([[1, 2], [2, 2]]),
           "union": np.array([[2, 3], [2, 2]]), "ap": np.array([0.5, 1.0]), "f1": np.array([[0.8, 0.5], [1.0, 0.0]])}
    res.update(ts.totals(res["correct"], res["labeled"], res["inter"], res["union"], res["ap"], res["f1"]))
    tot = oseg.totals(res["correct"], res["labeled"], list(res["inter"]), list(res["union"]), list(res["ap"]),
                      list(res["f1"]))
    for k in ("pixAcc", "mIoU", "mAP", "mF1"):
        assert res[k] == tot[k]
    res["precision"], res["recall"] = ts.precision_recall([1, 2, 2], [0, 1, 3])
    assert np.array_equal(res["precision"], [0.4, 2 / 3, 1.0, 1.0]) and np.array_equal(res["recall"], [1.0, 1.0, 0.5, 0.0])
    txt = ts.save(res, d0, "attn_gradcam")
    assert os.path.basename(txt) == "result_mIoU_%.4f.txt" % res["mIoU"]
    with open(txt) as fh:
        lines = fh.read().split("\n")
    assert lines[0] == "Mean IoU over 2 classes: %.4f" % res["mIoU"]
    assert lines[1] == "Pixel-wise Accuracy: %2.2f%%" % (res["pixAcc"] * 100)
    assert lines[2].startswith("Mean AP over 2 classes: ") and lines[3].startswith("Mean F1 over 2 classes: ")
    assert np.array_equal(np.load(os.path.join(d0, "precision.npy")), res["precision"])
    assert np.array_equal(np.load(os.path.join(d0, "recall.npy")), res["recall"])
    try:
        import matplotlib  # noqa: F401
        assert os.path.exists(os.path.join(d0, "PR_curve_attn_gradcam.png"))
    except ImportError:
        assert "matplotlib is not installed" in capsys.readouterr().out


def test_dataset_needs_h5py_with_a_clear_error(tmp_path):
    from transformer_explainability_b200 import segmentation as ts
    try:
        import h5py  # noqa: F401
        pytest.skip("h5py present")
    except ImportError:
        pass
    with pytest.raises(ImportError, match="h5py"):
        ts.ImagenetSegmentation(str(tmp_path / "gtsegs_ijcv.mat"))


def test_no_data_alias_is_installed():
    import sys
    import transformer_explainability_b200 as te
    te.install_aliases()
    assert "data" not in sys.modules or not getattr(sys.modules["data"], "__name__", "").startswith("transformer")


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the loud failure on a GPU-less host")
def test_segmentation_ops_have_no_cpu_fallback():
    from transformer_explainability_b200 import ops
    with pytest.raises(ValueError):
        ops.seg_metrics(torch.zeros(1, 196), torch.zeros(1, 224 * 224, dtype=torch.long))
    with pytest.raises(ValueError):
        ops.sort_keys(torch.zeros(8, dtype=torch.int32))
    with pytest.raises(ValueError):
        ops.pr_curve(torch.zeros(8, dtype=torch.int32))


def test_segmentation_entry_points_validate_arguments_without_gpu():
    import ctypes
    from transformer_explainability_b200 import _lib
    lib = _lib.load()
    assert lib.te_sort_workspace_bytes(10, 3) < 0 and lib.te_sort_workspace_bytes(12, 3) % 256 == 0
    assert lib.te_seg_workspace_bytes(2, 14, 16) > 2 * 2 * 50176 * 4 and lib.te_seg_workspace_bytes(0, 14, 16) < 0
    assert lib.te_pr_curve_workspace_bytes(0) < 0 and lib.te_pr_curve_workspace_bytes(5) > 0
    fake = ctypes.c_void_p(256)
    assert lib.te_sort_keys_u32(fake, fake, 10, 3, fake, 1 << 20, None) == -1
    assert lib.te_sort_keys_u32(fake, fake, 4096, 1, fake, 16, None) == -2
    big = lib.te_seg_workspace_bytes(1, 224, 1)
    assert lib.te_seg_metrics(fake, fake, 1, 200, 16, 0.0, fake, fake, fake, fake, fake, fake, None, fake, big, None) == -1
    assert b"45056" in lib.te_last_error()
    assert lib.te_seg_metrics(fake, fake, 1, 224, 1, float("nan"), fake, fake, fake, fake, fake, fake, None, fake, big, None) == -1
    assert lib.te_pr_curve(fake, 0, fake, fake, fake, fake, fake, 1 << 20, None) == -1
