"""CPU: the gradient-weighted attention rollout oracle (``oracle/attn_grad_rollout.py``) against the fixture made from the
reference's own attention maps and gradients (``oracle/make_golden_attn_grad_rollout.py``), and the ``attn_grad_rollout``
choice of every evaluation command, next to its unchanged methods."""
import os

import numpy as np
import pytest
import torch

from oracle import attn_grad_rollout as agr
from oracle import bert as obert
from oracle import vit as ovit

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "attn_grad_rollout.npz")
MODELS = {"vit": 3, "deit": 3, "bert": 3}          # blocks of each tiny model


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def _taps(z, key, L):
    return ([torch.from_numpy(z["%s.attn.%d" % (key, l)]) for l in range(L)],
            [torch.from_numpy(z["%s.grad.%d" % (key, l)]) for l in range(L)])


@pytest.mark.parametrize("model", sorted(MODELS))
@pytest.mark.parametrize("tag", ["f32", "f64"])
def test_rule_on_the_fixture_taps_is_bit_exact(z, model, tag):
    for s in range(2):
        key = "%s.%s.s%d" % (model, tag, s)
        attns, grads = _taps(z, key, MODELS[model])
        for sl in z["start_layers"]:
            want = torch.from_numpy(z["%s.map.sl%d" % (key, sl)])
            if model == "bert":
                got = agr.bert_map(attns, grads, int(sl))
            else:
                got = agr.vit_map(attns, grads, int(sl), prefix=2 if model == "deit" else 1)
            assert got.dtype == want.dtype and torch.equal(got, want), (key, int(sl))


def test_padded_bert_positions_are_zero(z):
    mask = z["mask"]
    for tag in ("f32", "f64"):
        for sl in z["start_layers"]:
            m = z["bert.%s.s1.map.sl%d" % (tag, sl)][0]
            assert (m[mask[1] == 0] == 0).all() and m[0] == 0
            assert (m[1:][mask[1][1:] == 1] > 0).all()


def _vit_params(z, model, dt):
    seed = int(z[model + ".param_seed"])
    p, h = ovit.init_params("vit_tiny_test", seed=seed, rand_affine=True, distilled=(model == "deit"))
    return {k: v.to(dt) for k, v in p.items()}, h


@pytest.mark.parametrize("model", ["vit", "deit"])
@pytest.mark.parametrize("tag", ["f32", "f64"])
def test_oracle_end_to_end_against_the_fixture(z, model, tag):
    """The oracle's own forward and class gradient give the fixture's maps and class index (fp64: to rounding, fp32:
    to the reference's fp32 forward)."""
    dt = torch.float64 if tag == "f64" else torch.float32
    p, h = _vit_params(z, model, dt)
    x = torch.from_numpy(z["x"]).to(dt)
    for sl in z["start_layers"]:
        maps, idx = agr.explain_vit(p, x, h, start_layer=int(sl))
        for s in range(2):
            key = "%s.%s.s%d" % (model, tag, s)
            assert int(idx[s]) == int(z[key + ".index"])
            want = torch.from_numpy(z["%s.map.sl%d" % (key, sl)])[0]
            err = (maps[s] - want).abs().max() / want.abs().max()
            assert err < (1e-12 if tag == "f64" else 1e-5), (key, float(err))


@pytest.mark.parametrize("tag", ["f32", "f64"])
def test_bert_oracle_end_to_end_against_the_fixture(z, tag):
    dt = torch.float64 if tag == "f64" else torch.float32
    p, h = obert.init_params(seed=int(z["bert.param_seed"]), vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128,
                             rand_affine=True)
    p = {k: v.to(dt) for k, v in p.items()}
    ids, mask = torch.from_numpy(z["ids"]), torch.from_numpy(z["mask"])
    for sl in z["start_layers"]:
        for s in range(2):
            key = "bert.%s.s%d" % (tag, s)
            n = int(mask[s].sum())
            # one sample at a time, unpadded and padded: the padded tail adds nothing
            for m in (mask[s:s + 1], None):
                i, mm = (ids[s:s + 1], m) if m is not None else (ids[s:s + 1, :n], mask[s:s + 1, :n])
                maps, idx = agr.explain_bert(p, i, mm, h, start_layer=int(sl))
                assert int(idx[0]) == int(z[key + ".index"])
                want = torch.from_numpy(z["%s.map.sl%d" % (key, sl)])[0, :maps.shape[1]]
                err = (maps[0] - want).abs().max() / want.abs().max()
                assert err < (1e-12 if tag == "f64" else 1e-5), (key, int(sl), float(err))


# ---- the evaluation commands -------------------------------------------------------------------------------------------------
def test_segmentation_accepts_the_method_and_keeps_its_methods():
    from transformer_explainability_b200 import segmentation as seg
    assert seg.METHODS == ("rollout", "transformer_attribution", "full_lrp", "lrp_last_layer", "attn_last_layer",
                           "attn_gradcam")
    args = seg.parse_args(["--method", "attn_grad_rollout", "--imagenet-seg-path", "x.mat"])
    assert args.method == "attn_grad_rollout"
    assert seg.runs_dir(args, "/r").endswith(os.path.join("run", "imagenet", "attn_grad_rollout_vgg"))
    seg.check_method("attn_grad_rollout")
    with pytest.raises(ValueError):
        seg.check_method("grad_rollout")


def test_hdf5_writer_accepts_the_method_and_keeps_its_methods():
    from transformer_explainability_b200 import hdf5_writer, perturbation
    assert hdf5_writer.METHODS == ("rollout", "lrp", "transformer_attribution", "full_lrp", "lrp_last_layer",
                                   "attn_last_layer", "attn_gradcam")
    assert set(hdf5_writer.MODEL_KIND) == set(hdf5_writer.METHODS)
    args = hdf5_writer.parse_args(["--method", "attn_grad_rollout", "--imagenet-validation-path", "v"])
    assert perturbation.vis_method_dir(args, "/r") == os.path.join("/r", "visualizations", "attn_grad_rollout", "top",
                                                                    "not_ablation")


def test_perturbation_accepts_the_method_and_keeps_its_methods():
    from transformer_explainability_b200 import perturbation
    assert perturbation.METHODS[:-1] == ['rollout', 'lrp', 'transformer_attribution', 'full_lrp', 'v_gradcam',
                                         'lrp_last_layer', 'lrp_second_layer', 'gradcam', 'attn_last_layer',
                                         'attn_gradcam', 'input_grads']
    args = perturbation.build_parser().parse_args(["--method", "attn_grad_rollout", "--neg", "False"])
    assert perturbation.runs_dir(args, "/r") == os.path.join("/r", "experiments", "perturbations", "attn_grad_rollout_pos",
                                                              "top", "not_ablation")
    assert perturbation.build_parser().parse_args([]).method == "grad_rollout"     # the reference's default, unchanged


def test_eraser_accepts_the_method_and_keeps_its_methods():
    from transformer_explainability_b200 import eraser as te
    assert te.METHODS == ("transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout")
    assert set(te.METHOD_FOLDER) == set(te.METHODS) == set(te.METHOD_GENERATOR)
    args = te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p.json", "--method",
                          "attn_grad_rollout", "--faithfulness", "--soft-scores", "--tokens-to-flip"])
    assert args.method == "attn_grad_rollout" and args.faithfulness and args.soft_scores and args.tokens_to_flip
    assert te.FOLLOW_UP_GENERATOR["attn_grad_rollout"] == ("ours", "generate_attn_grad_rollout")
    assert te.build_parser().parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p"]).method == \
        "transformer_attribution"


def test_visualization_accepts_the_method():
    from transformer_explainability_b200 import visualization as vis
    assert vis.parse_args(["--images", "a", "--output-dir", "o"]).method == "transformer_attribution"
    assert vis.parse_args(["--images", "a", "--output-dir", "o", "--method", "attn_grad_rollout"]).method == \
        "attn_grad_rollout"
    with pytest.raises(SystemExit):
        vis.parse_args(["--images", "a", "--output-dir", "o", "--method", "rollout"])


def test_generators_exist_on_every_facade():
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    import inspect
    for cls, first in ((LRP, "input"), (Generator, "input_ids")):
        sig = inspect.signature(cls.generate_attn_grad_rollout)
        assert list(sig.parameters)[1] == first
        assert sig.parameters["start_layer"].default == 0 and sig.parameters["index"].default is None


def test_flag_is_its_own_bit():
    from transformer_explainability_b200 import _lib
    assert _lib.FLAG_ATTN_GRAD_ROLLOUT == 65536
    assert not _lib.FLAG_BENCH_DEFAULT & _lib.FLAG_ATTN_GRAD_ROLLOUT
