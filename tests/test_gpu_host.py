"""GPU: ``_host.to_host`` on CUDA tensors, and the number of its calls (one device-to-host copy each) per command run.

- The round trip of every numpy dtype, 0-d, empty, non-contiguous and odd-sized tensors mixed with CPU tensors, bit for
  bit and aligned; a bfloat16 CUDA tensor is rejected.
- One call per batch for ``segmentation_eval``, ``text_visualization.run``, ``visualization.run``,
  ``compute_saliency_and_save`` and ``eraser.predictions``; for ``eraser_eval`` with every option on, one per batch, one
  per tokens-to-flip round and one at the end.
"""
import sys
from collections import Counter

import numpy as np
import pytest
import torch

from test_host import DTYPES, check, sample
from test_gpu_render import folder, small_model                                # noqa: F401 (fixtures)
from transformer_explainability_b200 import _host, eraser, hdf5_writer, segmentation, text_visualization, visualization

pytestmark = pytest.mark.gpu


def test_round_trip_on_cuda():
    for dtype in DTYPES:
        t = [sample(dtype, (3, 5), 1), sample(dtype, (), 2), sample(dtype, (0, 4), 3), sample(dtype, (7,), 4)[::2]]
        check(_host.to_host(*[x.cuda() for x in t]), t)
    t = [sample(torch.bool, (3,), 1), sample(torch.float64, (2, 3), 2), sample(torch.uint8, (5,), 3),
         sample(torch.float16, (3,), 4), sample(torch.int64, (4, 6), 5)[:, ::2], sample(torch.float64, (), 6),
         sample(torch.int32, (3, 4), 7).t(), sample(torch.float32, (0,), 8), sample(torch.float64, (3,), 9)]
    mixed = [x.cuda() if i % 3 else x for i, x in enumerate(t)]
    out = _host.to_host(*mixed)
    check(out, t)
    assert np.shares_memory(out[0], t[0].numpy()) and not np.shares_memory(out[1], t[1].numpy())
    with pytest.raises(ValueError, match="bfloat16"):
        _host.to_host(torch.zeros(2, device="cuda"), torch.zeros(2, dtype=torch.bfloat16, device="cuda"))


@pytest.fixture
def calls(monkeypatch):
    """Counter of ``to_host`` calls by the name of the calling function."""
    seen, to_host = Counter(), _host.to_host

    def counted(*tensors):
        seen[sys._getframe(1).f_code.co_name] += 1
        return to_host(*tensors)
    for mod in (eraser, segmentation, text_visualization, visualization):
        monkeypatch.setattr(mod, "to_host", counted)
    monkeypatch.setattr(_host, "to_host", counted)                        # hdf5_writer imports it at call time
    return seen


def test_segmentation_one_call_per_batch(calls):
    from test_gpu_segmentation import _generators, mgs
    images, labels = mgs.samples()
    lrp, _, _ = _generators()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(images, labels), batch_size=3)
    segmentation.segmentation_eval("transformer_attribution", loader, lrp=lrp)
    assert calls == {"segmentation_eval": len(loader)}


def test_text_visualization_one_call_per_batch(calls, tmp_path):
    from test_gpu_bert_pairs import PAIRS, TEXTS, save_model_dir
    model_dir = save_model_dir(tmp_path / "model")
    text_visualization.run(text_visualization.load_model(model_dir), text_visualization.load_tokenizer(model_dir), TEXTS,
                           PAIRS, batch_size=2, output_dir=str(tmp_path / "out"))
    assert calls == {"explain_batch": 2}


def test_visualization_one_call_per_batch(calls, small_model, folder, tmp_path):                  # noqa: F811
    paths = visualization.image_paths([folder])
    visualization.run(small_model, paths, str(tmp_path), class_indices=(3,), batch_size=3)
    assert calls == {"render_batch": -(-len(paths) // 3)}


def test_results_writer_one_call_per_batch(calls, small_model, tmp_path):                         # noqa: F811
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    g = torch.Generator().manual_seed(0)
    loader = [(torch.rand(b, 3, 224, 224, generator=g).to(dev), torch.arange(b)) for b, dev in ((2, "cuda"), (1, "cpu"))]
    hdf5_writer.compute_saliency_and_save(loader, str(tmp_path), "transformer_attribution", lrp=LRP(small_model),
                                          backend="builtin")
    assert calls == {"compute_saliency_and_save": 2}


def test_eraser_calls(calls, tmp_path):
    from test_gpu_eraser import _fixture
    from test_gpu_eraser_soft import FLIP_SHIFT, _generators
    g, docids, docs, anns, enc, te = _fixture()
    gen = _generators(FLIP_SHIFT)["transformer_attribution"]
    n = len(anns)
    eraser.predictions(te._generator_model(gen), anns, enc, batch_size=4)
    assert calls == {"predictions": -(-n // 4)}
    calls.clear()
    res = eraser.eraser_eval(gen, docs, anns, enc, {"NEG": 0, "POS": 1}, batch_size=4, same_length=False,
                             faithfulness=True, soft_scores=True, tokens_to_flip=True, flip_chunk=2, latex=True)
    assert calls["eraser_eval"] == -(-n // 4) and calls["result"] == 1
    assert calls["_flip_search"] >= -(-n // 4) and set(calls) == {"eraser_eval", "_flip_search", "result"}
    print("MEASURED eraser_eval: %d documents, %s to_host calls" % (n, dict(calls)))
    assert res["faithfulness"]["flipped"].any()
