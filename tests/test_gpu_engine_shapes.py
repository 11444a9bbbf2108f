"""GPU: the ViT and BERT engines at token counts the rest of the suite never runs, per layer against the fp64 oracle's taps.

Two-layer models of REAL width (D = 768, 12 heads, dh = 64, MLP 3072): every tensor-core predicate holds (the Linear / z+
kernels need widths that are multiples of 128, the attention kernels dh in {32, 64}), so the fast flag sets run the wgmma
kernels and not the SIMT fall-back, while the fp64 oracle stays fast.  Do not shrink the width below 128: the test would
silently become a SIMT test.

Token counts: BERT S = 37 (one ragged tile), 130 (two 128-row tiles, the second with 2 rows), 300 (ragged, above the fused
softmax's 256-key tile: scores + row softmax); ViT N = 50 (patch 32) and N = 577 (img 384: five 128-row tiles, ragged).
Tolerances (relative to the tensor maximum) are those of tests/test_gpu_tc.py::test_tc_attention_contractions_engine:
probabilities 1e-5, gradients 1e-4 (1e-3 with TE_FLAG_BACKWARD_TF32, as tests/test_gpu_parity_full.py states for the
single-pass TF32 backward), the top layer's attn_cam 5e-2.  Measured on one H100 80GB HBM3 at a 400 W power limit:
probabilities <= 3.7e-6, gradients <= 2.6e-6 (FLAG_ALL_FAST) / 6.8e-4 (FLAG_BENCH_DEFAULT), top attn_cam <= 2.2e-2 (ViT N = 577),
logits <= 1.8e-6.
"""
import pytest
import torch

from oracle import bert as obert
from oracle import cpu as ocpu
from oracle import vit as ovit
from transformer_explainability_b200 import _lib

pytestmark = pytest.mark.gpu

FLAG_SETS = [_lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT]


def rel(a, b):
    b = torch.as_tensor(b).double()
    return ((a.double().cpu() - b.cpu()).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def grad_tol(flags):
    return 1e-3 if flags & _lib.FLAG_BACKWARD_TF32 else 1e-4


@pytest.mark.parametrize("seq", [37, 130, 300])
def test_bert_engine_ragged_lengths(seq):
    from test_gpu_bert import make_model
    params, heads = obert.init_params(seed=3, vocab=1000, max_pos=512, dim=768, depth=2, heads=12, inter=3072,
                                      rand_affine=True)
    model = make_model(params, heads, hidden_size=768, num_hidden_layers=2, intermediate_size=3072, vocab_size=1000,
                       max_position_embeddings=512)
    eng = model.engine()
    g = torch.Generator().manual_seed(seq)
    ids = torch.randint(5, 1000, (3, seq), generator=g)
    ids[:, 0] = 101
    mask = torch.ones(3, seq, dtype=torch.long)
    pad = seq // 2
    mask[1, pad:] = 0                                              # sample 1 is padded from the middle on
    ocpu.set_torch_threads()
    ref, ridx, taps = obert.explain({k: v.double() for k, v in params.items()}, ids, mask, heads, start_layer=0,
                                    return_taps=True)
    layers = model.bert.encoder.layer
    for flags in FLAG_SETS:
        maps, idx, logits = eng.explain(ids.cuda(), mask.cuda(), start_layer=0, flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), ridx)
        el = rel(logits, taps["logits"])
        ea = [rel(layers[l].attention.self.get_attn(), taps["cache"]["layers"][l]["probs"]) for l in range(2)]
        eg = [rel(layers[l].attention.self.get_attn_gradients(), taps["grads"][l]) for l in range(2)]
        ec = rel(layers[1].attention.self.get_attn_cam(), taps["cams"][1])
        print("bert S %d flags %d: logits %.1e | attn %s | attn_grad %s | top attn_cam %.1e" % (
            seq, flags, el, ["%.1e" % e for e in ea], ["%.1e" % e for e in eg], ec))
        assert el < 1e-4
        assert max(ea) < 1e-5 and max(eg) < grad_tol(flags) and ec < 5e-2
        assert (maps[1, pad:] == 0).all(), "padded positions must get exactly zero relevance"
        for l in range(2):
            assert (layers[l].attention.self.get_attn()[1, :, :, pad:] == 0).all(), "a padded key got probability"


@pytest.mark.parametrize("img,patch", [(224, 32), (384, 16)])
def test_vit_engine_ragged_token_counts(img, patch):
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import VisionTransformer
    params, heads = ovit.init_params("vit_base_patch16_224", seed=4, img=img, patch=patch, depth=2, classes=10,
                                     rand_affine=True)
    m = VisionTransformer(img_size=img, patch_size=patch, embed_dim=768, depth=2, num_heads=heads, mlp_ratio=4.,
                          qkv_bias=True, num_classes=10)
    m.load_state_dict(params)
    m = m.cuda().eval()
    eng = m.engine()
    x = torch.randn(2, 3, img, img, generator=torch.Generator().manual_seed(img))
    ocpu.set_torch_threads()
    ref, ridx, taps = ovit.explain({k: v.double() for k, v in params.items()}, x.double(), heads, return_taps=True)
    n = (img // patch) ** 2 + 1
    assert taps["grads"][0].shape[-1] == n
    for flags in FLAG_SETS:
        maps, idx, logits = eng.explain(x.cuda(), flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), ridx)
        el = rel(logits, taps["logits"])
        ea = [rel(m.blocks[l].attn.get_attn(), taps["cache"]["blocks"][l]["attn"]) for l in range(2)]
        eg = [rel(m.blocks[l].attn.get_attn_gradients(), taps["grads"][l]) for l in range(2)]
        ec = rel(m.blocks[1].attn.get_attn_cam(), taps["cams"][1])
        print("vit N %d flags %d: logits %.1e | attn %s | attn_grad %s | top attn_cam %.1e" % (
            n, flags, el, ["%.1e" % e for e in ea], ["%.1e" % e for e in eg], ec))
        assert el < 1e-4
        assert max(ea) < 1e-5 and max(eg) < grad_tol(flags) and ec < 5e-2
