"""GPU: full-size parity at the benched kernel selection, with bounds that can fail.

Random-init ViT-B / BERT-base are ill-conditioned (``oracle/conditioned.py``): the reference's own fp32 result differs
from its fp64 result by 1e-5 ... 7e-1 of the map maximum, so a single-draw comparison at full size says nothing about the
kernels.  Three complementary checks replace the order statistics of ``test_gpu_vit.py::check_parity`` as the primary
full-size parity evidence:

1. **Conditioned full-size models** (``oracle.conditioned``: every ``safe_divide`` denominator bounded away from zero;
   the fp32 CPU oracle agrees with the fp64 oracle to ~1e-5 of the map maximum) at every BASELINE config — ViT-B/16,
   ViT-L/16, DeiT-B distilled (198 tokens), BERT-base S=512 ``start_layer=0`` with one padded row — single draws at
   flags 0 (fp32 SIMT), 51 (round-1 tensor-core selection), 4147 (51 with the fp16-split forward Linears), 307 (+ TF32
   backward), 1331 (+ TF32 relevance-side attention contractions), 3379 (+ bf16 z+ denominator term), 15667 (+ the opt-in
   fp16 second z+ contraction) and the bench default 7475 (3379 + fp16-split forward), against the fp64 oracle: class index
   bit-exact, logits, attention gradients and attn_cam of bottom / middle / top layers, final map.
2. **Teacher-forced rules at ViT-B size on the REAL (ill-conditioned) random-init data**: every rule kernel is fed the
   oracle's inputs for that step, so kernel error is separated from the chain's chaotic amplification.
3. z+ rule edge cases: all-zero activation rows and all-zero weight rows (the ``b != 0`` mask of ``safe_divide``,
   ``modules/layers_ours.py:10-13``) and the cancelled-denominator fallback of the single-pass tensor-core kernel.

Stated tolerances (relative to the tensor maximum unless noted): fp32 SIMT engine 2e-4 on maps / taps; tensor-core
selections 5e-3 (TF32 operands, 2^-11 relative rounding, on the z+ contractions; 3xTF32 elsewhere).
"""
import pytest
import torch

from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import rules
from oracle import vit as ovit

pytestmark = pytest.mark.gpu


def rel(a, b):
    b = torch.as_tensor(b).double()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def _flag_sets():
    from transformer_explainability_b200 import _lib
    out = [(0, 2e-4), (_lib.FLAG_ALL_FAST, 5e-3),
           (_lib.FLAG_ALL_FAST | _lib.FLAG_LINEAR_F16_SPLIT, 5e-3),     # 4147: fp32-grade forward Linears as the fp16 split
           (_lib.FLAG_ALL_FAST | _lib.FLAG_BACKWARD_TF32, 5e-3)]
    out.append((_lib.FLAG_ALL_FAST | _lib.FLAG_BACKWARD_TF32 | _lib.FLAG_RELPROP_TF32, 5e-3))        # 1331
    out.append((_lib.FLAG_ALL_FAST | _lib.FLAG_BACKWARD_TF32 | _lib.FLAG_RELPROP_TF32 | _lib.FLAG_ZPLUS_S1_BF16, 5e-3))   # 3379
    out.append((_lib.FLAG_ALL_FAST | _lib.FLAG_BACKWARD_TF32 | _lib.FLAG_RELPROP_TF32 | _lib.FLAG_ZPLUS_S1_BF16 |
                _lib.FLAG_LINEAR_F16_SPLIT | _lib.FLAG_ZPLUS_R_F16, 5e-3))                          # 15667: + fp16 R kernel
    if _lib.FLAG_BENCH_DEFAULT not in [f for f, _ in out]:
        out.append((_lib.FLAG_BENCH_DEFAULT, 5e-3))                     # 7475: 3379 + fp16-split forward Linears
    return out


VIT_CASES = {
    "vit_base_patch16_224": dict(seed=0, xseed=100),
    "vit_large_patch16_224": dict(seed=2, xseed=7),
    "deit_base_distilled_patch16_224": dict(seed=4, xseed=9),
}


@pytest.mark.parametrize("name", sorted(VIT_CASES))
def test_conditioned_vit_full_size(name):
    from transformer_explainability_b200.baselines.ViT import ViT_LRP
    c = VIT_CASES[name]
    params, heads = ovit.init_params(name, seed=c["seed"], rand_affine=True)
    params = conditioned.condition_vit(params)
    n = 2
    xs = torch.randn(n, 3, 224, 224, generator=torch.Generator().manual_seed(c["xseed"]))
    model = getattr(ViT_LRP, name)()
    model.load_state_dict(params)
    model = model.cuda().eval()
    eng = model.engine()
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    ref, ridx, taps = ovit.explain(p64, xs.double(), heads, return_taps=True)
    ref32, _ = ovit.explain(params, xs, heads)
    L = len(taps["grads"])
    err_ref = max(rel(ref32[s], ref[s]) for s in range(n))
    assert err_ref < 1e-4, "regime is not conditioned: fp32 oracle vs fp64 oracle %g" % err_ref
    for flags, tol in _flag_sets():
        maps, idx, logits = eng.explain(xs.cuda(), flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), ridx)                         # bit-exact class index
        e_logit = rel(logits, taps["logits"])
        e_map = max(rel(maps[s], ref[s]) for s in range(n))
        e_g = {l: rel(model.blocks[l].attn.get_attn_gradients(), taps["grads"][l]) for l in (0, L // 2, L - 1)}
        e_c = {l: rel(model.blocks[l].attn.get_attn_cam(), taps["cams"][l]) for l in (0, L // 2, L - 1)}
        print("%s conditioned flags %d: logits %.1e | attn_grad %s | attn_cam %s | map %.1e (fp32 CPU oracle %.1e)" % (
            name, flags, e_logit, {k: "%.1e" % v for k, v in e_g.items()}, {k: "%.1e" % v for k, v in e_c.items()},
            e_map, err_ref))
        assert e_logit < 2e-5
        assert max(e_g.values()) < tol and max(e_c.values()) < tol
        assert e_map < tol, "%s flags %d: map rel err %g" % (name, flags, e_map)
        assert (maps.cpu().double() - ref).abs().max().item() < 1e-4       # the north-star absolute tolerance


def _bert_model(params, heads):
    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    m = BertForSequenceClassification(BertConfig(num_attention_heads=heads, num_labels=2))
    res = m.load_state_dict({k: v.float() for k, v in params.items()}, strict=False)
    assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
    return m.cuda().eval()


def _bert_inputs(n, seq, pad_row=True):
    g = torch.Generator().manual_seed(seq)
    ids = torch.randint(1000, 5000, (n, seq), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones(n, seq, dtype=torch.long)
    if pad_row:
        mask[n - 1, seq * 3 // 4:] = 0                                     # last 25 % of one row is padding (SURVEY 8d config 5)
    return ids, mask


def test_conditioned_bert_s512_start_layer0():
    """BASELINE configs[4] as ``bench.py --workload bert_base`` times it: S=512, start_layer=0 (all 12 layers relprop'd),
    batch 3 with one padded row.  The conditioned map is nearly flat (row-normalised rollout), so its error is stated
    relative to the map's RANGE over the real tokens, not its maximum."""
    params, heads = obert.init_params(seed=0, rand_affine=True)
    params = conditioned.condition_bert(params)
    n, seq = 3, 512
    ids, mask = _bert_inputs(n, seq)
    model = _bert_model(params, heads)
    eng = model.engine()
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    ref, ridx, taps = obert.explain(p64, ids, mask, heads, start_layer=0, return_taps=True)
    ref32, _ = obert.explain(params, ids, mask, heads, start_layer=0)

    def range_err(m, s):
        live = mask[s].bool()
        live[0] = False                                                    # [0] is overwritten with the row minimum
        r = ref[s][live]
        return ((m.double().cpu()[live] - r).abs().max() / (r.max() - r.min()).clamp_min(1e-300)).item()

    err_ref = max(range_err(ref32[s], s) for s in range(n))
    assert err_ref < 5e-2, "regime is not conditioned: fp32 oracle vs fp64 oracle %g of the map range" % err_ref
    layers = model.bert.encoder.layer
    from transformer_explainability_b200 import _lib
    for flags, tol in [(0, 2e-4), (_lib.FLAG_ZPLUS_TENSOR_CORES, 5e-3)] + _flag_sets()[1:]:
        maps, idx, logits = eng.explain(ids.cuda(), mask.cuda(), start_layer=0, flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), ridx)
        e_logit = rel(logits, taps["logits"])
        e_g = {l: rel(layers[l].attention.self.get_attn_gradients(), taps["grads"][l]) for l in (0, 6, 11)}
        e_c = {l: rel(layers[l].attention.self.get_attn_cam(), taps["cams"][l]) for l in (0, 6, 11)}
        e_map = max(rel(maps[s], ref[s]) for s in range(n))
        e_rng = max(range_err(maps[s], s) for s in range(n))
        print("bert-base S=512 start 0 conditioned flags %d: logits %.1e | attn_grad %s | attn_cam %s | map %.1e of max, "
              "%.1e of range (fp32 CPU oracle %.1e of range)" % (flags, e_logit, {k: "%.1e" % v for k, v in e_g.items()},
                                                                  {k: "%.1e" % v for k, v in e_c.items()}, e_map, e_rng, err_ref))
        assert e_logit < 2e-5
        assert max(e_g.values()) < tol and max(e_c.values()) < tol
        assert e_map < tol
        # the conditioned BERT map is nearly flat (range ~ 1/300 of its maximum), so the range-relative number magnifies
        # every error ~300x: fp32 engine within 3x of the fp32 CPU oracle, TF32 z+ operands 5e-2, TF32 backward 0.3
        rng_tol = 3 * err_ref if flags == 0 else (0.3 if flags & _lib.FLAG_BACKWARD_TF32 else 5e-2)
        assert e_rng < rng_tol
        assert float(maps[n - 1, seq * 3 // 4:].abs().max()) == 0.0       # padded tokens: exactly zero relevance


def test_bert_s512_start_layer0_random_init():
    """The same config on the raw random-init model (what the bench times).  The reference itself is ill-conditioned here
    (its fp32 result deviates from its fp64 result by 0.1-0.7 of the map maximum), so the map is judged against that
    measured error; logits, class index and the attention gradients of the top and bottom layers (which chain through
    every forward / backward kernel of all 12 layers at S=512) are tight."""
    from transformer_explainability_b200 import _lib
    params, heads = obert.init_params(seed=0, rand_affine=True)
    n, seq = 3, 512
    ids, mask = _bert_inputs(n, seq)
    model = _bert_model(params, heads)
    eng = model.engine()
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    ref, ridx, taps = obert.explain(p64, ids, mask, heads, start_layer=0, return_taps=True)
    ref32, _ = obert.explain(params, ids, mask, heads, start_layer=0)
    err_ref = sorted(rel(ref32[s], ref[s]) for s in range(n))
    layers = model.bert.encoder.layer
    for flags in (0, _lib.FLAG_ZPLUS_TENSOR_CORES, _lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT):
        maps, idx, logits = eng.explain(ids.cuda(), mask.cuda(), start_layer=0, flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), ridx)
        assert rel(logits, taps["logits"]) < 1e-4
        gtol = 1e-3 if flags & _lib.FLAG_BACKWARD_TF32 else 2e-4
        assert rel(layers[11].attention.self.get_attn_gradients(), taps["grads"][11]) < gtol
        assert rel(layers[0].attention.self.get_attn_gradients(), taps["grads"][0]) < 5 * gtol
        cam = sorted(rel(layers[11].attention.self.get_attn_cam()[s], taps["cams"][11][s]) for s in range(n))
        errs = sorted(rel(maps[s], ref[s]) for s in range(n))
        print("bert-base S=512 start 0 random-init flags %d: top-cam %s | map %s | reference fp32-vs-fp64 %s" % (
            flags, ["%.1e" % e for e in cam], ["%.1e" % e for e in errs], ["%.1e" % e for e in err_ref]))
        assert cam[n // 2] < 5e-2
        assert errs[n // 2] <= max(5e-2, 3 * err_ref[n // 2])
        assert float(maps[n - 1, seq * 3 // 4:].abs().max()) == 0.0


# ---- teacher-forced rules at ViT-B size -------------------------------------------------------------------------------
def _g(t):
    return t.float().contiguous().cuda()


@pytest.mark.parametrize("tc", [False, True])
def test_rules_teacher_forced_at_vit_base_size(tc):
    """Every relprop rule of blocks 11, 10, 9 of a random-init ViT-B/16 (the ill-conditioned data the bench runs on), each
    kernel fed with the ORACLE's inputs for that step (batch 2).  Bounds: Add / Clone 1e-6; z+ Linear 1e-5 (fp32 SIMT) /
    3e-3 (tensor-core TF32, with the saved forward output: the single-pass kernel the engines run); matmul2 rule 5e-4; the
    matmul1 rule divides by signed near-zero Q K^T — its fp32 evaluation is itself ill-conditioned, so it is judged
    against the fp32 CPU oracle evaluated on the same inputs (error <= 10x that, or 1e-5)."""
    from transformer_explainability_b200 import ops
    nb = 2
    ocpu.set_torch_threads()
    params, heads = ovit.init_params("vit_base_patch16_224", seed=0)
    xs = torch.randn(nb, 3, 224, 224, generator=torch.Generator().manual_seed(100))
    with torch.enable_grad():
        logits, cache = ovit.forward(params, xs, heads, need_grad=True)
    blocks = [{k: v.detach() for k, v in c.items()} for c in cache["blocks"]]
    xf = cache["x_final_norm"].detach()
    seed = torch.zeros_like(logits)
    seed[torch.arange(nb), logits.argmax(-1)] = 1
    p = params
    D = lambda t: t.double()                                               # noqa: E731
    r_cls = rules.linear_relprop(D(xf[:, 0]), D(p["head.weight"]), D(seed.detach()))
    r = rules.index_select_relprop(D(xf), r_cls.unsqueeze(1), 0)
    lin_tol = 3e-3 if tc else 1e-5

    def lin(x, w, b, rr, what):
        o = rules.linear_relprop(D(x), D(w), D(rr))
        x2 = _g(x).reshape(-1, x.shape[-1])
        y = ops.linear_forward(x2, _g(w), _g(b), tensor_cores=tc) if tc else None
        gg = ops.linear_relprop(x2, _g(w), _g(rr).reshape(-1, rr.shape[-1]), tensor_cores=tc, y=y,
                                bias=_g(b) if tc else None).reshape(o.shape)
        e = rel(gg, o)
        assert e < lin_tol, "%s: %g" % (what, e)
        return o.float()

    for i in (11, 10, 9):
        pre = "blocks.%d." % i
        c = blocks[i]
        r32 = r.float()
        o1, o2 = rules.add_relprop(D(c["x_mid"]), D(c["mlp_out"]), D(r32))
        g1, g2 = ops.add_relprop(_g(c["x_mid"]), _g(c["mlp_out"]), _g(r32))
        assert rel(g1, o1) < 1e-6 and rel(g2, o2) < 1e-6, "L%d add2" % i
        r1, r2 = o1.float(), o2.float()
        rf = lin(c["g"], p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"], r2, "L%d fc2" % i)
        r2 = lin(c["xn2"], p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"], rf, "L%d fc1" % i)
        o = rules.clone_relprop(D(c["x_mid"]), (D(r1), D(r2)))
        assert rel(ops.clone_relprop(_g(c["x_mid"]), [_g(r1), _g(r2)]), o) < 1e-6, "L%d clone2" % i
        r32 = o.float()
        o1, o2 = rules.add_relprop(D(c["x_in"]), D(c["attn_out"]), D(r32))
        g1, g2 = ops.add_relprop(_g(c["x_in"]), _g(c["attn_out"]), _g(r32))
        assert rel(g1, o1) < 1e-6 and rel(g2, o2) < 1e-6, "L%d add1" % i
        r1, r2 = o1.float(), o2.float()
        o = lin(c["ctx"], p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"], r2, "L%d proj" % i)
        rc = ovit._split_heads(o, heads)
        op, ov = rules.matmul_av_relprop(D(c["attn"]), D(c["v"]), D(rc))
        gp, gv = ops.matmul_av_relprop(_g(c["attn"]), _g(c["v"]), _g(rc))
        assert rel(gp, op) < 5e-4 and rel(gv, ov) < 5e-4, "L%d matmul2 rule: %g %g" % (i, rel(gp, op), rel(gv, ov))
        cam1, cam_v = (op / 2).float(), (ov / 2).float()
        oq, ok = rules.matmul_qk_relprop(D(c["q"]), D(c["k"]), D(cam1))
        cq32, ck32 = rules.matmul_qk_relprop(c["q"].float(), c["k"].float(), cam1)
        gq, gk = ops.matmul_qk_relprop(_g(c["q"]), _g(c["k"]), _g(cam1))
        for got, want, cpu32, nm in ((gq, oq, cq32, "q"), (gk, ok, ck32, "k")):
            e, e32 = rel(got, want), rel(cpu32, want)
            print("L%d matmul1 rule R_%s: gpu %.1e, fp32 CPU oracle %.1e" % (i, nm, e, e32))
            assert e <= max(10 * e32, 1e-5), "L%d matmul1 rule R_%s: %g (fp32 CPU oracle %g)" % (i, nm, e, e32)
        cq, ck = (oq / 2).float(), (ok / 2).float()
        rqkv = torch.cat([ovit._merge_heads(cq), ovit._merge_heads(ck), ovit._merge_heads(cam_v)], dim=-1)
        r2 = lin(c["xn1"], p[pre + "attn.qkv.weight"], p[pre + "attn.qkv.bias"], rqkv, "L%d qkv" % i)
        o = rules.clone_relprop(D(c["x_in"]), (D(r1), D(r2)))
        assert rel(ops.clone_relprop(_g(c["x_in"]), [_g(r1), _g(r2)]), o) < 1e-6, "L%d clone1" % i
        r = o


# ---- z+ rule edge cases --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [False, True])
def test_zplus_zero_rows_and_cancelled_denominators(tc):
    """``safe_divide``'s ``b != 0`` mask (layers_ours.py:10-13) on the z+ rule: an all-zero activation row and an all-zero
    weight row give Z == 0 exactly -> S == 0 there (no inf / NaN, and no tiny spurious denominator from the single-pass
    identity ((y - b) + |x||W|^T)/2); and rows whose products are ALL negative (sign(x) != sign(W) everywhere: the
    identity cancels completely, true Z == 0) must not produce a sign-flipped or huge S."""
    from transformer_explainability_b200 import ops
    rows, inf, outf = 300, 768, 512
    g = torch.Generator().manual_seed(3)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    r = torch.rand(rows, outf, generator=g)
    b = torch.randn(outf, generator=g)
    x[5] = 0.0                                   # all-zero activation row
    x[131] = 0.0
    w[7] = 0.0                                   # all-zero weight row (one output feature)
    w[300] = 0.0
    w[9] = -w[9].abs()                           # output 9 x row 17: every product negative -> true Z == 0
    x[17] = x[17].abs()
    w[11] = w[11].abs()                          # output 11 x row 17: every product positive (control)
    x[18] = x[18].abs() * (torch.arange(inf) < 3)          # row 18: three non-zero entries -> tiny but non-zero Z
    xd, wd, rd, bd = x.cuda(), w.cuda(), r.cuda(), b.cuda()
    y = ops.linear_forward(xd, wd, bd, tensor_cores=tc)
    out = ops.linear_relprop(xd, wd, rd, tensor_cores=tc, y=y if tc else None, bias=bd if tc else None)
    torch.cuda.synchronize()
    ref = rules.linear_relprop(x.double(), w.double(), r.double())
    assert torch.isfinite(out).all()
    assert float(out[5].abs().max()) == 0.0 and float(out[131].abs().max()) == 0.0
    tol = 3e-3 if tc else 2e-5
    assert rel(out, ref) < tol, "rel err %g" % rel(out, ref)
    # row 17 alone (contains the fully cancelled column 9 and the fully positive column 11)
    assert rel(out[17], ref[17]) < tol
    assert rel(out[18], ref[18]) < tol
