"""GPU: every engine entry point and stand-alone op on poisoned workspaces, scratch and outputs, bit-identical to a normal run.

The other GPU tests compare results with fp64 or with a golden file, but none controls what device memory held before the
call.  A kernel that reads memory nothing wrote in this call (or writes past its buffer) passes them as long as the stale
bytes happen to be harmless, and ``torch.empty`` usually hands back exactly such bytes: zeros of a fresh block, or the
previous call's results for the same inputs.  Here every ``torch.empty`` / ``torch.empty_like`` that the package hands to
the C library (through ``engine``, ``ops``, ``visualization`` and ``parallel``) is replaced, per call, by an allocation of
``numel`` + a 2 MiB guard, filled byte-wise with a pattern:

- 0xFF: NaN in fp32 / fp16 / bf16 / fp64, -1 in integers: any stale read that reaches an output through arithmetic shows;
- 0x5A: finite (1.5e16 in fp32, 203.25 in fp16, large positive integers): what a NaN hides (relu / fmaxf of a NaN,
  NaN-ignoring min / max, select-style masks) shows.

``torch.zeros`` / ``torch.full`` stay untouched (callers rely on their values).  The engines' weight buffers are zeros, so
the alignment gaps between the tensors of ``weight_table`` are filled with the pattern too, and before every call the
engine drops its workspace, its CUDA graphs and its derived weight copies, so that each is a fresh poisoned allocation.
Each case runs four times: twice with the normal allocator (any difference between those two is a race: nothing here
is order-dependent, the only atomics are integer histograms), once under each pattern.  Every output must be
bit-identical (compared as integers, so NaN patterns must match too) to the first run, and every guard must still hold
its pattern.  Outputs are the maps, the logits, the pixel maps of ``full`` and every per-layer tensor the mode produces
(``attn``, ``attn_grad``, ``attn_cam``).

Phase poisoning: driven through the engine directly, the workspace from ``tmp_d0`` to its end is refilled with the
pattern between ``forward`` and ``attribute``, and from ``tmp_d1`` to its end between ``attribute(RELPROP_TO_INPUT)`` and
the pixel relprop, so that a phase that reads scratch the previous phase left behind fails.

Padding: the pad columns [N, NP) of the probabilities P must hold +0.0 after every call (TMA boxes of the tensor-core
contractions cover them), and so must those of the attention gradients G and ``attn_cam`` when the tensor-core
contractions produce them (TE_FLAG_ATTN_TENSOR_CORES, dh 32 / 64).  The SIMT producers of G and ``attn_cam`` leave their
pad columns unwritten; their consumers select the real columns (the head reductions, the rollout), which the
bit-identity of every output confirms (DESIGN.md §3).

Findings: no kernel read stale or unwritten memory, wrote past its allocation or differed between two normal runs.  The
one claim the test refuted was DESIGN.md §3's "every producer writes the pad columns as zeros": at flags 0 (and on the
tiny golden ViT, dh 16, at every flag set) G and ``attn_cam`` came back with the poison in all of their pad columns,
e.g. ``vit-b flags 0 transformer_attribution``.  The sentence now names the producers it holds for.

What it catches (each mutation tried once, not committed): dropping the ``te_launch_fill`` of R3 in the ViT top block
(the cls_row_top_block 0 / 1 comparison), writing only N of the NP columns in the fused-softmax epilogue (the P padding
check), and making the first write of the SIMT z+ rule or of the layers_lrp halves accumulate (the poisoned runs differ;
without the matching dispatch case the launch returns TE_ERR_UNSUPPORTED, which fails every case that reaches it).

Wall time: about 50 s on one H100 80GB HBM3 at a 400 W power limit.

Models: conditioned 3-block models as in test_gpu_methods_tc.py.  The full matrix (every entry point, flags 0, 51, 7475
with ``cls_row_top_block`` 1 and 0, 115, 32051) runs at ViT-B and BERT-base width; DeiT-distilled (N = 198), ViT-B at 384
(N = 577), ViT-Ti, D = 256 with MLP 128, BERT hidden 128 and 256 / intermediate 256 and the tiny golden ViT run
transformer_attribution / generate_LRP, ``full`` and a gradients-only baseline at flags 0 and 32051.  The stand-alone ops
run at the shapes where their kernels branch.
"""
import importlib
import math

import pytest
import torch

from oracle import bert as obert
from oracle import conditioned
from oracle import vit as ovit
from transformer_explainability_b200 import _lib, engine, ops, parallel, visualization

pytestmark = pytest.mark.gpu

GUARD_BYTES = 2 << 20
RUNS = ((None, "normal"), (None, "normal, again"), (0xFF, "0xFF"), (0x5A, "0x5A"))
POISONED_MODULES = (engine, ops, visualization, parallel)
BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}

BENCH = _lib.FLAG_BENCH_DEFAULT
FLAG_SETS = [0, _lib.FLAG_ALL_FAST, BENCH, _lib.FLAG_ALL_FAST | _lib.FLAG_ZPLUS_BF16,
             BENCH | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16]
NARROW_FLAG_SETS = [0, BENCH | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16]
TC = _lib.FLAG_RULES_LRP_TC


# ---- the poisoning allocator ---------------------------------------------------------------------------------------------
class PoisonTorch:
    """Stands in for ``torch`` in a module: ``empty`` / ``empty_like`` of CUDA tensors return the first numel elements
    (storage offset 0) of a buffer numel + 2 MiB long whose every byte holds the pattern; everything else is torch's."""

    def __init__(self, pattern):
        self.pattern = pattern
        self.guards = []

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *size, dtype=None, device=None, **kw):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        size = tuple(int(s) for s in size)
        dtype = dtype or torch.get_default_dtype()
        if device is None or torch.device(device).type != "cuda" or kw:
            return torch.empty(size, dtype=dtype, device=device, **kw)
        n = math.prod(size)
        item = torch.empty(0, dtype=dtype).element_size()
        flat = torch.empty(n + GUARD_BYTES // item, dtype=dtype, device=device)
        flat.view(torch.uint8).fill_(self.pattern)
        self.guards.append(flat[n:])
        return flat[:n].view(size)

    def empty_like(self, t, dtype=None, device=None, memory_format=None, **kw):
        return self.empty(tuple(t.shape), dtype=dtype or t.dtype, device=device or t.device, **kw)

    def broken_guards(self):
        return sum(int((g.view(torch.uint8) != self.pattern).any()) for g in self.guards)


def _items(out, key=""):
    if out is None:
        return []
    if torch.is_tensor(out):
        return [(key or "out", out)]
    if isinstance(out, dict):
        return [kv for k, v in out.items() for kv in _items(v, "%s%s" % (key + "." if key else "", k))]
    return [kv for i, v in enumerate(out) for kv in _items(v, "%s%d" % (key + "." if key else "", i))]


def _bits(t):
    return t.detach().contiguous().view(BITS[t.element_size()])


class Findings:
    """Every failure of one test, reported together."""

    def __init__(self):
        self.items = []
        self.cases = 0

    def add(self, msg):
        print("FINDING " + msg)
        self.items.append(msg)

    def check(self):
        print("%d cases" % self.cases)
        assert not self.items, "%d findings:\n%s" % (len(self.items), "\n".join(self.items[:80]))


def compare(found, tag, label, ref, out):
    for k, v in ref.items():
        w = out[k]
        if w.shape != v.shape or w.dtype != v.dtype:
            found.add("%s [%s]: %s shape / dtype differ" % (tag, label, k))
        elif not torch.equal(_bits(w), _bits(v)):
            d = _bits(w) != _bits(v)
            first = tuple(int(i) for i in d.nonzero()[0])
            found.add("%s [%s]: %s differs from the normal run in %d of %d entries, first at %s (%r vs %r)" % (
                tag, label, k, int(d.sum()), d.numel(), first, w[first].item(), v[first].item()))


def run_case(found, tag, fn, before=None, may_skip=False):
    """fn(pattern) -> tensors (tensor / tuple / dict); keys starting with 'pad:' must also be all +0.0.  before(pattern)
    resets state ahead of each run.  Returns the normal run's outputs.  may_skip: a diagnostic entry point that does not
    take the shape (TE_ERR_UNSUPPORTED in the normal run) skips the case; everywhere else that status is a failure."""
    ref = None
    for pattern, label in RUNS:
        if before is not None:
            before(pattern)
        proxy = PoisonTorch(pattern) if pattern is not None else None
        with pytest.MonkeyPatch.context() as mp:
            if proxy is not None:
                for m in POISONED_MODULES:
                    mp.setattr(m, "torch", proxy)
            try:
                out = fn(pattern)
            except _lib.TeError as e:
                if may_skip and ref is None and e.status == _lib.TE_ERR_UNSUPPORTED:
                    return None
                raise
            out = {k: v.detach().clone() for k, v in _items(out)}
        torch.cuda.synchronize()
        if proxy is not None and proxy.broken_guards():
            found.add("%s [%s]: %d allocations written past their end" % (tag, label, proxy.broken_guards()))
        for k, v in out.items():
            if k.startswith("pad:") and v.numel() and (_bits(v) != 0).any():
                found.add("%s [%s]: %s holds %d non-(+0.0) pad entries" % (tag, label, k[4:], int((_bits(v) != 0).sum())))
        if ref is None:
            ref = out
        else:
            compare(found, tag, label, ref, out)
    found.cases += 1
    return ref


# ---- engines ---------------------------------------------------------------------------------------------------------------
def _fill_value(pattern):
    return 0 if pattern is None else int.from_bytes(bytes([pattern] * 4), "little", signed=True)


class EngineState:
    """Before each run: drop the workspace, CUDA graphs and derived weights; fill the weight buffer's alignment gaps."""

    def __init__(self, eng):
        self.eng = eng
        ends = [(off + numel, nxt) for (_, numel, off), nxt in
                zip(eng.weight_table, [off for _, _, off in eng.weight_table[1:]] + [eng.weights.numel()])]
        idx = [i for a, b in ends for i in range(a, b)]
        self.gaps = torch.tensor(idx, dtype=torch.long, device=eng.weights.device)
        assert self.gaps.numel() > 0

    def __call__(self, pattern):
        e = self.eng
        e._ws, e._graphs, e.derived = None, None, None
        e.weights.view(torch.int32).index_fill_(0, self.gaps, _fill_value(pattern))


def _pads(eng, name, layer):
    v = eng.tensor(name, layer)
    B, H, N, _ = v.shape
    NP = v.stride(2)
    if NP == N:
        return {}
    return {"pad:%s%d" % (name, layer): torch.as_strided(eng._ws, (B, H, N, NP - N), v.stride(), v.storage_offset() + N)}


def tc_attention(eng):
    """whether the call's attention contractions (the producers of G and attn_cam) run on the tensor cores"""
    cfg = eng.cfg
    dh = (cfg.dim if hasattr(cfg, "dim") else cfg.hidden) // cfg.heads
    return bool(eng.flags & _lib.FLAG_ATTN_TENSOR_CORES) and dh in (32, 64)


def taps(eng, L, g0, c0):
    """logits and the per-layer tensors a call wrote: attn of every layer, attn_grad from layer g0, attn_cam from c0 on.
    The pad columns of P always, those of G and attn_cam when their producers are the tensor-core contractions: the SIMT
    producers leave them unwritten (DESIGN.md §3), and the bit-identity of every output shows that nothing reads them."""
    out = {"logits": eng.tensor("logits")}
    for name, first in (("attn", 0), ("attn_grad", g0), ("attn_cam", c0)):
        if first is None:
            continue
        for l in range(first, L):
            out["%s%d" % (name, l)] = eng.tensor(name, l)
            if name == "attn" or tc_attention(eng):
                out.update(_pads(eng, name, l))
    return out


def _poison_from(eng, name, pattern):
    if pattern is not None:
        eng._ws[eng.tensor(name).storage_offset():].view(torch.uint8).fill_(pattern)


class cls_rows:
    """te_set_option("cls_row_top_block", on) for the duration, restored to the default 1"""

    def __init__(self, on):
        self.on = on

    def __enter__(self):
        _lib.check(_lib.load().te_set_option(b"cls_row_top_block", self.on), "te_set_option")

    def __exit__(self, *exc):
        _lib.check(_lib.load().te_set_option(b"cls_row_top_block", 1), "te_set_option")


def flag_variants(flags):
    """(tag, flags, cls_row_top_block) of one flag set: at the bench default also the all-rows top block"""
    out = [("flags %d" % flags, flags, 1)]
    if flags == BENCH:
        out.append(("flags %d cls_row_top_block 0" % flags, flags, 0))
    return out


# ---- ViT ----
VIT_CASES = [("transformer_attribution", dict(start_layer=0)), ("transformer_attribution", dict(start_layer=1)),
             ("grad", {}), ("rollout", dict(start_layer=0)), ("rollout", dict(start_layer=1)), ("full", {}),
             ("last_layer", {}), ("last_layer", dict(is_ablation=True)), ("last_layer_attn", {}),
             ("second_layer", {}), ("second_layer", dict(is_ablation=True))]
ORIG_CASES = [("grad", {}), ("full", {}), ("last_layer", {}), ("rollout", dict(start_layer=0))]
NARROW_VIT_CASES = [("transformer_attribution", dict(start_layer=0)), ("full", {})]


def vit_layers(method, kw, L):
    """(first layer with attn_grad, first layer with attn_cam) that the façade's method writes"""
    if method in ("transformer_attribution", "grad"):
        return kw.get("start_layer", 0), kw.get("start_layer", 0)
    if method in ("rollout", "full"):
        return 0, 0
    if method == "last_layer":
        return L - 1, L - 1
    if method == "second_layer":
        return 1, 1
    return None, None


def vit_model(name="vit_base_patch16_224", module="ViT_LRP", seed=11, **over):
    params, heads = ovit.init_params(name, seed=seed, rand_affine=True, **over)
    params = conditioned.condition_vit(params, c_qkv=1.0)
    D = params["cls_token"].shape[-1]
    L = 1 + max(int(k.split(".")[1]) for k in params if k.startswith("blocks."))
    P = params["patch_embed.proj.weight"].shape[-1]
    img = P * int(round((params["pos_embed"].shape[1] - (2 if "dist_token" in params else 1)) ** 0.5))
    mod = importlib.import_module("transformer_explainability_b200.baselines.ViT." + module)
    m = mod.VisionTransformer(img_size=img, patch_size=P, embed_dim=D, depth=L, num_heads=heads,
                              mlp_ratio=params["blocks.0.mlp.fc1.weight"].shape[0] / D, qkv_bias=True,
                              num_classes=params["head.weight"].shape[0], distilled="dist_token" in params)
    m.load_state_dict(params)
    m = m.cuda().eval()
    x = torch.randn(2, 3, img, img, generator=torch.Generator().manual_seed(seed + 1)).cuda()
    return m, x, L


def _one_hot(logits):
    oh = torch.zeros_like(logits)
    oh[torch.arange(logits.shape[0], device=logits.device), logits.argmax(-1)] = 1
    return oh


def vit_method(model, x, L, method, kw, alpha=None):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP

    def fn(pattern):
        if alpha is None:
            out = LRP(model).generate_LRP(x, method=method, **kw)
        else:
            out = model.relprop(_one_hot(model(x)), method=method, alpha=alpha, **kw)
        return dict(map=out, **taps(model.engine(), L, *vit_layers(method, kw, L)))
    return fn


def vit_baseline_cam_attn(model, x, L, index=None):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import Baselines

    def fn(pattern):
        out = Baselines(model).generate_cam_attn(x, index=index)
        return dict(map=out, **taps(model.engine(), L, L - 1, None))
    return fn


def vit_baseline_rollout(model, x, L, start_layer):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import Baselines

    def fn(pattern):
        out = Baselines(model).generate_rollout(x, start_layer=start_layer)
        return dict(map=out, **taps(model.engine(), L, None, None))
    return fn


def vit_phases(model, x, L, start_layer=None):
    """forward | poison tmp_d0.. | attribute(RELPROP_TO_INPUT) | poison tmp_d1.. | pixel relprop; with start_layer:
    forward | poison tmp_d0.. | attribute(start_layer)"""
    def fn(pattern):
        eng = model.engine()
        eng.forward(x)
        _poison_from(eng, "tmp_d0", pattern)
        if start_layer is not None:
            maps, idx = eng.attribute(start_layer=start_layer)
            return dict(maps=maps, idx=idx, **taps(eng, L, start_layer, start_layer))
        got = {}
        attribute = eng.attribute

        def attribute_then_poison(*a, **k):
            got["maps"], got["idx"] = attribute(*a, **k)
            _poison_from(eng, "tmp_d1", pattern)
            return got["maps"], got["idx"]
        eng.attribute = attribute_then_poison
        try:
            pix = eng.relprop_pixels(per_channel=True)
        finally:
            del eng.attribute
        return dict(pix=pix, relevance_in=eng.tensor("relevance_in"), rtok=eng.tensor("tmp_d2"), **got,
                    **taps(eng, L, 0, 0))
    return fn


@pytest.fixture(scope="module")
def vit_b():
    return vit_model(depth=3, classes=100)


def sweep(found, model, prefix, cases, reset):
    """every case under every flag set; at the bench default also with cls_row_top_block 0, whose results must be the
    same bits: the top block's pooled-rows shortcut relies on the rows it skips holding zeros"""
    pooled = {}
    for flags in FLAG_SETS:
        for tag, fl, top in flag_variants(flags):
            model.engine_flags = fl
            with cls_rows(top):
                for name, fn in cases():
                    t = "%s %s %s" % (prefix, tag, name)
                    out = run_case(found, t, fn, reset)
                    if flags == BENCH and top:
                        pooled[name] = out
                    elif flags == BENCH:
                        compare(found, t, "all rows vs pooled rows", pooled[name], out)


def test_vit_b_entry_points(vit_b):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    model, x, L = vit_b
    x5 = torch.cat([x, x.flip(0), x[:1] * 0.5])

    def cases():
        out = [("%s %s" % (method, kw), vit_method(model, x, L, method, kw)) for method, kw in VIT_CASES]
        out += [("%s alpha 2" % method, vit_method(model, x, L, method, {}, alpha=2.0))
                for method in ("transformer_attribution", "full")]
        out += [("cam_attn index %s" % index, vit_baseline_cam_attn(model, x, L, index)) for index in (None, 7)]
        out += [("baseline rollout %d" % sl, vit_baseline_rollout(model, x, L, sl)) for sl in (0, 1)]
        out += [("phases full", vit_phases(model, x, L)), ("phases start_layer 1", vit_phases(model, x, L, start_layer=1))]
        # B = 5 in chunks of 2: the last chunk re-allocates the workspace
        out += [("generate_LRP_batched",
                 lambda p: dict(zip(("maps", "idx"), LRP(model).generate_LRP_batched(x5, chunk=2, return_index=True)),
                                **taps(model.engine(), L, 0, 0))),
                ("explain_graphed",
                 lambda p: dict(zip(("maps", "idx", "logits_out"), model.engine().explain_graphed(x, return_logits=True)),
                                **taps(model.engine(), L, 0, 0)))]
        return out
    found = Findings()
    sweep(found, model, "vit-b", cases, EngineState(model.engine()))
    found.check()


def test_vit_orig_lrp_entry_points():
    model, x, L = vit_model(module="ViT_orig_LRP", seed=15, depth=3, classes=100)
    reset = EngineState(model.engine())
    found = Findings()
    for flags in FLAG_SETS + [BENCH | TC, FLAG_SETS[-1] | TC]:
        model.engine_flags = flags
        for method, kw in ORIG_CASES:
            run_case(found, "vit-orig-lrp flags %d %s" % (flags, method), vit_method(model, x, L, method, kw), reset)
        run_case(found, "vit-orig-lrp flags %d grad alpha 2" % flags, vit_method(model, x, L, "grad", {}, alpha=2.0), reset)
    found.check()


VIT_GEOMETRIES = {
    "deit-b-dist": dict(name="deit_base_distilled_patch16_224", seed=13, depth=3, classes=100),
    "vit-b-384": dict(seed=19, depth=3, classes=100, img=384),
    "vit-ti": dict(seed=5, depth=3, classes=100, dim=192, heads=3, mlp=768),
    "vit-d256-mlp128": dict(seed=159, depth=3, classes=100, dim=256, heads=4, mlp=128),
    "vit-tiny-golden": dict(name="vit_tiny_test", seed=1),
}


@pytest.mark.parametrize("tag", list(VIT_GEOMETRIES))
def test_vit_geometry(tag):
    model, x, L = vit_model(**VIT_GEOMETRIES[tag])
    reset = EngineState(model.engine())
    found = Findings()
    for flags in NARROW_FLAG_SETS:
        model.engine_flags = flags
        for method, kw in NARROW_VIT_CASES:
            run_case(found, "%s flags %d %s" % (tag, flags, method), vit_method(model, x, L, method, kw), reset)
        run_case(found, "%s flags %d cam_attn" % (tag, flags), vit_baseline_cam_attn(model, x, L), reset)
        run_case(found, "%s flags %d phases full" % (tag, flags), vit_phases(model, x, L), reset)
    found.check()


# ---- BERT ----
BERT_GENERATORS = [("LRP", dict(start_layer=0)), ("LRP", dict(start_layer=1)), ("LRP_last_layer", {}),
                   ("full_lrp", {}), ("attn_last_layer", {}), ("rollout", dict(start_layer=0)), ("attn_gradcam", {})]


def bert_layers(which, kw, L):
    if which == "LRP":
        return kw["start_layer"], kw["start_layer"]
    if which == "LRP_last_layer":
        return L - 1, L - 1
    if which == "full_lrp":
        return 0, 0
    if which == "attn_gradcam":
        return L - 1, None
    return None, None


def bert_model(seed=22, dim=768, heads=12, inter=3072, cls_lrp=False, n=3, seq=130):
    params, heads = obert.init_params(seed=seed, vocab=1000, max_pos=512, dim=dim, depth=3, heads=heads, inter=inter,
                                      rand_affine=True)
    params = conditioned.condition_bert(params, c_qkv=3.0)
    from test_gpu_bert import make_model
    if cls_lrp:
        from test_gpu_bert_lrp import make_model
    model = make_model(params, heads, hidden_size=dim, num_hidden_layers=3, intermediate_size=inter, vocab_size=1000,
                       max_position_embeddings=512)
    g = torch.Generator().manual_seed(seed + 1)
    ids = torch.randint(5, 1000, (n, seq), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones(n, seq, dtype=torch.long)
    mask[1, seq // 2:] = 0                                     # sample 1 is padded from the middle on
    return model, ids.cuda(), mask.cuda(), 3


def bert_generator(model, ids, mask, L, which, kw):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator

    def fn(pattern):
        out = getattr(Generator(model), "generate_" + which)(ids, mask, **kw)
        return dict(map=out, **taps(model.engine(), L, *bert_layers(which, kw, L)))
    return fn


def bert_relprop(model, ids, mask, L, alpha):
    def fn(pattern):
        r = model.relprop(_one_hot(model(ids, mask)[0]), alpha=alpha)
        return dict(relevance_in=r, **taps(model.engine(), L, 0, 0))
    return fn


def bert_phases(model, ids, mask, L, to_input):
    """forward | poison tmp_d0.. | attribute (start_layer 0, RELPROP_TO_INPUT with to_input)"""
    def fn(pattern):
        eng = model.engine()
        eng.forward(ids, mask)
        _poison_from(eng, "tmp_d0", pattern)
        maps, idx = eng.attribute(start_layer=0, flags=eng.flags | (_lib.FLAG_RELPROP_TO_INPUT if to_input else 0))
        return dict(maps=maps, idx=idx, relevance_in=eng.tensor("relevance_in") if to_input else None, **taps(eng, L, 0, 0))
    return fn


@pytest.fixture(scope="module")
def bert_b():
    return bert_model()


def test_bert_b_entry_points(bert_b):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model, ids, mask, L = bert_b
    ids5, mask5 = torch.cat([ids, ids[:2]]), torch.cat([mask, mask[1:3]])

    def cases():
        out = [("%s %s" % (which, kw), bert_generator(model, ids, mask, L, which, kw)) for which, kw in BERT_GENERATORS]
        out += [("relprop alpha %g" % alpha, bert_relprop(model, ids, mask, L, alpha)) for alpha in (1.0, 2.0)]
        out += [("phases to_input %s" % t, bert_phases(model, ids, mask, L, t)) for t in (False, True)]
        # B = 5 in chunks of 2: the last chunk re-allocates the workspace
        out += [("generate_LRP_batched",
                 lambda p: dict(zip(("maps", "idx"), Generator(model).generate_LRP_batched(
                     ids5, mask5, start_layer=0, chunk=2, return_index=True)), **taps(model.engine(), L, 0, 0)))]
        return out
    found = Findings()
    sweep(found, model, "bert-b", cases, EngineState(model.engine()))
    found.check()


def test_bert_cls_lrp_entry_points():
    model, ids, mask, L = bert_model(seed=24, cls_lrp=True)
    reset = EngineState(model.engine())
    found = Findings()
    for flags in FLAG_SETS + [BENCH | TC, FLAG_SETS[-1] | TC]:
        model.engine_flags = flags
        for which, kw in [("LRP", dict(start_layer=0)), ("LRP_last_layer", {}), ("full_lrp", {})]:
            run_case(found, "bert-cls-lrp flags %d %s" % (flags, which), bert_generator(model, ids, mask, L, which, kw), reset)
        for alpha in (1.0, 2.0):
            run_case(found, "bert-cls-lrp flags %d relprop alpha %g" % (flags, alpha),
                     bert_relprop(model, ids, mask, L, alpha), reset)
    found.check()


BERT_GEOMETRIES = {"bert-tiny": dict(seed=51, dim=128, heads=2, inter=512),
                   "bert-d256-f256": dict(seed=41, dim=256, heads=4, inter=256)}


@pytest.mark.parametrize("tag", list(BERT_GEOMETRIES))
def test_bert_geometry(tag):
    model, ids, mask, L = bert_model(**BERT_GEOMETRIES[tag])
    reset = EngineState(model.engine())
    found = Findings()
    for flags in NARROW_FLAG_SETS:
        model.engine_flags = flags
        for which, kw in [("LRP", dict(start_layer=0)), ("attn_gradcam", {}), ("full_lrp", {})]:
            run_case(found, "%s flags %d %s" % (tag, flags, which), bert_generator(model, ids, mask, L, which, kw), reset)
        run_case(found, "%s flags %d phases" % (tag, flags), bert_phases(model, ids, mask, L, True), reset)
    found.check()


# ---- stand-alone ops ---------------------------------------------------------------------------------------------------------
ROWS = [1, 130, 394]                                                 # 394: a ragged 128-row tile
LINEAR_SHAPES = [(128, 128), (192, 768), (320, 128), (576, 192), (768, 3072), (3072, 768), (100, 128), (128, 100)]
ALPHAS = [1.0, 2.0, 0.5, 0.0]
NS_SAMPLE = [1, 5, 33, 65, 129, 197, 256, 257, 300, 577]           # test_gpu_attention_tc.py


def _rand(*shape, seed=0, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).cuda()


def test_ops_linear():
    found = Findings()
    for rows in ROWS:
        for K, N in LINEAR_SHAPES:
            x, w, b = _rand(rows, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5), _rand(N, seed=3)
            dy, e0f, e0b = _rand(rows, N, seed=4), _rand(rows, N, seed=5), _rand(rows, K, seed=6)
            y = x @ w.t() + b
            r = _rand(rows, N, seed=7)
            t = "rows %d K %d N %d" % (rows, K, N)
            for tc, f16 in ((False, False), (True, False), (True, True)):
                run_case(found, "%s linear_forward tc %s f16_split %s" % (t, tc, f16),
                         lambda p: ops.linear_forward(x, w, b, tensor_cores=tc, f16_split=f16))
            for tc in (False, True):
                run_case(found, "%s linear_backward tc %s" % (t, tc), lambda p: ops.linear_backward(dy, w, tensor_cores=tc))
            run_case(found, "%s linear_backward_f16" % t, lambda p: ops.linear_backward_f16(dy, w))
            run_case(found, "%s linear_backward_tf32" % t, lambda p: ops.linear_backward_tf32(dy, w))
            for family in ("simt", "3xtf32", "f16_split"):
                for epi in ("store", "bias", "bias_gelu", "bias_add"):
                    run_case(found, "%s linear_forward_epi %s %s" % (t, family, epi),
                             lambda p: ops.linear_forward_epi(x, w, None if epi == "store" else b,
                                                              e0f if epi == "bias_add" else None, epi=epi, family=family),
                             may_skip=True)
            for family in ("simt", "3xtf32", "tf32", "f16"):
                for epi in ("store", "gelu_bwd"):
                    run_case(found, "%s linear_backward_epi %s %s" % (t, family, epi),
                             lambda p: ops.linear_backward_epi(dy, w, e0b if epi == "gelu_bwd" else None, epi=epi, family=family),
                             may_skip=True)
            for f16 in (False, True) if N % 128 == 0 else (False,):      # the fp16 S has one scale per 128 columns
                for bf16 in (False, True):
                    run_case(found, "%s tc_zplus_s f16 %s bf16 %s" % (t, f16, bf16),
                             lambda p: ops.tc_zplus_s(x, w, r, y, bias=b, f16=f16, bf16=bf16), may_skip=True)
        for cols in (64, 100, 192, 320, 576, 768, 3072):
            x = _rand(rows, cols, seed=8)
            run_case(found, "rows %d f16_block_split %d" % (rows, cols), lambda p: ops.f16_block_split(x))
            run_case(found, "rows %d layernorm_split %d" % (rows, cols),
                     lambda p: ops.layernorm_split(x, _rand(cols, seed=9), _rand(cols, seed=10), 1e-6))
    found.check()


LINEAR_RELPROP_VARIANTS = [
    ("ours simt", dict()), ("ours tc", dict(tensor_cores=True)), ("ours tc y", dict(tensor_cores=True, y=True)),
    ("ours tc y bf16", dict(tensor_cores=True, y=True, bf16=True)), ("ours tc y s1", dict(tensor_cores=True, y=True, bf16="s1")),
    ("ours tc y r_f16", dict(tensor_cores=True, y=True, r_f16=True)), ("ours tc r_f16", dict(tensor_cores=True, r_f16=True)),
    ("lrp", dict(variant="lrp")), ("lrp_tc", dict(variant="lrp_tc"))]


def test_ops_linear_relprop():
    found = Findings()
    for rows in ROWS:
        for K, N in LINEAR_SHAPES:
            x, w, b = _rand(rows, K, seed=11), _rand(N, K, seed=12, scale=K ** -0.5), _rand(N, seed=13, scale=0.1)
            y = x @ w.t() + b
            r = _rand(rows, N, seed=14)
            for name, kw in LINEAR_RELPROP_VARIANTS:
                kw = dict(kw)
                if kw.pop("y", False):
                    kw.update(y=y, bias=b)
                for alpha in ALPHAS:
                    run_case(found, "rows %d K %d N %d linear_relprop %s alpha %g" % (rows, K, N, name, alpha),
                             lambda p: ops.linear_relprop(x, w, r, alpha=alpha, **kw))
    found.check()


def test_ops_rule_modules():
    """Linear / Add / Clone / einsum / IndexSelect / Conv2d .relprop of modules/layers_ours.py and modules/layers_lrp.py"""
    from transformer_explainability_b200.modules import layers_lrp, layers_ours
    found = Findings()
    for lib in (layers_ours, layers_lrp):
        t0 = lib.__name__.rsplit(".", 1)[1]
        for rows in ROWS:
            for K, N in [(768, 768), (768, 3072), (100, 128)]:
                lin = lib.Linear(K, N).cuda()
                x = _rand(rows, K, seed=15)
                lin(x)
                r = _rand(rows, N, seed=16)
                for alpha in ALPHAS:
                    run_case(found, "%s Linear rows %d %dx%d alpha %g" % (t0, rows, K, N, alpha),
                             lambda p: lin.relprop(r, alpha))
        for shape in [(1, 1, 768), (1, 130, 768), (2, 197, 768), (2, 197, 100)]:
            a, b, r = _rand(*shape, seed=17), _rand(*shape, seed=18), _rand(*shape, seed=19)
            add, clone, sel = lib.Add(), lib.Clone(), lib.IndexSelect()
            add([a, b])
            clone(a, 2)
            sel(a, 1, torch.tensor([0], device="cuda"))
            run_case(found, "%s Add %s" % (t0, shape), lambda p: add.relprop(r, 1))
            run_case(found, "%s Clone %s" % (t0, shape), lambda p: clone.relprop([r, b], 1))
            run_case(found, "%s IndexSelect %s" % (t0, shape), lambda p: sel.relprop(r[:, :1], 1))
        for n in NS_SAMPLE:
            q, k, v = (_rand(3, 12, n, 64, seed=20 + i) for i in range(3))
            p_ = torch.softmax(_rand(3, 12, n, n, seed=23), -1)
            av, qk = lib.einsum("bhij,bhjd->bhid"), lib.einsum("bhid,bhjd->bhij")
            av([p_, v])
            qk([q, k])
            r_av, r_qk = _rand(3, 12, n, 64, seed=24), _rand(3, 12, n, n, seed=25)
            run_case(found, "%s einsum av n %d" % (t0, n), lambda p: av.relprop(r_av, 1))
            run_case(found, "%s einsum qk n %d" % (t0, n), lambda p: qk.relprop(r_qk, 1))
        for B, C, S, P, D in [(2, 3, 32, 8, 64), (3, 3, 224, 16, 768), (1, 3, 48, 16, 40)]:
            conv = lib.Conv2d(C, D, P, P).cuda()
            conv(_rand(B, C, S, S, seed=26))
            r = _rand(B, D, S // P, S // P, seed=27)
            run_case(found, "%s Conv2d %s" % (t0, (B, C, S, P, D)), lambda p: conv.relprop(r, 1))
    found.check()


def _padded(shape, n, seed, positive=False):
    """a [..., n, n] view of a [..., n, round_up(n, 4)] buffer, and the buffer (its pad columns get the pattern)"""
    np_ = (n + 3) & ~3
    buf = _rand(*shape, n, np_, seed=seed)
    if positive:
        buf = buf.abs()
    return buf[..., :n], buf


def _fill_pads(buf, n, pattern):
    if buf.shape[-1] > n:
        buf[..., n:].view(torch.uint8).fill_(0 if pattern is None else pattern)


def test_ops_attention_shaped():
    """head_reduce (every mode, with and without g / head weights), head_region_mean, attribution_rollout (fused,
    want_joint, normalize), compute_rollout_attention and the two attention matmul rules at batch 3 x 12 heads; the inputs'
    row padding [N, NP) holds the pattern in the poisoned runs (it is never read)"""
    found = Findings()
    for n in NS_SAMPLE:
        a, abuf = _padded((3, 12), n, seed=30)
        g, gbuf = _padded((3, 12), n, seed=31)
        hw = _rand(3, 12, seed=32)

        def pads(pattern):
            _fill_pads(abuf, n, pattern)
            _fill_pads(gbuf, n, pattern)
        for mode in ("mean", "relu_mean", "mean_relu"):
            for with_g, with_w in ((False, False), (True, False), (False, True), (True, True)):
                run_case(found, "n %d head_reduce %s g %s w %s" % (n, mode, with_g, with_w),
                         lambda p: ops.head_reduce(a, g if with_g else None, hw if with_w else None, mode=mode), pads)
        for rr, cc in ((None, None), ((0, 1), (min(1, n - 1), n)), ((0, n), (0, n))):
            run_case(found, "n %d head_region_mean %s %s" % (n, rr, cc), lambda p: ops.head_region_mean(g, rr, cc), pads)
        # rollout over L = 3 layers, [L, B, H, N, NP] with the pad columns inside the tensor
        grad, gb = _padded((3, 3, 12), n, seed=33)
        cam, cb = _padded((3, 3, 12), n, seed=34, positive=True)

        def rpads(pattern):
            _fill_pads(gb, n, pattern)
            _fill_pads(cb, n, pattern)
        for fused in (False, True):
            for want_joint in (False, True):
                for normalize in (False, True):
                    for sl in (0, 1):
                        run_case(found, "n %d attribution_rollout fused %s joint %s normalize %s start %d" % (
                            n, fused, want_joint, normalize, sl),
                            lambda p: ops.attribution_rollout(gb, cb, start_layer=sl, normalize=normalize, fused=fused,
                                                              want_joint=want_joint), rpads)
        mats = [torch.softmax(_rand(3, n, n, seed=35 + i), -1) for i in range(3)]
        for normalize in (False, True):
            run_case(found, "n %d compute_rollout_attention normalize %s" % (n, normalize),
                     lambda p: ops.compute_rollout_attention(mats, start_layer=1, normalize=normalize))
        q, k, v = (_rand(3, 12, n, 64, seed=40 + i) for i in range(3))
        p_ = torch.softmax(_rand(3, 12, n, n, seed=43), -1)
        r_av, r_qk = _rand(3, 12, n, 64, seed=44), _rand(3, 12, n, n, seed=45)
        run_case(found, "n %d matmul_av_relprop" % n, lambda p: ops.matmul_av_relprop(p_, v, r_av))
        run_case(found, "n %d matmul_qk_relprop" % n, lambda p: ops.matmul_qk_relprop(q, k, r_qk))
    found.check()


def test_ops_pixels_and_heatmap():
    found = Findings()
    for B, C, S, P, D in [(2, 3, 32, 8, 64), (3, 3, 224, 16, 768), (1, 3, 48, 16, 40)]:
        images, weight = _rand(B, C, S, S, seed=50), _rand(D, C, P, P, seed=51, scale=0.05)
        r = _rand(B, (S // P) ** 2, D, seed=52)
        for per_channel in (False, True):
            run_case(found, "patch_embed_relprop %s per_channel %s" % ((B, C, S, P, D), per_channel),
                     lambda p: ops.patch_embed_relprop(images, weight, r, per_channel=per_channel))
    for B, grid, scale in [(1, 14, 16), (3, 14, 16), (2, 24, 16), (2, 7, 32)]:
        maps = _rand(B, grid * grid, seed=53)
        run_case(found, "relevance_to_heatmap %s" % ((B, grid, scale),),
                 lambda p: visualization.relevance_to_heatmap(maps, grid=grid, scale=scale))
    found.check()


def test_ops_evaluation():
    """perturb_images, logit_stats, seg_metrics (with PR keys), sort_keys and pr_curve"""
    found = Findings()
    images = torch.rand(3, 3, 224, 224, generator=torch.Generator().manual_seed(60)).cuda()
    sal = _rand(3, 224, 224, seed=61)
    sal[0, :3, :5] = float("nan")
    sal[1, 10:20] = 0.25                                            # ties
    for negate in (False, True):
        run_case(found, "perturb_images negate %s" % negate,
                 lambda p: ops.perturb_images(images, sal, [0, 1, 500, 25088, 50176], negate=negate))
    for R, K in [(1, 1000), (394, 1000), (130, 2)]:
        logits = _rand(R, K, seed=62)
        target = torch.randint(0, K, (R,), generator=torch.Generator().manual_seed(63)).cuda()
        run_case(found, "logit_stats %d x %d" % (R, K), lambda p: ops.logit_stats(logits, target))
    for B in (1, 3):
        maps = _rand(B, 196, seed=64)
        labels = (torch.rand(B, 224 * 224, generator=torch.Generator().manual_seed(65)) > 0.7).long().cuda()
        for pr_keys in (False, True):
            run_case(found, "seg_metrics B %d pr_keys %s" % (B, pr_keys),
                     lambda p: ops.seg_metrics(maps, labels, pr_keys=pr_keys))
        keys = ops.seg_metrics(maps, labels, pr_keys=True)["pr_keys"].reshape(-1).contiguous()
        for segments in (1, B):
            run_case(found, "sort_keys B %d segments %d" % (B, segments), lambda p: ops.sort_keys(keys, segments=segments))
        run_case(found, "pr_curve B %d" % B, lambda p: ops.pr_curve(ops.sort_keys(keys)))
    for n in (1, 1000, 3 * 50176 + 7):
        keys = torch.randint(-2 ** 31, 2 ** 31 - 1, (n,), generator=torch.Generator().manual_seed(66), dtype=torch.int32).cuda()
        run_case(found, "sort_keys n %d" % n, lambda p: ops.sort_keys(keys))
        run_case(found, "pr_curve n %d" % n, lambda p: ops.pr_curve(ops.sort_keys(keys)))
    found.check()
