"""GPU: the engines' cached state across weight reloads, CUDA-graph replay, chunking and streams, bit-identical to a fresh engine.

Every other engine test runs on an engine that is new or reset by hand, on the default stream.  A user's engine keeps six
kinds of device state between calls: the flat weight buffer, the derived tensor-core weight copies, the workspace of the
last shape, the CUDA graphs of ``explain_graphed``, the activations ``attribute`` / ``relprop_pixels`` / ``tensor()`` read,
and the façade's weights version.  Here each case compares a reused engine with a *fresh* engine (built on the same
weights, making the same call on the same shape), bit for bit on the integer views: the engines are deterministic run to
run (test_gpu_poison.py).  At flags 0 the fresh engine is tied to the fp64 oracle at the bounds the existing tests of these
models use, and every weight sequence checks that its two weight sets give different maps and logits.

Models: the tiny ViT of test_gpu_vit.py::test_cuda_graph_replay_matches_launches (img 32, patch 8, D 256, 4 heads, depth 2,
12 classes: 3xTF32 / fp16-split Linears, the tensor-core z+ rule and the dh-64 attention contractions at the bench flags)
and the hidden-256 conditioned BERT of test_gpu_poison.py (sequence 130, one padded row per batch).  Weights A and B are two
seeds of each.  Flag sets: 0, the bench default, the layers_lrp rule on the tensor cores, and the bench default with
alpha = 2 through ``attribute``.

A. Weight reloads through ``eng.load_state_dict``, ``model.load_state_dict`` + ``model.engine()``, an in-place parameter
   update under ``no_grad`` and ``broadcast_weights`` (with ``torch.distributed.broadcast`` replaced by a copy of B: a
   one-rank group cannot show staleness); after each, every entry point equals the fresh engine on B, then on A again.
B. Graph-cache transitions: re-capture after a reshape, eviction at the fifth key, index / start_layer / flags changes,
   ``attribute`` / ``tensor()`` after a replay.
C. Chunking against per-chunk fresh calls, and ``attribute`` after a reshape and back.
D. Streams.  A probe first shows that the test is not vacuous: work behind a ``torch.cuda._sleep`` on a side stream is
   still pending after the default stream has been synchronised, also once each call tested here has been issued.  Every
   engine entry point and every stand-alone op then runs on the side stream behind the sleep, on inputs that hold 0xFF
   until the side stream writes them, and must equal the call on the default stream: a launch or copy on another stream
   reads the poison.  The device-only calls are also captured in a CUDA graph (global capture mode), whose replay must
   equal the eager call.  Then the cross-stream order of one engine's calls: a call issued on the side stream behind the
   sleep, then one on the default stream; the later call's state is what stays (same shape, a shape change, derived
   weights built on the side stream and used on the default one).
E. Two engines interleaved on two streams equal each engine run alone.

Findings: three defects, each fixed in engine.py.  A graph captured on weights A replayed after a reload with the stale
tensor-core copies (A, ``explain_graphed`` on the graph captured on A; the old copies are kept referenced here so that the
unfixed engine replays from live memory), ``broadcast_weights`` kept the copies of the overwritten weights (A, broadcast),
and a call on another stream was not ordered after the engine's previous call (D: the same-shape cross-stream case, where
the side stream's activations stayed, and the derived copies built on the side stream, which the default stream read
before they were written).  E.g. ``vit bench after engine.load_state_dict to B: explain_graphed: maps differs in 48 of
48 entries``, ``bert bench after broadcast_weights to B: explain: maps differs in 324 of 390 entries``, ``vit flags 0
explain on the side stream, then on the default stream: attn0 differs in 3468 of 3468 entries``.

What it catches (each mutation tried once, not committed): launching the LayerNorm kernel that emits the fp16 split on the
legacy default stream (D: the side-stream cases of ``layernorm_split`` and of both engines at the bench flags, which read
the poison; the CUDA-graph replays of the ViT forward and the BERT explain at the bench flags; and the ViT cross-stream
order case), and not re-deriving the tensor-core copies in ``load_state_dict`` (A: every reload through it, the
``model.load_state_dict`` and in-place routes included, 74 mismatches per ViT sequence and 43 per BERT one).

Wall time: about 50 s for this file alone (half of it the first CUDA initialisation) on one H100 80GB HBM3 at a 700 W
power limit.
"""
import collections

import pytest
import torch

from oracle import bert as obert
from oracle import conditioned
from oracle import vit as ovit
from transformer_explainability_b200 import _lib, engine, ops, parallel, visualization

pytestmark = pytest.mark.gpu

BENCH = _lib.FLAG_BENCH_DEFAULT
LRP_TC = _lib.FLAG_RULES_LRP | _lib.FLAG_RULES_LRP_TC
FLAG_SETS = [("flags 0", 0, 1.0), ("bench", BENCH, 1.0), ("lrp_tc", LRP_TC, 1.0), ("bench alpha 2", BENCH, 2.0)]
TC_FLAG_SETS = [f for f in FLAG_SETS if f[1] & (_lib.FLAG_TENSOR_CORES | _lib.FLAG_RULES_LRP_TC)]
RELOADS = ["engine.load_state_dict", "model.load_state_dict", "in-place update", "broadcast_weights"]
BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
SLEEP_CYCLES = 100_000_000                        # ~50 ms at the H100's 1.98 GHz boost clock, longer below it


# ---- comparison ----------------------------------------------------------------------------------------------------------
def _items(out, key=""):
    if out is None:
        return []
    if torch.is_tensor(out):
        return [(key or "out", out)]
    if isinstance(out, dict):
        return [kv for k, v in out.items() for kv in _items(v, "%s%s" % (key + "." if key else "", k))]
    return [kv for i, v in enumerate(out) for kv in _items(v, "%s%d" % (key + "." if key else "", i))]


def snap(out):
    """the tensors of out (tensor / tuple / dict), cloned now: engine views and graph outputs are overwritten later"""
    return {k: v.detach().clone() for k, v in _items(out)}


def _bits(t):
    return t.detach().contiguous().view(BITS[t.element_size()])


class Findings:
    """every mismatch of one test, reported together"""

    def __init__(self):
        self.items = []

    def compare(self, tag, want, got):
        if want.keys() != got.keys():
            self.items.append("%s: outputs %s, expected %s" % (tag, sorted(got), sorted(want)))
            return
        for k, v in want.items():
            w = got[k]
            if w.shape != v.shape or w.dtype != v.dtype:
                self.items.append("%s: %s is %s %s, expected %s %s" % (tag, k, tuple(w.shape), w.dtype, tuple(v.shape), v.dtype))
            elif not torch.equal(_bits(w), _bits(v)):
                d = _bits(w) != _bits(v)
                first = tuple(int(i) for i in d.nonzero()[0])
                self.items.append("%s: %s differs in %d of %d entries, first at %s (%r, expected %r)" % (
                    tag, k, int(d.sum()), d.numel(), first, w[first].item(), v[first].item()))

    def check(self):
        for m in self.items:
            print("FINDING " + m)
        assert not self.items, "%d findings:\n%s" % (len(self.items), "\n".join(self.items[:60]))


# ---- models --------------------------------------------------------------------------------------------------------------
class Vit:
    name, L, seeds = "vit", 2, (2, 3)
    graphed = True

    def __init__(self):
        from test_gpu_vit import make_model
        self.params = {s: ovit.init_params("vit_tiny_test", seed=s, rand_affine=True, dim=256, heads=4, mlp=256, depth=2,
                                           classes=12) for s in self.seeds}
        self._make = lambda s: make_model(*self.params[s], img_size=32, patch_size=8, embed_dim=256, depth=2, mlp_ratio=1.,
                                          num_classes=12)
        self.models = {s: self._make(s) for s in self.seeds}
        self.x = torch.randn(7, 3, 32, 32, generator=torch.Generator().manual_seed(11)).cuda()

    def build(self, seed):
        return self._make(seed)

    def inputs(self, lo, hi):
        return (self.x[lo:hi].contiguous(),)

    def fresh(self, seed, flags=0):
        m = self.models[seed]
        return engine.ViTEngine(m._cfg, m.state_dict(), flags=flags)

    def oracle(self, seed, inp):
        p, heads = self.params[seed]
        return ovit.explain({k: v.double() for k, v in p.items()}, inp[0].cpu().double(), heads)


class Bert:
    name, L, seeds = "bert", 3, (41, 43)
    graphed = False

    def __init__(self):
        from test_gpu_bert import make_model
        self.params = {}
        for s in self.seeds:
            p, heads = obert.init_params(seed=s, vocab=1000, max_pos=512, dim=256, depth=3, heads=4, inter=256, rand_affine=True)
            self.params[s] = (conditioned.condition_bert(p, c_qkv=3.0), heads)
        self._make = lambda s: make_model(*self.params[s], hidden_size=256, num_hidden_layers=3, intermediate_size=256,
                                          vocab_size=1000, max_position_embeddings=512)
        self.models = {s: self._make(s) for s in self.seeds}
        g = torch.Generator().manual_seed(42)
        ids = torch.randint(5, 1000, (7, 130), generator=g)
        ids[:, 0], ids[:, -1] = 101, 102
        mask = torch.ones(7, 130, dtype=torch.long)
        mask[1, 65:], mask[4, 40:], mask[6, 100:] = 0, 0, 0           # a padded row in every batch of the tests
        self.ids, self.mask = ids.cuda(), mask.cuda()

    def build(self, seed):
        return self._make(seed)

    def inputs(self, lo, hi):
        return (self.ids[lo:hi].contiguous(), self.mask[lo:hi].contiguous())

    def fresh(self, seed, flags=0):
        m = self.models[seed]
        return engine.BertEngine(m._cfg, m.state_dict(), flags=flags)

    def oracle(self, seed, inp):
        p, heads = self.params[seed]
        return obert.explain({k: v.double() for k, v in p.items()}, inp[0].cpu(), inp[1].cpu(), heads, start_layer=0)


@pytest.fixture(scope="module")
def models():
    return {"vit": Vit(), "bert": Bert()}


# ---- entry points --------------------------------------------------------------------------------------------------------
def taps(m, eng, first=0):
    """the per-layer tensors a call with start_layer ``first`` writes: attn of every layer, attn_grad / attn_cam from first on"""
    out = {}
    for l in range(m.L):
        out["attn%d" % l] = eng.tensor("attn", l)
        if l >= first:
            out["attn_grad%d" % l] = eng.tensor("attn_grad", l)
            out["attn_cam%d" % l] = eng.tensor("attn_cam", l)
    return out


def ep_explain(m, inp, fl, **kw):
    def fn(eng):
        maps, idx, logits = eng.explain(*inp, start_layer=0, flags=fl, return_logits=True, **kw)
        return snap(dict(maps=maps, idx=idx, logits=logits, **taps(m, eng)))
    return fn


def ep_attribute(m, inp, fl, alpha):
    def fn(eng):
        logits = eng.forward(*inp, flags=fl)
        maps, idx = eng.attribute(start_layer=0, flags=fl, alpha=alpha)
        return snap(dict(logits=logits, maps=maps, idx=idx, **taps(m, eng)))
    return fn


def ep_pixels(m, inp, fl, alpha):
    def fn(eng):
        eng.forward(*inp, flags=fl)
        pix = eng.relprop_pixels(flags=fl, alpha=alpha, per_channel=True)
        return snap(dict(pix=pix, **taps(m, eng)))
    return fn


def ep_graphed(m, inp, fl, start_layer=0, index=None):
    def fn(eng):
        maps, idx, logits = eng.explain_graphed(*inp, index=index, start_layer=start_layer, flags=fl, return_logits=True)
        return snap(dict(maps=maps, idx=idx, logits=logits, **taps(m, eng, start_layer)))
    return fn


def ep_sharded(m, inp, fl):
    def fn(eng):
        eng.flags = fl
        maps, idx = parallel.explain_sharded(eng, inp[0], start_layer=0, graph=True)
        return snap(dict(maps=maps, idx=idx))
    return fn


def entry_points(m, inp, fl, alpha, new_key=False):
    """(name, fn(eng) -> outputs) of every entry point at one flag set; the graphed ones first, so that after a reload the
    graph captured on the old weights is the first thing that runs.  new_key: also a graph key no earlier call captured."""
    out = []
    if m.graphed and alpha == 1.0:
        out.append(("explain_graphed", ep_graphed(m, inp, fl)))
        if new_key:
            out.append(("explain_graphed, new key", ep_graphed(m, inp, fl, start_layer=1)))
    if alpha == 1.0:
        out += [("explain", ep_explain(m, inp, fl)), ("explain_sharded(graph=True)", ep_sharded(m, inp, fl))]
    alpha_tag = "" if alpha == 1.0 else " alpha %g" % alpha
    out.append(("forward + attribute" + alpha_tag, ep_attribute(m, inp, fl, alpha)))
    if m.name == "vit":
        out.append(("forward + relprop_pixels" + alpha_tag, ep_pixels(m, inp, fl, alpha)))
    return out


class References:
    """outputs of each call on a fresh engine, cached by (model, seed, flag set, call)"""

    def __init__(self):
        self.cache = {}

    def __call__(self, m, seed, fl, name, fn):
        key = (m.name, seed, fl, name)
        if key not in self.cache:
            self.cache[key] = fn(m.fresh(seed, fl))
        return self.cache[key]


@pytest.fixture(scope="module")
def refs():
    return References()


# ---- fp64 anchor and distinct weights --------------------------------------------------------------------------------------
def test_fresh_engine_matches_fp64_and_weights_differ(models, refs):
    """The fresh engine at flags 0 against the fp64 oracle on weights A, at the bounds of the existing tests of these models
    (the tiny ViTs of test_gpu_vit.py / smoke(): 1e-4 absolute and 2e-2 of the maximum; the hidden-256 BERT of
    test_gpu_methods_tc.py::test_bert_narrow_intermediate: 2e-4 of the maximum); the class index bit-exact.  Weights A and B
    give different maps and logits at every flag set, or the reload cases would prove nothing."""
    for m in models.values():
        a, b = m.seeds
        inp = m.inputs(0, 3)
        out = refs(m, a, 0, "explain", ep_explain(m, inp, 0))
        ref, ridx = m.oracle(a, inp)
        err = (out["maps"].cpu().double() - ref).abs().max().item()
        scale = ref.abs().max().item()
        print("%s flags 0 vs fp64: %.1e of the maximum" % (m.name, err / scale))
        assert torch.equal(out["idx"].cpu().long(), ridx.long()), m.name
        if m.name == "vit":
            assert err <= 1e-4 and err <= 2e-2 * scale, (m.name, err, scale)
        else:
            assert err < 2e-4 * scale, (m.name, err, scale)
        for tag, fl, alpha in FLAG_SETS:
            name, fn = [e for e in entry_points(m, inp, fl, alpha) if e[0].startswith("forward + attribute")][0]
            ra, rb = refs(m, a, fl, name, fn), refs(m, b, fl, name, fn)
            for k in ("maps", "logits"):
                assert not torch.equal(ra[k], rb[k]), "%s %s: weights A and B give the same %s" % (m.name, tag, k)


# ---- A. weight reloads -----------------------------------------------------------------------------------------------------
def reload(m, method, model, eng, seed, monkeypatch):
    target = m.models[seed]
    if method == "engine.load_state_dict":
        eng.load_state_dict(target.state_dict())
    elif method == "model.load_state_dict":
        model.load_state_dict(target.state_dict())
        assert model.engine() is eng
    elif method == "in-place update":
        with torch.no_grad():
            for p, q in zip(model.parameters(), target.parameters()):
                p.copy_(q)
        assert model.engine() is eng
    else:
        flat = m.fresh(seed).weights
        monkeypatch.setattr(torch.distributed, "broadcast", lambda t, src=0, group=None: t.copy_(flat))
        eng.broadcast_weights()


@pytest.mark.parametrize("method", RELOADS)
@pytest.mark.parametrize("kind", ["vit", "bert"])
def test_weight_reload(models, refs, kind, method, monkeypatch):
    """A, then B by ``method``, then A again, on one engine: every entry point equals the fresh engine on the current weights
    (explain_graphed both on the graph captured before the reload and on a new key)."""
    m = models[kind]
    a, b = m.seeds
    inp = m.inputs(0, 3)
    found = Findings()
    for tag, fl, alpha in FLAG_SETS:
        model = m.build(a)
        eng = model.engine()
        for name, fn in entry_points(m, inp, fl, alpha):
            found.compare("%s %s on A: %s" % (kind, tag, name), refs(m, a, fl, name, fn), fn(eng))
        kept = []
        for seed, label in ((b, "B"), (a, "A again")):
            # every derived buffer a graph may have captured stays referenced: an engine that dropped its buffer on a reload
            # then replays the graph from live memory and fails with a mismatch, not by reading a freed block
            kept.append(eng.derived)
            reload(m, method, model, eng, seed, monkeypatch)
            for name, fn in entry_points(m, inp, fl, alpha, new_key=True):
                found.compare("%s %s after %s to %s: %s" % (kind, tag, method, label, name), refs(m, seed, fl, name, fn), fn(eng))
        torch.cuda.synchronize()
        del kept
    found.check()


# ---- B. graph-cache transitions ------------------------------------------------------------------------------------------
def test_graph_cache_transitions(models, refs):
    m = models["vit"]
    a = m.seeds[0]
    x5, x3 = m.inputs(0, 5), m.inputs(0, 3)
    eng = m.build(a).engine()
    found = Findings()
    idx = torch.tensor([3, 1, 7, 0, 11], dtype=torch.int32)

    def step(tag, fl, fn):
        found.compare(tag, refs(m, a, fl, tag, fn), fn(eng))

    step("graphed B 5", BENCH, ep_graphed(m, x5, BENCH))
    step("explain B 3 (reshapes the workspace)", BENCH, ep_explain(m, x3, BENCH))
    first = eng._graphs[(5, 0, BENCH, (3, 32, 32))]
    step("graphed B 5 again (re-captures)", BENCH, ep_graphed(m, x5, BENCH))
    assert eng._graphs[(5, 0, BENCH, (3, 32, 32))] is not first
    step("graphed B 5 index", BENCH, ep_graphed(m, x5, BENCH, index=idx))
    step("graphed B 5 start_layer 1", BENCH, ep_graphed(m, x5, BENCH, start_layer=1))
    step("graphed B 5 flags 0", 0, ep_graphed(m, x5, 0))
    step("graphed B 5 lrp_tc", LRP_TC, ep_graphed(m, x5, LRP_TC))
    assert len(eng._graphs) == 4
    step("graphed B 5 flags all fast (a fifth key evicts)", _lib.FLAG_ALL_FAST, ep_graphed(m, x5, _lib.FLAG_ALL_FAST))
    assert len(eng._graphs) == 1
    step("graphed B 5 again after the eviction", BENCH, ep_graphed(m, x5, BENCH))
    step("graphed B 5 index after the eviction", BENCH, ep_graphed(m, x5, BENCH, index=idx))

    def replay_then_attribute(e):
        e.explain_graphed(*x5, start_layer=0, flags=BENCH)
        maps, i = e.attribute(start_layer=1, flags=BENCH)
        return snap(dict(maps=maps, idx=i, **taps(m, e, 1)))
    step("attribute and tensor() after a replay", BENCH, replay_then_attribute)
    found.check()


# ---- C. chunking and the shape-keyed workspace -----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["vit", "bert"])
def test_chunks_and_reshapes(models, kind):
    m = models[kind]
    a = m.seeds[0]
    found = Findings()
    for tag, fl, _ in FLAG_SETS[:3]:
        eng = m.build(a).engine()
        maps, idx, logits = eng.explain(*m.inputs(0, 7), start_layer=0, flags=fl, chunk=3, return_logits=True)
        got = snap(dict(maps=maps, idx=idx, logits=logits))
        parts = [m.fresh(a, fl).explain(*m.inputs(lo, hi), start_layer=0, flags=fl, return_logits=True)
                 for lo, hi in ((0, 3), (3, 6), (6, 7))]
        want = {k: torch.cat([p[i] for p in parts]) for i, k in enumerate(("maps", "idx", "logits"))}
        found.compare("%s %s explain(7, chunk=3)" % (kind, tag), want, got)

        eng.forward(*m.inputs(0, 5), flags=fl)
        eng.explain(*m.inputs(0, 2), start_layer=0, flags=fl)
        eng.forward(*m.inputs(0, 5), flags=fl)
        maps, idx = eng.attribute(start_layer=0, flags=fl)
        got = snap(dict(maps=maps, idx=idx, **taps(m, eng)))
        f = m.fresh(a, fl)
        f.forward(*m.inputs(0, 5), flags=fl)
        maps, idx = f.attribute(start_layer=0, flags=fl)
        found.compare("%s %s forward 5, explain 2, forward 5, attribute" % (kind, tag), snap(dict(maps=maps, idx=idx, **taps(m, f))), got)
    found.check()


# ---- D. streams ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def side():
    return torch.cuda.Stream()


def test_stream_probe(side):
    """work behind the sleep on the side stream is still pending once the default stream has run and been synchronised (the
    trivial op runs once first: its allocation and the lazy load of its kernel may each wait for the whole device)"""
    t = torch.ones(1, device="cuda")
    t.add_(1)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
    t.add_(1)
    torch.cuda.current_stream().synchronize()
    pending = not side.query()
    side.synchronize()
    assert pending, "the side stream finished its sleep before the default stream: the stream cases would be vacuous"


def _poisoned_like(t):
    b = torch.empty_like(t, memory_format=torch.contiguous_format)
    b.view(torch.uint8).fill_(0xFF)
    return b


def on_side_stream(side, fn, inputs, timed=True):
    """fn(*inputs) on the side stream behind the sleep, its inputs 0xFF until the side stream writes them; returns the
    outputs.  timed: the call must have been issued while the sleep is still pending (the probe's condition per call)."""
    bufs = [_poisoned_like(t) for t in inputs]
    cur = torch.cuda.current_stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, inputs):
            b.copy_(t)
        out = fn(*bufs)
        pending = not side.query()
        got = snap(out)
    cur.wait_stream(side)
    torch.cuda.synchronize()
    if timed:
        assert pending, "the sleep ended before the call was issued: raise SLEEP_CYCLES"
    return got


def stream_case(found, side, tag, make, inputs, timed=True):
    """make() -> fn, called for each of the two runs before either is issued: engines are built (their weights uploaded,
    which reads the state_dict back to the host) outside the timed window"""
    try:
        want = snap(make()(*[t.clone() for t in inputs]))
    except _lib.TeError as e:
        if e.status != _lib.TE_ERR_UNSUPPORTED:
            raise
        print("%s: the kernel does not take the shape" % tag)
        return
    torch.cuda.synchronize()
    got = on_side_stream(side, make(), inputs, timed)
    found.compare(tag + " on a side stream", want, got)


def capture_case(found, tag, fn, inputs):
    """fn(*inputs) eagerly and captured in a CUDA graph (global capture mode) whose outputs are poisoned before the replay"""
    try:
        want = snap(fn(*inputs))
    except _lib.TeError as e:
        if e.status != _lib.TE_ERR_UNSUPPORTED:
            raise
        return
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn(*inputs)
    outs = _items(out)
    for _, t in outs:
        t.fill_(float("nan") if t.is_floating_point() else -1)
    graph.replay()
    torch.cuda.synchronize()
    found.compare(tag + " replayed from a CUDA graph", want, snap(dict(outs)))


def engine_stream_cases(m, fl):
    """(tag, make() -> fn(*inputs) -> outputs, inputs) of every engine entry point; each run gets a new engine, except the
    graph replays, which share one whose graph is captured here (the capture synchronises the device)"""
    a = m.seeds[0]
    inp = m.inputs(0, 3)

    def explain():
        e = m.fresh(a, fl)
        return lambda *i: e.explain(*i, start_layer=0, flags=fl, return_logits=True)

    def attribute():
        e = m.fresh(a, fl)

        def fn(*i):
            logits = e.forward(*i, flags=fl)
            return dict(logits=logits, attribute=e.attribute(start_layer=0, flags=fl), **taps(m, e))
        return fn
    out = [("explain", explain, inp), ("forward + attribute + tensor()", attribute, inp)]
    if m.name == "vit":
        def pixels():
            e = m.fresh(a, fl)

            def fn(*i):
                e.forward(*i, flags=fl)
                return e.relprop_pixels(flags=fl, per_channel=True)
            return fn
        warm = m.fresh(a, fl)
        warm.flags = fl
        warm.explain_graphed(*inp)

        def graphed(*i):
            return dict(out=warm.explain_graphed(*i, return_logits=True), **taps(m, warm))

        def sharded(*i):
            return parallel.explain_sharded(warm, i[0], start_layer=0, graph=True)
        out += [("forward + relprop_pixels", pixels, inp), ("explain_graphed (replay)", lambda: graphed, inp),
                ("explain_sharded(graph=True)", lambda: sharded, inp)]
    else:
        def sharded():
            e = m.fresh(a, fl)
            return lambda *i: parallel.explain_sharded(e, i[0], start_layer=0)
        out.append(("explain_sharded", sharded, inp[:1]))
    return out


@pytest.mark.parametrize("kind", ["vit", "bert"])
def test_engine_launches_on_callers_stream(models, side, kind):
    m = models[kind]
    found = Findings()
    for fl in (0, BENCH, LRP_TC):
        for tag, fn, inputs in engine_stream_cases(m, fl):
            stream_case(found, side, "%s flags %d %s" % (kind, fl, tag), fn, inputs)
    found.check()


def _rand(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).cuda()


def op_cases():
    """(tag, fn(*inputs) -> outputs, inputs, capturable, timed) of every stand-alone op, at shapes the tensor-core kernels
    take (K 768, N 768 / 3072, 130 rows; attention batch 2 x 2 heads, n 65, dh 64)"""
    cases = []
    rows, K, N = 130, 768, 768
    x, w, b = _rand(rows, K, seed=1), _rand(N, K, seed=2, scale=K ** -0.5), _rand(N, seed=3)
    dy, e0f, e0b, r = _rand(rows, N, seed=4), _rand(rows, N, seed=5), _rand(rows, K, seed=6), _rand(rows, N, seed=7)
    y = x @ w.t() + b
    for tc, f16 in ((False, False), (True, False), (True, True)):
        cases.append(("linear_forward tc %s f16_split %s" % (tc, f16),
                      lambda x, w, b, tc=tc, f16=f16: ops.linear_forward(x, w, b, tensor_cores=tc, f16_split=f16), (x, w, b), tc))
    for tc in (False, True):
        cases.append(("linear_backward tc %s" % tc, lambda dy, w, tc=tc: ops.linear_backward(dy, w, tensor_cores=tc), (dy, w), tc))
    cases += [("linear_backward_f16", ops.linear_backward_f16, (dy, w), True),
              ("linear_backward_tf32", ops.linear_backward_tf32, (dy, w), True),
              ("linear_forward_epi 3xtf32 bias_gelu",
               lambda x, w, b: ops.linear_forward_epi(x, w, b, epi="bias_gelu", family="3xtf32"), (x, w, b), True),
              ("linear_forward_epi f16_split bias_add",
               lambda x, w, b, e: ops.linear_forward_epi(x, w, b, e, epi="bias_add", family="f16_split"), (x, w, b, e0f), True),
              ("linear_backward_epi simt gelu_bwd",
               lambda dy, w, e: ops.linear_backward_epi(dy, w, e, epi="gelu_bwd", family="simt"), (dy, w, e0b), False),
              ("linear_backward_epi tf32 gelu_bwd",
               lambda dy, w, e: ops.linear_backward_epi(dy, w, e, epi="gelu_bwd", family="tf32"), (dy, w, e0b), True),
              ("f16_block_split", ops.f16_block_split, (x,), False),
              ("layernorm_split", lambda x, g, c: ops.layernorm_split(x, g, c, 1e-6), (x, _rand(K, seed=8), _rand(K, seed=9)), False),
              ("tc_zplus_s", lambda x, w, r, y, b: ops.tc_zplus_s(x, w, r, y, bias=b), (x, w, r, y, b), True),
              ("tc_zplus_s f16", lambda x, w, r, y, b: ops.tc_zplus_s(x, w, r, y, bias=b, f16=True), (x, w, r, y, b), True)]
    for name, kw, tc in (("ours simt", {}, False), ("ours tc", dict(tensor_cores=True), True), ("lrp", dict(variant="lrp"), False),
                         ("lrp_tc", dict(variant="lrp_tc"), True)):
        for alpha in (1.0, 2.0):
            cases.append(("linear_relprop %s alpha %g" % (name, alpha),
                          lambda x, w, r, kw=kw, alpha=alpha: ops.linear_relprop(x, w, r, alpha=alpha, **kw), (x, w, r), tc))
    cases.append(("linear_relprop ours tc y", lambda x, w, r, y, b: ops.linear_relprop(x, w, r, tensor_cores=True, y=y, bias=b),
                  (x, w, r, y, b), True))
    a3, b3, r3 = _rand(2, 197, 64, seed=10), _rand(2, 197, 64, seed=11), _rand(2, 197, 64, seed=12)
    cases += [("add_relprop", ops.add_relprop, (a3, b3, r3), False),
              ("add_relprop lrp", lambda a, b, r: ops.add_relprop(a, b, r, variant="lrp"), (a3, b3, r3), False),
              ("clone_relprop", lambda x, r1, r2: ops.clone_relprop(x, [r1, r2]), (a3, b3, r3), False),
              ("index_select_relprop", ops.index_select_relprop, (a3, _rand(2, 1, 64, seed=13)), False)]
    n, H, dh = 65, 2, 64
    D, npad = H * dh, 68
    q, k, v = (_rand(2, H, n, dh, seed=14 + i) for i in range(3))
    p = torch.softmax(_rand(2, H, n, n, seed=17), -1)
    cases += [("matmul_av_relprop", ops.matmul_av_relprop, (p, v, _rand(2, H, n, dh, seed=18)), False),
              ("matmul_qk_relprop", ops.matmul_qk_relprop, (q, k, _rand(2, H, n, n, seed=19)), False)]
    qkv = _rand(2 * n, 3 * D, seed=20)
    amap = _rand(2, H, n, npad, seed=21)
    cases += [("tc_attention_nn", lambda qkv, out: ops.tc_attention_nn(qkv, 3 * D, qkv[:, D:], 3 * D, 2, H, n, dh, out, npad,
                                                                        None, 0.125, "store"),
               (qkv, torch.zeros(2 * H * n * npad, device="cuda")), True),
              ("tc_attention_nk", lambda amap, qkv, out: ops.tc_attention_nk(amap, npad, 0, qkv[:, 2 * D:], 3 * D, 2, H, n, out, D,
                                                                              None, 0.75, "store"),
               (amap, qkv, torch.zeros(2 * n, D, device="cuda")), True)]
    ga, gg = _rand(2, 4, n, n, seed=22), _rand(2, 4, n, n, seed=23)
    cases += [("head_reduce", lambda a, g, hw: ops.head_reduce(a, g, hw, mode="relu_mean"), (ga, gg, _rand(2, 4, seed=24)), False),
              ("head_region_mean", lambda g: ops.head_region_mean(g, (0, 1), (1, n)), (gg,), False)]
    grad, cam = _rand(2, 2, 4, n, npad, seed=25), _rand(2, 2, 4, n, npad, seed=26).abs()
    for fused in (False, True):
        cases.append(("attribution_rollout fused %s" % fused,
                      lambda g, c, fused=fused: ops.attribution_rollout(g, c, start_layer=0, normalize=True, fused=fused), (grad, cam),
                      True))
    mats = [torch.softmax(_rand(2, n, n, seed=27 + i), -1) for i in range(3)]
    cases.append(("compute_rollout_attention", lambda *ms: ops.compute_rollout_attention(list(ms), start_layer=1, normalize=True),
                  tuple(mats), True))
    images = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(30)).cuda()
    cases.append(("patch_embed_relprop", lambda im, w, r: ops.patch_embed_relprop(im, w, r, per_channel=True),
                  (images, _rand(64, 3, 8, 8, seed=31, scale=0.05), _rand(2, 16, 64, seed=32)), False))
    cases.append(("perturb_images", lambda im, s: ops.perturb_images(im, s, [0, 1, 500, 1024]), (images, _rand(2, 32, 32, seed=33)),
                  False))
    logits = _rand(130, 1000, seed=34)
    target = torch.randint(0, 1000, (130,), generator=torch.Generator().manual_seed(35)).cuda()
    cases += [("logit_stats", ops.logit_stats, (logits, target), False), ("class_probs", ops.class_probs, (logits,), False)]
    maps = _rand(2, 196, seed=36)
    labels = (torch.rand(2, 224 * 224, generator=torch.Generator().manual_seed(37)) > 0.7).long().cuda()
    keys = ops.seg_metrics(maps, labels, pr_keys=True)["pr_keys"].reshape(-1).contiguous()
    cases += [("seg_metrics", lambda m, l: ops.seg_metrics(m, l, pr_keys=True), (maps, labels), False),
              ("sort_keys", lambda k: ops.sort_keys(k, segments=2), (keys,), False),
              ("pr_curve", ops.pr_curve, (ops.sort_keys(keys),), None)]                       # reads its count back
    emaps = _rand(2, 40, seed=38)
    ids = torch.randint(5, 1000, (2, 40), generator=torch.Generator().manual_seed(39)).cuda()
    ranges, woff = [(1, 2), (3, 3), (4, 6), (7, 7), (1, 1), (2, 5)], [0, 4, 6]
    cases += [("eraser_rationales", lambda m: ops.eraser_rationales(m, ranges, woff, [(0, 1), (1, 1)], [0, 1, 2], (1, 3)), (emaps,),
               None),
              ("eraser_reduce_inputs", lambda m, i: ops.eraser_reduce_inputs(m, i, [40, 30], ranges, woff, [[1, 2], [0, 1]]),
               (emaps, ids), None),
              ("relevance_to_heatmap", lambda m: visualization.relevance_to_heatmap(m, grid=14, scale=16), (maps,), False)]
    return cases


def test_ops_launch_on_callers_stream(side):
    """every stand-alone op on the side stream behind the sleep, on inputs poisoned until the side stream writes them"""
    found = Findings()
    for tag, fn, inputs, capturable in op_cases():
        stream_case(found, side, tag, lambda fn=fn: fn, inputs, timed=tag != "pr_curve")
    found.check()


def test_capture_device_only_calls(models):
    """the device-only engine calls, the rollout ops and the tensor-core ops captured in a CUDA graph in the global capture
    mode (a launch on another stream, a synchronisation or a host read-back fails the capture) replay to the eager result;
    the calls with pageable host copies or host read-back (eraser_*, pr_curve) are left out"""
    found = Findings()
    for kind, m in models.items():
        inp = m.inputs(0, 3)
        for fl in (0, BENCH, LRP_TC):
            eng = m.fresh(m.seeds[0], fl)
            tag = "%s flags %d" % (kind, fl)
            capture_case(found, tag + " forward", lambda *i: eng.forward(*i, flags=fl), inp)
            capture_case(found, tag + " attribute", lambda: eng.attribute(start_layer=0, flags=fl), ())
            if kind == "vit":
                capture_case(found, tag + " relprop_pixels", lambda: eng.relprop_pixels(flags=fl, per_channel=True), ())
            else:
                capture_case(found, tag + " explain", lambda *i: eng.explain(*i, start_layer=0, flags=fl, chunk=3, return_logits=True),
                             inp)
    for tag, fn, inputs, capturable in op_cases():
        if capturable:
            capture_case(found, tag, fn, inputs)
    found.check()


def _order_case(m, eng, fl, x1, x2, side):
    """sleep on the side stream, eng.explain(x1) there, at once eng.explain(x2) on the default stream; then the state the
    engine keeps (tensor() views, attribute()) is that of x2"""
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        eng.explain(*x1, start_layer=0, flags=fl)
    maps, idx = eng.explain(*x2, start_layer=0, flags=fl)
    pending = not side.query()
    out = dict(maps=maps, idx=idx)
    torch.cuda.synchronize()
    assert pending, "the sleep ended before the default-stream call was issued: raise SLEEP_CYCLES"
    out.update(taps(m, eng))
    got = snap(out)
    got.update({"attribute." + k: v for k, v in snap(eng.attribute(start_layer=0, flags=fl)).items()})
    f = m.fresh(m.seeds[0], fl)
    maps, idx = f.explain(*x2, start_layer=0, flags=fl)
    want = snap(dict(maps=maps, idx=idx, **taps(m, f)))
    want.update({"attribute." + k: v for k, v in snap(f.attribute(start_layer=0, flags=fl)).items()})
    return want, got


@pytest.mark.parametrize("kind", ["vit", "bert"])
def test_cross_stream_order_same_shape(models, side, kind):
    m = models[kind]
    found = Findings()
    for fl in (0, BENCH):
        eng = m.build(m.seeds[0]).engine()
        eng.explain(*m.inputs(0, 3), start_layer=0, flags=fl)          # the workspace and derived weights exist
        torch.cuda.synchronize()
        want, got = _order_case(m, eng, fl, m.inputs(3, 6), m.inputs(0, 3), side)
        found.compare("%s flags %d explain on the side stream, then on the default stream" % (kind, fl), want, got)
    found.check()


@pytest.mark.parametrize("kind", ["vit", "bert"])
def test_cross_stream_order_shape_change(models, side, kind):
    """as above with a shape change between the two calls: the re-allocation must not hand out the workspace the side
    stream still uses"""
    m = models[kind]
    found = Findings()
    for fl in (0, BENCH):
        eng = m.build(m.seeds[0]).engine()
        eng.explain(*m.inputs(0, 3), start_layer=0, flags=fl)
        torch.cuda.synchronize()
        want, got = _order_case(m, eng, fl, m.inputs(2, 5), m.inputs(0, 5) if kind == "vit" else m.inputs(0, 2), side)
        found.compare("%s flags %d explain on the side stream, then another shape on the default stream" % (kind, fl), want, got)
    found.check()


@pytest.mark.parametrize("kind", ["vit", "bert"])
def test_derived_built_on_side_stream(models, side, kind):
    """the tensor-core copies are first built by a call on the side stream behind the sleep and used at once by a call on the
    default stream"""
    m = models[kind]
    found = Findings()
    eng = m.build(m.seeds[0]).engine()
    x = m.inputs(0, 3)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        eng.forward(*x, flags=BENCH)
    got = ep_explain(m, x, BENCH)(eng)
    torch.cuda.synchronize()
    found.compare("%s derived built on the side stream" % kind, ep_explain(m, x, BENCH)(m.fresh(m.seeds[0], BENCH)), got)
    found.check()


# ---- E. two engines at once ------------------------------------------------------------------------------------------------
def test_two_engines_interleaved(models, side):
    """a ViT and a BERT engine, and two ViT engines with different weights, interleaved on two streams: each equals the
    engine run alone (the library keeps no device globals; its host statics are per-device attributes and options)"""
    vit, bert = models["vit"], models["bert"]
    found = Findings()
    pairs = [(vit, vit.seeds[0], bert, bert.seeds[0]), (vit, vit.seeds[0], vit, vit.seeds[1])]
    for fl in (0, BENCH):
        for m1, s1, m2, s2 in pairs:
            alone = [ep_explain(m, m.inputs(0, 3), fl)(m.fresh(s, fl)) for m, s in ((m1, s1), (m2, s2))]
            e1, e2 = m1.fresh(s1, fl), m2.fresh(s2, fl)
            got = collections.defaultdict(list)
            side.wait_stream(torch.cuda.current_stream())
            for _ in range(2):
                with torch.cuda.stream(side):
                    got[0].append(ep_explain(m1, m1.inputs(0, 3), fl)(e1))
                got[1].append(ep_explain(m2, m2.inputs(0, 3), fl)(e2))
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for i, (m, s) in enumerate(((m1, s1), (m2, s2))):
                for r, out in enumerate(got[i]):
                    found.compare("flags %d %s seed %d (with %s) round %d" % (fl, m.name, s, (m2 if i == 0 else m1).name, r),
                                  alone[i], out)
    found.check()
