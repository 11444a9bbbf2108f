"""Host-side engine objects: flat frozen-weight buffer, workspace, and the explain call.

The engine is the CUDA replacement for the stateful hook machinery of the reference
(``modules/layers_ours.py:16-27`` forward hooks, ``retain_graph=True`` autograd graph): it owns one
flat fp32 weight buffer (the unit of the single NCCL broadcast), the tensor-core copies derived from it, and one
activation workspace (of the last shape), and issues O(1) launches per block per BATCH through the C ABI.

Every public call launches on the caller's current stream.  Calls to one engine are ordered in the order they are
issued, whatever their streams: each call ends by recording an event, and a call on another stream first waits on it,
so the state the later call leaves (workspace, ``tensor()`` views, ``attribute()`` inputs) is what stays.  The
workspace and the derived weights are marked as used by every stream that ran on them (``record_stream``), so a reshape
never hands their memory out while another stream's work still reads it.  Calls to one engine therefore never overlap
on the device; two engines are independent.
"""
import ctypes
import functools

import torch

from . import _lib
from ._lib import TeVitConfig, check, ptr


def _on_engine_device(fn):
    """Make the engine's device current for the duration of the call: the C library launches on the current device
    and neither it nor ``torch.cuda.current_stream(dev)`` switches devices (a model moved to ``cuda:1`` without
    ``torch.cuda.set_device(1)`` would otherwise fail with an invalid resource handle).  The call is ordered after the
    engine's previous call on any stream (the module docstring); not while a CUDA graph is being captured, where an
    event of outside work cannot be waited on and the graph's own order applies."""
    @functools.wraps(fn)
    def wrapped(self, *args, **kwargs):
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            if torch.cuda.is_current_stream_capturing():
                return fn(self, *args, **kwargs)
            if self._done_stream is not None and self._done_stream != stream:
                stream.wait_event(self._done)
            try:
                return fn(self, *args, **kwargs)
            finally:
                for t in (self._ws, self.derived):
                    if t is not None:
                        t.record_stream(stream)
                self._done.record(stream)
                self._done_stream = stream
    return wrapped


_VIT_ACTS = {"gelu": _lib.VIT_ACT_GELU, "quick_gelu": _lib.VIT_ACT_QUICK_GELU}


def vit_config(img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12, num_heads=12,
               mlp_ratio=4., distilled=False, eps_block=1e-6, eps_final=1e-5, pre_norm=False, act="gelu"):
    """``te_vit_config``.  pre_norm: a LayerNorm (``norm_pre``, eps_block) over the assembled tokens before block 0, as CLIP's
    ``ln_pre``; act: the MLP activation, "gelu" (erf) or "quick_gelu" (CLIP's x * sigmoid(1.702 x))."""
    if act not in _VIT_ACTS:
        raise ValueError("act must be one of %s, got %r" % (sorted(_VIT_ACTS), act))
    return TeVitConfig(img_size, patch_size, in_chans, num_classes, embed_dim, depth, num_heads,
                       int(embed_dim * mlp_ratio), int(bool(distilled)), eps_block, eps_final, int(bool(pre_norm)),
                       _VIT_ACTS[act])


class _Engine:
    """Host state the ViT and BERT engines share: the flat frozen-weight buffer described by the library's weight table, the
    derived tensor-core weight copies, and the workspace of the last shape.  ``_prefix`` names the model's C entry points."""
    _prefix = None
    _optional = ()                  # weight names a state_dict may leave out (zeros)

    def __init__(self, cfg, state_dict=None, device=None, flags=0):
        if not torch.cuda.is_available():
            raise RuntimeError("transformer_explainability_b200 needs a CUDA device (H100, sm_90a); "
                               "there is no CPU fallback")
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
        self.flags = flags
        c = ctypes.byref(cfg)
        n = check(self._fn("num_weights")(c), self._prefix + "num_weights")
        self.weight_table = [(self._fn("weight_name")(c, i).decode(), self._fn("weight_numel")(c, i),
                              self._fn("weight_offset")(c, i)) for i in range(n)]
        total = check(self._fn("weight_total")(c), self._prefix + "weight_total")
        self.weights = torch.zeros(total, dtype=torch.float32, device=self.device)
        self.derived = None                      # tensor-core weight copies, built on demand
        self._ws = None
        self._ws_key = None
        self._done = torch.cuda.Event()          # recorded at the end of every public call
        self._done_stream = None
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def _fn(self, name):
        return getattr(self.lib, self._prefix + name)

    # ---- weights ------------------------------------------------------------------------------
    @_on_engine_device
    def load_state_dict(self, sd):
        """Pack a reference-keyed ``state_dict`` into the flat device buffer."""
        host = torch.zeros(self.weights.numel(), dtype=torch.float32)
        for name, numel, off in self.weight_table:
            if name not in sd:
                if name.endswith(self._optional):
                    continue
                raise KeyError("state_dict is missing %r" % name)
            t = sd[name].detach().to(torch.float32).reshape(-1).cpu()
            if t.numel() != numel:
                raise ValueError("%s: expected %d values, got %d" % (name, numel, t.numel()))
            host[off:off + numel] = t
        self.weights.copy_(host)
        self._prepare_derived()

    def _prepare_derived(self):
        """Re-derive the tensor-core copies from the weights, in place: once built, the derived buffer keeps its address,
        so the CUDA graphs of ``explain_graphed`` that captured it stay valid after a weight reload."""
        if self.derived is not None:
            check(self._fn("prepare_derived")(ctypes.byref(self.cfg), ptr(self.weights), ptr(self.derived), self._stream()),
                  self._prefix + "prepare_derived")

    @_on_engine_device
    def _derived(self, flags):
        """W+/W-/W+^T/W-^T TF32 copies for the tensor-core paths (built on first use, kept current by every weight load)."""
        if not (flags & (_lib.FLAG_TENSOR_CORES | _lib.FLAG_RULES_LRP_TC)):
            return None
        if self.derived is None:
            n = check(self._fn("derived_total")(ctypes.byref(self.cfg)), self._prefix + "derived_total")
            self.derived = torch.empty(n, dtype=torch.float32, device=self.device)
            self._prepare_derived()
        return self.derived

    @_on_engine_device
    def broadcast_weights(self, src=0, group=None):
        """The one collective of the path: NCCL broadcast of the flat frozen-weight buffer (the derived copies follow)."""
        import torch.distributed as dist
        dist.broadcast(self.weights, src=src, group=group)
        self._prepare_derived()

    # ---- workspace: shape = (batch,) for ViT, (batch, seq) for BERT -----------------------------
    def _workspace_bytes(self, *shape):
        return check(self._fn("workspace_bytes")(ctypes.byref(self.cfg), *shape), self._prefix + "workspace_bytes")

    def _shaped_workspace(self, *shape):
        if self._ws is None or self._ws_key != shape:
            self._ws = None
            self._ws = torch.empty(self._workspace_bytes(*shape) // 4, dtype=torch.float32, device=self.device)
            self._ws_key = shape
        return self._ws

    def _max_batch(self, limit, reserve_bytes, *rest):
        free, _ = torch.cuda.mem_get_info(self.device)
        if self._ws is not None:
            free += self._ws.numel() * 4
        per = self._workspace_bytes(2, *rest) - self._workspace_bytes(1, *rest)
        b = max(1, int((free - reserve_bytes) // max(per, 1)))
        return min(b, limit) if limit else b

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _index_tensor(self, index, b):
        if index is None:
            return torch.full((b,), -1, dtype=torch.int32, device=self.device)
        t = torch.as_tensor(index, device=self.device).reshape(-1).to(torch.int32)
        if t.numel() == 1 and b > 1:
            t = t.expand(b)
        if t.numel() != b:
            raise ValueError("index must have one entry per sample")
        return t.contiguous().clone()

    def _view(self, name, layer, *shape):
        """The strided view of workspace tensor ``name`` that ``<prefix>tensor`` describes."""
        ws = self._shaped_workspace(*shape)
        p = ctypes.c_void_p()
        dims = (ctypes.c_longlong * 4)()
        strides = (ctypes.c_longlong * 4)()
        check(self._fn("tensor")(ctypes.byref(self.cfg), *shape, ptr(ws), name.encode(), layer, ctypes.byref(p), dims, strides),
              self._prefix + "tensor")
        off = (p.value - ws.data_ptr()) // 4
        nd = 4
        while nd > 2 and dims[nd - 1] == 1:
            nd -= 1
        return torch.as_strided(ws, [int(dims[i]) for i in range(nd)], [int(strides[i]) for i in range(nd)], off)


class ViTEngine(_Engine):
    """Runs ``generate_LRP(method='transformer_attribution')`` for batches of independent inputs."""
    _prefix = "te_vit_"
    # zeros when left out: qkv_bias=False models, and the bias-free patch embedding / projection head of CLIP image towers
    _optional = ("qkv.bias", "patch_embed.proj.bias", "head.bias")

    def __init__(self, cfg, state_dict=None, device=None, flags=0):
        super().__init__(cfg, state_dict, device, flags)
        self.tokens = (cfg.img_size // cfg.patch_size) ** 2 + (2 if cfg.distilled else 1)
        self.prefix = 2 if cfg.distilled else 1
        self.last_batch = 0
        self._seed_ready = False     # the workspace seed is the similarity gradient of the current forward's embeddings

    def workspace_bytes(self, batch):
        return self._workspace_bytes(batch)

    def _workspace(self, batch):
        return self._shaped_workspace(batch)

    def max_chunk(self, limit=None, reserve_bytes=4 << 30):
        """Largest per-call batch whose workspace fits in free HBM (activations of all blocks are kept)."""
        return self._max_batch(limit, reserve_bytes)

    # ---- the three calls ------------------------------------------------------------------------
    @_on_engine_device
    def forward(self, images, flags=None):
        """``model(x)``: logits [B,C]; leaves the activations in the workspace."""
        images = images.to(self.device, torch.float32).contiguous()
        b = images.shape[0]
        ws = self._workspace(b)
        fl = self.flags if flags is None else flags
        logits = torch.empty(b, self.cfg.num_classes, dtype=torch.float32, device=self.device)
        check(self.lib.te_vit_forward(ctypes.byref(self.cfg), ptr(self.weights), ptr(self._derived(fl)), ptr(images), b,
                                      fl, ptr(logits), ptr(ws), ws.numel() * 4, self._stream()), "te_vit_forward")
        self.last_batch = b
        self._last_images = images
        self._seed_ready = False
        return logits

    @_on_engine_device
    def relprop_pixels(self, index=None, per_channel=False, flags=None, alpha=1.0):
        """``method="full"`` (ViT_LRP.py:337-343) on the activations of the last ``forward``: the relprop is run to
        the encoder input, through ``self.add`` and the patch convolution's z^B rule.  Returns the relevance of every
        pixel, [B,H,W] (channels summed, what the reference returns) or [B,C,H,W] with ``per_channel``.
        alpha: as for ``attribute`` (the z^B rule of the patch convolution does not depend on it)."""
        fl = (self.flags if flags is None else flags) | _lib.FLAG_RELPROP_TO_INPUT
        self.attribute(index=index, start_layer=0, flags=fl, alpha=alpha)
        b = self.last_batch
        images = getattr(self, "_last_images", None)
        if images is None or images.shape[0] != b:
            raise RuntimeError("relprop_pixels() needs the images of the preceding forward()")
        ws = self._workspace(b)
        c, s = self.cfg.in_chans, self.cfg.img_size
        out = torch.empty((b, c, s, s) if per_channel else (b, s, s), dtype=torch.float32, device=self.device)
        check(self.lib.te_vit_relprop_pixels(ctypes.byref(self.cfg), ptr(self.weights), ptr(images), b, fl,
                                             None if per_channel else ptr(out), ptr(out) if per_channel else None,
                                             ptr(ws), ws.numel() * 4, self._stream()), "te_vit_relprop_pixels")
        return out

    @_on_engine_device
    def similarity(self, text_features, logit_scale):
        """CLIP's ``logits_per_image`` of each image of the last ``forward`` with its own text embedding: the engine's "logits"
        are then the projected image embeddings (num_classes = the embedding width).  text_features [B, E] (one row per
        image; one row [E] is used for every image), logit_scale = exp(the model's logit_scale).  Returns the similarities
        [B] and leaves their gradient in the workspace as the seed of ``attribute(similarity_seeded=True)``."""
        b = self.last_batch
        if b <= 0:
            raise RuntimeError("similarity() needs a preceding forward()")
        t = torch.as_tensor(text_features).to(self.device, torch.float32)
        if t.dim() == 1:
            t = t.unsqueeze(0)
        if t.shape[-1] != self.cfg.num_classes or t.shape[0] not in (1, b):
            raise ValueError("text_features must be [%d, %d] or [%d], got %s" % (b, self.cfg.num_classes, self.cfg.num_classes,
                                                                               tuple(t.shape)))
        t = t.expand(b, -1).contiguous()
        ws = self._workspace(b)
        sim = torch.empty(b, dtype=torch.float32, device=self.device)
        check(self.lib.te_vit_similarity_seed(ctypes.byref(self.cfg), b, ptr(t), float(logit_scale), ptr(sim), ptr(ws),
                                              ws.numel() * 4, self._stream()), "te_vit_similarity_seed")
        self._seed_ready = True
        return sim

    @_on_engine_device
    def attribute(self, index=None, start_layer=0, flags=None, alpha=1.0, similarity_seeded=False):
        """Backward + relprop + rollout on the activations of the last ``forward``.
        Returns (maps [B,N-prefix], index [B] int32).  alpha: ``model.relprop(..., alpha=alpha)``, the LRP-alpha-beta rule
        (beta = alpha - 1) in every Linear.relprop; 1 is the z+ rule every generator uses.
        similarity_seeded: the gradient-weighted attention rollout (FLAG_ATTN_GRAD_ROLLOUT) of the image-text similarity
        of the last ``similarity`` call (FLAG_SIMILARITY_SEED); index is not used and comes back as given (-1: none).  The
        seed must belong to the current forward: a seeded call after another ``forward`` / ``explain`` or after a class
        ``attribute`` (which overwrites the seed with a one-hot) without a new ``similarity`` raises RuntimeError."""
        if similarity_seeded:
            flags = (self.flags if flags is None else flags) | _lib.FLAG_SIMILARITY_SEED | _lib.FLAG_ATTN_GRAD_ROLLOUT
        b = self.last_batch
        if b <= 0:
            raise RuntimeError("attribute() needs a preceding forward()")
        seeded = bool((self.flags if flags is None else flags) & _lib.FLAG_SIMILARITY_SEED)
        if seeded and not self._seed_ready:
            raise RuntimeError("a similarity-seeded attribute() needs similarity() after the last forward() and class "
                               "attribute()")
        ws = self._workspace(b)
        idx = self._index_tensor(index, b)
        maps = torch.empty(b, self.tokens - self.prefix, dtype=torch.float32, device=self.device)
        fl = self.flags if flags is None else flags
        check(self.lib.te_vit_attribute(ctypes.byref(self.cfg), ptr(self.weights), ptr(self._derived(fl)), b, ptr(idx),
                                        int(start_layer), float(alpha), fl, ptr(maps), ptr(ws), ws.numel() * 4, self._stream()),
              "te_vit_attribute")
        self._seed_ready = seeded                # a class attribute() wrote its one-hot over the seed
        return maps, idx

    @_on_engine_device
    def explain(self, images, index=None, start_layer=0, flags=None, chunk=None, return_logits=False):
        """``LRP.generate_LRP`` for a batch of independent inputs (device-resident in, device-resident out)."""
        images = images.to(self.device, torch.float32).contiguous()
        B = images.shape[0]
        chunk = min(B, chunk or self.max_chunk(limit=B))
        maps = torch.empty(B, self.tokens - self.prefix, dtype=torch.float32, device=self.device)
        idx_all = self._index_tensor(index, B)
        logits = torch.empty(B, self.cfg.num_classes, dtype=torch.float32, device=self.device) if return_logits else None
        fl = self.flags if flags is None else flags
        derived = self._derived(fl)
        for s in range(0, B, chunk):
            e = min(B, s + chunk)
            ws = self._workspace(chunk if e - s == chunk else e - s)
            check(self.lib.te_vit_explain(ctypes.byref(self.cfg), ptr(self.weights), ptr(derived), ptr(images[s:e]), e - s,
                                          ptr(idx_all[s:e]), int(start_layer), fl, ptr(maps[s:e]),
                                          ptr(logits[s:e]) if logits is not None else None, ptr(ws), ws.numel() * 4,
                                          self._stream()), "te_vit_explain")
            self.last_batch = e - s
            self._last_images = images[s:e]
            self._seed_ready = False
        if return_logits:
            return maps, idx_all, logits
        return maps, idx_all

    # ---- CUDA-graph replay of the fixed-shape step ------------------------------------------------
    @_on_engine_device
    def explain_graphed(self, images, index=None, start_layer=0, flags=None, return_logits=False):
        """``explain`` with the whole step (~40 launches per block) captured once in a CUDA graph and replayed: the
        shapes, the workspace and every kernel argument are fixed for a given (batch, start_layer, flags), so small
        per-GPU batches (a fixed global batch sharded over 8 GPUs, SURVEY.md 8e) are not bound by launch gaps.
        Inputs are copied into static buffers; outputs are views of static buffers (overwritten by the next call)."""
        images = images.to(self.device, torch.float32)
        B = images.shape[0]
        fl = self.flags if flags is None else flags
        key = (B, int(start_layer), int(fl), tuple(images.shape[1:]))
        g = getattr(self, "_graphs", None)
        if g is None:
            g = self._graphs = {}
        if key not in g:
            if len(g) >= 4:
                g.clear()                                   # bounded cache: graphs pin their static buffers
            ws = self._workspace(B)
            derived = self._derived(fl)
            st = dict(images=torch.empty_like(images, memory_format=torch.contiguous_format),
                      idx_in=torch.full((B,), -1, dtype=torch.int32, device=self.device),
                      idx=torch.full((B,), -1, dtype=torch.int32, device=self.device),
                      maps=torch.empty(B, self.tokens - self.prefix, dtype=torch.float32, device=self.device),
                      logits=torch.empty(B, self.cfg.num_classes, dtype=torch.float32, device=self.device), ws=ws,
                      derived=derived)
            st["images"].copy_(images)

            def run():
                st["idx"].copy_(st["idx_in"])
                check(self.lib.te_vit_explain(ctypes.byref(self.cfg), ptr(self.weights), ptr(derived), ptr(st["images"]), B,
                                              ptr(st["idx"]), int(start_layer), fl, ptr(st["maps"]), ptr(st["logits"]),
                                              ptr(ws), ws.numel() * 4, self._stream()), "te_vit_explain")

            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                run()                                       # warm-up outside capture: per-device kernel attributes, allocator
            torch.cuda.current_stream(self.device).wait_stream(side)
            torch.cuda.synchronize(self.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                run()
            st["graph"] = graph
            g[key] = st
        st = g[key]
        # every pointer the graph captured besides its own buffers: the weights and the derived copies are rewritten in
        # place by a weight load, but the workspace is re-allocated for another batch size and the derived copies may
        # have been dropped (e.g. to free memory)
        if st["ws"] is not self._ws or st["derived"] is not self._derived(fl):
            del g[key]
            return self.explain_graphed(images, index=index, start_layer=start_layer, flags=flags,
                                        return_logits=return_logits)
        st["images"].copy_(images, non_blocking=True)
        st["idx_in"].copy_(self._index_tensor(index, B))
        st["graph"].replay()
        self.last_batch = B
        self._last_images = st["images"]
        self._seed_ready = False
        if return_logits:
            return st["maps"], st["idx"], st["logits"]
        return st["maps"], st["idx"]

    # ---- accessors (get_attn / get_attn_gradients / get_attn_cam ..., ViT_LRP.py:102-130) ---------
    def tensor(self, name, layer=0):
        return self._view(name, layer, self.last_batch)


def bert_config(vocab_size=30522, max_position_embeddings=512, type_vocab_size=2, hidden_size=768,
                num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, num_labels=2,
                layer_norm_eps=1e-12, arch=0, pad_token_id=0):
    """``te_bert_config``.  arch: ``_lib.BERT_ARCH_BERT`` / ``_ROBERTA`` / ``_DISTILBERT`` (type_vocab_size 0);
    pad_token_id: the id RoBERTa's position ids count from."""
    from ._lib import TeBertConfig
    return TeBertConfig(vocab_size, max_position_embeddings, type_vocab_size, hidden_size, num_hidden_layers,
                        num_attention_heads, intermediate_size, num_labels, layer_norm_eps, arch, pad_token_id)


class BertEngine(_Engine):
    """``Generator.generate_LRP`` (BERT_explainability/modules/BERT/ExplanationGenerator.py:28-59) for batches of
    independent sequences of one length."""
    _prefix = "te_bert_"

    def __init__(self, cfg, state_dict=None, device=None, flags=0):
        super().__init__(cfg, state_dict, device, flags)
        self.last = (0, 0)

    def workspace_bytes(self, batch, seq):
        return self._workspace_bytes(batch, seq)

    def _workspace(self, batch, seq):
        return self._shaped_workspace(batch, seq)

    def max_chunk(self, seq, limit=None, reserve_bytes=4 << 30):
        return self._max_batch(limit, reserve_bytes, seq)

    def _ids(self, input_ids, attention_mask, token_type_ids=None):
        if not input_ids.is_cuda and input_ids.numel() and (int(input_ids.min()) < 0 or
                                                            int(input_ids.max()) >= self.cfg.vocab_size):
            raise ValueError("input_ids outside [0, vocab_size)")     # device-resident ids: the kernel writes NaN rows
        ids = input_ids.to(self.device, torch.int64).contiguous()
        if attention_mask is None:
            attention_mask = torch.ones_like(ids)
        return ids, attention_mask.to(self.device, torch.int64).contiguous(), self._token_types(token_type_ids, ids.shape)

    def _token_types(self, token_type_ids, shape):
        """The segment of every token (BertEmbeddings' token_type_ids), int64 on the device; None: every token in segment 0
        (the kernel reads no table row but row 0)."""
        if token_type_ids is None:
            return None
        if self.cfg.arch == _lib.BERT_ARCH_DISTILBERT:
            raise ValueError("DistilBERT takes no token_type_ids: it has no token-type table")
        tt = torch.as_tensor(token_type_ids)
        if tuple(tt.shape) != tuple(shape):
            raise ValueError("token_type_ids must have the shape of input_ids %s, got %s" % (tuple(shape), tuple(tt.shape)))
        if not tt.is_cuda and tt.numel() and (int(tt.min()) < 0 or int(tt.max()) >= self.cfg.type_vocab):
            raise ValueError("token_type_ids outside [0, type_vocab_size)")   # device-resident: the kernel writes NaN rows
        return tt.to(self.device, torch.int64).contiguous()

    @_on_engine_device
    def forward(self, input_ids, attention_mask=None, flags=None, token_type_ids=None):
        """``model(input_ids, attention_mask, token_type_ids)``: logits [B,C]; leaves the activations in the workspace.
        token_type_ids: the segment of every token, the shape of input_ids; None puts every token in segment 0."""
        ids, mask, tt = self._ids(input_ids, attention_mask, token_type_ids)
        b, s = ids.shape
        ws = self._workspace(b, s)
        fl = self.flags if flags is None else flags
        logits = torch.empty(b, self.cfg.num_labels, dtype=torch.float32, device=self.device)
        check(self.lib.te_bert_forward(ctypes.byref(self.cfg), ptr(self.weights), ptr(self._derived(fl)), ptr(ids),
                                       ptr(mask), ptr(tt), b, s, fl, ptr(logits), ptr(ws), ws.numel() * 4, self._stream()),
              "te_bert_forward")
        self.last = (b, s)
        return logits

    @_on_engine_device
    def attribute(self, index=None, start_layer=11, flags=None, alpha=1.0):
        """Backward + relprop + normalised rollout on the activations of the last ``forward``; alpha as for
        ``ViTEngine.attribute``.  Returns (maps [B,S], index [B] int32)."""
        b, s = self.last
        if b <= 0:
            raise RuntimeError("attribute() needs a preceding forward()")
        ws = self._workspace(b, s)
        idx = self._index_tensor(index, b)
        maps = torch.empty(b, s, dtype=torch.float32, device=self.device)
        fl = self.flags if flags is None else flags
        check(self.lib.te_bert_attribute(ctypes.byref(self.cfg), ptr(self.weights), ptr(self._derived(fl)), b, s, ptr(idx),
                                         int(start_layer), float(alpha), fl, ptr(maps), ptr(ws), ws.numel() * 4,
                                         self._stream()), "te_bert_attribute")
        return maps, idx

    @_on_engine_device
    def explain(self, input_ids, attention_mask=None, index=None, start_layer=11, flags=None, chunk=None,
                return_logits=False, token_type_ids=None):
        """``Generator.generate_LRP`` of B independent sequences of one length: (maps [B,S], index [B] int32) and, with
        ``return_logits``, the logits [B,C].  token_type_ids as for ``forward``."""
        ids, mask, tt = self._ids(input_ids, attention_mask, token_type_ids)
        B, S = ids.shape
        chunk = min(B, chunk or self.max_chunk(S, limit=B))
        maps = torch.empty(B, S, dtype=torch.float32, device=self.device)
        idx_all = self._index_tensor(index, B)
        logits = torch.empty(B, self.cfg.num_labels, dtype=torch.float32, device=self.device) if return_logits else None
        fl = self.flags if flags is None else flags
        derived = self._derived(fl)
        for s0 in range(0, B, chunk):
            e = min(B, s0 + chunk)
            ws = self._workspace(e - s0, S)
            check(self.lib.te_bert_explain(ctypes.byref(self.cfg), ptr(self.weights), ptr(derived), ptr(ids[s0:e]),
                                           ptr(mask[s0:e]), ptr(tt[s0:e]) if tt is not None else None, e - s0, S,
                                           ptr(idx_all[s0:e]), int(start_layer), fl,
                                           ptr(maps[s0:e]), ptr(logits[s0:e]) if logits is not None else None, ptr(ws),
                                           ws.numel() * 4, self._stream()), "te_bert_explain")
            self.last = (e - s0, S)
        if return_logits:
            return maps, idx_all, logits
        return maps, idx_all

    def tensor(self, name, layer=0):
        return self._view(name, layer, *self.last)
