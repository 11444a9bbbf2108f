"""Batched driver + on-disk format of ``baselines/ViT/generate_visualizations.py:27-102`` (SURVEY.md 8f-2).

The reference loops over a loader, explains each batch with one of its methods, up-samples the 14 x 14 token map x16
(bilinear), min-max normalises and appends to ``results.hdf5`` with three datasets that
``dataset/expl_hdf5.py:23-28`` later reads by index:

    vis     float32 [N, 1, 224, 224]      image   float32 [N, 3, 224, 224]      target  int32 [N]

``compute_saliency_and_save`` is that loop on the engine (batched explanations, the x16 up-sampling + per-sample
min-max in one kernel, ``visualization.relevance_to_heatmap``).  ``ResultsWriter`` produces the file: with ``h5py``
when it is importable (then exactly the reference's resizable gzip datasets), otherwise with the built-in minimal HDF5
emitter below — same dataset names, shapes and dtypes in the simplest valid container (superblock version 0, version-1
object headers, one symbol-table group, CONTIGUOUS little-endian datasets; HDF5 File Format Specification v3, sections
II.A, III.A-D, IV.A.1-2).  ``h5py.File(path)['vis'][i]`` does not depend on the storage layout, so the consumer is
unchanged.  This image ships no HDF5 library at all: the emitter is checked against the specification by the independent
reader ``read_minimal_hdf5`` (``tests/test_hdf5_writer.py``), not against libhdf5 — stated here, in DESIGN.md and in the
test.

The command is the reference script itself: it explains every image of an ImageNet validation folder and writes
``visualizations/{method}/{vis_class}/{ablation}/results.hdf5`` (``visualizations/{method}/index_{class_id}`` for
``--vis-class index``), the directory ``python -m transformer_explainability_b200.perturbation`` reads.

    python -m transformer_explainability_b200.hdf5_writer --method transformer_attribution \\
        --imagenet-validation-path /data/imagenet --state-dict vit_base_patch16_224.pth --batch-size 32

The images are decoded on the host by PIL (the bits torchvision's ``pil_loader`` gives the reference), packed per batch
into one pinned buffer, and resized and scaled to [0, 1] on the GPU by ``ops.prepare_images``, bit for bit
``Resize((224, 224)) + ToTensor()`` of the reference.  Deviations from the script (DESIGN.md §1): ``--method`` is required
(the reference's default is not among its choices); an existing ``results.hdf5`` in the target directory is replaced;
``--vis-class index`` explains the top class, as the reference does; every sample is min-max normalised on its own.
"""
import argparse
import os
import struct
import tempfile

import numpy as np

UNDEF = 0xFFFFFFFFFFFFFFFF
_SIG = b"\x89HDF\r\n\x1a\n"


def _pad8(b):
    return b + b"\0" * (-len(b) % 8)


def _msg(mtype, data, flags=0):
    data = _pad8(data)
    return struct.pack("<HHB3x", mtype, len(data), flags) + data


def _object_header(messages):
    body = b"".join(messages)
    # version 1 prefix: version, reserved, #messages, reference count, header size, 4 bytes of padding (8-byte alignment)
    return struct.pack("<BBHII4x", 1, 0, len(messages), 1, len(body)) + body


def _dataspace(shape):
    return _msg(0x0001, struct.pack("<BBB5x", 1, len(shape), 0) + b"".join(struct.pack("<Q", int(d)) for d in shape))


def _datatype(dtype):
    dtype = np.dtype(dtype)
    if dtype == np.float32:
        # class 1 (floating point) version 1; little-endian, implied-msb mantissa normalisation, sign bit 31;
        # properties: bit offset 0, precision 32, exponent at 23 (8 bits), mantissa at 0 (23 bits), bias 127
        return _msg(0x0003, struct.pack("<BBBBI", 0x11, 0x20, 31, 0, 4) + struct.pack("<HHBBBBI", 0, 32, 23, 8, 0, 23, 127), 1)
    if dtype == np.int32:
        # class 0 (fixed point) version 1; little-endian, two's complement signed; bit offset 0, precision 32
        return _msg(0x0003, struct.pack("<BBBBI", 0x10, 0x08, 0, 0, 4) + struct.pack("<HH", 0, 32), 1)
    raise TypeError("minimal HDF5 emitter: float32 / int32 only")


def _dataset_header(shape, dtype, address, nbytes):
    fill = _msg(0x0005, struct.pack("<BBBB", 2, 2, 2, 0))                       # v2: late allocation, write-if-set, undefined
    layout = _msg(0x0008, struct.pack("<BBQQ", 3, 1, address, nbytes))         # v3, class 1 = contiguous
    return _object_header([_dataspace(shape), _datatype(dtype), fill, layout])


def write_minimal_hdf5(path, datasets):
    """datasets: ordered mapping name -> (shape, dtype, source) where source is an ndarray or a path of a raw
    little-endian file holding exactly prod(shape) elements.  Writes one root group with contiguous datasets."""
    names = sorted(datasets)                                                    # symbol-table entries are sorted by name
    if not 0 < len(names) <= 8:
        raise ValueError("minimal HDF5 emitter: 1..8 datasets (one symbol-table node)")
    # ---- local heap data segment: the empty string at offset 0, then the link names
    heap = bytearray(b"\0" * 8)
    name_off = {}
    for n in names:
        name_off[n] = len(heap)
        heap += _pad8(n.encode("ascii") + b"\0")
    heap_data = bytes(heap)
    # ---- layout of the file
    off = 96                                                                    # superblock (version 0, 8-byte offsets)
    root_hdr_addr = off
    root_hdr = _object_header([_msg(0x0011, struct.pack("<QQ", 0, 0))])         # patched below (needs addresses)
    off += len(root_hdr)
    btree_addr = off
    off += 24 + (2 * 16 + 1) * 8 + 2 * 16 * 8                                   # group B-tree node, internal K = 16
    heap_addr = off
    off += 32
    heap_data_addr = off
    off += len(heap_data)
    snod_addr = off
    off += 8 + 8 * 40                                                           # symbol-table node, leaf K = 4
    hdr_addr, hdr_len = {}, {}
    for n in names:
        shape, dtype, _ = datasets[n]
        hdr_addr[n] = off
        hdr_len[n] = len(_dataset_header(shape, dtype, 0, 0))
        off += hdr_len[n]
    data_addr = {}
    for n in names:
        shape, dtype, _ = datasets[n]
        off = (off + 7) & ~7
        data_addr[n] = off
        off += int(np.prod(shape, dtype=np.int64)) * np.dtype(dtype).itemsize
    eof = off
    with open(path, "wb") as f:
        # superblock v0 + root symbol-table entry (cache type 1: B-tree and heap addresses in the scratch pad)
        f.write(_SIG + struct.pack("<BBBBBBBBHHI", 0, 0, 0, 0, 0, 8, 8, 0, 4, 16, 0))
        f.write(struct.pack("<QQQQ", 0, UNDEF, eof, UNDEF))
        f.write(struct.pack("<QQII", 0, root_hdr_addr, 1, 0) + struct.pack("<QQ", btree_addr, heap_addr))
        assert f.tell() == 96
        f.write(_object_header([_msg(0x0011, struct.pack("<QQ", btree_addr, heap_addr))]))
        # B-tree: one leaf-level node (type 0 = group, level 0), one child: key0 = "" (heap offset 0), child, key1 = last name
        node = b"TREE" + struct.pack("<BBHQQ", 0, 0, 1, UNDEF, UNDEF) + struct.pack("<QQQ", 0, snod_addr, name_off[names[-1]])
        f.write(node)
        f.write(b"\0" * (heap_addr - f.tell()))                                  # unused key / child slots of the node
        f.write(b"HEAP" + struct.pack("<B3xQQQ", 0, len(heap_data), 1, heap_data_addr))      # free-list head 1 = none
        f.write(heap_data)
        snod = b"SNOD" + struct.pack("<BBH", 1, 0, len(names))
        for n in names:
            snod += struct.pack("<QQII16x", name_off[n], hdr_addr[n], 0, 0)
        f.write(snod + b"\0" * (8 + 8 * 40 - len(snod)))
        for n in names:
            shape, dtype, _ = datasets[n]
            nbytes = int(np.prod(shape, dtype=np.int64)) * np.dtype(dtype).itemsize
            h = _dataset_header(shape, dtype, data_addr[n], nbytes)
            assert f.tell() == hdr_addr[n] and len(h) == hdr_len[n]
            f.write(h)
        for n in names:
            shape, dtype, src = datasets[n]
            f.write(b"\0" * (data_addr[n] - f.tell()))
            if isinstance(src, str):
                with open(src, "rb") as r:
                    while True:
                        buf = r.read(1 << 24)
                        if not buf:
                            break
                        f.write(buf)
            else:
                f.write(np.ascontiguousarray(src, dtype=np.dtype(dtype).newbyteorder("<")).tobytes())
            want = int(np.prod(shape, dtype=np.int64)) * np.dtype(dtype).itemsize
            if f.tell() - data_addr[n] != want:
                raise ValueError("dataset %r: %d bytes written, %d expected" % (n, f.tell() - data_addr[n], want))
        assert f.tell() == eof


def read_minimal_hdf5(path):
    """Independent reader (test infrastructure for the emitter): walks superblock -> root symbol-table entry -> local
    heap + B-tree -> symbol-table node -> object headers -> contiguous data, following the specification field by field,
    and returns {name: ndarray}.  Handles exactly the subset ``write_minimal_hdf5`` emits."""
    with open(path, "rb") as f:
        raw = f.read()
    if raw[:8] != _SIG:
        raise ValueError("not an HDF5 file")
    ver, _, _, _, _, so, sl = struct.unpack_from("<BBBBBBB", raw, 8)
    if ver != 0 or so != 8 or sl != 8:
        raise ValueError("unsupported superblock")
    leaf_k, int_k = struct.unpack_from("<HH", raw, 16)
    base, _, eof, _ = struct.unpack_from("<QQQQ", raw, 24)
    if eof != len(raw) or base != 0:
        raise ValueError("bad end-of-file address")
    _, root_hdr, cache, _, btree, heap = struct.unpack_from("<QQIIQQ", raw, 56)
    # the root object header must carry the same symbol-table message
    v, _, nmsg, _, hsize = struct.unpack_from("<BBHII", raw, root_hdr)
    mt, ms = struct.unpack_from("<HH", raw, root_hdr + 16)
    if v != 1 or mt != 0x0011 or struct.unpack_from("<QQ", raw, root_hdr + 24) != (btree, heap):
        raise ValueError("root group header does not match the superblock entry")
    if raw[heap:heap + 4] != b"HEAP":
        raise ValueError("local heap signature")
    hsz, _, hdata = struct.unpack_from("<QQQ", raw, heap + 8)
    if raw[btree:btree + 4] != b"TREE":
        raise ValueError("B-tree signature")
    ntype, level, used = struct.unpack_from("<BBH", raw, btree + 4)
    if ntype != 0 or level != 0 or used != 1:
        raise ValueError("unexpected B-tree shape")
    snod = struct.unpack_from("<Q", raw, btree + 24 + 8)[0]
    if raw[snod:snod + 4] != b"SNOD":
        raise ValueError("symbol-table node signature")
    nsym = struct.unpack_from("<H", raw, snod + 6)[0]
    out = {}
    for i in range(nsym):
        noff, ohdr = struct.unpack_from("<QQ", raw, snod + 8 + 40 * i)
        end = raw.index(b"\0", hdata + noff)
        name = raw[hdata + noff:end].decode("ascii")
        v, _, nmsg, _, hsize = struct.unpack_from("<BBHII", raw, ohdr)
        pos, shape, dtype, addr, size = ohdr + 16, None, None, None, None
        for _ in range(nmsg):
            mt, ms = struct.unpack_from("<HH", raw, pos)
            d = pos + 8
            if mt == 0x0001:
                rank = raw[d + 1]
                shape = struct.unpack_from("<%dQ" % rank, raw, d + 8)
            elif mt == 0x0003:
                cls = raw[d] & 0x0F
                tsize = struct.unpack_from("<I", raw, d + 4)[0]
                dtype = np.dtype("<f4") if (cls == 1 and tsize == 4) else np.dtype("<i4") if (cls == 0 and tsize == 4) else None
            elif mt == 0x0008:
                lv, lc, addr, size = struct.unpack_from("<BBQQ", raw, d)
                if lv != 3 or lc != 1:
                    raise ValueError("layout")
            pos = d + ms
        n = int(np.prod(shape, dtype=np.int64))
        if dtype is None or size != n * dtype.itemsize:
            raise ValueError("dataset %r: inconsistent header" % name)
        out[name] = np.frombuffer(raw, dtype=dtype, count=n, offset=addr).reshape(shape).copy()
    return out


class ResultsWriter:
    """``results.hdf5`` of the reference: append batches of (image [B,3,H,W], vis [B,1,H,W], target [B]); datasets
    ``image`` / ``vis`` float32 and ``target`` int32 (``generate_visualizations.py:29-43``)."""

    def __init__(self, method_dir, size=224, backend=None):
        os.makedirs(method_dir, exist_ok=True)
        self.path = os.path.join(method_dir, "results.hdf5")
        self.size = size
        self.n = 0
        if backend is None:
            try:
                import h5py                                                     # noqa: F401
                backend = "h5py"
            except ImportError:
                backend = "builtin"
        self.backend = backend
        if backend == "h5py":
            import h5py
            self._f = h5py.File(self.path, "a")
            mk = lambda name, c, dt: self._f.create_dataset(name, (1,) + c, maxshape=(None,) + c, dtype=dt,       # noqa: E731
                                                            compression="gzip")
            self._d = {"vis": mk("vis", (1, size, size), np.float32), "image": mk("image", (3, size, size), np.float32),
                       "target": mk("target", (), np.int32)}
        else:
            self._tmp = {k: tempfile.NamedTemporaryFile(prefix="te_h5_%s_" % k, dir=method_dir, delete=False)
                         for k in ("vis", "image", "target")}

    def append(self, image, vis, target):
        image = np.ascontiguousarray(np.asarray(image, dtype=np.float32))
        vis = np.ascontiguousarray(np.asarray(vis, dtype=np.float32))
        target = np.ascontiguousarray(np.asarray(target, dtype=np.int32)).reshape(-1)
        b = image.shape[0]
        if image.shape != (b, 3, self.size, self.size) or vis.shape != (b, 1, self.size, self.size) or target.shape != (b,):
            raise ValueError("append: image [B,3,S,S], vis [B,1,S,S], target [B] expected")
        if self.backend == "h5py":
            for k, v in (("vis", vis), ("image", image), ("target", target)):
                self._d[k].resize(self.n + b, axis=0)
                self._d[k][self.n:self.n + b] = v
        else:
            self._tmp["vis"].write(vis.astype("<f4").tobytes())
            self._tmp["image"].write(image.astype("<f4").tobytes())
            self._tmp["target"].write(target.astype("<i4").tobytes())
        self.n += b

    def close(self):
        if self.backend == "h5py":
            self._f.close()
            return self.path
        for t in self._tmp.values():
            t.close()
        s = self.size
        try:
            write_minimal_hdf5(self.path, {"vis": ((self.n, 1, s, s), np.float32, self._tmp["vis"].name),
                                           "image": ((self.n, 3, s, s), np.float32, self._tmp["image"].name),
                                           "target": ((self.n,), np.int32, self._tmp["target"].name)})
        finally:
            for t in self._tmp.values():
                os.unlink(t.name)
        return self.path

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def normalize(tensor, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    """``generate_visualizations.py:18-24`` (out of place)."""
    import torch
    m = torch.as_tensor(mean, dtype=tensor.dtype, device=tensor.device)[None, :, None, None]
    s = torch.as_tensor(std, dtype=tensor.dtype, device=tensor.device)[None, :, None, None]
    return (tensor - m) / s


def compute_saliency_and_save(loader, method_dir, method, lrp=None, baselines=None, orig_lrp=None, vis_class="top",
                              is_ablation=False, device="cuda", backend=None):
    """The loop of ``compute_saliency_and_save`` (``generate_visualizations.py:27-102``) with batched engine calls.
    ``loader`` yields (images [B,3,224,224] in [0,1], targets [B]); ``lrp`` / ``baselines`` / ``orig_lrp`` are the
    generators of ``baselines/ViT/ViT_explanation_generator.py`` (here: this package's).  Every sample is normalised by
    its own min / max (the reference's ``Res.min()`` runs over the batch, which only equals this at its default
    batch size 1)."""
    import torch
    from . import visualization
    from ._host import to_host
    with ResultsWriter(method_dir, backend=backend) as out:
        for data, target in loader:
            x = normalize(data.to(device, torch.float32))
            index = target.to(device) if vis_class == "target" else None
            b = x.shape[0]
            if method == "rollout":
                res = baselines.generate_rollout(x, start_layer=1)
            elif method == "lrp":
                res = lrp.generate_LRP_batched(x, start_layer=1, index=index)
            elif method == "transformer_attribution":
                res = lrp.generate_LRP_batched(x, start_layer=1, index=index)       # method="grad" is the legacy alias
            elif method == "attn_grad_rollout":
                res = lrp.generate_attn_grad_rollout(x, index=index)
            elif method == "full_lrp":
                res = (orig_lrp or lrp).generate_LRP(x, method="full", index=index)
            elif method == "lrp_last_layer":
                res = (orig_lrp or lrp).generate_LRP(x, method="last_layer", is_ablation=is_ablation, index=index)
            elif method == "attn_last_layer":
                res = lrp.generate_LRP(x, method="last_layer_attn", is_ablation=is_ablation)
            elif method == "attn_gradcam":
                res = baselines.generate_cam_attn(x, index=index)
            else:
                raise ValueError("unknown method %r" % (method,))
            if method == "full_lrp":
                r = res.reshape(b, -1).float()
                lo, hi = r.amin(dim=1, keepdim=True), r.amax(dim=1, keepdim=True)
                vis = ((r - lo) / (hi - lo)).reshape(b, 1, data.shape[-2], data.shape[-1])
            else:
                vis = visualization.relevance_to_heatmap(res.reshape(b, -1).float().contiguous()).reshape(
                    b, 1, data.shape[-2], data.shape[-1])
            out.append(*to_host(data, vis, target))
    return out.path


# ---- command line: generate_visualizations.py ----------------------------------------------------------------------------
METHODS = ("rollout", "lrp", "transformer_attribution", "full_lrp", "lrp_last_layer", "attn_last_layer", "attn_gradcam")
# the façade model whose generator each method uses in generate_visualizations.py:180-192; only that one is built
MODEL_KIND = {"rollout": "new", "attn_gradcam": "new", "lrp": "lrp", "transformer_attribution": "lrp",
              "attn_last_layer": "lrp", "full_lrp": "orig", "lrp_last_layer": "orig"}
# one more choice besides the script's METHODS: the LRP-free gradient-weighted attention rollout of the authors' follow-up
# paper (Chefer, Gur, Wolf, ICCV 2021) on the ViT_LRP model, written to visualizations/attn_grad_rollout/...
FOLLOW_UP_KIND = {"attn_grad_rollout": "lrp"}
CHOICES = METHODS + tuple(FOLLOW_UP_KIND)


def read_rgb(path):
    """torchvision's ``pil_loader`` (``Image.open(f).convert("RGB")``), returning the decoded HWC uint8 array."""
    from PIL import Image
    with open(path, "rb") as f:
        return np.array(Image.open(f).convert("RGB"))


def pack_images(batch):
    """Collate of (HWC uint8 RGB array, target) samples -> (packed uint8 [sum of 3 h w], sizes int32 [B, 2] = (h, w),
    offsets int64 [B], targets int64 [B]): the images one after another in batch order, ``ops.prepare_images``' input."""
    import torch
    arrays = [np.ascontiguousarray(a, dtype=np.uint8) for a, _ in batch]
    for a in arrays:
        if a.ndim != 3 or a.shape[2] != 3:
            raise ValueError("pack_images: HWC RGB images expected, got shape %s" % (a.shape,))
    sizes = np.array([a.shape[:2] for a in arrays], dtype=np.int32).reshape(-1, 2)
    offsets = np.concatenate([[0], np.cumsum([a.size for a in arrays])[:-1]]).astype(np.int64)
    packed = torch.from_numpy(np.concatenate([a.reshape(-1) for a in arrays]))
    targets = torch.tensor([int(t) for _, t in batch], dtype=torch.int64)
    return packed, torch.from_numpy(sizes), torch.from_numpy(offsets), targets


def imagenet_val_loader(path, batch_size, num_workers=4):
    """The reference's ``ImageNet(path, split='val')`` in its sample order, decoded by ``read_rgb`` in ``num_workers``
    processes and packed by ``pack_images`` into pinned host buffers."""
    import torch
    from torchvision.datasets import ImageNet
    ds = ImageNet(path, split="val", loader=read_rgb)
    return torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=False, num_workers=num_workers,
                                       collate_fn=pack_images, pin_memory=torch.cuda.is_available())


def prepared_batches(loader, device="cuda", size=224):
    """(images [B, 3, size, size] fp32 in [0, 1] on ``device``, targets [B]) per packed batch of ``loader``: the copy of
    the pinned batch does not block the host, and ``ops.prepare_images`` resizes it on the device."""
    from . import ops
    for packed, sizes, offsets, target in loader:
        out01, _ = ops.prepare_images(packed.to(device, non_blocking=True), sizes.numpy(), offsets.numpy(), (size, size))
        yield out01, target


def build_parser():
    from .perturbation import str2bool
    p = argparse.ArgumentParser(description="Explain an ImageNet validation folder into results.hdf5")
    p.add_argument("--batch-size", type=int, default=1)
    p.add_argument("--method", type=str, required=True, choices=CHOICES)
    p.add_argument("--lmd", type=float, default=10, help="accepted for compatibility; unused, as in the reference")
    p.add_argument("--vis-class", type=str, default="top", choices=["top", "target", "index"])
    p.add_argument("--class-id", type=int, default=0, help="names the output directory of --vis-class index")
    for flag in ("--cls-agn", "--no-ia", "--no-fx", "--no-fgx", "--no-m", "--no-reg"):
        p.add_argument(flag, action="store_true", default=False, help="accepted for compatibility; unused")
    p.add_argument("--is-ablation", type=str2bool, default=False)
    p.add_argument("--imagenet-validation-path", type=str, required=True,
                   help="directory holding meta.bin and val/{wnid}/*.JPEG (torchvision's ImageNet layout)")
    p.add_argument("--state-dict", type=str, default=None,
                   help="ViT-B/16 weights (timm key names); pretrained weights are not downloaded")
    p.add_argument("--root", type=str, default=None,
                   help="directory holding visualizations/ (default: the current directory)")
    p.add_argument("--num-workers", type=int, default=4, help="decoding processes")
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    if args.num_workers < 0:
        p.error("--num-workers must not be negative")
    return args


def main(argv=None):
    args = parse_args(argv)
    from . import perturbation, segmentation
    method_dir = perturbation.vis_method_dir(args, args.root or os.getcwd())
    os.makedirs(method_dir, exist_ok=True)
    if os.path.exists(os.path.join(method_dir, "results.hdf5")):
        os.remove(os.path.join(method_dir, "results.hdf5"))
    kind = {**MODEL_KIND, **FOLLOW_UP_KIND}[args.method]
    lrp, orig_lrp, baselines = segmentation.build_generators(args.method, args.state_dict, kind=kind)
    loader = imagenet_val_loader(args.imagenet_validation_path, args.batch_size, args.num_workers)
    path = compute_saliency_and_save(prepared_batches(loader), method_dir, args.method, lrp=lrp, baselines=baselines,
                                     orig_lrp=orig_lrp, vis_class=args.vis_class, is_ablation=args.is_ablation)
    print(path)
    return path


if __name__ == "__main__":
    main()
