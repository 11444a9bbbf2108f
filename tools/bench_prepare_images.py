"""Input preparation of the generate_visualizations command: ``te_prepare_images`` against torchvision's CPU transform.

    python tools/bench_prepare_images.py [--batch 32] [--iters 200] [--images 160] [--methods all]

Reports one JSON line:
* ``kernel``: ``ops.prepare_images`` on a packed batch already on the device (CUDA events over ``--iters`` calls, host
  work of each call included): images/s, and the bytes the two passes move (input read, uint8 intermediate written and
  read, fp32 output written) over the time, as a share of the H100 SXM's 3.35 TB/s;
* ``kernel_h2d``: the same with the non-blocking copy of the pinned packed batch in each call;
* ``cpu_per_core``: torchvision ``Resize((224, 224)) + ToTensor()`` on the decoded PIL images, one host thread, host clock;
* ``command``: the command's pipeline (``imagenet_val_loader`` -> ``prepared_batches`` -> ``compute_saliency_and_save``)
  per method on a synthetic JPEG tree written here, with random-init ViT-B weights: images/s after the first batch and the
  share of that time the main loop waits for the loader;
* ``gpu`` / ``power_limit_w``: the card, read in the same run.
Every timed batch of the kernel runs is compared bit for bit with the CPU transform; a difference aborts the run.

Images: synthetic uint8 at ImageNet-val sizes (500 x 375, 375 x 500, 500 x 333, 333 x 500, 500 x 500) and a few over
1000 px, the mix of the validation set's common shapes.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from transformer_explainability_b200 import _lib, hdf5_writer, ops, segmentation   # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZES = [(375, 500), (500, 375), (333, 500), (500, 333), (500, 500)] * 5 + [(1024, 768), (1200, 1600), (1365, 1024)]


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def synthetic_batches(n_batches, batch, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for b in range(n_batches):
        sizes = [SIZES[(b * batch + i) % len(SIZES)] for i in range(batch)]
        out.append([rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes])
    return out


def moved_bytes(arrays, oh=224, ow=224):
    """Bytes the two passes read and write: input, uint8 intermediate (written once, read once), fp32 output."""
    n = 0
    for a in arrays:
        h, w = a.shape[:2]
        mid = 3 * (oh * w if (h > 100 * w and oh < h) else h * ow)
        n += a.size + 2 * mid + 12 * oh * ow
    return n


def cpu_transform(arrays):
    import torchvision.transforms as T
    from PIL import Image
    t = T.Compose([T.Resize((224, 224)), T.ToTensor()])
    return torch.stack([t(Image.fromarray(a)) for a in arrays])


def bench_kernel(batches, refs, iters, h2d):
    packs = [hdf5_writer.pack_images([(a, 0) for a in arrs]) for arrs in batches]
    host = [(p.pin_memory(), s.numpy(), o.numpy()) for p, s, o, _ in packs]
    dev = [p.cuda() for p, _, _ in host]

    def call(i):
        p, s, o = host[i % len(host)]
        src = p.to("cuda", non_blocking=True) if h2d else dev[i % len(dev)]
        return ops.prepare_images(src, s, o)[0]
    for i in range(len(host)):                                    # warm-up, and the bit check of every batch
        if not torch.equal(call(i).cpu(), refs[i]):
            raise SystemExit("prepare_images differs from the CPU transform on batch %d" % i)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    outs = {}
    start.record()
    for i in range(iters):
        outs[i % len(host)] = call(i)
    end.record()
    torch.cuda.synchronize()
    for i, o in outs.items():
        if not torch.equal(o.cpu(), refs[i]):
            raise SystemExit("prepare_images differs from the CPU transform on timed batch %d" % i)
    s = start.elapsed_time(end) / 1e3
    imgs = sum(len(batches[i % len(batches)]) for i in range(iters))
    nbytes = sum(moved_bytes(batches[i % len(batches)]) for i in range(iters))
    res = {"images_per_s": imgs / s, "ms_per_batch": 1e3 * s / iters, "bytes_per_s": nbytes / s,
           "share_of_hbm_peak": nbytes / s / HBM_BYTES_PER_S}
    if h2d:
        res["h2d_bytes_per_s"] = sum(host[i % len(host)][0].numel() for i in range(iters)) / s
    return res


def bench_cpu(batches, reps=3):
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    from PIL import Image
    import torchvision.transforms as T
    t = T.Compose([T.Resize((224, 224)), T.ToTensor()])
    pil = [Image.fromarray(a) for arrs in batches for a in arrs]
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        for im in pil:
            t(im)
        best = min(best, time.perf_counter() - t0)
    torch.set_num_threads(threads)
    return {"images_per_s": len(pil) / best, "ms_per_image": 1e3 * best / len(pil)}


def write_tree(root, n, seed=1):
    from PIL import Image
    rng = np.random.default_rng(seed)
    wnids = ["n%08d" % (1440764 + i) for i in range(4)]
    torch.save(({w: ("class %d" % i,) for i, w in enumerate(wnids)}, []), os.path.join(root, "meta.bin"))
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        d = os.path.join(root, "val", wnids[i % 4])
        os.makedirs(d, exist_ok=True)
        y, x = np.mgrid[0:h, 0:w]
        a = np.stack([x * 255 // (w - 1), y * 255 // (h - 1), (x + y) * 127 // (h + w - 2)], -1)
        a = a + rng.integers(-30, 31, (h, w, 3))
        Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(os.path.join(d, "ILSVRC2012_val_%08d.JPEG" % (i + 1)),
                                                                  quality=90)


class TimedLoader:
    """Iterates a loader and adds the time spent waiting in ``next`` (from the second batch on) to ``wait``."""

    def __init__(self, loader):
        self.loader, self.wait, self.t_start, self.n_after_first = loader, 0.0, None, 0

    def __iter__(self):
        it = iter(self.loader)
        first = True
        while True:
            t0 = time.perf_counter()
            try:
                b = next(it)
            except StopIteration:
                return
            if first:
                first = False
            else:
                if self.t_start is None:
                    self.t_start = t0
                self.wait += time.perf_counter() - t0
                self.n_after_first += len(b[3])
            yield b


def bench_command(methods, n_images, batch, workers):
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224
    out = {}
    with tempfile.TemporaryDirectory(prefix="te_bench_prepare_") as tmp:
        tree = os.path.join(tmp, "imagenet")
        os.makedirs(tree)
        write_tree(tree, n_images)
        torch.manual_seed(0)
        sd = os.path.join(tmp, "vit_b.pth")
        torch.save({k: v.detach().clone() for k, v in vit_base_patch16_224().state_dict().items()}, sd)
        for method in methods:
            lrp, orig_lrp, baselines = segmentation.build_generators(method, sd, kind=hdf5_writer.MODEL_KIND[method])
            timed = TimedLoader(hdf5_writer.imagenet_val_loader(tree, batch, workers))
            hdf5_writer.compute_saliency_and_save(hdf5_writer.prepared_batches(timed), os.path.join(tmp, "vis", method),
                                                  method, lrp=lrp, baselines=baselines, orig_lrp=orig_lrp)
            torch.cuda.synchronize()
            total = time.perf_counter() - timed.t_start
            out[method] = {"images_per_s": timed.n_after_first / total, "loader_wait_share": timed.wait / total}
            del lrp, orig_lrp, baselines
            torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--batch", type=int, default=32)
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--images", type=int, default=160, help="JPEGs in the synthetic tree of the command runs")
    p.add_argument("--workers", type=int, default=4)
    p.add_argument("--methods", type=str, default="all", help="comma-separated, 'all' or 'none'")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prepare_images needs a GPU")
    _lib.load()
    batches = synthetic_batches(4, args.batch)
    refs = [cpu_transform(b) for b in batches]
    res = {"gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "batch": args.batch,
           "kernel": bench_kernel(batches, refs, args.iters, h2d=False),
           "kernel_h2d": bench_kernel(batches, refs, args.iters, h2d=True),
           "cpu_per_core": bench_cpu(batches)}
    methods = {"all": list(hdf5_writer.METHODS), "none": []}.get(args.methods, args.methods.split(","))
    res["command"] = bench_command(methods, args.images, args.batch, args.workers) if methods else {}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
