"""Time the attention-shaped tensor-core contractions of one ViT-B/16 attention block at the bench shapes (batch 256, 12
heads, N = 197 tokens, head dim 64, maps padded to NP = 200 columns) through ``ops.tc_attention_nn`` / ``ops.tc_attention_nk``,
with the operand forms flags 7475 selects, and the dense rollout chain (``ops.attribution_rollout(..., fused=True,
want_joint=True)``, whose chain steps are ``NkProb<0, AT_RESID>``).

    python tools/bench_attention_ops.py [--batch 256] [--iters 20]

Per op: CUDA-event time per launch (mean over --iters launches after a warm-up), the algorithmic bytes (every operand read
once, every output written once, computed from the shapes), the achieved GB/s and its share of the 3.35 TB/s HBM3
data-sheet bandwidth of the H100 SXM.  The card's name, power limit and SM clock are printed with the numbers.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import _lib, ops  # noqa: E402

HBM_TBS = 3.35


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the card name still comes from torch
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    _lib.load()
    B, H, N, dh, NP = args.batch, 12, 197, 64, 200
    D = H * dh
    print("card:", card(), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)

    def rnd(*shape):
        return torch.randn(*shape, device="cuda", generator=g)

    qkv = rnd(B * N, 3 * D)                                 # packed q | k | v rows, as the engine stores them
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    act = [rnd(B * N, D) for _ in range(3)]                 # dctx / S (relevance) / an output row block
    out_act = torch.empty(B * N, D, device="cuda")
    maps = [torch.softmax(rnd(B, H, N, NP)[..., :N], -1) for _ in range(2)]
    P, E = [torch.nn.functional.pad(m, (0, NP - N)).contiguous() for m in maps]
    out_map = torch.empty(B, H, N, NP, device="cuda")
    A, M = B * N * D * 4, B * H * N * NP * 4               # bytes of one activation block, of one N x N map

    def nn(a, b, epi, sp, e=None):
        return lambda: ops.tc_attention_nn(a, a.stride(0), b, b.stride(0), B, H, N, dh, out_map, NP, e=e, alpha=0.125, epi=epi,
                                           single_pass=sp)

    def nk(amap, amn, x, epi, sp, e=None):
        return lambda: ops.tc_attention_nk(amap, NP, amn, x, x.stride(0), B, H, N, out_act, D, e=e, alpha=0.5, epi=epi,
                                           single_pass=sp)

    # (label, problem, launch, algorithmic bytes)
    cases = [
        ("P = softmax(QK^T)", "NnProb<SOFTMAX, 3xTF32, 256>", nn(q, k, "softmax", False), 2 * A + M),
        ("ctx = P V", "NkProb<0, STORE, 3xTF32>", nk(P, 0, v, "store", False), M + 2 * A),
        ("G = dctx V^T", "NnProb<STORE, SP, 128>", nn(act[0], v, "store", True), 2 * A + M),
        ("dV = P^T dctx", "NkProb<1, STORE, SP>", nk(P, 1, act[0], "store", True), M + 2 * A),
        ("dQ = dS K", "NkProb<0, STORE, SP>", nk(E, 0, k, "store", True), M + 2 * A),
        ("dK = dS^T Q", "NkProb<1, STORE, SP>", nk(E, 1, q, "store", True), M + 2 * A),
        ("cam = P * (S V^T)/2", "NnProb<MUL, SP, 128>", nn(act[1], v, "mul", True, e=P), 2 * A + 2 * M),
        ("R_v = V * (P^T S)/2", "NkProb<1, MUL, SP>", nk(P, 1, act[1], "mul", True, e=v.contiguous()), M + 3 * A),
        ("S1 = sd(cam, QK^T)", "NnProb<SD, 3xTF32, 128>", nn(q, k, "sd", False, e=E), 2 * A + 2 * M),
        ("R_q = Q * (S1 K)", "NkProb<0, MUL, SP>", nk(E, 0, k, "mul", True, e=act[2]), M + 3 * A),
        ("R_k = K * (S1^T Q)", "NkProb<1, MUL, SP>", nk(E, 1, q, "mul", True, e=act[2]), M + 3 * A),
    ]
    print("batch %d, heads %d, N %d, dh %d, NP %d: one N x N map = %.0f MB" % (B, H, N, dh, NP, M / 1e6))
    print("%-22s %-30s %9s %9s %9s %8s" % ("op", "problem", "ms", "MB", "GB/s", "of HBM"))
    tot_ms = tot_b = 0.0
    for label, prob, fn, nbytes in cases:
        ms = timed(fn, args.iters)
        tot_ms += ms
        tot_b += nbytes
        gbs = nbytes / ms / 1e6
        print("%-22s %-30s %9.3f %9.0f %9.0f %7.1f%%" % (label, prob, ms, nbytes / 1e6, gbs, 100 * gbs / (HBM_TBS * 1e3)),
              flush=True)
    gbs = tot_b / tot_ms / 1e6
    print("%-53s %9.3f %9.0f %9.0f %7.1f%%" % ("all of the above", tot_ms, tot_b / 1e6, gbs, 100 * gbs / (HBM_TBS * 1e3)))

    # dense rollout: L = 12 layers of G / cam, one-launch aggregation + the N^3 chain in residual form
    L = 12
    Bd = max(1, B // 8)
    grad, cam = rnd(L, Bd, H, N, NP), rnd(L, Bd, H, N, NP)
    ms = timed(lambda: ops.attribution_rollout(grad, cam, fused=True, want_joint=True), max(1, args.iters // 4))
    nbytes = 2 * L * Bd * H * N * NP * 4 + (L - 1) * 3 * Bd * N * NP * 4 + Bd * N * N * 4
    gbs = nbytes / ms / 1e6
    print("%-22s %-30s %9.3f %9.0f %9.0f %7.1f%%  (batch %d)" % ("dense rollout", "aggregate + NkProb<0, RESID>", ms,
                                                                 nbytes / 1e6, gbs, 100 * gbs / (HBM_TBS * 1e3), Bd))
    print("flags default", _lib.FLAG_BENCH_DEFAULT)


if __name__ == "__main__":
    main()
