"""Time the dense-joint rollout (aggregation + N x N x N chain): SIMT fp32 chain vs tensor-core 3xTF32 chain.

    python tools/bench_dense_rollout.py [L B H N]
"""
import sys
import json
import torch

sys.path.insert(0, ".")
from transformer_explainability_b200 import ops  # noqa: E402


def main():
    L, B, H, N = (int(a) for a in sys.argv[1:5]) if len(sys.argv) >= 5 else (12, 256, 12, 197)
    ld = (N + 3) // 4 * 4
    g = torch.Generator(device="cuda").manual_seed(0)
    grad = torch.randn(L, B, H, N, ld, device="cuda", generator=g) * 0.05
    cam = torch.randn(L, B, H, N, ld, device="cuda", generator=g) * 0.05
    grad, cam = grad[..., :N], cam[..., :N]
    if ld != N:
        grad, cam = grad.contiguous(), cam.contiguous()
    res = {"L": L, "B": B, "H": H, "N": N}
    outs = {}
    for name, fused in (("simt", False), ("tensor_cores", True)):
        for _ in range(2):
            j, r = ops.attribution_rollout(grad, cam, fused=fused, want_joint=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            j, r = ops.attribution_rollout(grad, cam, fused=fused, want_joint=True)
        e1.record()
        torch.cuda.synchronize()
        res[name + "_ms"] = e0.elapsed_time(e1) / 5
        outs[name] = j
    res["max_abs_diff"] = (outs["simt"] - outs["tensor_cores"]).abs().max().item()
    res["chain_flops"] = 2.0 * (L - 1) * B * N ** 3
    print(json.dumps(res))


if __name__ == "__main__":
    main()
