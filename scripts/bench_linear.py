#!/usr/bin/env python
"""Per-piece timing of the K8 tensor-core dense-layer path at the config-3 decoder shapes
(R = K*N = 262 144 rows; 500 -> 784 output layer, 500 -> 500 hidden layer)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402
from zhusuan_b200 import fused as Fz  # noqa: E402


def timeit(fn, n=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    dev = "cuda"
    R = 64 * 4096
    out = {}
    for K, J in ((500, 784), (500, 500), (40, 500)):
        h = torch.relu(torch.randn(R, K, device=dev))
        W = torch.randn(J, K, device=dev) / K ** 0.5
        b = torch.zeros(J, device=dev)
        x = (torch.rand(4096, J, device=dev) < 0.13).float()
        g = torch.randn(R, device=dev)
        gy = torch.randn(R, J, device=dev)
        wp, ws = Fz._tc_split(W)
        hp, hs = Fz._tc_split(h)
        flops = 2.0 * R * K * J
        t = {}
        t["split_h"] = timeit(lambda: Fz._tc_split(h))
        t["split_gy"] = timeit(lambda: Fz._tc_split(gy))
        t["gemm_epi0_store"] = timeit(lambda: Fz._tc_linear(0, wp, ws, hp, hs, b, None, None, R, J, K, True))
        t["gemm_epi1_bernoulli"] = timeit(lambda: Fz._tc_linear(1, wp, ws, hp, hs, b, x, None, R, J, K))
        t["gemm_epi2_dlogits"] = timeit(lambda: Fz._tc_linear(2, wp, ws, hp, hs, b, x, g, R, J, K))
        t["dual_split_gy"] = timeit(lambda: Fz._tc_split_dual(gy))
        t["dual_split_h"] = timeit(lambda: Fz._tc_split_dual(h))
        t["relu_mask_mul"] = timeit(lambda: gy * (gy > 0))
        torch.backends.cuda.matmul.allow_tf32 = False
        t["cublas_fp32_fwd"] = timeit(lambda: torch.nn.functional.linear(h, W, b))
        torch.backends.cuda.matmul.allow_tf32 = True
        t["cublas_tf32_fwd"] = timeit(lambda: torch.nn.functional.linear(h, W, b))
        torch.backends.cuda.matmul.allow_tf32 = False
        lg = torch.nn.functional.linear(h, W, b).reshape(64, 4096, J)
        t["unfused_bernoulli_logprob"] = timeit(
            lambda: zs.distributions.Bernoulli(lg, group_ndims=1).log_prob(x))
        t = {k: round(v, 4) for k, v in t.items()}
        t["gemm_fp32_equiv_tflops_epi0"] = round(flops / (t["gemm_epi0_store"] * 1e-3) / 1e12, 1)
        t["mma_issued_tflops_epi0"] = round(3 * 2.0 * R * (-(-K // 64) * 64) * (-(-J // 256) * 256)
                                            / (t["gemm_epi0_store"] * 1e-3) / 1e12, 1)
        out["K%d_J%d" % (K, J)] = t
    print(json.dumps(out))


if __name__ == "__main__":
    main()
