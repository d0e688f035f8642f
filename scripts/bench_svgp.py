"""Sparse variational GP (examples/gaussian_process/svgp.py) on zs.fused.gp_conditional against the
generic path (RBFKernel.__call__ plus torch ops, the reference's arithmetic), on seeded synthetic
data.  Cases:
  train_boston   the training step (sample, bound, sgvb().backward(), Adam): B = 455, d = 13
  train_protein  the same at B = 5000, d = 9
  predict_test   log_likelihood and pred_mse at 100 particles over 4573 rows, d = 9
  predict_1e5    the same over 1e5 rows at M = 256
M = 100 and K = 20 (training) unless stated.  The arms alternate in one process; each prints the
median over windows.  Launches per call come from a separate torch.profiler pass.  One JSON line
per case and arm, with the card's name and power limit.

    python scripts/bench_svgp.py [--windows 7] [--steps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

CASES = {
    "train_boston": dict(B=455, d=13, M=100, K=20, train=True),
    "train_protein": dict(B=5000, d=9, M=100, K=20, train=True),
    "predict_test": dict(B=4573, d=9, M=100, K=100, train=False),
    "predict_1e5": dict(B=100000, d=9, M=256, K=100, train=False),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def model_cost(c, fused):
    """FLOPs and HBM bytes of the B-sized work from the shapes (the M x M algebra is excluded)."""
    B, d, M, K = c["B"], c["d"], c["M"], c["K"]
    flops = 3 * B * M * d + B * M * (M + 1) + 2 * K * B * M + 2 * B * M
    byts = 4 * (B * d + K * B + B + M * d + M * M + K * M)
    if c["train"]:
        flops *= 3
        byts += 4 * (2 * B * M + K * B + B)          # A kept for backward, upstream grads
    if not fused:
        byts += 4 * 2 * B * M * d + 4 * 4 * B * M     # [B, M, d] broadcast and [B, M] products
    return flops, byts


def setup(c, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, d, M, K = c["B"], c["d"], c["M"], c["K"]
    kern = zs.fused.RBFKernel(d)
    p = {
        "z_pos": (torch.rand(M, d, generator=g, device="cuda") * 2 - 1).requires_grad_(True),
        "z_mean": torch.zeros(M, device="cuda", requires_grad=True),
        "z_cov_raw": torch.eye(M, device="cuda", requires_grad=True),
        "noise_level": torch.tensor(0.05, device="cuda", requires_grad=True),
    }
    x = torch.randn(B, d, generator=g, device="cuda")
    y = torch.randn(B, generator=g, device="cuda")
    params = list(p.values()) + [kern.k_raw_scale]
    return kern, p, x, y, params, g


def step_fn(c, fused):
    kern, p, x, y, params, g = setup(c)
    cond = zs.fused.gp_conditional if fused else zs.fused._gp_conditional_generic
    opt = torch.optim.Adam(params, lr=1e-2)
    B, M, K = c["B"], c["M"], c["K"]
    n_train = 10 * B
    sp = torch.nn.functional.softplus

    def variational():
        raw = p["z_cov_raw"]
        tril = torch.tril(raw, -1) + torch.diag(sp(torch.diagonal(raw)))
        q = zs.distributions.MultivariateNormalCholesky(p["z_mean"], tril)
        fz = q.sample(K)
        return fz, q.log_prob(fz)

    def train():
        fz, log_qfz = variational()
        fx = cond(p["z_pos"], fz, x, False, kern).sample()
        Kzz_chol = torch.linalg.cholesky_ex(kern(p["z_pos"], p["z_pos"]))[0]
        prior = zs.distributions.MultivariateNormalCholesky(
            torch.zeros(M, device="cuda"), Kzz_chol).log_prob(fz)
        log_py = zs.distributions.Normal(fx, std=sp(p["noise_level"]), group_ndims=1).log_prob(y)
        bound = (prior + log_py / B * n_train - log_qfz).mean()
        opt.zero_grad()
        (-bound).backward()
        opt.step()
        return bound

    def predict():
        with torch.no_grad():
            fz, _ = variational()
            fx = cond(p["z_pos"], fz, x, False, kern).sample()
            ll = zs.distributions.Normal(fx, std=sp(p["noise_level"]), group_ndims=1).log_prob(y)
            ll = zs.log_mean_exp(ll, 0) / B
            mse = ((fx.mean(0) - y) ** 2).mean()
            return ll, mse

    return train if c["train"] else predict


def launches(fn):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    name, power = card()
    for case in args.cases.split(","):
        c = CASES[case]
        fns = {arm: step_fn(c, arm == "fused") for arm in ("fused", "generic")}
        for fn in fns.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {arm: [] for arm in fns}
        for _ in range(args.windows):
            for arm, fn in fns.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) / args.steps * 1e3)
        for arm, fn in fns.items():
            ts = sorted(times[arm])
            flops, byts = model_cost(c, arm == "fused")
            print(json.dumps({
                "case": case, "arm": arm, "B": c["B"], "d": c["d"], "M": c["M"], "K": c["K"],
                "ms_median": round(ts[len(ts) // 2], 4), "ms_min": round(ts[0], 4),
                "ms_max": round(ts[-1], 4), "flops": flops, "bytes": byts,
                "launches_per_call": launches(fn), "gpu": name, "power_limit": power}),
                flush=True)


if __name__ == "__main__":
    main()
