#!/usr/bin/env python
"""The Bernoulli-latent VAE of examples/variational_autoencoders/bernoulli_latent_vae.py on two
arms, run in one process and alternating.  Prints one JSON line per case and arm, with the card's
name and power limit read in the same run.

    generic   F.linear + F.batch_norm (momentum 0.01: TF's 0.99) + the registry Bernoulli.
              F.batch_norm moves running_var towards the unbiased (Bessel-corrected) batch
              variance where TF and bn_linear use the population variance, so this arm's
              evaluation cases normalise with slightly different statistics; the work timed is
              the same
    fused     zs.fused.bn_linear, zs.fused.LinearBernoulli and zs.fused.linear

    layer     one dense + batch-norm layer, 500 -> 500, forward and backward in training mode at
              400,000 rows (a layer of the IS estimate at 1000 particles x 400 rows)
    train     the example's training step: 128 rows, S = 1, [784, 500, 500], z 40, REINFORCE with
              the baseline net, backward, torch.optim.Adam(1e-3)
    test      the test lower bound at 400 rows, S = 1, evaluation mode, under torch.no_grad()
    is_ll     the IS log-likelihood at 1000 particles x 400 rows, evaluation mode, no_grad

Each window is `--iters` calls between device synchronises; median, fastest and slowest of
`--windows` windows are printed in ms per call.  `launches` is the number of device kernels per
call, counted in a separate torch.profiler pass.  `flop` is the dense-layer work (2 R K J per
product, three products per layer with a gradient); `bytes` counts each layer's fp32 input read
and output written once (4 (R K + R J)), times 3 with a gradient.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

X, H, Z, C = 784, 500, 40, 100
MOMENTUM, EPS = 0.99, 1e-3
ARMS = ("generic", "fused")


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def bn_layer(arm, h, W, g, b, mm, mv, training):
    if arm == "fused":
        return zs.fused.bn_linear(h, W, g, b, mm, mv, training)
    a = F.linear(h.to(torch.float32), W)
    lead = a.shape[:-1]
    y = F.batch_norm(a.reshape(-1, a.shape[-1]), mm, mv, g, b, training, 1.0 - MOMENTUM, EPS)
    return F.relu(y).reshape(tuple(lead) + (W.shape[0],))


def dense(arm, h, W, b, relu=False):
    if arm == "fused":
        return zs.fused.linear(h, W, b, relu=relu)
    y = F.linear(h, W, b)
    return F.relu(y) if relu else y


def model(arm, x, P, stats, training, S):
    """(log q(z) [S, n], the model's log_joint, cx [1, n]) of bernoulli_latent_vae.py:18-55."""
    q, p, c = P
    qs, ps = stats
    xf = x.to(torch.float32)
    bn = zs.BayesianNet()
    h = bn_layer(arm, xf, *q[0:3], *qs[0], training)
    h = bn_layer(arm, h, *q[3:6], *qs[1], training)
    if arm == "fused":
        z = bn.stochastic("z", zs.fused.LinearBernoulli(h, q[6], q[7], dtype=torch.float32),
                          n_samples=S)
    else:
        z = bn.bernoulli("z", F.linear(h, q[6], q[7]), group_ndims=1, n_samples=S,
                         dtype=torch.float32)

    def log_joint(obs):
        m = zs.BayesianNet(observed=obs)
        zn = m.bernoulli("z", torch.zeros(x.shape[0], Z, device=x.device), group_ndims=1,
                         n_samples=S, dtype=torch.float32)
        hh = bn_layer(arm, zn.tensor, *p[0:3], *ps[0], training)
        hh = bn_layer(arm, hh, *p[3:6], *ps[1], training)
        if arm == "fused":
            m.stochastic("x", zs.fused.LinearBernoulli(hh, p[6], p[7]))
        else:
            m.bernoulli("x", F.linear(hh, p[6], p[7]), group_ndims=1)
        return m.log_joint()

    cx = dense(arm, dense(arm, xf, c[0], c[1], relu=True), c[2], c[3]).squeeze(-1)
    return {"z": [z.tensor, z.cond_log_p]}, log_joint, cx.unsqueeze(0)


def params(dev, seed=0):
    g = torch.Generator().manual_seed(seed)

    def r(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).to(dev).requires_grad_(True)

    def bnp(J, K):
        return [r(J, K, scale=(2.0 / K) ** 0.5), r(J, scale=0.1).detach().add_(1.0)
                .requires_grad_(True), r(J, scale=0.1)]

    def dn(J, K):
        return [r(J, K, scale=K ** -0.5), r(J, scale=0.1)]
    return (bnp(H, X) + bnp(H, H) + dn(Z, H), bnp(H, Z) + bnp(H, H) + dn(X, H),
            dn(C, X) + dn(1, C))


def fresh_stats(dev):
    return [[(torch.zeros(H, device=dev), torch.ones(H, device=dev)) for _ in range(2)]
            for _ in range(2)]


def layer_flops(rows, grad):
    """(flop, bytes) of the eight dense layers (encoder, decoder and baseline net) of one pass
    over `rows` rows."""
    shapes = [(X, H), (H, H), (H, Z), (Z, H), (H, H), (H, X), (X, C), (C, 1)]
    f = sum(2 * rows * k * j for k, j in shapes) * (3 if grad else 1)
    b = sum(4 * (rows * k + rows * j) for k, j in shapes) * (3 if grad else 1)
    return f, b


def make_cases(dev):
    gen = torch.Generator(device=dev).manual_seed(1)

    def binarized(n):
        xin = torch.rand(n, X, device=dev, generator=gen) ** 3
        return (torch.rand(n, X, device=dev, generator=gen) < xin).to(torch.int32)

    cases = {}
    P = {arm: params(dev) for arm in ARMS}
    opt = {arm: torch.optim.Adam([t for l in P[arm] for t in l], lr=1e-3) for arm in ARMS}
    st = {arm: fresh_stats(dev) for arm in ARMS}
    x128, x400 = binarized(128), binarized(400)
    mmean = {arm: torch.zeros((), device=dev) for arm in ARMS}

    def train(arm):
        latent, lj, cx = model(arm, x128, P[arm], st[arm], True, 1)
        lb = zs.variational.elbo(lj, {"x": x128}, latent=latent, axis=0)
        cost, bcost = lb.reinforce(baseline=cx, moving_mean=mmean[arm])
        opt[arm].zero_grad(set_to_none=True)
        (cost + bcost).mean().backward()
        opt[arm].step()
    cases["train"] = (train, layer_flops(128, True))

    def test(arm):
        with torch.no_grad():
            latent, lj, _ = model(arm, x400, P[arm], st[arm], False, 1)
            return zs.variational.elbo(lj, {"x": x400}, latent=latent, axis=0).tensor.mean()
    cases["test"] = (test, layer_flops(400, False))

    def is_ll(arm):
        with torch.no_grad():
            latent, lj, _ = model(arm, x400, P[arm], st[arm], False, 1000)
            return zs.is_loglikelihood(lj, {"x": x400}, latent=latent, axis=0).mean()
    cases["is_ll"] = (is_ll, layer_flops(400 * 1000, False))

    R = 400000
    hl = torch.randn(R, H, device=dev, generator=gen)
    Wl = (torch.randn(H, H, device=dev, generator=gen) * H ** -0.5).requires_grad_(True)
    gl = torch.ones(H, device=dev, requires_grad=True)
    bl = torch.zeros(H, device=dev, requires_grad=True)
    sl = {arm: (torch.zeros(H, device=dev), torch.ones(H, device=dev)) for arm in ARMS}
    gy = torch.randn(R, H, device=dev, generator=gen)

    def layer(arm):
        h = hl.detach().requires_grad_(True)     # a new tensor: no operand split cached on it
        y = bn_layer(arm, h, Wl, gl, bl, *sl[arm], True)
        torch.autograd.grad(y, (h, Wl, gl, bl), gy)
    cases["layer"] = (layer, (3 * 2 * R * H * H, 3 * 4 * (2 * R * H)))
    return cases


def windows(fn, arm, iters, n):
    out = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            fn(arm)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3 / iters)
    return out


def launches(fn, arm):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(arm)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == "CUDA" and
               not e.name.startswith(("Memcpy", "Memset")))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--cases", default="layer,train,test,is_ll")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_blvae.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda")
    info = card()
    cases = make_cases(dev)
    for name in args.cases.split(","):
        fn, (flop, nbytes) = cases[name]
        iters = max(1, args.iters // (10 if name in ("layer", "is_ll") else 1))
        for arm in ARMS:                      # warm-up of every shape
            windows(fn, arm, 2, 1)
        res = {arm: [] for arm in ARMS}
        for _ in range(args.windows):         # the arms alternate window by window
            for arm in ARMS:
                res[arm] += windows(fn, arm, iters, 1)
        for arm in ARMS:
            w = res[arm]
            print(json.dumps(dict(case=name, arm=arm, ms_median=round(statistics.median(w), 4),
                                  ms_min=round(min(w), 4), ms_max=round(max(w), 4),
                                  iters_per_window=iters, windows=len(w),
                                  launches=launches(fn, arm), flop=flop, bytes=nbytes, **info)),
                  flush=True)


if __name__ == "__main__":
    main()
