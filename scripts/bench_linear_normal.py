#!/usr/bin/env python
"""The Gaussian dense layer zs.fused.LinearNormal against the registry's Normal fed two dense heads.
Prints one JSON line per case and arm, with the card's name and power limit read in the same run.

    head        z ~ N(dense(h), exp(dense(h))) at the config-3 IWAE shape (R = 4096 rows, K = 64
                draws, 500 -> 40): the draw, log q of it summed over the features, and the
                gradients of sum(z * c) + sum(log q) w.r.t. h and the four parameters
    iwae_step   the config-3 IWAE training step (scripts/bench_iwae.py: VAE 784-(500,500)-40, K =
                64, batch 4096, SGVB), forward + backward
    ssl_ais_step / ssl_ais_test
                vae_ssl_adaptive_is.py at the example's shape (500 hidden units, z 100, K 10,
                100 labeled + 100 unlabeled rows of 784 pixels): one training step (both bounds,
                both gradient lists, one Adam update) and one test batch (both bounds and the
                accuracy), on tests/ssl_ais_models.py's fused and generic arms

Arms.  head: fused (LinearNormal), fused_linear_registry (Normal on two zs.fused.linear heads) and
torch_linear_registry (Normal on two F.linear heads).  iwae_step: fused (every dense layer on the
wgmma kernel, the encoder's z head on LinearNormal) and fused_linear_registry
(bench_iwae.step_fn(fused=True), the same step with the head on Normal of two zs.fused.linear).
The arms alternate window by window in one process; each line gives the median, fastest and slowest
window in ms per call, and, from a separate torch.profiler pass, kernel launches per call.  FLOPs
and bytes come from the shapes: head flops = 3 products of 2 R H 2D (forward, input and weight
gradients); bytes = z, its upstream gradient and, for the registry arms, the eps tensor they keep
(written once, read once), in fp32, plus h and its gradient.  iwae_step flops = 3 * 3.97e6 K N
(bench_iwae.py's forward count, times three for the backward products).  The ssl_ais lines carry
no flops: at 100 rows per batch the step is bound by launches and host work, not arithmetic.
"""
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zhusuan_b200 as zs  # noqa: E402
import bench_iwae  # noqa: E402
import ssl_ais_models as SM  # noqa: E402

R, K, H, D = 4096, 64, 500, 40


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def head_dist(arm, h, Wm, bm, Wl, bl):
    if arm == "fused":
        return zs.fused.LinearNormal(h, Wm, bm, Wl, bl, group_ndims=1)
    lin = zs.fused.linear if arm == "fused_linear_registry" else F.linear
    return zs.distributions.Normal(lin(h, Wm, bm), logstd=lin(h, Wl, bl), group_ndims=1)


def head_case(arm, params, c):
    def fn():
        d = head_dist(arm, *params)
        z = d.sample(K)
        return torch.autograd.grad((z * c).sum() + d.log_prob(z).sum(), params)
    return fn


def iwae_step_fn(W, x, Kp, dev):
    """bench_iwae.step_fn(fused=True) with the encoder's z head on LinearNormal."""
    n = x.shape[0]
    z_dim = W["em"].shape[0]
    lin = zs.fused.linear

    def step():
        Wd = {k: v.detach().requires_grad_(True) for k, v in W.items()}

        @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
        def build_gen(n, n_particles):
            bn = zs.BayesianNet()
            z = bn.normal("z", torch.zeros(n, z_dim, device=dev), std=1., group_ndims=1,
                          n_samples=n_particles)
            hh = lin(z.tensor, Wd["d1"], Wd["d1_b"], relu=True)
            hh = lin(hh, Wd["d2"], Wd["d2_b"], relu=True)
            bn.stochastic("x", zs.fused.LinearBernoulli(hh, Wd["d3"], Wd["d3_b"]))
            return bn

        def build_q_net(x, n_particles):
            bn = zs.BayesianNet()
            hh = lin(x.float(), Wd["e1"], Wd["e1_b"], relu=True)
            hh = lin(hh, Wd["e2"], Wd["e2_b"], relu=True)
            bn.stochastic("z", zs.fused.LinearNormal(hh, Wd["em"], Wd["em_b"], Wd["es"],
                                                     Wd["es_b"], group_ndims=1),
                          n_samples=n_particles)
            return bn

        model = build_gen(n, Kp)
        variational = build_q_net(x, Kp)
        lb = zs.variational.iw_objective(model, {'x': x}, variational=variational, axis=0)
        cost = torch.mean(lb.sgvb())
        grads = torch.autograd.grad(cost, list(Wd.values()))
        return cost.detach(), grads
    return step


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return len([e for e in prof.events() if e.device_type.name == "CUDA"])


def measure(fns, reps):
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    windows = {a: [] for a in fns}
    for _ in range(7):
        for a, fn in fns.items():
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            windows[a].append(e0.elapsed_time(e1) / reps)
    return windows


def report(info, case, fns, windows, flops, nbytes, **shape):
    for a in fns:
        ms = statistics.median(windows[a])
        line = dict(info, case=case, arm=a, **shape, ms=round(ms, 4),
                    ms_min=round(min(windows[a]), 4), ms_max=round(max(windows[a]), 4),
                    launches=launches(fns[a]), flops=flops,
                    tflops=round(flops / ms / 1e9, 2) if flops else None)
        if flops is None:
            line.pop("flops"), line.pop("tflops")
        if nbytes is not None:
            line.update(bytes=nbytes[a], gbps=round(nbytes[a] / ms / 1e6, 1))
        print(json.dumps(line), flush=True)


def main():
    torch.manual_seed(0)
    info = card()
    dev = torch.device("cuda")

    h = torch.randn(R, H, device=dev).requires_grad_()
    params = [h] + [t.requires_grad_() for t in (
        torch.randn(D, H, device=dev) / H ** 0.5, torch.zeros(D, device=dev),
        0.1 * torch.randn(D, H, device=dev) / H ** 0.5, torch.zeros(D, device=dev))]
    c = torch.randn(K, R, D, device=dev)
    arms = ("fused", "fused_linear_registry", "torch_linear_registry")
    fns = {a: head_case(a, params, c) for a in arms}
    z_bytes = 4 * K * R * D
    base = 2 * z_bytes + 2 * 4 * R * H
    nbytes = {a: base + (2 * z_bytes if a != "fused" else 0) for a in arms}
    report(info, "head", fns, measure(fns, 10), 3 * 2 * R * H * 2 * D, nbytes, rows=R,
           n_samples=K, H=H, D=D)

    rng = np.random.Generator(np.random.PCG64(4))
    x = torch.tensor(rng.random((R, 784)) < 0.13, dtype=torch.int32, device=dev)
    W = bench_iwae.build(dev)
    fns = {"fused": iwae_step_fn(W, x, K, dev),
           "fused_linear_registry": bench_iwae.step_fn(W, x, K, dev, fused=True)}
    report(info, "iwae_step", fns, measure(fns, 3), int(3 * 3.97e6 * K * R), None, batch=R,
           n_samples=K)

    x_dim, z_dim, C, Ks, N = 784, 100, 10, 10, 100
    xp_l, xp_u = torch.rand(N, x_dim, device=dev), torch.rand(N, x_dim, device=dev)
    y_l = F.one_hot(torch.randint(C, (N,), device=dev), C).float()
    x_t = (torch.rand(N, x_dim, device=dev) < 0.3).float()
    fns, tests = {}, {}
    for a in ("fused", "generic"):
        P = SM.init_params(np.random.default_rng(3), x_dim, z_dim, C)
        opt = SM.Adam(P)
        fused = a == "fused"
        fns[a] = (lambda P=P, opt=opt, fused=fused:
                  SM.train_step(zs, P, opt, xp_l, y_l, xp_u, Ks, fused))
        tests[a] = lambda P=P, fused=fused: SM.test_batch(zs, P, x_t, y_l, Ks, fused)
    report(info, "ssl_ais_step", fns, measure(fns, 10), None, None, rows=N, n_samples=Ks)
    report(info, "ssl_ais_test", tests, measure(tests, 10), None, None, rows=N, n_samples=Ks)


if __name__ == "__main__":
    main()
