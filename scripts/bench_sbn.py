#!/usr/bin/env python
"""The sigmoid belief nets of examples/sigmoid_belief_nets on fused Bernoulli-sampling layers
(zs.fused.LinearBernoulli: one launch per proposal layer, two-product mainloop on 0/1 activations)
against the generic path (F.linear + bn.bernoulli).  Prints one JSON line per case and path, with
the card's name and power limit read in the same run.

    vimco_step     sbn_vimco.py's training step: N = 24, K = 10, [784, 200, 200, 200],
                   vimco() cost, backward, torch.optim.Adam; ms per step
    rws_step       sbn_adaptive_is.py's step: -mean(IW bound) for the model and
                   klpq(...).importance() for the proposal, backward, Adam; ms per step
    test_bound     the test-set bound under torch.no_grad() at ll_samples = 1000 over 100 rows
                   (1e5 particle rows); particle rows / s and the dense-layer FLOP rate (2 R K J
                   per layer, the six layers of the proposal and the model)
"""
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

X, H = 784, 200


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def timed(fn, iters, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def params(seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def dense(J, K):
        return [(torch.randn(J, K, device="cuda", generator=g) / K ** 0.5).requires_grad_(True),
                torch.zeros(J, device="cuda").requires_grad_(True)]
    q = [dense(H, X), dense(H, H), dense(H, H)]
    m = [dense(H, H), dense(H, H), dense(X, H)]
    return q, m


def objective(fused, x, q, m, K):
    N = int(x.shape[0])

    def layer(bn, name, h, Wb, n_samples=None, dtype=torch.float32):
        if fused:
            return bn.stochastic(name, zs.fused.LinearBernoulli(h, Wb[0], Wb[1], dtype=dtype),
                                 n_samples=n_samples)
        return bn.bernoulli(name, F.linear(h.to(torch.float32), Wb[0], Wb[1]), group_ndims=1,
                            n_samples=n_samples, dtype=dtype)

    qn = zs.BayesianNet()
    h1 = layer(qn, "h1", x.to(torch.float32), q[0], n_samples=K)
    h2 = layer(qn, "h2", h1.tensor, q[1])
    h3 = layer(qn, "h3", h2.tensor, q[2])

    def log_joint(obs):
        bn = zs.BayesianNet(observed=obs)
        z3 = bn.bernoulli("h3", torch.zeros(N, H, device="cuda"), group_ndims=1, n_samples=K,
                          dtype=torch.float32)
        z2 = layer(bn, "h2", z3.tensor, m[0])
        z1 = layer(bn, "h1", z2.tensor, m[1])
        layer(bn, "x", z1.tensor, m[2], dtype=torch.int32)
        return bn.log_joint()

    latent = {n: [t.tensor, t.cond_log_p] for n, t in (("h1", h1), ("h2", h2), ("h3", h3))}
    return log_joint, latent


def data(N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(N, X, device="cuda", generator=g) < 0.2).to(torch.int32)


def step_case(kind, fused, iters=200, warm=20):
    q, m = params()
    qp = [p for l in q for p in l]
    mp = [p for l in m for p in l]
    opt = torch.optim.Adam(qp + mp, lr=1e-3, eps=1e-4)
    xs = [data(24, s) for s in range(16)]
    it = [0]

    def step():
        x = xs[it[0] % len(xs)]
        it[0] += 1
        lj, latent = objective(fused, x, q, m, 10)
        opt.zero_grad()
        if kind == "vimco_step":
            lb = zs.variational.iw_objective(lj, {"x": x}, latent=latent, axis=0)
            lb.vimco().mean().backward()
        else:
            lb = zs.variational.iw_objective(lj, {"x": x}, latent=latent, axis=0)
            gm = torch.autograd.grad(-lb.tensor.mean(), mp)
            kl = zs.variational.klpq(lj, {"x": x}, latent=latent, axis=0)
            gq = torch.autograd.grad(kl.importance().mean(), qp)
            for p, g in zip(mp + qp, list(gm) + list(gq)):
                p.grad = g
        opt.step()
    ms = timed(step, iters, warm)
    return {"case": kind, "path": "fused" if fused else "generic", "N": 24, "K": 10,
            "layers": [X, H, H, H], "ms_per_step": round(ms, 4)}


def bound_case(fused, iters=20, warm=3):
    q, m = params()
    x = data(100, 99)
    K = 1000

    def run():
        with torch.no_grad():
            lj, latent = objective(fused, x, q, m, K)
            return zs.variational.iw_objective(lj, {"x": x}, latent=latent, axis=0).tensor.mean()
    ms = timed(run, iters, warm)
    rows = 100 * K
    flops = sum(2.0 * rows * k * j for k, j in ((X, H), (H, H), (H, H), (H, H), (H, H), (H, X)))
    return {"case": "test_bound", "path": "fused" if fused else "generic", "ll_samples": K,
            "rows": 100, "ms": round(ms, 4), "particle_rows_per_s": round(rows / ms * 1e3, 1),
            "dense_tflops": round(flops / ms * 1e-9, 2)}


def main():
    c = card()
    zs.set_random_seed(1234)
    for run in (lambda f: step_case("vimco_step", f), lambda f: step_case("rws_step", f),
                bound_case):
        for fused in (True, False):            # both paths in the same process, back to back
            print(json.dumps(dict(run(fused), **c)), flush=True)


if __name__ == "__main__":
    main()
