#!/usr/bin/env python
"""The semi-supervised VAE (M2) of examples/semi_supervised_vae/vae_ssl.py on three arms, run in one
process and alternating.  Prints one JSON line per case and arm, with the card's name and power
limit read in the same run.

    generic        the reference's layout: unlabeled rows tiled C times, concat([x, onehot(y)]),
                   F.linear and a torch Bernoulli log-probability
    fused-tiled    the same layout on zs.fused.linear and zs.fused.LinearBernoulli
    fused-class    zs.fused.class_linear: the one-hot block gathered in the epilogue, the classes
                   enumerated from one product over the unlabeled rows (class-major)

    step           the training step at the example's shape: 100 labeled and 100 unlabeled rows,
                   K = 10, z = 100, cost, backward, torch.optim.Adam(3e-4); ms per step
    unlabeled      the unlabeled bound forward and backward at 1000 rows (1e5 decoder particle rows)
    eval           the test-set evaluation of a batch of 100 rows (both bounds and the accuracy)
                   under torch.no_grad()

`flop` is the dense-layer work the arm does per call (2 R K J per product, times 3 with the
backward's two products), computed from the shapes below.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

XD, ZD, C, H, K = 784, 100, 10, 500, 10
ARMS = ("generic", "fused-tiled", "fused-class")
SHAPES = dict(g_z=(H, ZD), g_y=(H, C), g_h=(H, H), g_x=(XD, H), q_h1=(H, XD + C), q_h2=(H, H),
              q_mean=(ZD, H), q_logstd=(ZD, H), c_h1=(H, XD), c_h2=(H, H), c_logits=(C, H))


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def params(seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {n: ((torch.randn(s, device="cuda", generator=g) / s[1] ** 0.5).requires_grad_(True),
                torch.zeros(s[0], device="cuda").requires_grad_(True))
            for n, s in SHAPES.items()}


def normal_lp(z, mean, logstd):
    return (-0.5 * math.log(2 * math.pi) - logstd
            - 0.5 * torch.exp(-2 * logstd) * (z - mean) ** 2).sum(-1)


def bounds(arm, P, x_l, y_l, x_u, eps_l, eps_u, labeled=True, classifier=True):
    """(labeled bound, unlabeled bound, classifier cost, accuracy) of vae_ssl.py:86-136 on `arm`.
    y_l: class indices; eps_u [K, N C, z] (tiled arms, row n C + c) or [K, C, N, z] (fused-class)."""
    fused = arm != "generic"

    def lin(h, Wb, relu=False):
        if fused:
            return zs.fused.linear(h, *Wb, relu=relu)
        y = F.linear(h, *Wb)
        return F.relu(y) if relu else y

    def x_lp(h, x):
        if fused:
            return zs.fused.LinearBernoulli(h, *P["g_x"]).log_prob(x)
        logits = F.linear(h, *P["g_x"])
        return -F.binary_cross_entropy_with_logits(logits, x.expand_as(logits),
                                                   reduction="none").sum(-1)

    Wq, bq = P["q_h1"]

    def elbo(x, y, eps):
        """per-row ELBO; y: indices (fused-class, or None to enumerate) or one-hot rows"""
        if arm == "fused-class":
            h1 = zs.fused.class_linear(x, Wq[:, :XD], Wq[:, XD:], y, b=bq, relu=True)
        else:
            h1 = lin(torch.cat([x, y], -1), P["q_h1"], relu=True)
        h = lin(h1, P["q_h2"], relu=True)
        mean, logstd = lin(h, P["q_mean"]), lin(h, P["q_logstd"])
        z = mean + torch.exp(logstd) * eps
        log_q = normal_lp(z, mean, logstd)
        if arm == "fused-class":
            if y is None:
                y = torch.arange(C, device=x.device).view(C, 1).expand(C, x.shape[0])
            h = zs.fused.class_linear(z, P["g_z"][0], P["g_y"][0], y,
                                      b=P["g_z"][1] + P["g_y"][1], relu=True)
        else:
            h = F.relu(lin(z, P["g_z"]) + lin(y, P["g_y"]))
        h = lin(h, P["g_h"], relu=True)
        log_p = normal_lp(z, torch.zeros_like(z), torch.zeros_like(z)) - math.log(C) + x_lp(h, x)
        return (log_p - log_q).mean(0)

    def clf(x):
        return lin(lin(lin(x, P["c_h1"], relu=True), P["c_h2"], relu=True), P["c_logits"])

    out = [None, None, None, None]
    if labeled:
        y = y_l if arm == "fused-class" else F.one_hot(y_l, C).float()
        out[0] = elbo(x_l, y, eps_l).mean()
    N = x_u.shape[0]
    if arm == "fused-class":
        lb_z = elbo(x_u, None, eps_u).t()                                    # [N, C]
    else:
        y_t = torch.eye(C, device=x_u.device).repeat(N, 1)
        lb_z = elbo(x_u.repeat_interleave(C, 0), y_t, eps_u).reshape(N, C)
    qy = torch.softmax(clf(x_u), -1) + 1e-8
    qy = qy / qy.sum(1, keepdim=True)
    out[1] = (qy * (lb_z - torch.log(qy))).sum(1).mean()
    if classifier:
        logits = clf(x_l)
        out[2] = -1200.0 * torch.log_softmax(logits, -1).gather(1, y_l.view(-1, 1)).mean()
        out[3] = (logits.argmax(1) == y_l).float().mean()
    return out


def flops(arm, n_l, n_u, train, labeled=True, classifier=True):
    """Dense-layer FLOPs of one call of `bounds` (x3 when trained: the two backward products)."""
    d = lambda r, k, j: 2 * r * k * j                                       # noqa: E731
    f = 0
    for n, unl in ((n_l, False), (n_u, True)):
        if n == 0 or (not unl and not labeled):
            continue
        rows = n * C if unl else n                 # encoder rows after the class expansion
        if arm == "fused-class":
            f += d(n, XD, H)                       # the one-hot block is a gather
        else:
            f += d(rows, XD + C, H)
        f += d(rows, H, H) + 2 * d(rows, H, ZD)
        rz = K * rows
        f += d(rz, ZD, H) + (0 if arm == "fused-class" else d(rz, C, H)) + d(rz, H, H) + \
            d(rz, H, XD)
    nc = n_u + (n_l if classifier else 0)
    f += d(nc, XD, H) + d(nc, H, H) + d(nc, H, C)
    return f * (3 if train else 1)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ssl.py needs a CUDA device")
    info = card()
    g = torch.Generator(device="cuda").manual_seed(1)

    def batch(n_l, n_u):
        x_l = (torch.rand(n_l, XD, device="cuda", generator=g) < 0.3).float()
        x_u = (torch.rand(n_u, XD, device="cuda", generator=g) < 0.3).float()
        y_l = torch.randint(0, C, (n_l,), device="cuda", generator=g)
        eps_l = torch.randn(K, n_l, ZD, device="cuda", generator=g)
        eps_u = torch.randn(K, n_u * C, ZD, device="cuda", generator=g)
        return x_l, y_l, x_u, eps_l, eps_u

    def for_arm(arm, b):
        x_l, y_l, x_u, eps_l, eps_u = b
        if arm == "fused-class":                       # the same noise, class-major
            n = x_u.shape[0]
            eps_u = eps_u.reshape(K, n, C, ZD).permute(0, 2, 1, 3).contiguous()
        return x_l, y_l, x_u, eps_l, eps_u

    cases = []
    b_step = batch(100, 100)
    for arm in ARMS:
        P = params()
        opt = torch.optim.Adam([p for l in P.values() for p in l], lr=3e-4)
        a = for_arm(arm, b_step)

        def step(arm=arm, P=P, opt=opt, a=a):
            lab, unl, clf, _ = bounds(arm, P, *a)
            opt.zero_grad(set_to_none=True)
            (-(lab + unl - clf) / 2.0).backward()
            opt.step()
        cases.append(("step", arm, step, flops(arm, 100, 100, True), 200))

    b_unl = batch(1, 1000)
    for arm in ARMS:
        P = params()
        a = for_arm(arm, b_unl)
        ps = [p for l in P.values() for p in l]

        def unl(arm=arm, P=P, a=a, ps=ps):
            _, u, _, _ = bounds(arm, P, *a, labeled=False, classifier=False)
            torch.autograd.grad(u, ps, allow_unused=True)
        cases.append(("unlabeled", arm, unl, flops(arm, 0, 1000, True, False, False), 1000))

    b_eval = batch(100, 100)
    for arm in ARMS:
        P = params()
        a = for_arm(arm, b_eval)

        def ev(arm=arm, P=P, a=a):
            with torch.no_grad():
                bounds(arm, P, *a)
        cases.append(("eval", arm, ev, flops(arm, 100, 100, False), 200))

    times = {(c, arm): [] for c, arm, _, _, _ in cases}
    for _ in range(args.rounds):                       # arms alternate within each round
        for c, arm, fn, _, _ in cases:
            times[(c, arm)].append(timed(fn, args.iters, args.warmup))
    for c, arm, _, fl, rows in cases:
        ts = sorted(times[(c, arm)])
        ms = ts[len(ts) // 2]
        rec = dict(case=c, arm=arm, ms=round(ms, 4), ms_min=round(ts[0], 4),
                   ms_max=round(ts[-1], 4), rows=rows, flop=fl,
                   tflops=round(fl / (ms * 1e-3) / 1e12, 3), **info)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
