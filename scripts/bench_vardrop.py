#!/usr/bin/env python
"""The variational-dropout classifier of examples/bayesian_neural_nets/variational_dropout.py on two
arms, run in one process and alternating.  Prints one JSON line per case and arm, with the card's
name and power limit read in the same run.

    generic   the reference's formulation in torch: x tiled over the particles, h * eps, F.linear,
              batch-norm moments as separate reductions, the affine step and ReLU
    fused     zs.fused.noisy_bn_linear: x broadcast over the particles, h * eps split straight into
              operand planes, the moments from the product's epilogue

    train     the training step at the example's shape: S = 10 particles x 1000 rows through
              [784, 100, 100, 100, 10], cost, backward, torch.optim.Adam(1e-3, eps=1e-4); ms/step
    eval      the test bound and accuracy at S = 100 particles x 1000 rows (1e5 particle rows), in
              evaluation mode under torch.no_grad(); ms per batch

`flop` is the dense-layer work per call (2 R K J per product, times 3 in training for the two
backward products).  `bytes` is computed from the shapes: the fp32 noise of every layer read once,
plus, in the generic arm, layer 0's tiled x and x * eps, each written and read once.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

NET = [784, 100, 100, 100, 10]
N, S_TRAIN, S_EVAL, N_TRAIN = 1000, 10, 100, 60000
DECAY, EPS = 0.999, 1e-3
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


def generic_layer(h, eps, W, beta, mm, mv, training):
    """variational_dropout.py:26-37 in torch, as TF builds it."""
    a = F.linear(h * eps, W)
    if training:
        mean = a.mean((0, 1))
        var = (a - mean.detach()).square().mean((0, 1))
        with torch.no_grad():
            mm.sub_((mm - mean) * (1.0 - DECAY))
            mv.sub_((mv - var) * (1.0 - DECAY))
    else:
        mean, var = mm, mv
    return F.relu((a - mean) * torch.rsqrt(var + EPS) + beta)


def fused_layer(h, eps, W, beta, mm, mv, training):
    return zs.fused.noisy_bn_linear(h, eps, W, beta, mm, mv, training)


def run(arm, P, x, y, z, training):
    """(bound, cost, accuracy) of variational_dropout.py:86-114 given the standard-normal draws z."""
    Ws, betas, alphas, mms, mvs = P
    layer = fused_layer if arm == "fused" else generic_layer
    S = z[0].shape[0]
    h = x if arm == "fused" else x.unsqueeze(0).expand(S, -1, -1)      # x_obs = tile(x, [S, 1, 1])
    lp, lq = 0.0, 0.0
    for i in range(len(Ws)):
        std = torch.sqrt(torch.sigmoid(alphas[i]) + 1e-10)
        eps = 1.0 + std * z[i]
        d = eps - 1.0
        lp = lp + (-0.5 * d * d).sum(-1)
        lq = lq + (-torch.log(std) - 0.5 * z[i] * z[i]).sum(-1)      # the 2 pi terms cancel
        h = layer(h, eps, Ws[i], betas[i], mms[i], mvs[i], training)
    log_py = torch.log_softmax(h, -1).gather(-1, y.expand(S, -1).unsqueeze(-1)).squeeze(-1)
    lb = (lp + log_py * N_TRAIN - lq).mean(0)
    acc = (torch.softmax(h, -1).mean(0).argmax(1) == y).float().mean()
    return lb.mean() / N_TRAIN, -lb.mean() / N_TRAIN, acc


def params(seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Ws = [(torch.randn(o, i, device="cuda", generator=g) / i ** 0.5).requires_grad_(True)
          for i, o in zip(NET[:-1], NET[1:])]
    betas = [torch.zeros(o, device="cuda").requires_grad_(True) for o in NET[1:]]
    alphas = [torch.zeros(i, device="cuda").requires_grad_(True) for i in NET[:-1]]
    mms = [torch.zeros(o, device="cuda") for o in NET[1:]]
    mvs = [torch.ones(o, device="cuda") for o in NET[1:]]
    return Ws, betas, alphas, mms, mvs


def flops(S, train):
    f = sum(2 * S * N * i * o for i, o in zip(NET[:-1], NET[1:]))
    return f * (3 if train else 1)


def noise_bytes(S):
    return 4 * S * N * sum(NET[:-1])


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
        sys.exit("bench_vardrop.py needs a CUDA device")
    info = card()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(N, NET[0], device="cuda", generator=g)
    y = torch.randint(0, 10, (N,), device="cuda", generator=g)
    z_tr = [torch.randn(S_TRAIN, N, k, device="cuda", generator=g) for k in NET[:-1]]
    z_ev = [torch.randn(S_EVAL, N, k, device="cuda", generator=g) for k in NET[:-1]]
    cases = []
    for arm in ARMS:
        P = params()
        opt = torch.optim.Adam(P[0] + P[1] + P[2], lr=1e-3, eps=1e-4)

        def step(arm=arm, P=P, opt=opt):
            _, cost, _ = run(arm, P, x, y, z_tr, True)
            opt.zero_grad(set_to_none=True)
            cost.backward()
            opt.step()
        cases.append(("train", arm, step, flops(S_TRAIN, True), S_TRAIN * N,
                      noise_bytes(S_TRAIN)))
    for arm in ARMS:
        P = params()

        def ev(arm=arm, P=P):
            with torch.no_grad():
                bound, _, acc = run(arm, P, x, y, z_ev, False)
            return bound, acc
        cases.append(("eval", arm, ev, flops(S_EVAL, False), S_EVAL * N, noise_bytes(S_EVAL)))

    # the two arms compute the same bound: check it once before timing
    with torch.no_grad():
        b = [run(arm, params(), x, y, z_ev, False)[0].item() for arm in ARMS]
    assert abs(b[0] - b[1]) <= 1e-4 * max(1.0, abs(b[0])), b

    times = {(c, arm): [] for c, arm, *_ in cases}
    for _ in range(args.rounds):                       # arms alternate within each round
        for c, arm, fn, *_ in cases:
            times[(c, arm)].append(timed(fn, args.iters, args.warmup))
    for c, arm, _, fl, rows, nb in cases:
        ts = sorted(times[(c, arm)])
        ms = ts[len(ts) // 2]
        tiled = 2 * 2 * 4 * rows * NET[0] if arm == "generic" else 0
        rec = dict(case=c, arm=arm, ms=round(ms, 4), ms_min=round(ts[0], 4),
                   ms_max=round(ts[-1], 4), particle_rows=rows, flop=fl,
                   tflops=round(fl / (ms * 1e-3) / 1e12, 3), bytes=nb + tiled, **info)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
