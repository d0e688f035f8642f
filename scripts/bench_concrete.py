#!/usr/bin/env python
"""ExpConcrete sampling and scoring on the kernels of csrc/concrete.cu against the composition the
class ran before them (elementwise torch ops and the library's reduce kernel), both arms
alternating in one process.  One JSON line per case and arm: the median, fastest and slowest of
several timed windows (ms per call, CUDA events), kernel launches and kernel device time per call
(from torch.profiler, in a separate pass), the least bytes the step must move (from the shapes),
and the card's name and power limit.

One call is the inner step of a relaxed categorical model at IWAE-like particle counts:
y = q.sample(S), log q(y) grouped over the last two axes, and the gradient of its mean w.r.t. the
logits and the temperature (through the sample and the density).  Cases: S x 100 rows x 20 groups
x C with about 2e7 elements each: S = 1000 at C = 10, S = 40 at C = 256, S = 10 at C = 1024.
prior_k1000 scores z [1000, 100, 20, 10] under a prior whose logits [20, 10] broadcast over the
first two axes, with the gradients w.r.t. z, the logits and the temperature.

    python scripts/bench_concrete.py [--windows 5] [--case NAME ...]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402
from zhusuan_b200 import ops  # noqa: E402


def composition_step(logits, t, S, seed, it):
    """ExpConcrete._sample and ._log_prob as composed before the kernels (group_ndims = 2)."""
    C = logits.shape[-1]
    u = ops.base_noise(0, (S,) + tuple(logits.shape), logits.device, seed, it)
    u = u.clamp(1e-7, 1.0 - 1e-7)
    y = torch.log_softmax((logits + (-torch.log(-torch.log(u)))) / t, -1)
    temp = (logits - t * y).contiguous()
    lp = math.lgamma(C) + (C - 1.0) * torch.log(t) + ops.reduce_axes(temp, ops.OP_SUM, -1) - \
        C * ops.reduce_axes(temp, ops.OP_LSE, -1)
    return ops.group_sum(lp, 2)


def case(S, C, N=100, G=20):
    g = torch.Generator(device="cuda").manual_seed(C)
    logits = torch.randn(N, G, C, device="cuda", generator=g).requires_grad_(True)
    t = torch.tensor(0.5, device="cuda", requires_grad=True)

    def fused():
        d = zs.distributions.ExpConcrete(t, logits, group_ndims=2, seed=1)
        lp = d.log_prob(d.sample(S))
        return torch.autograd.grad(lp.mean(), [logits, t])

    def generic():
        lp = composition_step(logits, t, S, 1, zs.random.next_counter())
        return torch.autograd.grad(lp.mean(), [logits, t])

    n = S * N * G * C
    # sample write; log q reads y; its backward reads y, writes dgiven; the sample's backward
    # reads y and gy
    return dict(fused=fused, generic=generic), dict(bytes=24 * n, elements=n, S=S, N=N, G=G, C=C)


def prior_case(K=1000, N=100, G=20, C=10):
    """log p(z) of the relaxed categorical VAE's prior, ExpConcrete(t, zeros [G, C]), on z
    [K, N, G, C] with the gradient w.r.t. z, the (broadcast) logits and the temperature."""
    g = torch.Generator(device="cuda").manual_seed(3)
    z = torch.log_softmax(torch.randn(K, N, G, C, device="cuda", generator=g), -1)
    z.requires_grad_(True)
    logits = torch.zeros(G, C, device="cuda", requires_grad=True)
    t = torch.tensor(0.5, device="cuda", requires_grad=True)

    def fused():
        lp = zs.distributions.ExpConcrete(t, logits, group_ndims=2).log_prob(z)
        return torch.autograd.grad(lp.mean(), [z, logits, t])

    def generic():
        temp = (logits - t * z).contiguous()
        lp = math.lgamma(C) + (C - 1.0) * torch.log(t) + ops.reduce_axes(temp, ops.OP_SUM, -1) - \
            C * ops.reduce_axes(temp, ops.OP_LSE, -1)
        return torch.autograd.grad(ops.group_sum(lp, 2).mean(), [z, logits, t])

    n = K * N * G * C
    # log p reads z; its backward reads z and writes dz
    return dict(fused=fused, generic=generic), dict(bytes=12 * n, elements=n, S=K, N=N, G=G, C=C)


CASES = {"step_c10": lambda: case(1000, 10), "step_c256": lambda: case(40, 256),
         "step_c1024": lambda: case(10, 1024), "prior_k1000": prior_case}


def timed(fn, n):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def profile_call(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(ev), sum(e.device_time_total for e in ev) / 1e3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--window-ms", type=float, default=200.)
    ap.add_argument("--case", nargs="*", default=list(CASES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_concrete.py needs a CUDA device")
    info = card()
    for name in a.case:
        arms, shape = CASES[name]()
        for fn in arms.values():                   # warm-up: modules, allocator
            fn()
            fn()
        torch.cuda.synchronize()
        n = {k: max(2, int(a.window_ms / max(timed(fn, 2), 1e-3))) for k, fn in arms.items()}
        win = {k: [] for k in arms}
        for _ in range(a.windows):
            for k, fn in arms.items():
                win[k].append(timed(fn, n[k]))
        for k, fn in arms.items():
            ms = statistics.median(win[k])
            nl, dev_ms = profile_call(fn)
            print(json.dumps(dict(
                case=name, arm=k, ms_median=round(ms, 4), ms_min=round(min(win[k]), 4),
                ms_max=round(max(win[k]), 4), calls_per_window=n[k], launches_per_call=nl,
                kernel_ms_per_call=round(dev_ms, 4),
                gbps_min_bytes=round(shape["bytes"] / (ms * 1e-3) / 1e9, 1),
                speedup_vs_generic=round(statistics.median(win["generic"]) / ms, 3),
                **shape, **info)), flush=True)


if __name__ == "__main__":
    main()
