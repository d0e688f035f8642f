#!/usr/bin/env python
"""Bayesian neural nets with L >= 3 weight layers (csrc/bnn_deep.cu) against the generic autograd
path, both arms alternating in one process.  One JSON line per case and arm: the median, fastest
and slowest of several timed windows (ms per call, CUDA events), kernel launches per call (from
torch.profiler, in a separate pass), FLOPs and bytes from the shapes, and the card's name and
power limit.

Cases: every SG-MCMC method at K = 8192, B = 100, [10, 50, 50, 1] (bnn_sgmcmc.py with
n_hiddens = [50, 50]); the bnn_vi.py training step at K = 10, B = 10, [13, 50, 50, 1]; value and
gradient at K = 8192; predictive at K = 5000 over 4096 rows; one full-batch HMC iteration
(1024 chains, 455 rows, 10 leapfrog steps); an SGHMC step at the UCI Year shape [90, 100, 100, 1].

    python scripts/bench_bnn_deep.py [--windows 5] [--case NAME ...]
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

SGMCMC = {
    "sghmc": ("SGHMC", dict(learning_rate=2e-6, friction=0.2, n_iter_resample_v=1000)),
    "sgld": ("SGLD", dict(learning_rate=4e-6)),
    "psgld": ("PSGLD", dict(learning_rate=4e-6)),
    "sgnht": ("SGNHT", dict(learning_rate=1e-5, tune_rate=50.)),
    "sgnht_scalar": ("SGNHT", dict(learning_rate=1e-5, tune_rate=50., use_vector_alpha=False)),
}
# bytes each method moves per weight and chain-step (as scripts/bench_bnn.py counts them)
STATE_BYTES = {"sghmc": 16, "sgld": 8, "psgld": 16, "sgnht": 28, "sgnht_scalar": 20}


def n_weights(sizes):
    return sum(sizes[i + 1] * (sizes[i] + 1) for i in range(len(sizes) - 1))


def fwd_bwd_flops(sizes, B):
    """forward 2BP, weight gradient 2BP, activation gradient 2B(P - first layer)."""
    P = n_weights(sizes)
    return 2 * B * P * 3 - 2 * B * sizes[1] * (sizes[0] + 1)


def problem(sizes, K, B, seed=0, scale=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, sizes[0], device="cuda", generator=g)
    y = torch.sin(x.sum(1)) + 0.1 * torch.randn(B, device="cuda", generator=g)
    ws = [scale * torch.randn(K, sizes[i + 1], sizes[i] + 1, device="cuda", generator=g)
          for i in range(len(sizes) - 1)]
    names = ["w%d" % i for i in range(len(ws))]
    ls = [torch.zeros((), device="cuda") for _ in ws]
    return x, y, ws, names, ls


def case_sgmcmc(method, sizes=(10, 50, 50, 1), K=8192, B=100):
    sizes = list(sizes)
    x, y, ws, names, ls = problem(sizes, K, B)
    lj = zs.fused.BNNRegressionLogJoint(x, y, ls, 10000, names=names)
    cls, kw = SGMCMC[method]
    arms = {}
    for fused in (True, False):
        sg = getattr(zs, cls)(seed=1, use_fused=fused, **kw)
        op, _ = sg.sample(lj, {}, dict(zip(names, [w.clone() for w in ws])))
        if fused:
            assert sg._fused_bnn() is lj
        arms["fused" if fused else "generic"] = op
    P = n_weights(sizes)
    return arms, dict(flops=K * (fwd_bwd_flops(sizes, B) + 10 * P),
                      bytes=K * P * STATE_BYTES[method], K=K, B=B, sizes=sizes)


def case_value_grad(sizes=(10, 50, 50, 1), K=8192, B=100):
    sizes = list(sizes)
    x, y, ws, names, ls = problem(sizes, K, B)
    lj = zs.fused.BNNRegressionLogJoint(x, y, ls, 10000, names=names)
    ws = [w.requires_grad_(True) for w in ws]
    obs = dict(zip(names, ws))

    def fused():
        torch.autograd.grad(lj.fused_log_joint(obs).sum(), ws)

    def generic():
        torch.autograd.grad(lj(obs).sum(), ws)
    P = n_weights(sizes)
    return {"fused": fused, "generic": generic}, dict(
        flops=K * fwd_bwd_flops(sizes, B), bytes=K * P * 8, K=K, B=B, sizes=sizes)


def case_predictive(sizes=(10, 50, 50, 1), K=5000, B=4096):
    sizes = list(sizes)
    x, y, ws, names, ls = problem(sizes, K, B)
    lj = zs.fused.BNNRegressionLogJoint(x, y, ls, B, names=names)
    obs = dict(zip(names, ws))

    def generic():
        with torch.no_grad():
            h = x.unsqueeze(0).expand(K, -1, -1)
            for i, w in enumerate(ws):
                h = torch.cat([h, torch.ones(h.shape[:-1] + (1,), device="cuda")], -1)
                h = torch.einsum("imk,ijk->ijm", w, h) / (h.shape[2] ** 0.5)
                if i < len(ws) - 1:
                    h = torch.relu(h)
            ym = h.squeeze(2)
            ys = lj.y_logstd                        # the default -0.95
            return ym, -0.5 * math.exp(-2 * ys) * (y - ym) ** 2 - ys - 0.5 * math.log(2 * math.pi)
    P = n_weights(sizes)
    return {"fused": lambda: lj.predictive(obs), "generic": generic}, dict(
        flops=K * 2 * B * P, bytes=K * P * 4 + 2 * K * B * 4, K=K, B=B, sizes=sizes)


def case_vi_step(sizes=(13, 50, 50, 1), K=10, B=10):
    """bnn_vi.py's training step: elbo(...).sgvb() and its backward (no optimizer update)."""
    sizes = list(sizes)
    x, y, ws, names, _ = problem(sizes, K, B)
    means = [torch.zeros(w.shape[1:], device="cuda", requires_grad=True) for w in ws]
    logstds = [torch.full(w.shape[1:], -3., device="cuda", requires_grad=True) for w in ws]
    ys = torch.zeros((), device="cuda", requires_grad=True)
    zero = torch.zeros((), device="cuda")
    lj = zs.fused.BNNRegressionLogJoint(x, y, [zero] * len(ws), 455, y_logstd=ys, names=names)
    params = means + logstds + [ys]

    def variational():
        bn = zs.BayesianNet()
        for n, m, s in zip(names, means, logstds):
            bn.normal(n, m, logstd=s, n_samples=K, group_ndims=2)
        return bn

    def arm(model):
        def step():
            lb = zs.variational.elbo(model, {"y": y}, variational=variational(), axis=0)
            torch.autograd.grad(lb.sgvb(), params)
        return step
    P = n_weights(sizes)
    return {"fused": arm(lj), "generic": arm(lambda o: lj(o))}, dict(
        flops=K * fwd_bwd_flops(sizes, B), bytes=K * P * 8, K=K, B=B, sizes=sizes)


def case_hmc(sizes=(13, 50, 50, 1), K=1024, B=455, n_leapfrogs=10):
    sizes = list(sizes)
    x, y, ws, names, ls = problem(sizes, K, B, scale=0.2)
    lj = zs.fused.BNNRegressionLogJoint(x, y, ls, B, names=names)
    arms = {}
    for fused in (True, False):
        h = zs.HMC(step_size=1e-3, n_leapfrogs=n_leapfrogs)
        op, _ = h.sample(lj if fused else (lambda o: lj(o)), {},
                         dict(zip(names, [w.clone() for w in ws])))
        assert (h._provider is not None) == fused
        arms["fused" if fused else "generic"] = op
    P = n_weights(sizes)
    calls = n_leapfrogs + 2
    return arms, dict(flops=K * calls * fwd_bwd_flops(sizes, B), bytes=K * P * 8 * calls, K=K,
                      B=B, sizes=sizes, n_leapfrogs=n_leapfrogs)


CASES = dict(
    {"sgmcmc_" + m: (lambda m=m: case_sgmcmc(m)) for m in SGMCMC},
    vi_step=case_vi_step, value_grad=case_value_grad, predictive=case_predictive, hmc=case_hmc,
    year_sghmc=lambda: case_sgmcmc("sghmc", sizes=(90, 100, 100, 1), K=2048))


def timed(fn, n):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


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
        raise SystemExit("bench_bnn_deep.py needs a CUDA device")
    info = card()
    for name in a.case:
        arms, shape = CASES[name]()
        for fn in arms.values():                   # warm-up: modules, allocator, algorithms
            fn()
            fn()
        torch.cuda.synchronize()
        # calls per window from one probe call each, so a window lasts about --window-ms
        n = {k: max(2, int(a.window_ms / max(timed(fn, 2), 1e-3))) for k, fn in arms.items()}
        win = {k: [] for k in arms}
        for _ in range(a.windows):
            for k, fn in arms.items():
                win[k].append(timed(fn, n[k]))
        for k, fn in arms.items():
            ms = statistics.median(win[k])
            print(json.dumps(dict(
                case=name, arm=k, ms_median=round(ms, 4), ms_min=round(min(win[k]), 4),
                ms_max=round(max(win[k]), 4), calls_per_window=n[k],
                launches_per_call=launches(fn), flops=shape["flops"], bytes=shape["bytes"],
                tflops=round(shape["flops"] / (ms * 1e-3) / 1e12, 3),
                speedup_vs_generic=round(statistics.median(win["generic"]) / ms, 3),
                **{k2: v for k2, v in shape.items() if k2 not in ("flops", "bytes")}, **info)),
                flush=True)


if __name__ == "__main__":
    main()
