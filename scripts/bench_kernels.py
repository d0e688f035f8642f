#!/usr/bin/env python
"""Micro-benchmarks of the HBM-bound kernels vs the measured copy bandwidth
(MEASURED_PEAKS.json hbm_gbs).  Each line: algorithmic bytes / CUDA-event time.
Inputs are > L2 (50 MB) so nothing is cache-resident."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402
from zhusuan_b200._lib import lib, ptr, stream  # noqa: E402

PEAK = 6570.0
p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
if os.path.exists(p):
    PEAK = json.load(open(p))["hbm_gbs"]


def timeit(fn, n=10, warm=3):
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


def report(name, nbytes, ms, extra=""):
    gbs = nbytes / (ms * 1e-3) / 1e9
    print(json.dumps({"kernel": name, "ms": round(ms, 4), "GBps": round(gbs, 1),
                      "frac_of_hbm_peak": round(gbs / PEAK, 3), "note": extra}))


def main():
    dev = "cuda"
    s = stream()
    C, D = 65536, 1024
    n = C * D
    q = torch.randn(C, D, device=dev); p_ = torch.randn(C, D, device=dev)
    g = torch.randn(C, D, device=dev); out = torch.empty(C, device=dev)
    mass = torch.ones(D, device=dev); state = torch.zeros(16, device=dev); state[7] = 0.01
    eps_ptr = state.data_ptr() + 28

    ms = timeit(lambda: q.copy_(p_))
    report("torch copy (reference point)", 8 * n, ms)
    # hmc elementwise
    ms = timeit(lambda: lib.call("zsb_hmc_leapfrog_q_f32", ptr(q), ptr(p_), ptr(mass), D, D, eps_ptr, 1.0, n, s))
    report("hmc_leapfrog_q", 12 * n, ms, "read q,p write q")
    ms = timeit(lambda: lib.call("zsb_hmc_leapfrog_p_f32", ptr(p_), ptr(g), eps_ptr, 1.0, n, s))
    report("hmc_leapfrog_p", 12 * n, ms)
    ms = timeit(lambda: lib.call("zsb_hmc_momentum_f32", ptr(p_), None, ptr(mass), D, C, D, 1, 1, 1, 0, ptr(out), 0, None, s))
    report("hmc_momentum (Philox)", 4 * n, ms, "write p only")
    ms = timeit(lambda: lib.call("zsb_hmc_kinetic_f32", ptr(p_), ptr(mass), D, C, D, ptr(out), 0, s))
    report("hmc_kinetic", 4 * n, ms)
    acc = torch.ones(C, dtype=torch.int32, device=dev)
    ms = timeit(lambda: lib.call("zsb_hmc_select_f32", ptr(q), ptr(p_), ptr(acc), C, D, s))
    report("hmc_select", 8 * n, ms, "all accepted: read q_new write q")
    part = torch.empty(lib.load().zsb_hmc_mass_parts() * 2 * D, device=dev); st2 = torch.empty(2 * D, device=dev); mean = torch.zeros(D, device=dev)
    ms = timeit(lambda: lib.call("zsb_hmc_mass_stats_f32", ptr(q), ptr(mean), C, D, ptr(part), ptr(st2), s))
    report("hmc_mass_stats", 4 * n, ms)
    lo = torch.empty(2, C, D, dtype=torch.float16, device=dev); sc = torch.zeros(8 + 4 * 3, device=dev); sc[3] = 1.0
    ms = timeit(lambda: lib.call("zsb_hmc_dense_traj_prepare_f32", ptr(q), ptr(p_), ptr(mass), ptr(lo), ptr(sc), C, D, s))
    report("dense_traj_prepare (absmax+split)", 16 * n, ms, "read q twice and p, write 2 fp16 planes")
    # record 0 has no overflow flag: the planes are read, never the spare
    ms = timeit(lambda: lib.call("zsb_hmc_dense_select_traj_planes_f32", ptr(q), ptr(lo), ptr(lo), ptr(sc[8:]), ptr(acc), C, D, s))
    report("dense_select_traj_planes", 8 * n, ms, "all accepted: read 2 fp16 planes, write q")
    # sgmcmc
    ms = timeit(lambda: lib.call("zsb_sgmcmc_sgld_f32", ptr(q), ptr(g), None, 1e-6, C, D, 1, 1, 0, s))
    report("sgmcmc_sgld (Philox)", 12 * n, ms)
    v = torch.zeros(C, D, device=dev); prt = torch.empty(148 * 8, device=dev); mk = torch.empty(1, device=dev)
    ms = timeit(lambda: lib.call("zsb_sgmcmc_sghmc_f32", ptr(q), ptr(v), ptr(g), None, 1e-6, 0.2, 0.0, 1, C, D, 1, 1, 0, ptr(prt), ptr(mk), s))
    report("sgmcmc_sghmc (Philox)", 20 * n, ms, "read q,v,g write q,v")
    # distributions / reductions at config-3 shapes
    K, N, X = 64, 4096, 784
    logits = torch.randn(K, N, X, device=dev); x = (torch.rand(N, X, device=dev) < 0.13).float()
    d = zs.distributions.Bernoulli(logits, group_ndims=1)
    ms = timeit(lambda: d.log_prob(x))
    report("bernoulli_log_prob [64,4096,784]", 4 * K * N * X, ms, "reads logits (x is L2 resident)")
    lr = logits.clone().requires_grad_(True)
    dd = zs.distributions.Bernoulli(lr, group_ndims=1)

    def fb():
        lp = dd.log_prob(x)
        lp.backward(torch.ones_like(lp))
        lr.grad = None
    ms = timeit(fb, n=5)
    report("bernoulli fwd+bwd", 12 * K * N * X, ms, "fwd read; bwd read + write dlogits")
    z = torch.randn(K, N, 40, device=dev); mu = torch.randn(N, 40, device=dev); ls = torch.randn(N, 40, device=dev) * 0.1
    dn = zs.distributions.Normal(mu, logstd=ls, group_ndims=1)
    big = torch.randn(64, 4096 * 64, 16, device=dev)
    dn2 = zs.distributions.Normal(torch.zeros(16, device=dev), logstd=torch.zeros(16, device=dev), group_ndims=1)
    ms = timeit(lambda: dn2.log_prob(big))
    report("normal_log_prob group=16 (268 MB)", 4 * big.numel(), ms)
    lw = torch.randn(64, 4096 * 256, device=dev)
    ms = timeit(lambda: zs.log_mean_exp(lw, 0))
    report("log_mean_exp [64, 1M] axis 0", 4 * lw.numel(), ms, "two passes over x, second from L2 only if < 50 MB")
    # fused diag-normal HMC iteration, C1' = 1M chains x 100
    C1, D1, L = 1 << 20, 100, 10
    std = torch.tensor(1.0 / (1.0 + np.arange(D1)), dtype=torch.float32, device=dev)

    @zs.meta_bayesian_net()
    def gaussian():
        bn = zs.BayesianNet()
        bn.normal('x', torch.zeros(D1, device=dev), std=std, group_ndims=1)
        return bn
    xq = torch.zeros(C1, D1, device=dev)
    h = zs.HMC(step_size=0.05, n_leapfrogs=L, seed=3)
    op, info = h.sample(gaussian(), {}, {"x": xq})
    ms = timeit(lambda: op(), n=10)
    report("fused diag HMC iteration C1' (1M x 100, L=10)", 12 * C1 * D1, ms,
           "actual traffic: read q, write q + init_momentum; %.3e chain-steps/s; ALGORITHMIC "
           "(SURVEY 8d: 16 D B per chain-step) %.0f GB/s = %.3f of the HBM peak" % (
               C1 * L / (ms * 1e-3), 16 * D1 * C1 * L / (ms * 1e-3) / 1e9,
               16 * D1 * C1 * L / (ms * 1e-3) / 1e9 / PEAK))
    # config 1 proper: 64 chains x 100, L=10 (launch-latency bound)
    xq2 = torch.zeros(64, D1, device=dev)
    h2 = zs.HMC(step_size=1e-3, n_leapfrogs=10, adapt_step_size=True, adapt_mass=True,
                target_acceptance_rate=0.9, seed=3)
    op2, info2 = h2.sample(gaussian(), {}, {"x": xq2})
    for i in range(12):
        op2(adapt_step_size=True, adapt_mass=True)
    ms = timeit(lambda: op2(adapt_step_size=True, adapt_mass=True), n=100)
    report("config 1 (64 x 100, L=10, adaptation on)", 12 * 64 * D1, ms,
           "launch bound: %.3e chain-steps/s, %.1f us per iteration" % (64 * 10 / (ms * 1e-3), ms * 1e3))
    # the same, replayed from a CUDA graph (device-driven iteration scalars)
    xq3 = torch.zeros(64, D1, device=dev)
    h3 = zs.HMC(step_size=1e-3, n_leapfrogs=10, adapt_step_size=True, adapt_mass=True,
                target_acceptance_rate=0.9, seed=3, use_cuda_graph=True)
    op3, info3 = h3.sample(gaussian(), {}, {"x": xq3})
    for i in range(12):
        op3(adapt_step_size=True, adapt_mass=True)
    ms = timeit(lambda: op3(adapt_step_size=True, adapt_mass=True), n=100)
    report("config 1 via CUDA graph", 12 * 64 * D1, ms,
           "%.3e chain-steps/s, %.1f us per iteration" % (64 * 10 / (ms * 1e-3), ms * 1e3))
    # dense D=64, 4096 chains, L=10: small-problem regime for the dense path
    from bench import make_dense_gaussian_problem
    P, _ = make_dense_gaussian_problem(64, seed=2)
    for graph in (False, True):
        xd = torch.randn(4096, 64, device=dev)
        hd = zs.HMC(step_size=0.05, n_leapfrogs=10, adapt_step_size=True, seed=3,
                    use_cuda_graph=graph)
        opd, _i = hd.sample(zs.fused.GaussianLogJoint(P), {}, {"x": xd})
        for i in range(5):
            opd()
        ms = timeit(lambda: opd(), n=100)
        report("dense 4096 x 64, L=10, graph=%s" % graph, 0, ms,
               "%.3e chain-steps/s, %.1f us per iteration" % (4096 * 10 / (ms * 1e-3), ms * 1e3))


if __name__ == "__main__":
    main()
