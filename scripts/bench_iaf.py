#!/usr/bin/env python
"""Inverse autoregressive flows with the linear autoregressive network, and the normalizing-flow VAE
of examples/normalizing_flows/vae_nf.py with two IAF stacks, arms run in one process and
alternating.  Prints one JSON line per case and arm, with the card's name and power limit read in
the same run.

    flows     two stacks of 10 IAF flows (update 'normal') at d = 40 (vae_nf.py's z_dim) and at
              d = 128, forward ("fwd") and forward plus backward ("fwd_bwd"), at 128 rows (a
              training batch) and 4e5 rows (the IS evaluation's 1000 particles x 400 rows).  Arms:
                kernel  zs.inv_autoregressive_flow with a LinearAR (one launch per stack forward,
                        two backward)
                torch   the reference's loop (transform.py:262-275) in float32 torch through
                        LinearAR.__call__
              `launches` is the number of GPU kernels per call, counted with torch.profiler in a
              run of its own; the same run gives `flow_kernel_us`, the device time per call of the
              IAF kernels (forward, backward sweep, merge), summed over both stacks.  `flops`
              counts the two strictly triangular products, 2 d (d - 1) per row and flow; the
              backward counts four times that (the forward, the recomputation of m and t, the
              input gradient and the weight gradients).  `bytes` is the least traffic from the
              shapes, the same for both arms: z and log_q read and written once per stack, the
              weights read once, and in the backward the gradients of z and log_q as well.
              `gflops` = flops / ms and `gbps` = bytes / ms.
    train     the vae_nf.py training step with IAF: 128 rows, 1 particle, [784, 500, 500],
              z_dim 40, 2 x 10 flows, elbo(...).sgvb(), backward, Adam(1e-3); ms per step
    test      the test-set bound (1 particle) plus the IS estimate at 1000 particles over 400 rows,
              under torch.no_grad(); ms per batch
              Arms of train and test: zs.fused layers with the flows as above ("kernel" or
              "torch").
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

X_DIM, H, Z_DIM, N_FLOWS = 784, 500, 40, 10


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def kernel_flow(z, log_q, ar):
    return zs.inv_autoregressive_flow(z, None, log_q, ar, ar.n_iters)


def torch_flow(z, log_q, ar):
    # a plain callable, so the call runs the reference's loop in torch
    return zs.inv_autoregressive_flow(z, None, log_q, lambda *a: ar(*a), ar.n_iters)


FLOWS = {"kernel": kernel_flow, "torch": torch_flow}


def make_ar(d, g, scale):
    ar = zs.LinearAR(d, N_FLOWS, generator=g)
    with torch.no_grad():
        ar.m_w.mul_(scale / 0.005 / math.sqrt(d))
        ar.s_w.mul_(0.3 * scale / 0.005 / math.sqrt(d))
    return ar


def example(x, eps, P, flow):
    """vae_nf.py:19-85 on zs.fused layers with two IAF stacks; returns (elbo objective,
    is_loglikelihood thunk)."""
    q, p, flows = P
    lin = lambda h, W, b, relu=False: zs.fused.linear(h, W, b, relu=relu)   # noqa: E731
    S, n, z_dim = eps.shape

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, z_dim, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        h = lin(lin(z, p[0], p[1], True), p[2], p[3], True)
        bn.stochastic("x", zs.fused.LinearBernoulli(h, p[4], p[5], dtype=torch.float32))
        return bn

    h = lin(lin(x, q[0], q[1], True), q[2], q[3], True)
    mean, logstd = lin(h, q[4], q[5]), lin(h, q[6], q[7])
    qz = mean + torch.exp(logstd) * eps
    log_qz = zs.distributions.Normal(mean, logstd=logstd, group_ndims=1).log_prob(qz)
    for ar in flows:
        qz, log_qz = flow(qz, log_qz, ar)
    model = build_gen(n, z_dim, S)
    lb = zs.variational.elbo(model, {"x": x}, latent={"z": [qz, log_qz]}, axis=0)
    return lb, lambda: zs.is_loglikelihood(model, {"x": x}, {"z": [qz, log_qz]}, axis=0)


def params(seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def dense(i, o):
        return [(torch.randn(o, i, device="cuda", generator=g) / math.sqrt(i)).requires_grad_(True),
                torch.zeros(o, device="cuda").requires_grad_(True)]
    q = dense(X_DIM, H) + dense(H, H) + dense(H, Z_DIM) + dense(H, Z_DIM)
    p = dense(Z_DIM, H) + dense(H, H) + dense(H, X_DIM)
    flows = [make_ar(Z_DIM, g, 0.1) for _ in range(2)]
    return q, p, flows


def flat(P):
    return P[0] + P[1] + [t for ar in P[2] for t in (ar.m_w, ar.s_w)]


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


def profiled(fn):
    """(GPU kernels per call, {IAF kernel: device microseconds per call}) from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset"))]
    us = {}
    for e in kernels:
        for part in ("fwd", "bwd", "merge"):
            if "iaf_%s_kernel" % part in e.name:
                us[part] = us.get(part, 0.0) + e.time_range.elapsed_us()
    return len(kernels), {k: round(v, 1) for k, v in us.items()}


def flow_cases(d, rows_list):
    cases = []
    g = torch.Generator(device="cuda").manual_seed(3)
    ars = [make_ar(d, g, 0.3) for _ in range(2)]
    w_bytes = 2 * 2 * 4 * N_FLOWS * d * d
    for R in rows_list:
        z = torch.randn(R, d, device="cuda", generator=g)
        lq = torch.randn(R, device="cuda", generator=g)
        gz, gl = torch.randn_like(z), torch.randn_like(lq)
        for arm, flow in FLOWS.items():
            def fwd(flow=flow, z=z, lq=lq):
                with torch.no_grad():
                    a, b_ = z, lq
                    for ar in ars:
                        a, b_ = flow(a, b_, ar)
                return a, b_

            zi, li = z.clone().requires_grad_(True), lq.clone().requires_grad_(True)

            def fwd_bwd(flow=flow, zi=zi, li=li, gz=gz, gl=gl):
                a, b_ = zi, li
                for ar in ars:
                    a, b_ = flow(a, b_, ar)
                torch.autograd.backward((a, b_), (gz, gl))
            flops = 2 * N_FLOWS * 2 * d * (d - 1) * R
            base = 2 * (8 * R * d + 8 * R) + w_bytes
            cases.append(dict(case="flows_fwd", arm=arm, d=d, rows=R, fn=fwd, flops=flops,
                              bytes=base))
            cases.append(dict(case="flows_fwd_bwd", arm=arm, d=d, rows=R, fn=fwd_bwd,
                              flops=4 * flops, bytes=2 * base - 8 * R))
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_iaf.py needs a CUDA device")
    info = card()
    g = torch.Generator(device="cuda").manual_seed(1)
    x_tr = (torch.rand(128, X_DIM, device="cuda", generator=g) < 0.3).float()
    eps_tr = torch.randn(1, 128, Z_DIM, device="cuda", generator=g)
    x_te = (torch.rand(400, X_DIM, device="cuda", generator=g) < 0.3).float()
    eps_lb = torch.randn(1, 400, Z_DIM, device="cuda", generator=g)
    eps_is = torch.randn(1000, 400, Z_DIM, device="cuda", generator=g)

    # both arms compute the same bound: check it once before timing
    with torch.no_grad():
        got = {a: example(x_te, eps_lb, params(), fl)[0].tensor.mean().item()
               for a, fl in FLOWS.items()}
    assert abs(got["kernel"] - got["torch"]) <= 1e-4 * max(1.0, abs(got["torch"])), got

    cases = flow_cases(Z_DIM, [128, 400000]) + flow_cases(128, [128, 400000])
    for arm, flow in FLOWS.items():
        P = params()
        opt = torch.optim.Adam(flat(P), lr=1e-3)

        def step(P=P, opt=opt, flow=flow):
            lb, _ = example(x_tr, eps_tr, P, flow)
            cost = lb.sgvb().mean()
            opt.zero_grad(set_to_none=True)
            cost.backward()
            opt.step()
        cases.append(dict(case="train", arm=arm, d=Z_DIM, rows=128, fn=step))
    for arm, flow in FLOWS.items():
        P = params()

        def test(P=P, flow=flow):
            with torch.no_grad():
                lb, _ = example(x_te, eps_lb, P, flow)
                _, is_ll = example(x_te, eps_is, P, flow)
                return lb.tensor.mean(), is_ll().mean()
        cases.append(dict(case="test", arm=arm, d=Z_DIM, rows=400, fn=test))

    for c in cases:
        c["launches"], c["flow_kernel_us"] = profiled(c["fn"])
        c["times"] = []
    for _ in range(args.rounds):                       # arms alternate within each round
        for c in cases:
            c["times"].append(timed(c["fn"], args.iters, args.warmup))
    for c in cases:
        ts = sorted(c["times"])
        ms = ts[len(ts) // 2]
        rec = dict(case=c["case"], arm=c["arm"], d=c["d"], rows=c["rows"], ms=round(ms, 4),
                   ms_min=round(ts[0], 4), ms_max=round(ts[-1], 4), launches=c["launches"])
        if c["flow_kernel_us"]:
            rec["flow_kernel_us"] = c["flow_kernel_us"]
        if "flops" in c:
            rec.update(flops=c["flops"], gflops=round(c["flops"] / (ms * 1e-3) / 1e9, 1),
                       bytes=c["bytes"], gbps=round(c["bytes"] / (ms * 1e-3) / 1e9, 1))
        rec.update(info)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
