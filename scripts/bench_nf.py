#!/usr/bin/env python
"""Planar normalizing flows and the normalizing-flow VAE of examples/normalizing_flows/vae_nf.py,
arms run in one process and alternating.  Prints one JSON line per case and arm, with the card's
name and power limit read in the same run.

    flows     two stacks of 10 planar flows at d = 40 (vae_nf.py's z_dim), forward ("fwd") and
              forward plus backward ("fwd_bwd"), at 128 rows (a training batch) and 4e5 rows (the IS
              evaluation's 1000 particles x 400 rows).  Arms:
                kernel  zs.planar_normalizing_flow (one launch per stack forward, two backward)
                torch   the reference's op sequence (transform.py:161-194) in float32 torch
              `launches` is the number of GPU kernels per call, counted with torch.profiler in a
              run of its own; the same run gives `flow_kernel_us`, the device time per call of the
              flow kernels (forward, backward sweep, merge), summed over both stacks.  `bytes` is
              the least traffic from the shapes, the same for both arms: z and log_q read and
              written once per stack, and in the backward their gradients.
              `bytes_kernel` adds what the kernels keep for the backward pass (every flow's input
              z, written forward and read backward).  `gbps` = bytes / ms against 3350 GB/s.
    train     the vae_nf.py training step: 128 rows, 1 particle, [784, 500, 500], z_dim 40, 2 x 10
              flows, elbo(...).sgvb(), backward, Adam(1e-3); ms per step
    test      the test-set bound (1 particle) plus the IS estimate at 1000 particles over 400 rows,
              under torch.no_grad(); ms per batch
              Arms of train and test:
                fused        zs.fused.linear / LinearBernoulli and zs.planar_normalizing_flow
                fused_torch  zs.fused layers and the flows in torch (isolates the flow)
                generic      F.linear and the flows in torch
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

X_DIM, H, Z_DIM, N_FLOWS = 784, 500, 40, 10
HBM_GBPS = 3350.0


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def torch_flow(z, log_q, b, aux_u, w):
    """transform.py:161-194 op for op in torch."""
    d = z.shape[-1]
    lead = z.shape[:-1]
    z = z.reshape(-1, d)
    log_q = log_q.reshape(-1)
    for k in range(b.shape[0]):
        wk, ak = w[k].unsqueeze(1), aux_u[k].unsqueeze(1)
        dot = wk.t() @ ak
        u = (ak + wk / (wk.t() @ wk) * (torch.log(torch.exp(dot) + 1) - 1 - dot)).t()
        scalar = (u @ wk).reshape(())
        a = torch.tanh(z @ wk + b[k])
        ra = a.sum(-1)
        log_q = log_q - torch.log(scalar * (1 - ra * ra) + 1)
        z = z + a @ u
    return z.reshape(lead + (d,)), log_q.reshape(lead)


def kernel_flow(z, log_q, b, aux_u, w):
    return zs.planar_normalizing_flow(z, log_q, int(b.shape[0]), b, aux_u, w)


FLOWS = {"kernel": kernel_flow, "torch": torch_flow}


def lin_of(fused):
    if fused:
        return lambda h, W, b, relu=False: zs.fused.linear(h, W, b, relu=relu)
    return lambda h, W, b, relu=False: torch.relu(F.linear(h, W, b)) if relu else F.linear(h, W, b)


def example(x, eps, P, fused, flow):
    """vae_nf.py:19-85 on zs; returns (elbo objective, is_loglikelihood thunk)."""
    q, p, flows = P
    lin = lin_of(fused)
    S, n, z_dim = eps.shape

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, z_dim, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        h = lin(lin(z, p[0], p[1], True), p[2], p[3], True)
        if fused:
            bn.stochastic("x", zs.fused.LinearBernoulli(h, p[4], p[5], dtype=torch.float32))
        else:
            bn.bernoulli("x", F.linear(h, p[4], p[5]), group_ndims=1, dtype=torch.float32)
        return bn

    h = lin(lin(x, q[0], q[1], True), q[2], q[3], True)
    mean, logstd = lin(h, q[4], q[5]), lin(h, q[6], q[7])
    qz = mean + torch.exp(logstd) * eps
    log_qz = zs.distributions.Normal(mean, logstd=logstd, group_ndims=1).log_prob(qz)
    for b, u, w in flows:
        qz, log_qz = flow(qz, log_qz, b, u, w)
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
    flows = [zs.planar_flow_parameters(Z_DIM, N_FLOWS, generator=g) for _ in range(2)]
    return q, p, flows


def flat(P):
    return P[0] + P[1] + [t for f in P[2] for t in f]


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
    """(GPU kernels per call, {flow kernel: device microseconds per call}) from torch.profiler."""
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
            if "planar_flow_%s_kernel" % part in e.name:
                us[part] = us.get(part, 0.0) + e.time_range.elapsed_us()
    return len(kernels), {k: round(v, 1) for k, v in us.items()}


def flow_cases(rows_list):
    cases = []
    g = torch.Generator(device="cuda").manual_seed(3)
    fl = [[t.detach() for t in zs.planar_flow_parameters(Z_DIM, N_FLOWS, generator=g)]
          for _ in range(2)]
    for R in rows_list:
        z = torch.randn(R, Z_DIM, device="cuda", generator=g)
        lq = torch.randn(R, device="cuda", generator=g)
        gz, gl = torch.randn_like(z), torch.randn_like(lq)
        for arm, flow in FLOWS.items():
            def fwd(flow=flow, z=z, lq=lq):
                with torch.no_grad():
                    a, b_ = z, lq
                    for f in fl:
                        a, b_ = flow(a, b_, *f)
                return a, b_

            ps = [[t.clone().requires_grad_(True) for t in f] for f in fl]
            zi, li = z.clone().requires_grad_(True), lq.clone().requires_grad_(True)

            def fwd_bwd(flow=flow, ps=ps, zi=zi, li=li, gz=gz, gl=gl):
                a, b_ = zi, li
                for f in ps:
                    a, b_ = flow(a, b_, *f)
                torch.autograd.backward((a, b_), (gz, gl))
            base = 2 * (8 * R * Z_DIM + 8 * R)
            ck = 2 * 4 * N_FLOWS * R * Z_DIM
            cases.append(("flows_fwd", arm, R, fwd, base, base))
            cases.append(("flows_fwd_bwd", arm, R, fwd_bwd, 2 * base - 8 * R,
                          2 * base - 8 * R + 2 * ck))
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_nf.py needs a CUDA device")
    info = card()
    g = torch.Generator(device="cuda").manual_seed(1)
    x_tr = (torch.rand(128, X_DIM, device="cuda", generator=g) < 0.3).float()
    eps_tr = torch.randn(1, 128, Z_DIM, device="cuda", generator=g)
    x_te = (torch.rand(400, X_DIM, device="cuda", generator=g) < 0.3).float()
    eps_lb = torch.randn(1, 400, Z_DIM, device="cuda", generator=g)
    eps_is = torch.randn(1000, 400, Z_DIM, device="cuda", generator=g)
    arms = {"fused": (True, kernel_flow), "fused_torch": (True, torch_flow),
            "generic": (False, torch_flow)}

    # every arm computes the same bound: check it once before timing
    with torch.no_grad():
        got = {a: example(x_te, eps_lb, params(), f, fl)[0].tensor.mean().item()
               for a, (f, fl) in arms.items()}
    assert max(got.values()) - min(got.values()) <= 1e-4 * max(1.0, abs(got["generic"])), got

    cases = []
    for c, arm, rows, fn, nb, nbk in flow_cases([128, 400000]):
        cases.append(dict(case=c, arm=arm, rows=rows, fn=fn, bytes=nb, bytes_kernel=nbk))
    for arm, (fused, flow) in arms.items():
        P = params()
        opt = torch.optim.Adam(flat(P), lr=1e-3)

        def step(P=P, opt=opt, fused=fused, flow=flow):
            lb, _ = example(x_tr, eps_tr, P, fused, flow)
            cost = lb.sgvb().mean()
            opt.zero_grad(set_to_none=True)
            cost.backward()
            opt.step()
        cases.append(dict(case="train", arm=arm, rows=128, fn=step))
    for arm, (fused, flow) in arms.items():
        P = params()

        def test(P=P, fused=fused, flow=flow):
            with torch.no_grad():
                lb, _ = example(x_te, eps_lb, P, fused, flow)
                _, is_ll = example(x_te, eps_is, P, fused, flow)
                return lb.tensor.mean(), is_ll().mean()
        cases.append(dict(case="test", arm=arm, rows=400, fn=test))

    for c in cases:
        c["launches"], c["flow_kernel_us"] = profiled(c["fn"])
        c["times"] = []
    for _ in range(args.rounds):                       # arms alternate within each round
        for c in cases:
            c["times"].append(timed(c["fn"], args.iters, args.warmup))
    for c in cases:
        ts = sorted(c["times"])
        ms = ts[len(ts) // 2]
        rec = dict(case=c["case"], arm=c["arm"], rows=c["rows"], ms=round(ms, 4),
                   ms_min=round(ts[0], 4), ms_max=round(ts[-1], 4), launches=c["launches"])
        if c["flow_kernel_us"]:
            rec["flow_kernel_us"] = c["flow_kernel_us"]
        if "bytes" in c:
            gbps = c["bytes"] / (ms * 1e-3) / 1e9
            rec.update(bytes=c["bytes"], bytes_kernel=c["bytes_kernel"], gbps=round(gbps, 1),
                       hbm_share=round(gbps / HBM_GBPS, 4))
        rec.update(info)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
