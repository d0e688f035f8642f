#!/usr/bin/env python
"""Config 3 (BASELINE.json): VAE 784-(500,500)-40, IWAE K=64 particles, batch
4096, SGVB reparameterised gradient (examples/variational_autoencoders/
iwae.py:23-78).  Unit: particle-ELBOs/s = K*N per step, forward + backward.

Generic path of this repo: BayesianNet / StochasticTensor wiring, the Normal
and Bernoulli log-prob kernels (+ analytic backward), the reparameterised
sampler and the log_mean_exp kernel are libzsb200; the dense layers are
torch.nn.functional.linear (cuBLAS = library code).  A fused decoder GEMM with
a Bernoulli epilogue is round-2 work (DESIGN.md section 6).
"""
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402


def glorot(rng, n_in, n_out, dev):
    lim = np.sqrt(6.0 / (n_in + n_out))          # tf.layers.dense default init
    return torch.tensor(rng.uniform(-lim, lim, (n_out, n_in)), dtype=torch.float32,
                        device=dev).requires_grad_(True)


def build(dev, seed=5, x_dim=784, z_dim=40, h=500):
    rng = np.random.Generator(np.random.PCG64(seed))
    W = {}
    for name, (i, o) in dict(e1=(x_dim, h), e2=(h, h), em=(h, z_dim), es=(h, z_dim),
                             d1=(z_dim, h), d2=(h, h), d3=(h, x_dim)).items():
        W[name] = glorot(rng, i, o, dev)
        W[name + "_b"] = torch.zeros(o, device=dev, requires_grad=True)
    return W


def step_fn(W, x, K, dev, fused=False):
    n, x_dim = x.shape
    z_dim = W["em"].shape[0]
    if fused:      # every dense layer on the wgmma kernel; Bernoulli fused into the last GEMM
        lin = lambda h, w, b, relu=False: zs.fused.linear(h, w, b, relu=relu)
    else:
        lin = lambda h, w, b, relu=False: (F.relu(F.linear(h, w, b)) if relu
                                           else F.linear(h, w, b))

    def step():
        # fresh leaves every step (views of the parameters, no copy): under CUDA-graph capture the
        # autograd engine then works on the capturing stream only (a leaf created on the legacy
        # stream would make that stream depend on the capture)
        Wd = {k: v.detach().requires_grad_(True) for k, v in W.items()}

        @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
        def build_gen(n, n_particles):                                   # iwae.py:23-32
            bn = zs.BayesianNet()
            z = bn.normal("z", torch.zeros(n, z_dim, device=dev), std=1., group_ndims=1,
                          n_samples=n_particles)
            hh = lin(z.tensor, Wd["d1"], Wd["d1_b"], True)
            hh = lin(hh, Wd["d2"], Wd["d2_b"], True)
            if fused:
                bn.stochastic("x", zs.fused.LinearBernoulli(hh, Wd["d3"], Wd["d3_b"]))
            else:
                bn.bernoulli("x", F.linear(hh, Wd["d3"], Wd["d3_b"]), group_ndims=1)
            return bn

        def build_q_net(x, n_particles):                                 # iwae.py:35-44
            bn = zs.BayesianNet()
            hh = lin(x.float(), Wd["e1"], Wd["e1_b"], True)
            hh = lin(hh, Wd["e2"], Wd["e2_b"], True)
            bn.normal("z", lin(hh, Wd["em"], Wd["em_b"]), logstd=lin(hh, Wd["es"], Wd["es_b"]),
                      group_ndims=1, n_samples=n_particles)
            return bn

        model = build_gen(n, K)
        variational = build_q_net(x, K)
        lb = zs.variational.iw_objective(model, {'x': x}, variational=variational, axis=0)
        cost = torch.mean(lb.sgvb())                                     # iwae.py:72-75
        grads = torch.autograd.grad(cost, list(Wd.values()))
        return cost.detach(), grads
    return step


def main():
    # one process per GPU under torchrun: the batch axis is sharded (weak scaling: 4096 data per
    # GPU), particles stay local, ONE all-reduce of the packed gradient + bound per step
    # (SURVEY 8e; zhusuan_b200/dist.py)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        import torch.distributed as td
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        td.init_process_group("nccl")
    dev = torch.device("cuda")
    K, N = 64, 4096
    rng = np.random.Generator(np.random.PCG64(4 + rank))
    x = torch.tensor(rng.random((N, 784)) < 0.13, dtype=torch.int32, device=dev)
    out = {"n_gpus": world, "batch_per_gpu": N}
    grads = {}
    for mode in ("fp32_matmul", "tf32_matmul", "wgmma_split_fused"):
        tf32 = mode == "tf32_matmul"
        torch.backends.cuda.matmul.allow_tf32 = tf32
        W = build(dev)
        zs.set_random_seed(1234)           # same eps in every mode
        local_step = step_fn(W, x, K, dev, fused=(mode == "wgmma_split_fused"))

        def step():
            cost, g = local_step()
            if world > 1:
                g, (cost,) = zs.dist.all_reduce_mean_gradients(g, [cost.detach()], n_local=N)
            return cost, g
        for _ in range(3):
            cost, g = step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        steps = 10
        e0.record()
        for _ in range(steps):
            cost, g = step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        if world > 1:                      # max over ranks, whole-job throughput
            t = torch.tensor([ms], device=dev)
            td.all_reduce(t, op=td.ReduceOp.MAX)
            ms = float(t.item())
        grads[mode] = torch.cat([t.reshape(-1) for t in g]).double()
        out[mode] = {
            "ms_per_step": ms, "particle_elbos_per_s": world * K * N / (ms * 1e-3),
            "tflops_dense_layers": world * 3.97e6 * K * N / (ms * 1e-3) / 1e12,
            "bound_value": float(-cost)}
    ref = grads["fp32_matmul"]
    for mode in ("tf32_matmul", "wgmma_split_fused"):
        out[mode]["grad_rel_err_vs_fp32"] = float((grads[mode] - ref).norm() / ref.norm())
    if rank != 0:
        td.destroy_process_group()
        return
    # CPU baseline: the same graph in torch-CPU (restatement of the TF graph), small batch
    torch.backends.cuda.matmul.allow_tf32 = False
    Nc = 128
    cpu_step = make_cpu_step(x[:Nc].cpu().float(), K)
    cpu_step()
    t0 = time.perf_counter()
    for _ in range(3):
        cpu_step()
    dt = (time.perf_counter() - t0) / 3
    out["cpu_port"] = {"particle_elbos_per_s": K * Nc / dt, "cores": torch.get_num_threads(),
                       "sample": "batch %d of 4096, K=64, torch-CPU restatement of iwae.py" % Nc}
    print(json.dumps(out))
    if world > 1:
        td.destroy_process_group()


def make_cpu_step(xc, K, seed=5):
    """The graph of iwae.py:23-78 op by op in torch-CPU (forward + SGVB backward): the CPU arm
    of bench.py --workload iwae (TensorFlow is not installable here, so kind = "port")."""
    Nc = xc.shape[0]
    Wc = {k: v.detach().cpu().requires_grad_(True)
          for k, v in build(torch.device("cpu"), seed=seed).items()}
    eps = torch.randn(K, Nc, 40)

    def cpu_step():
        h = F.relu(F.linear(xc, Wc["e1"], Wc["e1_b"])); h = F.relu(F.linear(h, Wc["e2"], Wc["e2_b"]))
        zm, zl = F.linear(h, Wc["em"], Wc["em_b"]), F.linear(h, Wc["es"], Wc["es_b"])
        z = zm + torch.exp(zl) * eps
        c = -0.5 * np.log(2 * np.pi)
        log_q = (c - zl - 0.5 * torch.exp(-2 * zl) * (z - zm) ** 2).sum(-1)
        log_pz = (c - 0.5 * z ** 2).sum(-1)
        hh = F.relu(F.linear(z, Wc["d1"], Wc["d1_b"])); hh = F.relu(F.linear(hh, Wc["d2"], Wc["d2_b"]))
        logits = F.linear(hh, Wc["d3"], Wc["d3_b"])
        log_px = -F.binary_cross_entropy_with_logits(logits, xc.expand(K, -1, -1), reduction="none").sum(-1)
        lw = log_pz + log_px - log_q
        cost = -(torch.logsumexp(lw, 0) - np.log(K)).mean()
        return torch.autograd.grad(cost, list(Wc.values()))
    return cpu_step


if __name__ == "__main__":
    main()
