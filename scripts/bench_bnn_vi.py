#!/usr/bin/env python
"""The fused BNN log-joint (csrc/bnn_logjoint.cu) in the four uses it was built for, each on the
fused path and on the generic path (``lambda o: lj(o)``: the torch restatement under autograd).
Prints one JSON line per case, with the card's name and power limit read in the same run.

    bnn_vi_step   examples/bayesian_neural_nets/bnn_vi.py's training step: K = 10 particles,
                  B = 10 rows, [13, 50, 1], n_train = 455; sample, ELBO, .sgvb().backward()
                  and torch.optim.Adam, ms per step
    value_grad    value and gradient at config 4's shape: K = 8192, B = 100, [10, 50, 1];
                  particle-gradients / s, beside the fused SGHMC step (scripts/bench_bnn.py),
                  which does the same forward and backward work plus an update
    predictive    test-set evaluation: y_mean and log-likelihood at K = 5000, N = 4096 rows
    hmc           one full-batch HMC iteration: 1024 chains, B = 455, L = 10
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402


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


def problem(n_in, H, B, n_train, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, n_in, device="cuda", generator=g)
    y = torch.sin(x.sum(1)) + 0.1 * torch.randn(B, device="cuda", generator=g)
    return x, y


def bnn_vi_step(fused, iters=300, warm=30):
    n_in, H, K, B, n_train = 13, 50, 10, 10, 455
    x_all, y_all = problem(n_in, H, n_train, n_train)
    batches = [(x_all[i:i + B].contiguous(), y_all[i:i + B].contiguous())
               for i in range(0, n_train - B + 1, B)]
    y_logstd = torch.zeros((), device="cuda", requires_grad=True)          # bnn_vi.py:32-34
    params = [torch.zeros(H, n_in + 1, device="cuda", requires_grad=True),
              torch.zeros(H, n_in + 1, device="cuda", requires_grad=True),
              torch.zeros(1, H + 1, device="cuda", requires_grad=True),
              torch.zeros(1, H + 1, device="cuda", requires_grad=True)]
    zero = torch.zeros((), device="cuda")
    lj = zs.fused.BNNRegressionLogJoint(batches[0][0], batches[0][1], [zero, zero], n_train,
                                        y_logstd=y_logstd)
    model = lj if fused else (lambda o: lj(o))
    opt = torch.optim.Adam(params + [y_logstd], lr=0.01)                  # bnn_vi.py:91
    state = {"i": 0, "lb": None}

    def step():
        xb, yb = batches[state["i"] % len(batches)]
        state["i"] += 1
        q = zs.BayesianNet()                                               # bnn_vi.py:38-50
        for i in range(2):
            q.normal("w%d" % i, params[2 * i], logstd=params[2 * i + 1], n_samples=K,
                     group_ndims=2)
        lb = zs.variational.elbo(model, {"x": xb, "y": yb}, variational=q, axis=0)
        cost = lb.sgvb()
        opt.zero_grad()
        cost.backward()
        opt.step()
        state["lb"] = lb.tensor
    ms = timed(step, iters, warm)
    return {"case": "bnn_vi_step", "path": "fused" if fused else "generic", "K": K, "B": B,
            "layers": [n_in, H, 1], "ms_per_step": ms,
            "lower_bound": float(state["lb"].detach()),
            "finite": bool(torch.isfinite(y_logstd).all())}


def value_grad(fused, iters=200, warm=20):
    n_in, H, K, B, n_train = 10, 50, 8192, 100, 10000
    x, y = problem(n_in, H, B, n_train, seed=1)
    zero = torch.zeros((), device="cuda")
    lj = zs.fused.BNNRegressionLogJoint(x, y, [zero, zero], n_train)
    g = torch.Generator(device="cuda").manual_seed(2)
    w0 = (torch.rand(K, H, n_in + 1, device="cuda", generator=g) * 4 - 2).requires_grad_(True)
    w1 = (torch.rand(K, 1, H + 1, device="cuda", generator=g) * 4 - 2).requires_grad_(True)
    obs = {"w0": w0, "w1": w1}

    def step():
        lp = lj.fused_log_joint(obs) if fused else lj(obs)
        torch.autograd.grad(lp.sum(), [w0, w1])
    ms = timed(step, iters if fused else iters // 10, warm if fused else 3)
    out = {"case": "value_grad", "path": "fused" if fused else "generic", "K": K, "B": B,
           "layers": [n_in, H, 1], "ms_per_call": ms, "particle_grads_per_s": K / (ms * 1e-3)}
    if fused:
        # the kernel alone (one zsb_bnn_logjoint_f32 launch writing lp, g0 and g1)
        ys = lj._y_logstd_dev(w0.device)
        kern = timed(lambda: lj._launch(w0, w1, x, y, ys, lp=True, g0=True, g1=True), iters,
                     warm)
        out.update(kernel_ms=kern, kernel_particle_grads_per_s=K / (kern * 1e-3))
        # the fused SGHMC step of scripts/bench_bnn.py on the same shape, in the same run
        sg = zs.SGHMC(learning_rate=2e-6, friction=0.2, n_iter_resample_v=1000,
                      second_order=True, seed=1)
        q0, q1 = w0.detach().clone(), w1.detach().clone()
        op, _ = sg.sample(lj, {}, {"w0": q0, "w1": q1})
        assert sg._fused_bnn() is not None
        out["sghmc_step_ms"] = timed(op, iters, warm)
    return out


def predictive(fused, iters=50, warm=5):
    n_in, H, K, N, n_train = 13, 50, 5000, 4096, 455
    x, y = problem(n_in, H, N, n_train, seed=3)
    zero = torch.zeros((), device="cuda")
    lj = zs.fused.BNNRegressionLogJoint(x, y, [zero, zero], n_train, y_logstd=-1.0)
    g = torch.Generator(device="cuda").manual_seed(4)
    obs = {"w0": torch.randn(K, H, n_in + 1, device="cuda", generator=g),
           "w1": torch.randn(K, 1, H + 1, device="cuda", generator=g)}

    def fused_eval():
        return lj.predictive(obs)

    def generic_eval():
        with torch.no_grad():                 # bnn_vi.py:98-103 in torch
            w0, w1 = obs["w0"], obs["w1"]
            h = torch.cat([x, torch.ones(N, 1, device="cuda")], -1)
            h = torch.relu(torch.einsum("imk,jk->ijm", w0, h) / (n_in + 1) ** 0.5)
            h = torch.cat([h, torch.ones(K, N, 1, device="cuda")], -1)
            ym = torch.einsum("imk,ijk->ijm", w1, h).squeeze(2) / (H + 1) ** 0.5
            ll = zs.distributions.Normal(ym, logstd=torch.full_like(ym, -1.0)).log_prob(y)
            return ym, ll
    fn = fused_eval if fused else generic_eval
    ms = timed(fn, iters, warm)
    ym, ll = fn()
    return {"case": "predictive", "path": "fused" if fused else "generic", "K": K, "N": N,
            "layers": [n_in, H, 1], "ms_per_call": ms,
            "particle_rows_per_s": K * N / (ms * 1e-3),
            "test_ll": float((torch.logsumexp(ll, 0) - torch.log(torch.tensor(float(K)))).mean())}


def hmc(fused, iters=20, warm=3):
    n_in, H, C, B, L = 13, 50, 1024, 455, 10
    x, y = problem(n_in, H, B, B, seed=5)
    zero = torch.zeros((), device="cuda")
    lj = zs.fused.BNNRegressionLogJoint(x, y, [zero, zero], B, y_logstd=-1.0)
    g = torch.Generator(device="cuda").manual_seed(6)
    w0 = 0.3 * torch.randn(C, H, n_in + 1, device="cuda", generator=g)
    w1 = 0.3 * torch.randn(C, 1, H + 1, device="cuda", generator=g)
    h = zs.HMC(step_size=1e-3, n_leapfrogs=L)
    op, info = h.sample(lj if fused else (lambda o: lj(o)), {}, {"w0": w0, "w1": w1})
    assert (h._provider is not None) == fused
    ms = timed(op, iters, warm)
    return {"case": "hmc", "path": "fused" if fused else "generic", "chains": C, "B": B, "L": L,
            "layers": [n_in, H, 1], "ms_per_iter": ms,
            "acceptance_mean": float(info.acceptance_rate.mean())}


if __name__ == "__main__":
    c = card()
    for case in (bnn_vi_step, value_grad, predictive, hmc):
        for fused in (True, False):
            print(json.dumps(dict(case(fused), **c)), flush=True)
