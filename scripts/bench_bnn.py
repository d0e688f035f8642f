#!/usr/bin/env python
"""Config 4 (BASELINE.json): BNN regression [10 -> 50 -> 1], SGHMC 2nd order,
8192 chains, minibatch 100 (examples/bayesian_neural_nets/bnn_sgmcmc.py).
Times the fused kernel and the generic path; unit = chains*steps / s.

    --method sgld | psgld | sgnht | sgnht_scalar   the example's alternative samplers
    (bnn_sgmcmc.py:81-84; PSGLD takes SGLD's learning rate), same problem and output."""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402


# sampler per --method (bnn_sgmcmc.py:81-84) and the bytes each must move per weight and
# chain-step: q r+w (SGLD); q and aux / v r+w (PSGLD, SGHMC); q, v r+w and k written (scalar
# SGNHT); q, v, alpha r+w and k written (vector SGNHT)
METHODS = {
    "sghmc": (lambda: zs.SGHMC, dict(learning_rate=2e-6, friction=0.2, n_iter_resample_v=1000,
                                     second_order=True), 16),
    "sgld": (lambda: zs.SGLD, dict(learning_rate=4e-6), 8),
    "psgld": (lambda: zs.PSGLD, dict(learning_rate=4e-6), 16),
    "sgnht": (lambda: zs.SGNHT, dict(learning_rate=1e-5, variance_extra=0., tune_rate=50.,
                                     second_order=True), 28),
    "sgnht_scalar": (lambda: zs.SGNHT, dict(learning_rate=1e-5, variance_extra=0., tune_rate=50.,
                                            second_order=True, use_vector_alpha=False), 20),
}


def run(fused, C=8192, steps=200, warm=20, method="sghmc"):
    torch.manual_seed(8)
    n_in, H, B, n_train = 10, 50, 100, 10000
    x_all = torch.randn(n_train, n_in, device="cuda")
    y_all = torch.sin(x_all.sum(1)) + 0.1 * torch.randn(n_train, device="cuda")
    ls = [torch.zeros(H, n_in + 1, device="cuda"), torch.zeros(1, H + 1, device="cuda")]
    w0 = torch.rand(C, H, n_in + 1, device="cuda") * 4 - 2          # bnn_sgmcmc.py:68-69
    w1 = torch.rand(C, 1, H + 1, device="cuda") * 4 - 2
    lj = zs.fused.BNNRegressionLogJoint(x_all[:B], y_all[:B], ls, n_train)
    cls, kw, bytes_per_weight = METHODS[method]
    sg = cls()(seed=1, use_fused=fused, **kw)                          # bnn_sgmcmc.py:81-84
    op, info = sg.sample(lj, {}, {"w0": w0, "w1": w1})
    batches = [(x_all[i * B:(i + 1) * B].contiguous(), y_all[i * B:(i + 1) * B].contiguous())
               for i in range(n_train // B)]
    for i in range(warm):
        xb, yb = batches[i % len(batches)]
        op(observed={"x": xb, "y": yb})
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for i in range(steps):
        xb, yb = batches[i % len(batches)]
        op(observed={"x": xb, "y": yb})
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    out = {"path": "fused" if fused else "generic", "chains": C, "ms_per_step": ms,
           "chain_steps_per_s": C / (ms * 1e-3),
           "hbm_GBps_algorithmic": C * bytes_per_weight * 601 / (ms * 1e-3) / 1e9}
    if method == "sghmc":
        out["mean_k_w0"] = float(info.mean_k["w0"])
    else:
        out = dict({"method": method}, **out)
        if hasattr(info, "mean_k"):
            out["mean_k_w0"] = float(info.mean_k["w0"].mean())
    out["finite"] = bool(torch.isfinite(w0).all())
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--method", choices=sorted(METHODS), default="sghmc")
    m = ap.parse_args().method
    print(json.dumps(run(True, method=m)))
    print(json.dumps(run(False, steps=20, warm=3, method=m)))
