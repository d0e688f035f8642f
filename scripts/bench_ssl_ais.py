#!/usr/bin/env python
"""The one-hot categorical layer of examples/semi_supervised_vae/vae_ssl_adaptive_is.py
(qy_x's last layer, 500 -> 10 classes) on zs.fused.LinearOnehotCategorical against the registry's
OnehotCategorical fed by the fused dense layer and by F.linear.  Prints one JSON line per case and
arm, with the card's name and power limit read in the same run.

    sample_logq   y = onehot_categorical(dense(h)) at R = 4e5 rows, H = 500, C = 10: the draw, its
                  log q, and the gradients of sum(log q) w.r.t. h, W and b
    classifier    the classifier cost -mean(log p(y_label | x)) at R = 4e5 rows and its gradients

Arms: fused (LinearOnehotCategorical), fused_linear_registry (OnehotCategorical(zs.fused.linear))
and torch_linear_registry (OnehotCategorical(F.linear)).  The arms alternate window by window in
one process; each line gives the median, fastest and slowest window in ms per call, and, from a
separate torch.profiler pass, kernel launches per call and the device time of each tensor-core
product launch (product_ms, keyed by epilogue family and number: CatEpi12 / 13 sample or score and
CatEpi14 forms d/dlogits, RowsEpi0 is the dense layer's forward product, _mn1 / _mn3 the input and
weight gradients).  FLOPs and bytes come from the shapes: model_flops = 6 R H C (a forward product
of 2 R H C and two gradient products); flops, the work the arm does, adds 2 R H C for the fused arm,
whose backward pass forms the logits a second time (CatEpi14); tflops is flops over the median
time.  Bytes: h and its gradient, the one-hot rows, labels and log q, in fp32.
"""
import json
import os
import re
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

R, H, C = 400000, 500, 10
ARMS = ("fused", "fused_linear_registry", "torch_linear_registry")


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": name, "power_limit": pl or "unknown"}


def dist(arm, h, W, b):
    if arm == "fused":
        return zs.fused.LinearOnehotCategorical(h, W, b)
    lin = zs.fused.linear if arm == "fused_linear_registry" else F.linear
    return zs.distributions.OnehotCategorical(lin(h, W, b))


def make_case(case, arm, h, W, b, labels):
    params = (h, W, b)

    def sample_logq():
        d = dist(arm, h, W, b)
        y = d.sample()
        return torch.autograd.grad(d.log_prob(y).sum(), params)

    def classifier():
        cost = -dist(arm, h, W, b).log_prob(labels).mean()
        return torch.autograd.grad(cost, params)
    return sample_logq if case == "sample_logq" else classifier


def profile_pass(fn):
    """Kernel launches per call, and the device time per call (ms) of each tensor-core product,
    keyed by its epilogue family and number (e.g. CatEpi12, RowsEpi0), from one torch.profiler
    pass."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type.name == "CUDA"]
    products = {}
    for e in kernels:
        # demangled: ...LinW<(anonymous namespace)::CatEpi, 12, 0, 0>...
        m = re.search(r"LinW<(?:\(anonymous namespace\)::)?(\w+Epi), (\d+), (\d+)", e.name)
        if m:
            mn = "" if m.group(3) == "0" else "_mn" + m.group(3)
            key = m.group(1) + m.group(2) + mn
            products[key] = products.get(key, 0.0) + e.time_range.elapsed_us() / 1e3
    return len(kernels), {k: round(v, 4) for k, v in sorted(products.items())}


def main():
    torch.manual_seed(0)
    info = card()
    h = torch.randn(R, H, device="cuda").requires_grad_()
    W = (torch.randn(C, H, device="cuda") / H ** 0.5).requires_grad_()
    b = torch.zeros(C, device="cuda").requires_grad_()
    labels = F.one_hot(torch.randint(C, (R,), device="cuda"), C).to(torch.float32)
    for case in ("sample_logq", "classifier"):
        fns = {a: make_case(case, a, h, W, b, labels) for a in ARMS}
        nbytes = 4 * (2 * R * H + 2 * R * C + R)
        for fn in fns.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        windows = {a: [] for a in ARMS}
        for _ in range(7):
            for a in ARMS:
                e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                e0.record()
                for _ in range(10):
                    fns[a]()
                e1.record()
                torch.cuda.synchronize()
                windows[a].append(e0.elapsed_time(e1) / 10)
        for a in ARMS:
            ms = statistics.median(windows[a])
            n_launch, products = profile_pass(fns[a])
            flops = (8 if a == "fused" else 6) * R * H * C
            print(json.dumps(dict(info, case=case, arm=a, rows=R, H=H, C=C,
                                  ms=round(ms, 4), ms_min=round(min(windows[a]), 4),
                                  ms_max=round(max(windows[a]), 4), launches=n_launch,
                                  product_ms=products, model_flops=6 * R * H * C, flops=flops,
                                  bytes=nbytes, tflops=round(flops / ms / 1e9, 2),
                                  gbps=round(nbytes / ms / 1e6, 1))), flush=True)


if __name__ == "__main__":
    main()
