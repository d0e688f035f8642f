"""The GANs of examples/generative_adversarial_nets (dcgan.py, wasserstein_gan.py) on
zs.fused.bn_conv2d / bn_conv2d_transpose / sigmoid_conv2d_transpose against cuDNN convolutions with
the same TF pads, on seeded synthetic data.  Arms (alternating in one process):
  fused       the fused layers (tests/gan_models.py on zs.fused)
  cudnn_fp32  F.conv2d / F.conv_transpose2d with TF's asymmetric pads (F.pad, crop), allow_tf32 =
              False, batch norm and activations in torch: the accuracy-matched arm
  cudnn_tf32  the same with cuDNN in TF32: NOT accuracy-matched
Cases:
  {dcgan,wgan}_<layer>_{fwd,fwdbwd}_{batch,4096}  every conv layer of both networks, at the
      example's batch (32 / 64) and at 4096 images
  {dcgan,wgan}_step       one training step (DCGAN: batch 32, Adam(2e-4, beta1 0.5); WGAN: batch
                          64, TF-form RMSProp(decay 0.5) and weight clipping)
  {dcgan,wgan}_gen100     eval_x_gen: 100 images from the prior in evaluation mode
  {dcgan,wgan}_gen1e5     1e5 images, in chunks of 10,000
  conv3x3_64_fwdbwd_4096  a 3x3, 64-channel, stride-1 SAME layer at 4096 images of 14x14, on
                          bn_conv2d (fused) beside the FFMA zs.fused.conv2d + torch batch norm
                          (arm ffma_conv2d); reported only
Each prints the median, min and max over windows; launches per call and device time come from a
separate torch.profiler pass; conv FLOPs (2 * output pixels * k * k * Cin * Cout per product,
three products with the backward) and the bytes of the layer's tensors from the shapes.  One
JSON line per case and arm, with the card's name and power limit.

    python scripts/bench_gan.py [--windows 5] [--steps 10] [--cases a,b]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
import zhusuan_b200 as zs  # noqa: E402
import gan_models as GM  # noqa: E402

ARMS = ("fused", "cudnn_fp32", "cudnn_tf32")
Z_DIM = 40


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def _pads(big, small, k, s, padding):
    if padding == "VALID":
        return 0, 0
    t = max((small - 1) * s + k - big, 0)
    return t // 2, t - t // 2


class Cudnn(object):
    """The layers on cuDNN in NCHW (permuted NHWC views), batch norm in torch.  F.batch_norm
    moves the running variance with the Bessel-corrected batch variance: the fused rule."""

    def __init__(self, tf32):
        self.tf32 = tf32

    def _conv(self, x, W, s, padding):
        torch.backends.cudnn.allow_tf32 = self.tf32
        k = int(W.shape[0])
        H, Wd = int(x.shape[1]), int(x.shape[2])
        Ho = -(-H // s) if padding == "SAME" else -(-(H - k + 1) // s)
        Wo = -(-Wd // s) if padding == "SAME" else -(-(Wd - k + 1) // s)
        (pt, pb), (pl, pr) = _pads(H, Ho, k, s, padding), _pads(Wd, Wo, k, s, padding)
        xc = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
        return F.conv2d(xc, W.permute(3, 2, 0, 1), stride=s)[:, :, :Ho, :Wo]

    def _deconv(self, x, W, s, padding):
        torch.backends.cudnn.allow_tf32 = self.tf32
        k = int(W.shape[0])
        Hi, Wi = int(x.shape[1]), int(x.shape[2])
        grow = 0 if padding == "SAME" else max(k - s, 0)
        Ho, Wo = Hi * s + grow, Wi * s + grow
        pt, pl = _pads(Ho, Hi, k, s, padding)[0], _pads(Wo, Wi, k, s, padding)[0]
        y = F.conv_transpose2d(x.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1), stride=s)
        y = F.pad(y, (0, max(pl + Wo - int(y.shape[3]), 0), 0, max(pt + Ho - int(y.shape[2]), 0)))
        return y[:, :, pt:pt + Ho, pl:pl + Wo]

    @staticmethod
    def _bn(a, gamma, beta, mm, mv, training, relu, momentum, epsilon):
        if gamma is None:                   # scale=False (F.batch_norm's backward needs a weight)
            gamma = torch.ones_like(beta)
        y = F.batch_norm(a, mm, mv, gamma, beta, training, 1.0 - momentum, epsilon)
        return (torch.relu(y) if relu else y).permute(0, 2, 3, 1)

    def bn_conv2d(self, x, W, gamma, beta, mm, mv, training, stride=1, padding="SAME", relu=True,
                  momentum=0.99, epsilon=1e-3):
        return self._bn(self._conv(x, W, stride, padding), gamma, beta, mm, mv, training, relu,
                        momentum, epsilon)

    def bn_conv2d_transpose(self, x, W, gamma, beta, mm, mv, training, stride=1, padding="SAME",
                            relu=True, momentum=0.99, epsilon=1e-3):
        return self._bn(self._deconv(x, W, stride, padding), gamma, beta, mm, mv, training, relu,
                        momentum, epsilon)

    def sigmoid_conv2d_transpose(self, x, W, b=None, stride=1, padding="SAME"):
        y = self._deconv(x, W, stride, padding).permute(0, 2, 3, 1)
        return torch.sigmoid(y if b is None else y + b)

    @staticmethod
    def bn_linear(h, W, gamma, beta, mm, mv, training, relu=True, momentum=0.99, epsilon=1e-3):
        torch.backends.cuda.matmul.allow_tf32 = False
        a = F.linear(h, W)
        if training:
            mean, var = a.mean(0), a.var(0, unbiased=False)
            with torch.no_grad():
                mm.sub_((mm - mean) * (1 - momentum))
                mv.sub_((mv - var) * (1 - momentum))
        else:
            mean, var = mm, mv
        y = (a - mean) * torch.rsqrt(var + epsilon) * gamma + beta
        return torch.relu(y) if relu else y

    @staticmethod
    def linear(h, W, b=None, relu=False):
        y = F.linear(h, W, b)
        return torch.relu(y) if relu else y


def ops(arm):
    return zs.fused if arm == "fused" else Cudnn(arm == "cudnn_tf32")


# (name, transpose, k, stride, padding, in HWC, Cout, gamma) of every conv layer, at the examples'
# widths (DCGAN ngf 64, ndf 32; WGAN ngf 32, ndf 16)
LAYERS = {
    "dcgan": [("g1", True, 5, 2, "SAME", (4, 4, 512), 256, True),
              ("g2", True, 5, 2, "SAME", (8, 8, 256), 128, True),
              ("g3", True, 5, 2, "SAME", (16, 16, 128), 3, None),
              ("d0", False, 5, 2, "SAME", (32, 32, 3), 64, True),
              ("d1", False, 5, 2, "SAME", (16, 16, 64), 128, True),
              ("d2", False, 5, 2, "SAME", (8, 8, 128), 256, True)],
    "wgan": [("g0", True, 3, 1, "VALID", (1, 1, 40), 128, False),
             ("g1", True, 5, 1, "VALID", (3, 3, 128), 64, False),
             ("g2", True, 5, 2, "SAME", (7, 7, 64), 32, False),
             ("g3", True, 5, 2, "SAME", (14, 14, 32), 1, None),
             ("d0", False, 5, 2, "SAME", (28, 28, 1), 16, False),
             ("d1", False, 5, 2, "SAME", (14, 14, 16), 32, False),
             ("d2", False, 5, 1, "VALID", (7, 7, 32), 64, False)],
}
BATCH = {"dcgan": 32, "wgan": 64}


def _out_hw(transpose, k, s, pad, h):
    if transpose:
        return h * s + (0 if pad == "SAME" else max(k - s, 0))
    return -(-h // s) if pad == "SAME" else -(-(h - k + 1) // s)


def layer_cost(spec, n, backward):
    _, transpose, k, s, pad, (h, w, cin), cout, _ = spec
    ho, wo = _out_hw(transpose, k, s, pad, h), _out_hw(transpose, k, s, pad, w)
    small = n * (h * w if transpose else ho * wo)
    flops = 2 * small * k * k * cin * cout * (3 if backward else 1)
    byts = 4 * n * (h * w * cin + ho * wo * cout) * (3 if backward else 1)
    return flops, byts


def layer_fn(spec, n, arm, backward):
    name, transpose, k, s, pad, (h, w, cin), cout, gamma = spec
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand((n, h, w, cin), generator=g, device="cuda").requires_grad_(backward)
    shape = (k, k, cout, cin) if transpose else (k, k, cin, cout)
    W = (torch.randn(shape, generator=g, device="cuda") / np.sqrt(k * k * cin)).requires_grad_(
        backward)
    gm = torch.ones(cout, device="cuda", requires_grad=backward) if gamma else None
    bt = torch.zeros(cout, device="cuda", requires_grad=backward)
    mm, mv = torch.zeros(cout, device="cuda"), torch.ones(cout, device="cuda")
    L = ops(arm)
    ins = [t for t in (x, W, gm, bt) if t is not None]

    def fn():
        if gamma is None:
            y = L.sigmoid_conv2d_transpose(x, W, bt, stride=s, padding=pad)
        else:
            f = L.bn_conv2d_transpose if transpose else L.bn_conv2d
            y = f(x, W, gm, bt, mm, mv, True, stride=s, padding=pad)
        if backward:
            torch.autograd.grad(y.sum(), ins)
    return fn, layer_cost(spec, n, backward)


def model_cost(kind, n, backward):
    f = b = 0
    for spec in LAYERS[kind]:
        ff, bb = layer_cost(spec, n, backward)
        f, b = f + ff, b + bb
    return f, b


def step_fn(kind, arm):
    n = BATCH[kind]
    gen, disc = (GM.dcgan_params if kind == "dcgan" else GM.wgan_params)(0)
    opt_g, opt_d = GM.optimizers(kind, gen, disc)
    g = torch.Generator(device="cuda").manual_seed(2)
    hwc = (32, 32, 3) if kind == "dcgan" else (28, 28, 1)
    x = torch.rand((n,) + hwc, generator=g, device="cuda")
    L = ops(arm)

    def fn():
        GM.L = L
        GM.train_step(kind, gen, disc, x, opt_g, opt_d)
    # generator forward + backward, three discriminator passes (one without weight gradients)
    f, b = model_cost(kind, n, True)
    return fn, (int(f * 1.5), int(b * 1.5))


def gen_fn(kind, arm, total):
    gen, _ = (GM.dcgan_params if kind == "dcgan" else GM.wgan_params)(0)
    G = GM.dcgan_generator if kind == "dcgan" else GM.wgan_generator
    L = ops(arm)
    chunk = min(total, 10000)

    def fn():
        GM.L = L
        with torch.no_grad():
            for i in range(0, total, chunk):
                G(gen, min(chunk, total - i), False)
    f, b = model_cost(kind, total, False)
    gl = [s for s in LAYERS[kind] if s[0].startswith("g")]
    f = sum(layer_cost(s, total, False)[0] for s in gl)
    b = sum(layer_cost(s, total, False)[1] for s in gl)
    return fn, (f, b)


def conv3x3_fn(arm, n=4096):
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand((n, 14, 14, 64), generator=g, device="cuda").requires_grad_(True)
    W = (torch.randn((3, 3, 64, 64), generator=g, device="cuda") / 24.).requires_grad_(True)
    gm = torch.ones(64, device="cuda", requires_grad=True)
    bt = torch.zeros(64, device="cuda", requires_grad=True)
    mm, mv = torch.zeros(64, device="cuda"), torch.ones(64, device="cuda")

    def fn():
        if arm == "ffma_conv2d":
            a = zs.fused.conv2d(x, W)
            y = F.batch_norm(a.permute(0, 3, 1, 2), mm, mv, gm, bt, True, 0.01, 1e-3).relu()
        else:
            y = ops(arm).bn_conv2d(x, W, gm, bt, mm, mv, True)
        torch.autograd.grad(y.sum(), (x, W, gm, bt))
    spec = ("c", False, 3, 1, "SAME", (14, 14, 64), 64, True)
    return fn, layer_cost(spec, n, True)


def all_cases():
    out = []
    for kind in ("dcgan", "wgan"):
        for spec in LAYERS[kind]:
            for mode in ("fwd", "fwdbwd"):
                for size in ("batch", "4096"):
                    out.append("%s_%s_%s_%s" % (kind, spec[0], mode, size))
        out += [kind + "_step", kind + "_gen100", kind + "_gen1e5"]
    return out + ["conv3x3_64_fwdbwd_4096"]


def case_fns(case):
    parts = case.split("_")
    if case.startswith("conv3x3"):
        return {arm: conv3x3_fn(arm) for arm in ("fused", "ffma_conv2d", "cudnn_fp32",
                                                 "cudnn_tf32")}
    kind = parts[0]
    if parts[1] == "step":
        return {arm: step_fn(kind, arm) for arm in ARMS}
    if parts[1].startswith("gen"):
        total = 100 if parts[1] == "gen100" else 100000
        return {arm: gen_fn(kind, arm, total) for arm in ARMS}
    spec = [s for s in LAYERS[kind] if s[0] == parts[1]][0]
    n = BATCH[kind] if parts[3] == "batch" else 4096
    return {arm: layer_fn(spec, n, arm, parts[2] == "fwdbwd") for arm in ARMS}


def profile(fn):
    """(kernel launches, device ms of all kernels) of one call."""
    from torch.profiler import profile as prof_, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with prof_(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(evs), round(sum(e.device_time_total for e in evs) / 1e3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--cases", default=",".join(all_cases()))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gan.py measures on a CUDA device"
    name, power = card()
    tf32_default = torch.backends.cudnn.allow_tf32
    for case in args.cases.split(","):
        pairs = case_fns(case)
        fns = {arm: p[0] for arm, p in pairs.items()}
        for fn in fns.values():
            for _ in range(2):
                fn()
        torch.cuda.synchronize()
        steps = 1 if case.endswith("gen1e5") else args.steps
        times = {arm: [] for arm in fns}
        for _ in range(args.windows):
            for arm, fn in fns.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(steps):
                    fn()
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) / steps * 1e3)
        for arm, fn in fns.items():
            ts = sorted(times[arm])
            launches, dev_ms = profile(fn)
            flops, byts = pairs[arm][1]
            print(json.dumps({
                "case": case, "arm": arm, "accuracy_matched": arm != "cudnn_tf32",
                "ms_median": round(ts[len(ts) // 2], 4), "ms_min": round(ts[0], 4),
                "ms_max": round(ts[-1], 4), "launches_per_call": launches, "device_ms": dev_ms,
                "conv_flops": flops, "bytes": byts,
                "tflops_at_median": round(flops / ts[len(ts) // 2] / 1e9, 2),
                "gpu": name, "power_limit": power}), flush=True)
        del pairs, fns
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = tf32_default


if __name__ == "__main__":
    main()
