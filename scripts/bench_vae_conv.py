"""Convolutional VAE (examples/variational_autoencoders/vae_conv.py) on zs.fused.conv2d /
conv2d_transpose and on zs.fused.conv2d_tc / conv2d_transpose_tc against cuDNN convolutions with
the same SAME padding, on seeded synthetic data.
Arms (alternating in one process; dense layers are zs.fused.linear in every arm):
  fused       zs.fused.conv2d / conv2d_transpose (FFMA): one launch per layer, bias, residual and
              ReLU fused; 3 x 3 kernels and 1 - 64 channels only, so it prints nothing elsewhere
  fused_tc    zs.fused.conv2d_tc / conv2d_transpose_tc: the tensor-core products with the gather
              split, col2im, bias, residual and ReLU passes around them
  cudnn_fp32  F.conv2d / F.conv_transpose2d with the asymmetric pads, allow_tf32 = False, then
              bias, residual add and ReLU as separate ops: the accuracy-matched arm
  cudnn_tf32  the same with torch's defaults (cuDNN in TF32): NOT accuracy-matched
Cases (nf = 16 unless --nf says otherwise):
  {enc,dec}_{plain,resize}_{fwd,fwdbwd}_{128,4096}  one resnet block of the example:
      enc_plain 28x28xnf -> 28x28xnf, enc_resize 28x28xnf -> 14x14x2nf,
      dec_plain 28x28xnf -> 28x28xnf, dec_resize 14x14x2nf -> 28x28xnf
  layer_{conv,deconv}_{k3c128,k5c64}_{fwd,fwdbwd}_4096  one stride-1 SAME layer with bias and ReLU
      outside the FFMA range: 3 x 3 with 128 -> 128 channels and 5 x 5 with 64 -> 64, at 14 x 14
  train_step   one training step at 128 images (bound, sgvb().backward(), Adam(1e-4, beta1 0.5))
  test_bound   the bound over 400 images without a gradient
  generate     x_mean of 100 images from the prior
Each prints the median, min and max over windows and the CUDA-event time of one call
(`stream_ms`); launches per call and conv-kernel device time come from a separate torch.profiler
pass, checked against the FFMA conv kernels the library launched: when the profiler recorded a
different number of them (`conv_kernels_profiled` against `conv_kernels_launched`),
`profile_complete` is false and its device columns are null.  In the fused_tc arm the conv device
time counts every tensor-core product, so in train_step, test_bound and generate it includes the
products of the dense layers too.
FLOPs and bytes of the convolutions are computed from the shapes.  One JSON line per case and arm, with the card's name and power limit.

    python scripts/bench_vae_conv.py [--windows 7] [--steps 20] [--cases a,b] [--nf 16]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zhusuan_b200 as zs  # noqa: E402

NF, Z_DIM = 16, 32
ARMS = ("fused", "fused_tc", "cudnn_fp32", "cudnn_tf32")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def _pads(big, small, s, k=3):
    total = max((small - 1) * s + k - big, 0)
    return total // 2, total - total // 2


class Fused(object):
    conv = staticmethod(zs.fused.conv2d)
    deconv = staticmethod(zs.fused.conv2d_transpose)


class FusedTC(object):
    conv = staticmethod(zs.fused.conv2d_tc)
    deconv = staticmethod(zs.fused.conv2d_transpose_tc)


class Cudnn(object):
    """SAME convolutions on cuDNN: NHWC tensors are passed as channels_last NCHW views."""

    def __init__(self, tf32):
        self.tf32 = tf32

    def conv(self, x, W, b=None, stride=1, relu=False, residual=None):
        torch.backends.cudnn.allow_tf32 = self.tf32
        H, Wd, k = int(x.shape[-3]), int(x.shape[-2]), int(W.shape[0])
        Ho, Wo = -(-H // stride), -(-Wd // stride)
        (pt, pb), (pl, pr) = _pads(H, Ho, stride, k), _pads(Wd, Wo, stride, k)
        xc = x.reshape((-1,) + tuple(x.shape[-3:])).permute(0, 3, 1, 2)
        if pt == pb and pl == pr:
            y = F.conv2d(xc, W.permute(3, 2, 0, 1), stride=stride, padding=(pt, pl))
        else:
            y = F.conv2d(F.pad(xc, (pl, pr, pt, pb)), W.permute(3, 2, 0, 1), stride=stride)
        return self._epilogue(y.permute(0, 2, 3, 1), b, relu, residual)

    def deconv(self, x, W, out_shape, stride=1, b=None, relu=False, residual=None):
        torch.backends.cudnn.allow_tf32 = self.tf32
        Ho, Wo, k = int(out_shape[0]), int(out_shape[1]), int(W.shape[0])
        pt, _ = _pads(Ho, int(x.shape[-3]), stride, k)
        pl, _ = _pads(Wo, int(x.shape[-2]), stride, k)
        xc = x.reshape((-1,) + tuple(x.shape[-3:])).permute(0, 3, 1, 2)
        y = F.conv_transpose2d(xc, W.permute(3, 2, 0, 1), stride=stride)
        return self._epilogue(y[:, :, pt:pt + Ho, pl:pl + Wo].permute(0, 2, 3, 1), b, relu,
                              residual)

    @staticmethod
    def _epilogue(y, b, relu, residual):
        if b is not None:
            y = y + b
        if residual is not None:
            y = y + residual
        return torch.relu(y) if relu else y


def make_ops(arm):
    if arm in ("fused", "fused_tc"):
        return Fused() if arm == "fused" else FusedTC()
    return Cudnn(arm == "cudnn_tf32")


# ---- the example's blocks (vae_conv.py:20-53) ------------------------------------------------------

def conv_resnet_block(ops, h, ps, resize):
    if not resize:
        t = ops.conv(h, ps[0], ps[1], relu=True)
        return ops.conv(t, ps[2], ps[3], relu=True, residual=h)
    t = ops.conv(h, ps[0], ps[1], stride=2, relu=True)
    r = ops.conv(h, ps[4], ps[5], stride=2)
    return ops.conv(t, ps[2], ps[3], relu=True, residual=r)


def deconv_resnet_block(ops, h, ps, out_shape, resize):
    if not resize:
        t = ops.deconv(h, ps[0], out_shape, b=ps[1], relu=True)
        return ops.deconv(t, ps[2], out_shape, b=ps[3], relu=True, residual=h)
    t = ops.deconv(h, ps[0], tuple(h.shape[1:]), b=ps[1], relu=True)
    r = ops.deconv(h, ps[4], out_shape, 2, b=ps[5])
    return ops.deconv(t, ps[2], out_shape, 2, b=ps[3], relu=True, residual=r)


def set_nf(nf):
    """The example's filter count: the encoder / decoder blocks and the block cases."""
    global NF, ENC, DEC, BLOCKS
    NF = nf
    ENC = [(NF, False), (2 * NF, True), (2 * NF, False), (2 * NF, True), (2 * NF, False)]
    DEC = [((7, 7, 2 * NF), False), ((14, 14, 2 * NF), True), ((14, 14, 2 * NF), False),
           ((28, 28, NF), True), ((28, 28, NF), False)]
    BLOCKS = {   # name: (transpose, resize, in [H, W, C], out [H, W, C])
        "enc_plain": (False, False, (28, 28, NF), (28, 28, NF)),
        "enc_resize": (False, True, (28, 28, NF), (14, 14, 2 * NF)),
        "dec_plain": (True, False, (28, 28, NF), (28, 28, NF)),
        "dec_resize": (True, True, (14, 14, 2 * NF), (28, 28, NF)),
    }


def _param(g, shape, fan_in=None):
    if len(shape) == 1:
        t = 0.1 * torch.randn(shape, generator=g, device="cuda")
    else:
        t = torch.randn(shape, generator=g, device="cuda") / math.sqrt(fan_in)
    return t.requires_grad_(True)


def block_params(g, cin, cout, resize, transpose):
    """Weights of one block: conv [3, 3, Cin, Cout], transposed conv [3, 3, Cout, Cin]."""
    def w(i, o):
        return _param(g, (3, 3, o, i) if transpose else (3, 3, i, o), 9 * i)
    if not resize:
        return [w(cin, cout), _param(g, (cout,)), w(cout, cout), _param(g, (cout,))]
    mid = cin if transpose else cout
    return [w(cin, mid), _param(g, (mid,)), w(mid, cout), _param(g, (cout,)), w(cin, cout),
            _param(g, (cout,))]


def model_params(g):
    q = [_param(g, (3, 3, 1, NF), 9), _param(g, (NF,))]
    c = NF
    for co, resize in ENC:
        q += block_params(g, c, co, resize, False)
        c = co
    q += [_param(g, (500, 7 * 7 * 2 * NF), 7 * 7 * 2 * NF), _param(g, (500,)),
          _param(g, (Z_DIM, 500), 500), _param(g, (Z_DIM,)), _param(g, (Z_DIM, 500), 500),
          _param(g, (Z_DIM,))]
    p = [_param(g, (7 * 7 * 2 * NF, Z_DIM), Z_DIM), _param(g, (7 * 7 * 2 * NF,))]
    c = 2 * NF
    for (ho, wo, co), resize in DEC:
        p += block_params(g, c, co, resize, True)
        c = co
    p += [_param(g, (3, 3, 1, NF), 9 * NF), _param(g, (1,))]
    return q, p


def decoder(ops, z, p, n, n_particles):
    h = zs.fused.linear(z, p[0], p[1], relu=True).reshape(-1, 7, 7, 2 * NF)
    i = 2
    for out, resize in DEC:
        k = 6 if resize else 4
        h = deconv_resnet_block(ops, h, p[i:i + k], out, resize)
        i += k
    return ops.deconv(h, p[i], (28, 28, 1), b=p[i + 1]).reshape(n_particles, -1, 784)


def example(ops, x, q, p):
    """vae_conv.py:56-114: build_q_net, build_gen and elbo(..., axis=0) on zs, one particle."""
    n = int(x.shape[0])

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, z_dim, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        x_logits = decoder(ops, z, p, n, n_particles)
        bn.deterministic("x_mean", torch.sigmoid(x_logits))
        bn.bernoulli("x", x_logits, group_ndims=1, dtype=torch.float32)
        return bn

    h = ops.conv((2 * x - 1).reshape(-1, 28, 28, 1), q[0], q[1], relu=True)
    i = 2
    for co, resize in ENC:
        k = 6 if resize else 4
        h = conv_resnet_block(ops, h, q[i:i + k], resize)
        i += k
    h = zs.fused.linear(h.reshape(n, -1), q[i], q[i + 1], relu=True)
    mean, logstd = zs.fused.linear(h, q[i + 2], q[i + 3]), zs.fused.linear(h, q[i + 4], q[i + 5])
    qz = mean + torch.exp(logstd) * torch.randn((1,) + tuple(mean.shape), device="cuda")
    log_qz = zs.distributions.Normal(mean, logstd=logstd, group_ndims=1).log_prob(qz)
    return zs.variational.elbo(build_gen(n, Z_DIM, 1), {"x": x}, latent={"z": [qz, log_qz]},
                               axis=0)


# ---- cases -------------------------------------------------------------------------------------

set_nf(NF)
LAYERS = {"k3c128": (3, 128), "k5c64": (5, 64)}   # single layers at 14 x 14: (k, channels)
LAYER_HW = 14


def model_layers(encoder, decoder_):
    """(Cin, Cout, small pixels) of every (3 x 3) convolution of the example."""
    out = []
    if encoder:
        out.append((1, NF, 784))
        c, hw = NF, 784
        for co, resize in ENC:
            if resize:
                out += [(c, co, hw // 4), (co, co, hw // 4), (c, co, hw // 4)]
                hw //= 4
            else:
                out += [(c, co, hw), (co, co, hw)]
            c = co
    if decoder_:
        c, hw = 2 * NF, 49
        for (ho, wo, co), resize in DEC:
            if resize:
                out += [(c, c, hw), (c, co, hw), (c, co, hw)]
                hw = ho * wo
            else:
                out += [(c, co, hw), (co, co, hw)]
            c = co
        out.append((1, NF, 784))
    return out


def conv_cost(layers, R, backward, k=3):
    flops = sum(2 * k * k * ci * co * px * R for ci, co, px in layers)
    byts = sum(4 * (R * px * (ci + 2 * co) + k * k * ci * co) for ci, co, px in layers)
    return (3 * flops, 3 * byts) if backward else (flops, byts)


def case_fn(case, arm):
    ops = make_ops(arm)
    g = torch.Generator(device="cuda").manual_seed(0)
    if case in ("train_step", "test_bound", "generate"):
        q, p = model_params(g)
        if case == "generate":
            def gen():
                with torch.no_grad():
                    z = torch.randn(1, 100, Z_DIM, device="cuda", generator=g)
                    return torch.sigmoid(decoder(ops, z, p, 100, 1))
            return gen, conv_cost(model_layers(False, True), 100, False)
        n = 128 if case == "train_step" else 400
        x = (torch.rand(n, 784, generator=g, device="cuda") < 0.3).float()
        if case == "test_bound":
            def bound():
                with torch.no_grad():
                    return example(ops, x, q, p).tensor.mean()
            return bound, conv_cost(model_layers(True, True), n, False)
        opt = torch.optim.Adam(q + p, lr=1e-4, betas=(0.5, 0.999))

        def step():
            lb = example(ops, x, q, p)
            cost = lb.sgvb().mean()
            opt.zero_grad()
            cost.backward()
            opt.step()
            return lb.tensor.mean()
        return step, conv_cost(model_layers(True, True), n, True)
    block, kind, R = case.rsplit("_", 2)
    R = int(R)
    backward = kind == "fwdbwd"
    if block.startswith("layer_"):
        return layer_case(ops, g, block, R, backward)
    transpose, resize, (hi, wi, ci), out = BLOCKS[block]
    ps = block_params(g, ci, out[2], resize, transpose)
    h = torch.randn(R, hi, wi, ci, generator=g, device="cuda")
    if backward:
        h.requires_grad_(True)

    def run():
        if transpose:
            y = deconv_resnet_block(ops, h, ps, out, resize)
        else:
            y = conv_resnet_block(ops, h, ps, resize)
        if backward:
            torch.autograd.grad(y.sum(), [h] + ps)
        return y
    if not backward:
        run0 = run

        def run():
            with torch.no_grad():
                return run0()
    layers = model_layers_block(block)
    return run, conv_cost(layers, R, backward)


def layer_case(ops, g, name, R, backward):
    """One stride-1 SAME layer with bias and ReLU: layer_{conv,deconv}_{k3c128,k5c64}."""
    _, kind, size = name.split("_")
    k, c = LAYERS[size]
    W = _param(g, (k, k, c, c), k * k * c)
    b = _param(g, (c,))
    h = torch.randn(R, LAYER_HW, LAYER_HW, c, generator=g, device="cuda")
    if backward:
        h.requires_grad_(True)

    def run():
        with torch.set_grad_enabled(backward):
            if kind == "deconv":
                y = ops.deconv(h, W, (LAYER_HW, LAYER_HW, c), 1, b=b, relu=True)
            else:
                y = ops.conv(h, W, b, 1, True)
            if backward:
                torch.autograd.grad(y.sum(), [h, W, b])
        return y
    return run, conv_cost([(c, c, LAYER_HW * LAYER_HW)], R, backward, k)


def model_layers_block(block):
    transpose, resize, (hi, wi, ci), (ho, wo, co) = BLOCKS[block]
    small = min(hi * wi, ho * wo)
    if not resize:
        return [(ci, co, hi * wi), (co, co, hi * wi)]
    if transpose:
        return [(ci, ci, hi * wi), (ci, co, small), (ci, co, small)]
    return [(ci, co, small), (co, co, small), (ci, co, small)]


CONV_NAMES = ("conv3x3", "conv", "cudnn", "xmma", "implicit", "dgrad", "wgrad", "cutlass",
              "winograd", "fft")


def profile(fn, arm):
    """(kernel launches, device ms of all kernels, device ms of convolution kernels, FFMA conv
    kernels the library launched, FFMA conv kernels the profiler recorded) of one call.  In the
    fused_tc arm every tensor-core product counts as a convolution kernel."""
    from torch.profiler import profile as prof_, ProfilerActivity
    from zhusuan_b200._lib import lib
    fn()
    torch.cuda.synchronize()
    launched = [0]
    call = lib.call

    def counting_call(name, *args):
        if name.startswith("zsb_conv3x3"):
            launched[0] += lib._KERNELS.get(name, 1)
        return call(name, *args)
    lib.call = counting_call
    try:
        with prof_(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
    finally:
        lib.call = call
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    seen = sum(1 for e in evs if "conv3x3" in e.name)
    total = sum(e.device_time_total for e in evs) / 1e3
    names = CONV_NAMES + (("tc_pipeline_kernel",) if arm == "fused_tc" else ())
    conv = sum(e.device_time_total for e in evs
               if any(k in e.name.lower() for k in names)
               and "zsb_linear" not in e.name and "split16" not in e.name) / 1e3
    return len(evs), round(total, 4), round(conv, 4), launched[0], seen


def stream_ms(fn, reps=5):
    """Median over `reps` calls of the CUDA-event time of one call on the current stream (kernels
    and the gaps between them)."""
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return round(sorted(ts)[len(ts) // 2], 4)


def all_cases():
    out = []
    for block in BLOCKS:
        for kind in ("fwd", "fwdbwd"):
            for R in (128, 4096):
                out.append("%s_%s_%d" % (block, kind, R))
    for layer in ("conv_k3c128", "deconv_k3c128", "conv_k5c64", "deconv_k5c64"):
        for kind in ("fwd", "fwdbwd"):
            out.append("layer_%s_%s_4096" % (layer, kind))
    return out + ["train_step", "test_bound", "generate"]


def fused_supports(case):
    """The FFMA layers take 3 x 3 kernels and at most 64 channels."""
    if case.startswith("layer_"):
        return False
    return 2 * NF <= 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--cases", default=",".join(all_cases()))
    ap.add_argument("--nf", type=int, default=NF, help="the example's filter count (16)")
    args = ap.parse_args()
    set_nf(args.nf)
    assert torch.cuda.is_available(), "bench_vae_conv.py measures on a CUDA device"
    name, power = card()
    tf32_default = torch.backends.cudnn.allow_tf32
    for case in args.cases.split(","):
        fns, costs = {}, {}
        for arm in ARMS:
            if arm == "fused" and not fused_supports(case):
                continue
            fns[arm], costs[arm] = case_fn(case, arm)
        for fn in fns.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {arm: [] for arm in fns}
        for _ in range(args.windows):
            for arm, fn in fns.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) / args.steps * 1e3)
        for arm, fn in fns.items():
            ts = sorted(times[arm])
            launches, dev_ms, conv_ms, zsb, seen = profile(fn, arm)
            complete = seen == zsb
            flops, byts = costs[arm]
            print(json.dumps({
                "case": case, "arm": arm, "nf": NF, "accuracy_matched": arm != "cudnn_tf32",
                "ms_median": round(ts[len(ts) // 2], 4), "ms_min": round(ts[0], 4),
                "ms_max": round(ts[-1], 4), "stream_ms": stream_ms(fn),
                "launches_per_call": launches, "conv_kernels_launched": zsb,
                "conv_kernels_profiled": seen,
                "profile_complete": complete, "device_ms": dev_ms if complete else None,
                "conv_device_ms": conv_ms if complete else None, "conv_flops": flops,
                "conv_bytes": byts, "conv_tflops": round(flops / conv_ms / 1e9, 2)
                if complete and conv_ms > 0 else None, "gpu": name, "power_limit": power}),
                flush=True)
    torch.backends.cudnn.allow_tf32 = tf32_default


if __name__ == "__main__":
    main()
