"""Float64 torch restatement of the convolutional VAE of
examples/variational_autoencoders/vae_conv.py, with TensorFlow's SAME padding written out: F.pad with
the asymmetric pads, then F.conv2d; F.conv_transpose2d, then a crop of the leading pads.  It shares
no code with zs.fused.conv2d / conv2d_transpose, so one misreading of SAME cannot hide in both.
Runs on whatever device its inputs are on.

Parameters are lists of tensors in a fixed order (see `param_shapes`): conv weights
[3, 3, Cin, Cout] (tf.layers.conv2d), transposed-conv weights [3, 3, Cout, Cin]
(examples/utils/utils.py:94), dense weights [out, in] (torch / zs.fused.linear layout)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

LOG_2PI = math.log(2 * math.pi)


def same_pads(big, small, stride):
    """(before, after) of TensorFlow's SAME rule for a 3x3 window."""
    total = max((small - 1) * stride + 3 - big, 0)
    return total // 2, total - total // 2


def conv2d(x, W, b=None, stride=1):
    """tf.layers.conv2d(x, Cout, 3, strides=stride, padding="same") on NHWC x [N, H, W, Cin]."""
    H, Wd = int(x.shape[1]), int(x.shape[2])
    Ho, Wo = -(-H // stride), -(-Wd // stride)
    pt, pb = same_pads(H, Ho, stride)
    pl, pr = same_pads(Wd, Wo, stride)
    xp = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(xp, W.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)
    return y if b is None else y + b


def conv2d_transpose(x, W, out_shape, stride=1, b=None):
    """tf.nn.conv2d_transpose(x, W, [N] + out_shape, stride, "SAME") (+ bias_add): the adjoint of
    conv2d from [Ho, Wo, Cout] to [Hi, Wi, Cin]; W [3, 3, Cout, Cin]."""
    Ho, Wo = int(out_shape[0]), int(out_shape[1])
    Hi, Wi = int(x.shape[1]), int(x.shape[2])
    assert -(-Ho // stride) == Hi and -(-Wo // stride) == Wi, (out_shape, tuple(x.shape))
    pt, _ = same_pads(Ho, Hi, stride)
    pl, _ = same_pads(Wo, Wi, stride)
    y = F.conv_transpose2d(x.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1), stride=stride)
    y = y[:, :, pt:pt + Ho, pl:pl + Wo].permute(0, 2, 3, 1)
    return y if b is None else y + b


# ---- vae_conv.py -------------------------------------------------------------------------------

def enc_blocks(nf):
    """(out_channel, resize) of the five conv_resnet_blocks (vae_conv.py:82-86)."""
    return [(nf, False), (2 * nf, True), (2 * nf, False), (2 * nf, True), (2 * nf, False)]


def dec_blocks(nf):
    """(out_shape, resize) of the five deconv_resnet_blocks (vae_conv.py:63-67)."""
    return [((7, 7, 2 * nf), False), ((14, 14, 2 * nf), True), ((14, 14, 2 * nf), False),
            ((28, 28, nf), True), ((28, 28, nf), False)]


def param_shapes(nf, z_dim):
    """(q shapes, p shapes), in the order the networks read them."""
    q = [(3, 3, 1, nf), (nf,)]
    c = nf
    for co, resize in enc_blocks(nf):
        q += [(3, 3, c, co), (co,), (3, 3, co, co), (co,)]
        if resize:
            q += [(3, 3, c, co), (co,)]
        c = co
    q += [(500, 7 * 7 * 2 * nf), (500,), (z_dim, 500), (z_dim,), (z_dim, 500), (z_dim,)]
    p = [(7 * 7 * 2 * nf, z_dim), (7 * 7 * 2 * nf,)]
    c = 2 * nf
    for (ho, wo, co), resize in dec_blocks(nf):
        if resize:
            p += [(3, 3, c, c), (c,), (3, 3, co, c), (co,), (3, 3, co, c), (co,)]
        else:
            p += [(3, 3, co, c), (co,), (3, 3, co, co), (co,)]
        c = co
    p += [(3, 3, 1, nf), (1,)]
    return q, p


def init_params(rng, nf, z_dim):
    """Random parameters (NumPy float64): weights scaled by 1/sqrt(fan-in), small biases."""
    out = []
    for shapes in param_shapes(nf, z_dim):
        ps = []
        for s in shapes:
            if len(s) == 1:
                ps.append(0.1 * rng.standard_normal(s))
            else:
                fan_in = s[2] * 9 if len(s) == 4 else s[1]
                ps.append(rng.standard_normal(s) / math.sqrt(fan_in))
        out.append(ps)
    return out


def encode(x, q, nf, relu=torch.relu):
    """build_q_net (vae_conv.py:76-93) up to the z heads: x [n, 784] (0/1) -> (mean, logstd).
    ``relu`` is applied at every ReLU in order (a test may pass one that replays given masks)."""
    h = (2 * x - 1).reshape(-1, 28, 28, 1)
    h = relu(conv2d(h, q[0], q[1]))
    i = 2
    for co, resize in enc_blocks(nf):
        if not resize:
            t = relu(conv2d(h, q[i], q[i + 1]))
            t = conv2d(t, q[i + 2], q[i + 3]) + h
            i += 4
        else:
            t = relu(conv2d(h, q[i], q[i + 1], 2))
            t = conv2d(t, q[i + 2], q[i + 3]) + conv2d(h, q[i + 4], q[i + 5], 2)
            i += 6
        h = relu(t)
    h = relu(F.linear(h.reshape(h.shape[0], -1), q[i], q[i + 1]))
    return F.linear(h, q[i + 2], q[i + 3]), F.linear(h, q[i + 4], q[i + 5])


def decode(z, p, nf, relu=torch.relu):
    """build_gen (vae_conv.py:56-73) up to the logits: z [S, n, z_dim] -> logits [S, n, 784]."""
    S, n = int(z.shape[0]), int(z.shape[1])
    h = relu(F.linear(z, p[0], p[1])).reshape(-1, 7, 7, 2 * nf)
    i = 2
    for out, resize in dec_blocks(nf):
        if not resize:
            t = relu(conv2d_transpose(h, p[i], out, 1, p[i + 1]))
            t = conv2d_transpose(t, p[i + 2], out, 1, p[i + 3]) + h
            i += 4
        else:
            t = relu(conv2d_transpose(h, p[i], tuple(h.shape[1:]), 1, p[i + 1]))
            t = conv2d_transpose(t, p[i + 2], out, 2, p[i + 3]) + \
                conv2d_transpose(h, p[i + 4], out, 2, p[i + 5])
            i += 6
        h = relu(t)
    h = conv2d_transpose(h, p[i], (28, 28, 1), 1, p[i + 1])
    return h.reshape(S, n, 784)


def normal_lp(x, mean, logstd):
    return (-0.5 * LOG_2PI - logstd - 0.5 * (x - mean) ** 2 * torch.exp(-2 * logstd)).sum(-1)


def bernoulli_lp(x, logits):
    return (x * logits - F.softplus(logits)).sum(-1)


def vae_conv(x, eps, q, p, nf, relu=torch.relu):
    """log p(x, z) - log q(z | x) [S, n] with z = mean + exp(logstd) eps, and x_mean [S, n, 784]."""
    mean, logstd = encode(x, q, nf, relu)
    z = mean + torch.exp(logstd) * eps
    logits = decode(z, p, nf, relu)
    lw = normal_lp(z, torch.zeros_like(z), torch.zeros_like(z)) + bernoulli_lp(x, logits) - \
        normal_lp(z, mean, logstd)
    return lw, torch.sigmoid(logits)


def bound_and_cost(lw):
    """(mean ELBO, cost): tf.reduce_mean of elbo(..., axis=0) and of its sgvb() (vae_conv.py:
    111-114); for a reparameterised q the surrogate cost is the negative bound."""
    lb = lw.mean(0)
    return lb.mean(), -lb.mean()


def as_torch(ps, device="cpu"):
    return [torch.as_tensor(np.asarray(a), dtype=torch.float64, device=device) for a in ps]
