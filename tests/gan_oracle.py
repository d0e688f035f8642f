"""Float64 torch restatement of the layers of examples/generative_adversarial_nets (dcgan.py,
wasserstein_gan.py): k x k convolutions with TensorFlow's SAME / VALID padding written out (F.pad
with the asymmetric pads, then F.conv2d; F.conv_transpose2d, then a crop), and the batch norm of
4-D inputs as TF 1.x's fused path computes it.  It shares no code with zs.fused, so one misreading
of TF's padding or batch-norm rules cannot hide in both.  Runs on whatever device its inputs are
on.  Tensors are NHWC; conv kernels [k, k, Cin, Cout] (tf.layers.conv2d), transposed-conv kernels
[k, k, Cout, Cin] (tf.layers.conv2d_transpose)."""
import numpy as np
import torch
import torch.nn.functional as F


def conv_out_size(n, k, stride, padding):
    """tf.layers.conv2d's output length (conv_utils.conv_output_length)."""
    if padding == "SAME":
        return -(-n // stride)
    return -(-(n - k + 1) // stride)


def deconv_out_size(n, k, stride, padding):
    """tf.layers.conv2d_transpose's output length (conv_utils.deconv_output_length)."""
    if padding == "SAME":
        return n * stride
    return n * stride + max(k - stride, 0)


def tf_pads(big, small, k, stride, padding):
    """(before, after) pads of a convolution from `big` to `small` rows: SAME pads
    max((small - 1) stride + k - big, 0) rows, the smaller half before; VALID pads nothing."""
    if padding != "SAME":
        return 0, 0
    total = max((small - 1) * stride + k - big, 0)
    return total // 2, total - total // 2


def conv2d(x, W, stride=1, padding="SAME"):
    """tf.layers.conv2d(x, Cout, k, stride, padding, use_bias=False) on x [N, H, W, Cin]."""
    k = int(W.shape[0])
    H, Wd = int(x.shape[1]), int(x.shape[2])
    Ho, Wo = conv_out_size(H, k, stride, padding), conv_out_size(Wd, k, stride, padding)
    pt, pb = tf_pads(H, Ho, k, stride, padding)
    pl, pr = tf_pads(Wd, Wo, k, stride, padding)
    xp = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(xp, W.permute(3, 2, 0, 1).contiguous(), stride=stride)[:, :, :Ho, :Wo]
    return y.permute(0, 2, 3, 1)


def conv2d_transpose(x, W, stride=1, padding="SAME"):
    """tf.layers.conv2d_transpose(x, Cout, k, stride, padding, use_bias=False) on x [N, Hi, Wi,
    Cin], W [k, k, Cout, Cin]: the adjoint of conv2d from the output grid to x's grid."""
    k = int(W.shape[0])
    Hi, Wi = int(x.shape[1]), int(x.shape[2])
    Ho, Wo = deconv_out_size(Hi, k, stride, padding), deconv_out_size(Wi, k, stride, padding)
    pt, _ = tf_pads(Ho, Hi, k, stride, padding)
    pl, _ = tf_pads(Wo, Wi, k, stride, padding)
    y = F.conv_transpose2d(x.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1).contiguous(),
                           stride=stride)
    # full output (Hi - 1) stride + k rows; drop pt before, and pad with zeros rows no tap reaches
    y = F.pad(y, (0, max(pl + Wo - int(y.shape[3]), 0), 0, max(pt + Ho - int(y.shape[2]), 0)))
    return y[:, :, pt:pt + Ho, pl:pl + Wo].permute(0, 2, 3, 1)


def batch_norm_4d(a, gamma, beta, moving_mean, moving_variance, training, momentum=0.99,
                  epsilon=1e-3):
    """tf.layers.batch_normalization on a 4-D input (TF 1.x's fused path): returns (y,
    new_moving_mean, new_moving_variance).  Training normalises with the mean and the population
    variance over N*H*W; the moving variance moves towards the Bessel-corrected variance
    var * R / (R - 1), with the factor 1 at R = 1.  gamma None is scale=False."""
    if training:
        R = a.shape[0] * a.shape[1] * a.shape[2]
        mean = a.mean((0, 1, 2))
        var = ((a - mean) ** 2).mean((0, 1, 2))
        corr = R / (R - 1.0) if R > 1 else 1.0
        new_m = moving_mean - (moving_mean - mean) * (1 - momentum)
        new_v = moving_variance - (moving_variance - var * corr) * (1 - momentum)
    else:
        mean, var = moving_mean, moving_variance
        new_m, new_v = moving_mean, moving_variance
    y = (a - mean) / torch.sqrt(var + epsilon)
    if gamma is not None:
        y = y * gamma
    return y + beta, new_m, new_v


def bn_conv2d(x, W, gamma, beta, mm, mv, training, stride=1, padding="SAME", relu=True,
              momentum=0.99, epsilon=1e-3):
    y, m, v = batch_norm_4d(conv2d(x, W, stride, padding), gamma, beta, mm, mv, training,
                            momentum, epsilon)
    return (torch.relu(y) if relu else y), m, v


def bn_conv2d_transpose(x, W, gamma, beta, mm, mv, training, stride=1, padding="SAME", relu=True,
                        momentum=0.99, epsilon=1e-3):
    y, m, v = batch_norm_4d(conv2d_transpose(x, W, stride, padding), gamma, beta, mm, mv,
                            training, momentum, epsilon)
    return (torch.relu(y) if relu else y), m, v


def sigmoid_conv2d_transpose(x, W, b=None, stride=1, padding="SAME"):
    y = conv2d_transpose(x, W, stride, padding)
    return torch.sigmoid(y if b is None else y + b)


# ---- the two examples' networks and one training step, in float64 ------------------------------
# Parameters are dicts: W0..W3 (the generator's kernels; DCGAN's W0 is the dense kernel [out, in]),
# W0..W2, Wd, bd (the discriminator's), b3 (the generator's output bias), bn0..bn2 (bn3 for none)
# each {"gamma" (absent for scale=False), "beta", "mm", "mv"}.

def params_from_golden(g, kind, role):
    """The parameter dict of one network from the arrays of tests/golden/ref_gan.npz, in the
    order the network reads them."""
    pre = "%s/%s/" % (kind, role)
    names = sorted((k for k in g if k.startswith(pre)), key=lambda k: int(k[len(pre):].split("_")[0]))
    p, n_w, n_bn, cur = {}, 0, 0, None
    dense_last = role == "disc"
    for k in names:
        a = g[k]
        tail = k[len(pre):].split("_", 1)[1]
        if tail == "kernel":
            if dense_last and a.ndim == 2:
                p["Wd"] = a
            else:
                p["W%d" % n_w] = a
                n_w += 1
            cur = None
        elif tail in ("gamma", "beta"):
            if cur is None:
                cur = {"mm": np.zeros(a.shape[0], np.float32),
                       "mv": np.ones(a.shape[0], np.float32)}
                p["bn%d" % n_bn] = cur
                n_bn += 1
            cur[tail] = a
        else:
            p["bd" if role == "disc" else "b3"] = a
    return p


def _bn(fn, h, W, b, training, **kw):
    y, m, v = fn(h, W, b.get("gamma"), b["beta"], b["mm"], b["mv"], training, **kw)
    return y, (m, v)


def dense_bn_relu(z, W, b, training, momentum=0.99, epsilon=1e-3):
    """tf.layers.dense(use_bias=False) + batch_normalization on a 2-D input (the non-fused rule:
    the population variance normalises AND moves the moving variance) + relu."""
    a = z @ W.t()
    if training:
        mean, var = a.mean(0), a.var(0, unbiased=False)
        nm = b["mm"] - (b["mm"] - mean) * (1 - momentum)
        nv = b["mv"] - (b["mv"] - var) * (1 - momentum)
    else:
        mean, var, nm, nv = b["mm"], b["mv"], b["mm"], b["mv"]
    y = (a - mean) / torch.sqrt(var + epsilon) * b["gamma"] + b["beta"]
    return torch.relu(y), (nm, nv)


def generator(kind, p, z, training):
    """dcgan.py:20-40 / wasserstein_gan.py:20-43; returns (x, [new moving statistics per layer])."""
    new = []
    if kind == "dcgan":
        h, s = dense_bn_relu(z, p["W0"], p["bn0"], training)
        new.append(s)
        h = h.reshape(-1, 4, 4, int(p["W1"].shape[3]))
        geo = [(1, 2, "SAME"), (2, 2, "SAME")]
    else:
        h = z.reshape(-1, 1, 1, int(z.shape[-1]))
        geo = [(0, 1, "VALID"), (1, 1, "VALID"), (2, 2, "SAME")]
    for i, s_, pad in geo:
        h, s = _bn(bn_conv2d_transpose, h, p["W%d" % i], p["bn%d" % i], training, stride=s_,
                   padding=pad)
        new.append(s)
    return sigmoid_conv2d_transpose(h, p["W3"], p["b3"], 2, "SAME"), new


def discriminator(kind, p, x, training):
    """dcgan.py:43-60 / wasserstein_gan.py:46-62; returns (logits [n, 1], [new statistics])."""
    geo = [(2, "SAME")] * 3 if kind == "dcgan" else [(2, "SAME"), (2, "SAME"), (1, "VALID")]
    h, new = x, []
    for i, (s_, pad) in enumerate(geo):
        h, s = _bn(bn_conv2d, h, p["W%d" % i], p["bn%d" % i], training, stride=s_, padding=pad)
        new.append(s)
    return h.reshape(h.shape[0], -1) @ p["Wd"].t() + p["bd"], new


def with_stats(p, new):
    q = dict(p)
    for i, (m, v) in enumerate(new):
        q["bn%d" % i] = dict(p["bn%d" % i], mm=m.detach(), mv=v.detach())
    return q


def step(kind, gen, disc, x, z):
    """One training step's graph (dcgan.py:79-100, wasserstein_gan.py:82-96): gen_loss,
    disc_loss, x_gen and the moving statistics after it -- the generator's moved once, the
    discriminator's twice, on the real batch and then on the fake one."""
    x_gen, gnew = generator(kind, gen, z, True)
    real, dnew = discriminator(kind, disc, x, True)
    fake, dnew2 = discriminator(kind, with_stats(disc, dnew), x_gen, True)
    if kind == "dcgan":
        ce = F.binary_cross_entropy_with_logits
        gen_loss = ce(fake, torch.ones_like(fake))
        disc_loss = (ce(real, torch.ones_like(real)) + ce(fake, torch.zeros_like(fake))) / 2.
    else:
        gen_loss, disc_loss = -fake.mean(), -(real - fake).mean()
    return gen_loss, disc_loss, x_gen, gnew, dnew2
