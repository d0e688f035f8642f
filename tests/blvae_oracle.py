"""Float64 restatement of the Bernoulli-latent VAE of
examples/variational_autoencoders/bernoulli_latent_vae.py, in torch so that autograd gives its
gradients.

Layer (:25-30, 39-44): y = relu(BN(h W^T) * gamma + beta), tf.layers.dense(use_bias=False) and
tf.layers.batch_normalization with its defaults (momentum 0.99, epsilon 1e-3, center and scale).
Training normalises with the batch moments over every row (population variance) and moves the
moving statistics by m -= (m - batch) * (1 - momentum); evaluation normalises with the moving
statistics.

q (:37-48): two layers from x, then z ~ Bernoulli(dense(h, z_dim)) with S draws.  p (:18-33):
z ~ Bernoulli(0), two layers from z, x ~ Bernoulli(dense(h, x_dim)).  Baseline (:51-55):
dense(relu(dense(x, 100)), 1).  elbo(...).reinforce(baseline=cx) follows
zhusuan/variational/exclusive_kl.py:161-231 with axis 0.
"""
import math

import torch
import torch.nn.functional as F

MOMENTUM, EPSILON = 0.99, 1e-3


def bn_layer(h, W, gamma, beta, mm, mv, training, relu=True, momentum=MOMENTUM, epsilon=EPSILON):
    """(y, new moving mean, new moving variance) of one dense + batch-norm layer."""
    a = h @ W.t()
    if training:
        rows = a.reshape(-1, a.shape[-1])
        mean = rows.mean(0)
        var = ((rows - mean.detach()) ** 2).mean(0)
        d = 1.0 - momentum
        new_mm = mm - (mm - mean.detach()) * d
        new_mv = mv - (mv - var.detach()) * d
    else:
        mean, var, new_mm, new_mv = mm, mv, mm, mv
    y = (a - mean) * torch.rsqrt(var + epsilon) * gamma + beta
    return (torch.relu(y) if relu else y), new_mm, new_mv


def bern_lp(logits, x):
    """sum over the last axis of Bernoulli(logits).log_prob(x)."""
    return (x * logits - F.softplus(logits)).sum(-1)


def encoder(x, q, stats, training):
    """q = (W1, g1, b1, W2, g2, b2, Wz, bz); stats = [(mm, mv)] * 2.  Returns the z logits and the
    new moving statistics."""
    W1, g1, b1, W2, g2, b2, Wz, bz = q
    h, m1, v1 = bn_layer(x, W1, g1, b1, *stats[0], training)
    h, m2, v2 = bn_layer(h, W2, g2, b2, *stats[1], training)
    return h @ Wz.t() + bz, [(m1, v1), (m2, v2)]


def decoder_log_joint(x, z, p, stats, training):
    """log p(x, z) [S, n] for z [S, n, z_dim] and the new moving statistics; p = (W1, g1, b1, W2,
    g2, b2, Wx, bx)."""
    W1, g1, b1, W2, g2, b2, Wx, bx = p
    h, m1, v1 = bn_layer(z, W1, g1, b1, *stats[0], training)
    h, m2, v2 = bn_layer(h, W2, g2, b2, *stats[1], training)
    log_pz = bern_lp(torch.zeros_like(z), z)
    return log_pz + bern_lp(h @ Wx.t() + bx, x), [(m1, v1), (m2, v2)]


def baseline(x, c):
    W1, b1, W2, b2 = c
    return (torch.relu(x @ W1.t() + b1) @ W2.t() + b2).squeeze(-1)


def reinforce(log_pxz, log_qz, cx, moving_mean):
    """(cost, lower bound, bc) of exclusive_kl.py:161-231 with axis 0 and a baseline, and the
    final tf.reduce_mean(cost + baseline_cost) of :80-81: ``moving_mean`` is the value before this
    step's update; bc = mean(l_signal - cx) is what the update moves it towards."""
    l_signal = log_pxz - log_qz
    ls = l_signal - cx
    bc = ls.detach().mean()
    ls = ls - moving_mean
    cost = (-log_pxz + ls.detach() * (-log_qz)).mean(0)
    return (cost + baseline_cost(log_pxz, log_qz, cx)).mean(), l_signal.mean(0).mean(), bc


def baseline_cost(log_pxz, log_qz, cx):
    """The baseline net's cost [n]: 0.5 (l_signal - cx)^2 averaged over the particles, with no
    gradient through l_signal (exclusive_kl.py:200-204)."""
    return (0.5 * ((log_pxz - log_qz).detach() - cx) ** 2).mean(0)


def is_loglikelihood(log_pxz, log_qz):
    """mean over rows of log mean_s exp(log p(x, z_s) - log q(z_s)) (axis 0)."""
    w = log_pxz - log_qz
    return (torch.logsumexp(w, 0) - math.log(w.shape[0])).mean()
