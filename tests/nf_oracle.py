"""Float64 restatement of the planar normalizing flow of zhusuan/transform.py:70-198 and of the
normalizing-flow VAE of examples/normalizing_flows/vae_nf.py, in torch so that autograd gives their
gradients.

planar_flow follows the reference's op sequence (transform.py:161-194), with its softplus
log(exp(t) + 1) and u.w formed as a product, so within the finite range it is the reference.

vae_nf (:19-85): q(z | x) = N(mean(x), exp(logstd(x))) through two ReLU layers, two calls of the
flow stack, and p(x, z) = N(z; 0, 1) Bernoulli(x; logits(z)) through two ReLU layers.  Dense
weights are [out, in] (the kernel transposed, the layout of zs.fused).  The ELBO is
mean over particles of log p(x, z_K) - log q_K; the IS estimate is log_mean_exp over particles.
"""
import math

import torch
import torch.nn.functional as F

LOG_2PI = math.log(2 * math.pi)


def planar_flow(z, log_q, b, aux_u, w):
    """z [..., d], log_q [...], b [n], aux_u / w [n, d] -> (z, log_q) after n flows."""
    d = z.shape[-1]
    lead = z.shape[:-1]
    z = z.reshape(-1, d)
    log_q = log_q.reshape(-1)
    for k in range(b.shape[0]):
        wk, ak = w[k], aux_u[k]
        t = wk @ ak
        u = ak + wk / (wk @ wk) * (torch.log(torch.exp(t) + 1) - 1 - t)
        psi = u @ wk
        a = torch.tanh(z @ wk + b[k])
        log_q = log_q - torch.log(psi * (1 - a * a) + 1)
        z = z + a[:, None] * u
    return z.reshape(lead + (d,)), log_q.reshape(lead)


def normal_lp(x, mean, logstd):
    """Normal(mean, exp(logstd)).log_prob(x) summed over the last axis."""
    return (-0.5 * LOG_2PI - logstd - 0.5 * (x - mean) ** 2 * torch.exp(-2 * logstd)).sum(-1)


def bernoulli_lp(x, logits):
    """Bernoulli(logits).log_prob(x) summed over the last axis."""
    return (x * logits - F.softplus(logits)).sum(-1)


def encode(x, q, linear=F.linear):
    """q = [W1, b1, W2, b2, Wm, bm, Ws, bs] -> (z_mean, z_logstd) [n, z_dim]."""
    h = torch.relu(linear(x, q[0], q[1]))
    h = torch.relu(linear(h, q[2], q[3]))
    return linear(h, q[4], q[5]), linear(h, q[6], q[7])


def log_px_z(x, z, p, linear=F.linear):
    """p = [W1, b1, W2, b2, Wx, bx]; log p(z) + log p(x | z), z [S, n, z_dim]."""
    h = torch.relu(linear(z, p[0], p[1]))
    h = torch.relu(linear(h, p[2], p[3]))
    logits = linear(h, p[4], p[5])
    return normal_lp(z, torch.zeros_like(z), torch.zeros_like(z)) + bernoulli_lp(x, logits)


def vae_nf(x, eps, q, p, flows, flow=planar_flow, linear=F.linear):
    """x [n, x_dim] (0/1), eps [S, n, z_dim]; flows: a list of (b, aux_u, w), one per flow call.
    Returns (log p(x, z_K) - log q_K) [S, n]: the per-particle log weights."""
    mean, logstd = encode(x, q, linear)
    z = mean + torch.exp(logstd) * eps
    log_q = normal_lp(z, mean, logstd)
    for b, aux_u, w in flows:
        z, log_q = flow(z, log_q, b, aux_u, w)
    return log_px_z(x, z, p, linear) - log_q


def bound_and_cost(lw):
    """(mean ELBO, cost = -mean ELBO): elbo(..., axis=0).sgvb() of the reparameterised q."""
    lb = lw.mean(0)
    return lb.mean(), -lb.mean()


def is_loglikelihood(lw):
    """mean over rows of log_mean_exp over particles (evaluation.py:22-54)."""
    return (torch.logsumexp(lw, 0) - math.log(lw.shape[0])).mean()
