"""Float64 restatement of the Inverse Autoregressive Flow of zhusuan/transform.py:200-282 with the
linear autoregressive network of :17-67, and of the normalizing-flow VAE of
examples/normalizing_flows/vae_nf.py with two IAF stacks in place of the planar ones, in torch so
that autograd gives their gradients.

linear_iaf follows the reference's op sequence: m = z (mask * m_w), s = exp(z (mask * s_w)), then
the update with log(s) or log(sigmoid(s)) taken literally, then the reversal.
"""
import torch

import nf_oracle as NF


def linear_iaf(z, log_q, m_w, s_w, update="normal"):
    """z [..., d], log_q [...], m_w / s_w [n, d, d] -> (z, log_q) after n flows."""
    d = z.shape[-1]
    lead = z.shape[:-1]
    mask = torch.ones(d, d, dtype=z.dtype, device=z.device).triu(1)
    z = z.reshape(-1, d)
    log_q = log_q.reshape(-1)
    for k in range(m_w.shape[0]):
        m = z @ (mask * m_w[k])
        s = torch.exp(z @ (mask * s_w[k]))
        if update == "gru":
            sigma = torch.sigmoid(s)
            z = sigma * z + (1 - sigma) * m
            log_q = log_q - torch.log(sigma).sum(-1)
        else:
            z = s * z + m
            log_q = log_q - torch.log(s).sum(-1)
        z = torch.flip(z, [-1])
    return z.reshape(lead + (d,)), log_q.reshape(lead)


def vae_iaf(x, eps, q, p, flows, update="normal", linear=torch.nn.functional.linear):
    """x [n, x_dim] (0/1), eps [S, n, z_dim]; flows: a list of (m_w, s_w), one per flow call.
    Returns (log p(x, z_K) - log q_K) [S, n]: the per-particle log weights."""
    mean, logstd = NF.encode(x, q, linear)
    z = mean + torch.exp(logstd) * eps
    log_q = NF.normal_lp(z, mean, logstd)
    for m_w, s_w in flows:
        z, log_q = linear_iaf(z, log_q, m_w, s_w, update)
    return NF.log_px_z(x, z, p, linear) - log_q
