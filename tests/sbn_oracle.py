"""Float64 restatement of the sigmoid belief nets of examples/sigmoid_belief_nets (sbn_vimco.py:19-44,
sbn_adaptive_is.py): the model log-joint, the proposal's log q, the VIMCO cost and the importance
(reweighted wake-sleep) cost, on the CPU in torch float64 so that autograd gives their gradients.
The samples are inputs: a test evaluates the oracle on the samples the GPU drew.

Layers are ``(W [J, K], b [J])`` pairs (tf.layers.dense: logits = h W^T + b).
model:    h3 ~ Bernoulli(0), h2 | h3, h1 | h2, x | h1      (model_layers = [W_h2, W_h1, W_x])
proposal: h1 | x, h2 | h1, h3 | h2                        (q_layers = [W_h1, W_h2, W_h3])
"""
import math

import torch


def bern_lp(x, logits):
    """sum over the last axis of Bernoulli(logits).log_prob(x) (univariate.py:398-403)."""
    x, logits = torch.broadcast_tensors(x.to(logits.dtype), logits)
    return -torch.nn.functional.binary_cross_entropy_with_logits(
        logits, x, reduction="none").sum(-1)


def dense(h, layer):
    W, b = layer
    return h.to(W.dtype) @ W.t() + b


def log_q(x, hs, q_layers):
    """[K, N] log q(h1, h2, h3 | x) of the samples hs = (h1, h2, h3), each [K, N, H]."""
    h1, h2, h3 = hs
    return (bern_lp(h1, dense(x, q_layers[0])) + bern_lp(h2, dense(h1, q_layers[1]))
            + bern_lp(h3, dense(h2, q_layers[2])))


def log_joint(x, hs, model_layers):
    """[K, N] log p(x, h1, h2, h3) of the model."""
    h1, h2, h3 = hs
    lp_h3 = -h3.shape[-1] * math.log(2.0) * torch.ones(h3.shape[:-1], dtype=torch.float64)
    return (lp_h3 + bern_lp(h2, dense(h3, model_layers[0])) + bern_lp(h1, dense(h2, model_layers[1]))
            + bern_lp(x, dense(h1, model_layers[2])))


def log_mean_exp(x, axis):
    return torch.logsumexp(x, axis) - math.log(x.shape[axis])


def iw_bound(lp, lq):
    """[N] importance-weighted bound log mean_k exp(log p - log q) (monte_carlo.py:137-141)."""
    return log_mean_exp(lp - lq, 0)


def vimco_cost(lp, lq):
    """[N] vimco() of monte_carlo.py:166-227 over the sample axis 0: the learning signal of sample k is
    LME(log w) - LME(log w with entry k replaced by the mean of the others), held constant."""
    log_w = lp - lq
    K = log_w.shape[0]
    lw = log_w.detach()
    mean_except = (lw.sum(0, keepdim=True) - lw) / (K - 1)
    tiled = lw.unsqueeze(0).expand(K, K, -1).clone()        # [k, k', N]
    idx = torch.arange(K)
    tiled[idx, idx] = mean_except
    signal = log_mean_exp(lw, 0).unsqueeze(0) - log_mean_exp(tiled, 1)
    fake = (lq * signal).sum(0)
    return -fake - log_mean_exp(log_w, 0)


def importance_cost(lp, lq):
    """[N] klpq(...).importance() of inclusive_kl.py:119-151: sum_k w~_k * (-log q_k) with the
    self-normalised weights w~ held constant."""
    w = torch.softmax((lp - lq).detach(), 0)
    return (w * -lq).sum(0)
