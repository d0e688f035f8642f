"""Float64 restatement of the variational-dropout classifier of
examples/bayesian_neural_nets/variational_dropout.py, in torch on the CPU so that autograd gives its
gradients (the same code in float32 on the GPU is the generic path: F.linear and a batch-norm
restatement).

Layer i (:26-37): y = relu(BN((h * eps_i) W_i^T)), tf.contrib.layers.fully_connected with
layers.batch_norm: no bias, beta_i and no gamma, epsilon 1e-3.  Training normalises with the batch
moments over every particle row (population variance) and moves the moving statistics by
m -= (m - batch) * (1 - decay); evaluation normalises with the moving statistics.  The ReLU applies
to every layer, the logits layer included.

q (:40-50): eps_i = 1 + sqrt(sigmoid(logit_alpha_i) + 1e-10) z_i with z_i ~ N(0, 1) [S, n, n_in]
given.  log_joint = sum_i log N(eps_i; 1, 1) + N_train log Categorical(logits).log_prob(y), the
bound is mean over particles of log_joint - log q, and the cost is -mean(bound) / N_train.
"""
import math

import torch

DECAY, EPSILON = 0.999, 1e-3


def bn_layer(h, eps, W, beta, mm, mv, training, relu=True, decay=DECAY, epsilon=EPSILON):
    """(y, new moving mean, new moving variance) of one layer; h broadcasts against eps."""
    a = (h * eps) @ W.t()
    if training:
        rows = a.reshape(-1, a.shape[-1])
        mean = rows.mean(0)
        var = ((rows - mean.detach()) ** 2).mean(0)
        d = 1.0 - decay
        new_mm = mm - (mm - mean.detach()) * d
        new_mv = mv - (mv - var.detach()) * d
    else:
        mean, var, new_mm, new_mv = mm, mv, mm, mv
    y = (a - mean) * torch.rsqrt(var + epsilon) + beta
    return (torch.relu(y) if relu else y), new_mm, new_mv


def normal_lp(x, mean, std):
    """sum over the last axis of Normal(mean, std).log_prob(x)."""
    return (-0.5 * math.log(2 * math.pi) - torch.log(std)
            - 0.5 * ((x - mean) / std) ** 2).sum(-1)


def q_std(logit_alpha):
    return torch.sqrt(torch.sigmoid(logit_alpha) + 1e-10)


def vardrop_run(x, y, z, Ws, betas, logit_alphas, mms, mvs, training, n_train, layer=bn_layer):
    """x [n, K0], y int [n], z: per layer [S, n, n_in]; returns a dict of bound, cost, acc, logits
    [S, n, C], and the moving statistics after the run (lists).  ``layer(h, eps, W, beta, mm, mv,
    training)`` -> (y, moving mean, moving variance) computes one layer (default: bn_layer)."""
    h = x
    lp_eps, lq_eps = 0.0, 0.0
    new_m, new_v = [], []
    for i, (W, beta) in enumerate(zip(Ws, betas)):
        std = q_std(logit_alphas[i])
        eps = 1.0 + std * z[i]
        lq_eps = lq_eps + normal_lp(eps, torch.ones_like(eps), std.expand_as(eps))
        lp_eps = lp_eps + normal_lp(eps, torch.ones_like(eps), torch.ones_like(eps))
        h, m, v = layer(h, eps, W, beta, mms[i], mvs[i], training)
        new_m.append(m)
        new_v.append(v)
    logits = h
    log_py = torch.log_softmax(logits, -1).gather(-1, y.long().expand(
        logits.shape[:-1]).unsqueeze(-1)).squeeze(-1)
    lower_bound = (lp_eps + log_py * n_train - lq_eps).mean(0)
    pred = torch.softmax(logits, -1).mean(0).argmax(1)
    acc = (pred == y.long()).to(logits.dtype).mean()
    return dict(bound=lower_bound.mean() / n_train, cost=-lower_bound.mean() / n_train, acc=acc,
                logits=logits, moving_mean=new_m, moving_variance=new_v)
