"""Float64 restatement of the semi-supervised VAE (M2) of examples/semi_supervised_vae/vae_ssl.py: the
labeled bound, the unlabeled bound summed over the classes, the classifier cost and the total cost,
in torch float64 on the CPU so that autograd gives their gradients (the same code in float32 on
the GPU is the generic path, in the reference's tiled layout).  The normal noise of the two z
draws is an input, in the reference's row order (the unlabeled rows tiled as row n C + c).

Layers are ``(W [J, K], b [J])`` pairs (tf.layers.dense: h W^T + b), keyed by name, with H
hidden units (500 in the example):
  model (build_gen, :19-33)        g_z: z -> H, g_y: onehot(y) -> H, g_h: H -> H,
                                   g_x: H -> x_dim  (h = relu(g_z(z) + g_y(y)))
  q(z | x, y) (qz_xy, :36-46)      q_h1: [x, y] -> H (ReLU), q_h2 (ReLU), q_mean, q_logstd
  q(y | x) (qy_x, :49-54)          c_h1: x -> H (ReLU), c_h2 (ReLU), c_logits: H -> C
"""
import math

import torch
import torch.nn.functional as F

MODEL = ["g_z", "g_y", "g_h", "g_x"]
ENCODER = ["q_h1", "q_h2", "q_mean", "q_logstd"]
CLASSIFIER = ["c_h1", "c_h2", "c_logits"]
NAMES = MODEL + ENCODER + CLASSIFIER


def dense(h, layer, relu=False):
    W, b = layer
    y = h.to(W.dtype) @ W.t() + b
    return torch.relu(y) if relu else y


def bern_lp(x, logits):
    """sum over the last axis of Bernoulli(logits).log_prob(x) (univariate.py:398-403)."""
    x, logits = torch.broadcast_tensors(x.to(logits.dtype), logits)
    return -F.binary_cross_entropy_with_logits(logits, x, reduction="none").sum(-1)


def normal_lp(z, mean, logstd):
    """sum over the last axis of Normal(mean, logstd).log_prob(z) (univariate.py)."""
    return (-0.5 * math.log(2 * math.pi) - logstd
            - 0.5 * torch.exp(-2 * logstd) * (z - mean) ** 2).sum(-1)


def elbo(x, y1h, eps, L):
    """[M] per-row ELBO of vae_ssl.py's labeled term (elbo(..., axis=0): the mean over the K
    particles of log p(x, y, z) - log q(z | x, y)) for x [M, x_dim], y1h [M, C], eps [K, M, z]."""
    C = y1h.shape[-1]
    dt = L["q_h1"][0].dtype
    h = dense(torch.cat([x.to(dt), y1h.to(dt)], -1), L["q_h1"], True)
    h = dense(h, L["q_h2"], True)
    mean, logstd = dense(h, L["q_mean"]), dense(h, L["q_logstd"])
    z = mean + torch.exp(logstd) * eps
    log_q = normal_lp(z, mean, logstd)
    h = torch.relu(dense(z, L["g_z"]) + dense(y1h, L["g_y"]))
    h = dense(h, L["g_h"], True)
    log_p = (normal_lp(z, torch.zeros_like(z), torch.zeros_like(z)) - math.log(C)
             + bern_lp(x, dense(h, L["g_x"])))
    return (log_p - log_q).mean(0)


def classifier_logits(x, L):
    h = dense(x, L["c_h1"], True)
    return dense(dense(h, L["c_h2"], True), L["c_logits"])


def ssl_step(x_l, y_l, x_u, eps_l, eps_u, L, beta=1200.0):
    """The step of vae_ssl.py:86-141: dict of the labeled bound, the per-datum unlabeled lb_z
    [N, C], the unlabeled bound, the classifier cost, the total cost and the accuracy.
    x_l [N_l, x_dim], y_l one-hot [N_l, C], x_u [N, x_dim], eps_l [K, N_l, z],
    eps_u [K, N C, z] (row n C + c: x_u[n] with class c)."""
    C = y_l.shape[-1]
    N = x_u.shape[0]
    dt = L["g_x"][0].dtype
    lab = elbo(x_l, y_l, eps_l, L).mean()
    x_t = x_u.repeat_interleave(C, 0)
    y_t = torch.eye(C, dtype=dt, device=x_u.device).repeat(N, 1)
    lb_z = elbo(x_t, y_t, eps_u, L).reshape(N, C)
    qy = torch.softmax(classifier_logits(x_u, L), -1) + 1e-8
    qy = qy / qy.sum(1, keepdim=True)
    unl = (qy * (lb_z - torch.log(qy))).sum(1).mean()
    logits_l = classifier_logits(x_l, L)
    log_qy_x = (y_l.to(dt) * torch.log_softmax(logits_l, -1)).sum(-1)
    clf = -beta * log_qy_x.mean()
    acc = (logits_l.argmax(1) == y_l.argmax(1)).to(dt).mean()
    cost = -(lab + unl - clf) / 2.0
    return dict(labeled_lb=lab, lb_z=lb_z, unlabeled_lb=unl, classifier_cost=clf, cost=cost,
                acc=acc)
