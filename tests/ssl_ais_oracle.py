"""Float64 restatement of the semi-supervised VAE trained by adaptive importance sampling
(examples/semi_supervised_vae/vae_ssl_adaptive_is.py), in torch float64 on the CPU so that autograd
gives its gradients.  Its noise is an input: the uniforms that binarise x, the unlabeled class draws
(indices) and the standard normals of both z draws.

Layers are ``(W [J, K], b [J])`` pairs keyed by the names of tests/ssl_oracle.py: the model
(build_gen, :19-33) g_z, g_y, g_h, g_x; q(z | x, y) (qz_xy, :36-43) q_h1 ([x, y] -> H), q_h2, q_mean,
q_logstd; q(y | x) (qy_x, :46-51) c_h1, c_h2, c_logits.  Both proposals draw z without
reparameterisation (:53-68), so z is a constant and log q keeps its partials.
"""
import math

import torch

from ssl_oracle import CLASSIFIER, ENCODER, MODEL, NAMES, bern_lp, dense, normal_lp  # noqa: F401

PROPOSAL = CLASSIFIER + ENCODER


def qz_xy(x, y1h, L):
    dt = L["q_h1"][0].dtype
    h = dense(torch.cat([x.to(dt), y1h.to(dt)], -1), L["q_h1"], True)
    h = dense(h, L["q_h2"], True)
    return dense(h, L["q_mean"]), dense(h, L["q_logstd"])


def qy_logits(x, L):
    h = dense(x, L["c_h1"], True)
    return dense(dense(h, L["c_h2"], True), L["c_logits"])


def log_joint(x, y1h, z, L):
    """log p(x, y, z) of build_gen [K, N]: N(0, 1) prior on z, uniform prior on the C classes."""
    C = y1h.shape[-1]
    h = torch.relu(dense(z, L["g_z"]) + dense(y1h, L["g_y"]))
    h = dense(h, L["g_h"], True)
    return (normal_lp(z, torch.zeros_like(z), torch.zeros_like(z)) - math.log(C)
            + bern_lp(x, dense(h, L["g_x"])))


def objectives(log_p, log_q):
    """(importance_weighted_objective, klpq(...).importance()) over axis 0, each averaged over the
    rows: log_mean_exp(log w) and sum_k w~_k (-log q_k), w~ the constant normalised weights."""
    log_w = log_p - log_q
    K = log_w.shape[0]
    lb = (torch.logsumexp(log_w, 0) - math.log(K)).mean()
    w = torch.softmax(log_w, 0).detach()
    return lb, (w * -log_q).sum(0).mean()


def ais_step(x_l, y_l, x_u, eps_l, eps_u, y_u, L, beta=1200.0):
    """Bounds, costs and accuracy of one step of :75-159 on binarised x_l [N_l, x_dim], one-hot y_l
    [N_l, C], binarised x_u [N_u, x_dim], eps_l [K, N_l, z], eps_u [K, N_u, z] and the unlabeled
    class draws y_u [N_u] (indices)."""
    dt = L["g_x"][0].dtype
    C = y_l.shape[-1]
    y_l = y_l.to(dt)
    mean, logstd = qz_xy(x_l, y_l, L)
    z = (mean + torch.exp(logstd) * eps_l).detach()
    lab_lb, lab_q = objectives(log_joint(x_l, y_l, z, L), normal_lp(z, mean, logstd))
    logits_u = qy_logits(x_u, L)
    y1h = torch.nn.functional.one_hot(y_u.long(), C).to(dt)
    log_qy = (y1h * torch.log_softmax(logits_u, -1)).sum(-1)
    mean, logstd = qz_xy(x_u, y1h, L)
    z = (mean + torch.exp(logstd) * eps_u).detach()
    unl_lb, unl_q = objectives(log_joint(x_u, y1h, z, L), normal_lp(z, mean, logstd) + log_qy)
    logits_l = qy_logits(x_l, L)
    clf = -beta * (y_l * torch.log_softmax(logits_l, -1)).sum(-1).mean()
    acc = (logits_l.argmax(1) == y_l.argmax(1)).to(dt).mean()
    return dict(labeled_lb=lab_lb, unlabeled_lb=unl_lb, labeled_q_cost=lab_q,
                unlabeled_q_cost=unl_q, classifier_cost=clf, acc=acc,
                model_cost=-lab_lb - unl_lb, proposal_cost=lab_q + unl_q + clf)


def step_grads(out, L):
    """{name: (dW, db)}: model_cost w.r.t. the model's layers, proposal_cost w.r.t. qy_x's and
    qz_xy's (:148-156)."""
    res = {}
    for cost, names in ((out["model_cost"], MODEL), (out["proposal_cost"], PROPOSAL)):
        gs = torch.autograd.grad(cost, [p for n in names for p in L[n]], retain_graph=True)
        for i, n in enumerate(names):
            res[n] = (gs[2 * i], gs[2 * i + 1])
    return res
