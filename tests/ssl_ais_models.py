"""The semi-supervised VAE trained by adaptive importance sampling
(examples/semi_supervised_vae/vae_ssl_adaptive_is.py) on the GPU, in two arms: ``fused`` runs every
dense layer on the project's dense-layer kernels -- build_gen's ``relu(dense(z) + dense(y))`` and
qz_xy's ``dense(concat([x, y]))`` as ``class_linear``, qy_x's last layer as
``LinearOnehotCategorical`` and both proposals' z heads as ``LinearNormal(..., group_ndims=1,
is_reparameterized=False)``; ``generic`` runs ``F.linear`` and the registry's distributions.
Imported by the GPU tests and scripts/bench_linear_normal.py.

Parameters are ``{name: (W [J, K], b [J])}`` with the names of tests/ssl_ais_oracle.py.  The noise
can be injected (the uniforms that binarise x, the uniforms of the unlabeled class draws, the
normals of both z draws) or drawn from ``zs.random``.
"""
import math

import torch
import torch.nn.functional as F

MODEL = ["g_z", "g_y", "g_h", "g_x"]
ENCODER = ["q_h1", "q_h2", "q_mean", "q_logstd"]
CLASSIFIER = ["c_h1", "c_h2", "c_logits"]
NAMES = MODEL + ENCODER + CLASSIFIER
PROPOSAL = CLASSIFIER + ENCODER
HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)


def init_params(rng, x_dim, z_dim, C, H=500, device="cuda"):
    """Glorot-uniform kernels (tf.layers.dense's default) and zero biases, as float32 leaves."""
    fans = dict(g_z=(z_dim, H), g_y=(C, H), g_h=(H, H), g_x=(H, x_dim), q_h1=(x_dim + C, H),
                q_h2=(H, H), q_mean=(H, z_dim), q_logstd=(H, z_dim), c_h1=(x_dim, H),
                c_h2=(H, H), c_logits=(H, C))
    P = {}
    for n in NAMES:
        i, o = fans[n]
        lim = math.sqrt(6.0 / (i + o))
        W = torch.tensor(rng.uniform(-lim, lim, (o, i)), dtype=torch.float32, device=device)
        P[n] = (W.requires_grad_(True), torch.zeros(o, device=device, requires_grad=True))
    return P


class Arm(object):
    def __init__(self, zs, P, fused):
        self.zs, self.P, self.fused = zs, P, fused

    def lin(self, h, name, relu=False):
        if self.fused:
            return self.zs.fused.linear(h, *self.P[name], relu=relu)
        y = F.linear(h, *self.P[name])
        return F.relu(y) if relu else y

    def qy(self, x):
        """q(y | x): the layer of qy_x (:46-51) as a distribution."""
        h = self.lin(self.lin(x, "c_h1", True), "c_h2", True)
        if self.fused:
            return self.zs.fused.LinearOnehotCategorical(h, *self.P["c_logits"])
        return self.zs.distributions.OnehotCategorical(self.lin(h, "c_logits"))

    def qz(self, x, y):
        """q(z | x, y) of qz_xy (:36-43); y is one-hot [N, C] (or a LinearOnehotCategorical draw)."""
        xd = int(x.shape[-1])
        Wq, bq = self.P["q_h1"]
        if self.fused:
            h = self.zs.fused.class_linear(x, Wq[:, :xd], Wq[:, xd:], y, b=bq, relu=True)
            h = self.lin(h, "q_h2", True)
            return self.zs.fused.LinearNormal(h, *self.P["q_mean"], *self.P["q_logstd"],
                                              group_ndims=1, is_reparameterized=False)
        h = F.relu(F.linear(torch.cat([x, y.to(x.dtype)], -1), Wq, bq))
        h = self.lin(h, "q_h2", True)
        return self.zs.distributions.Normal(self.lin(h, "q_mean"), logstd=self.lin(h, "q_logstd"),
                                            group_ndims=1, is_reparameterized=False)

    def log_joint(self, x, y, z):
        """log p(x, y, z) of build_gen (:19-33), [K, N]."""
        C = int(self.P["g_y"][0].shape[1])
        lp_z = -HALF_LOG_2PI * int(z.shape[-1]) - 0.5 * (z * z).sum(-1)
        if self.fused:
            Wz, bz = self.P["g_z"]
            Wy, by = self.P["g_y"]
            h = self.zs.fused.class_linear(z, Wz, Wy, y, b=bz + by, relu=True)
            h = self.lin(h, "g_h", True)
            lp_x = self.zs.fused.LinearBernoulli(h, *self.P["g_x"]).log_prob(x)
        else:
            h = F.relu(self.lin(z, "g_z") + self.lin(y.to(z.dtype), "g_y"))
            h = self.lin(h, "g_h", True)
            lp_x = self.zs.distributions.Bernoulli(self.lin(h, "g_x"), group_ndims=1).log_prob(x)
        return lp_z - math.log(C) + lp_x

    def objectives(self, log_p, log_q):
        """importance_weighted_objective and klpq(...).importance() over axis 0, row means."""
        ops = self.zs.ops
        log_w = log_p - log_q
        lb = ops.reduce_axes(log_w, ops.OP_LME, 0).mean()
        w = ops.normalized_weights(log_w, 0)
        return lb, (w * -log_q).sum(0).mean()


def _draw_z(q, K, eps, fused):
    """K draws of z with the injected normals eps (or from zs.random when None)."""
    return q.sample(K, eps=eps) if fused else q._sample(K, eps=eps)


def ais_step(zs, P, x_l, y_l, x_u, K, fused, u_l=None, u_u=None, u_y=None, eps_l=None,
             eps_u=None, beta=1200.0):
    """Bounds, costs and accuracy of one step (:75-146).  x_l / x_u: the pixel probabilities,
    binarised here as u < x with the uniforms u_l / u_u (drawn from zs.random when None; u = 0
    keeps an already binary x).  y_l one-hot [N_l, C] float.  u_y: the uniforms of the unlabeled
    class draws [N_u]; eps_l [K, N_l, z], eps_u [K, N_u, z] (drawn when None)."""
    arm = Arm(zs, P, fused)

    def binarise(p, u):
        if u is None:
            u = zs.ops.base_noise(0, p.shape, p.device, seed=zs.random.get_seed(),
                                  it=zs.random.next_counter())
        return (u < p).to(torch.float32)
    x_l, x_u = binarise(x_l, u_l), binarise(x_u, u_u)
    C = int(y_l.shape[-1])
    # labeled proposal and its objectives (:53-58, :84-95)
    q = arm.qz(x_l, y_l)
    z = _draw_z(q, K, eps_l, fused)
    lab_lb, lab_q = arm.objectives(arm.log_joint(x_l, y_l, z), q.log_prob(z))
    # unlabeled proposal (:61-68, :105-116): one class draw per row, K z draws
    qy = arm.qy(x_u)
    if fused:
        y = qy.sample(u=u_y)
    else:
        draws = zs.ops.sample_categorical(qy.logits, 1, u=u_y, seed=zs.random.get_seed(),
                                          it=zs.random.next_counter())
        y = F.one_hot(draws[0].long(), C).to(torch.int32)
    log_qy = qy.log_prob(y)
    q = arm.qz(x_u, y)
    z = _draw_z(q, K, eps_u, fused)
    unl_lb, unl_q = arm.objectives(arm.log_joint(x_u, y, z), q.log_prob(z) + log_qy)
    # classifier (:119-128)
    ql = arm.qy(x_l)
    clf = -beta * ql.log_prob(y_l).mean()
    acc = (ql.logits.argmax(1) == y_l.argmax(1)).float().mean()
    return dict(labeled_lb=lab_lb, unlabeled_lb=unl_lb, labeled_q_cost=lab_q,
                unlabeled_q_cost=unl_q, classifier_cost=clf, acc=acc,
                model_cost=-lab_lb - unl_lb, proposal_cost=lab_q + unl_q + clf,
                y_u=y.argmax(-1))


def step_grads(out, P):
    """{name: (dW, db)}: model_cost w.r.t. the model's layers, proposal_cost w.r.t. qy_x's and
    qz_xy's (:148-156)."""
    res = {}
    for cost, names in ((out["model_cost"], MODEL), (out["proposal_cost"], PROPOSAL)):
        gs = torch.autograd.grad(cost, [p for n in names for p in P[n]], retain_graph=True)
        for i, n in enumerate(names):
            res[n] = (gs[2 * i], gs[2 * i + 1])
    return res


class Adam(object):
    """tf.train.AdamOptimizer(3e-4) (epsilon 1e-8) applied to both gradient lists (:156-159)."""

    def __init__(self, P, lr=3e-4, b1=0.9, b2=0.999, eps=1e-8):
        self.P, self.lr, self.b1, self.b2, self.eps, self.t = P, lr, b1, b2, eps, 0
        self.m = {n: [torch.zeros_like(p) for p in P[n]] for n in P}
        self.v = {n: [torch.zeros_like(p) for p in P[n]] for n in P}

    @torch.no_grad()
    def step(self, grads):
        self.t += 1
        lr = self.lr * math.sqrt(1 - self.b2 ** self.t) / (1 - self.b1 ** self.t)
        for n, gs in grads.items():
            for p, g, m, v in zip(self.P[n], gs, self.m[n], self.v[n]):
                m.mul_(self.b1).add_(g, alpha=1 - self.b1)
                v.mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
                p.sub_(lr * m / (v.sqrt() + self.eps))


def train_step(zs, P, opt, x_l, y_l, x_u, K, fused, **noise):
    """One training step: the step's bounds, both gradient lists, one Adam update."""
    out = ais_step(zs, P, x_l, y_l, x_u, K, fused, **noise)
    opt.step(step_grads(out, P))
    return out


def test_batch(zs, P, x, y, K, fused, **noise):
    """The test-batch evaluation (:190-200): both bounds and the accuracy of binary x [N, x_dim]
    with labels y [N, C], at K = ll_samples particles."""
    zero = torch.zeros_like(x)
    with torch.no_grad():
        out = ais_step(zs, P, x, y, x, K, fused, u_l=zero, u_u=zero, **noise)
    return dict(labeled_lb=out["labeled_lb"], unlabeled_lb=out["unlabeled_lb"], acc=out["acc"])
