"""The generators and discriminators of examples/generative_adversarial_nets (dcgan.py:20-60,
wasserstein_gan.py:20-62) ported line for line onto the fused layers, with their parameters and
the two training steps.  Test and benchmark code, not library code.

Both losses of the examples backpropagate through discriminator(x_gen).  The fused layers release
their saved operand planes after one backward, so a step here runs the discriminator three times:
on the real batch and on x_gen.detach() for disc_loss, then on x_gen again for gen_loss with the
discriminator's moving statistics swapped for throwaway copies and its parameters detached.  In
training mode the batch
moments are the same and the kernels are deterministic, so the logits are the same bits as the
first fake pass.  The discriminator's moving statistics therefore move exactly twice per step:
first on the real batch, then on the fake one.  The reference also updates them twice per step (two
discriminator calls in one graph), in an order TF leaves unspecified."""
import numpy as np
import torch
import torch.nn.functional as F

import zhusuan_b200 as zs

L = zs.fused


def _w(rng, shape, fan_in):
    return torch.tensor(rng.uniform(-1, 1, shape) * np.sqrt(3.0 / fan_in), dtype=torch.float32,
                        device="cuda").requires_grad_(True)


def _bn(c, gamma=True):
    d = {"beta": torch.zeros(c, device="cuda", requires_grad=True),
         "mm": torch.zeros(c, device="cuda"), "mv": torch.ones(c, device="cuda")}
    if gamma:
        d["gamma"] = torch.ones(c, device="cuda", requires_grad=True)
    return d


def dcgan_params(seed=0, z_dim=40, ngf=64, ndf=32):
    rng = np.random.RandomState(seed)
    gen = {"W0": _w(rng, (ngf * 8 * 16, z_dim), z_dim), "bn0": _bn(ngf * 8 * 16),
           "W1": _w(rng, (5, 5, ngf * 4, ngf * 8), 25 * ngf * 8), "bn1": _bn(ngf * 4),
           "W2": _w(rng, (5, 5, ngf * 2, ngf * 4), 25 * ngf * 4), "bn2": _bn(ngf * 2),
           "W3": _w(rng, (5, 5, 3, ngf * 2), 25 * ngf * 2),
           "b3": torch.zeros(3, device="cuda", requires_grad=True)}
    disc = {"W0": _w(rng, (5, 5, 3, ndf * 2), 75), "bn0": _bn(ndf * 2),
            "W1": _w(rng, (5, 5, ndf * 2, ndf * 4), 25 * ndf * 2), "bn1": _bn(ndf * 4),
            "W2": _w(rng, (5, 5, ndf * 4, ndf * 8), 25 * ndf * 4), "bn2": _bn(ndf * 8),
            "Wd": _w(rng, (1, ndf * 8 * 16), ndf * 8 * 16),
            "bd": torch.zeros(1, device="cuda", requires_grad=True)}
    return gen, disc


def wgan_params(seed=0, z_dim=40, ngf=32, ndf=16):
    rng = np.random.RandomState(seed)
    gen = {"W0": _w(rng, (3, 3, ngf * 4, z_dim), 9 * z_dim), "bn0": _bn(ngf * 4, False),
           "W1": _w(rng, (5, 5, ngf * 2, ngf * 4), 25 * ngf * 4), "bn1": _bn(ngf * 2, False),
           "W2": _w(rng, (5, 5, ngf, ngf * 2), 25 * ngf * 2), "bn2": _bn(ngf, False),
           "W3": _w(rng, (5, 5, 1, ngf), 25 * ngf),
           "b3": torch.zeros(1, device="cuda", requires_grad=True)}
    disc = {"W0": _w(rng, (5, 5, 1, ndf), 25), "bn0": _bn(ndf, False),
            "W1": _w(rng, (5, 5, ndf, ndf * 2), 25 * ndf), "bn1": _bn(ndf * 2, False),
            "W2": _w(rng, (5, 5, ndf * 2, ndf * 4), 25 * ndf * 2), "bn2": _bn(ndf * 4, False),
            "Wd": _w(rng, (1, ndf * 4 * 9), ndf * 4 * 9),
            "bd": torch.zeros(1, device="cuda", requires_grad=True)}
    return gen, disc


def trainable(p):
    out = []
    for v in p.values():
        if isinstance(v, dict):
            out += [v[k] for k in ("gamma", "beta") if k in v]
        else:
            out.append(v)
    return out


def _bnl(fn, h, W, b, training, **kw):
    return fn(h, W, b.get("gamma"), b["beta"], b["mm"], b["mv"], training, **kw)


def prior_z(n, z_dim, z=None):
    """z of the examples' registry node bn.uniform("z", -1, 1); a given z is observed."""
    bn = zs.BayesianNet(observed=None if z is None else {"z": z})
    node = bn.uniform("z", -torch.ones(n, z_dim, device="cuda"),
                      torch.ones(n, z_dim, device="cuda"))
    return node.tensor


def dcgan_generator(p, n, training, z=None):
    """dcgan.py:20-40; z from the prior node (or the given value of it)"""
    ngf8 = int(p["W1"].shape[3])
    z = prior_z(n, int(p["W0"].shape[1]), z)
    h = _bnl(L.bn_linear, z, p["W0"], p["bn0"], training)
    h = h.reshape(-1, 4, 4, ngf8)
    h = _bnl(L.bn_conv2d_transpose, h, p["W1"], p["bn1"], training, stride=2, padding="SAME")
    h = _bnl(L.bn_conv2d_transpose, h, p["W2"], p["bn2"], training, stride=2, padding="SAME")
    return L.sigmoid_conv2d_transpose(h, p["W3"], p["b3"], stride=2, padding="SAME")


def dcgan_discriminator(p, x, training):
    """dcgan.py:43-60"""
    h = _bnl(L.bn_conv2d, x, p["W0"], p["bn0"], training, stride=2, padding="SAME")
    h = _bnl(L.bn_conv2d, h, p["W1"], p["bn1"], training, stride=2, padding="SAME")
    h = _bnl(L.bn_conv2d, h, p["W2"], p["bn2"], training, stride=2, padding="SAME")
    return L.linear(h.reshape(h.shape[0], -1), p["Wd"], p["bd"])


def wgan_generator(p, n, training, z=None):
    """wasserstein_gan.py:20-43; z from the prior node (or the given value of it)"""
    z = prior_z(n, int(p["W0"].shape[3]), z)
    h = z.reshape(-1, 1, 1, int(z.shape[-1]))
    h = _bnl(L.bn_conv2d_transpose, h, p["W0"], p["bn0"], training, padding="VALID")
    h = _bnl(L.bn_conv2d_transpose, h, p["W1"], p["bn1"], training, padding="VALID")
    h = _bnl(L.bn_conv2d_transpose, h, p["W2"], p["bn2"], training, stride=2, padding="SAME")
    return L.sigmoid_conv2d_transpose(h, p["W3"], p["b3"], stride=2, padding="SAME")


def wgan_discriminator(p, x, training):
    """wasserstein_gan.py:46-62"""
    h = _bnl(L.bn_conv2d, x, p["W0"], p["bn0"], training, stride=2, padding="SAME")
    h = _bnl(L.bn_conv2d, h, p["W1"], p["bn1"], training, stride=2, padding="SAME")
    h = _bnl(L.bn_conv2d, h, p["W2"], p["bn2"], training, padding="VALID")
    return L.linear(h.reshape(h.shape[0], -1), p["Wd"], p["bd"])


def _gen_pass_params(p):
    """The discriminator as the gen_loss pass sees it: detached parameters (gen_loss's gradient
    is taken w.r.t. the generator only, so no weight-gradient product runs for them) and
    throwaway copies of the moving statistics."""
    q = {}
    for k, v in p.items():
        if isinstance(v, dict):
            q[k] = {kk: (vv.clone() if kk in ("mm", "mv") else vv.detach())
                    for kk, vv in v.items()}
        else:
            q[k] = v.detach()
    return q


def losses(kind, gen, disc, x, z=None):
    """(gen_loss, disc_loss, x_gen, fake logits of the disc_loss pass, of the gen_loss pass) of
    one training step (dcgan.py:79-100, wasserstein_gan.py:82-96), each loss a graph over its
    own parameter list only.  z None: drawn from the prior."""
    G, D = (dcgan_generator, dcgan_discriminator) if kind == "dcgan" else \
        (wgan_generator, wgan_discriminator)
    x_gen = G(gen, int(x.shape[0]), True, z)
    real = D(disc, x, True)
    fake = D(disc, x_gen.detach(), True)
    fake_g = D(_gen_pass_params(disc), x_gen, True)
    if kind == "dcgan":
        ce = F.binary_cross_entropy_with_logits
        gen_loss = ce(fake_g, torch.ones_like(fake_g))
        disc_loss = (ce(real, torch.ones_like(real)) + ce(fake, torch.zeros_like(fake))) / 2.
    else:
        gen_loss = -fake_g.mean()
        disc_loss = -(real - fake).mean()
    return gen_loss, disc_loss, x_gen, fake, fake_g


class TFRMSProp(object):
    """tf.train.RMSPropOptimizer(lr, decay) with its defaults (momentum 0, epsilon 1e-10): the mean
    square starts at ONE and epsilon sits inside the square root,
        ms = decay ms + (1 - decay) g^2,   w -= lr g / sqrt(ms + epsilon)
    unlike torch.optim.RMSprop (zero start, epsilon outside the root)."""

    def __init__(self, params, lr=2e-4, decay=0.5, epsilon=1e-10):
        self.params, self.lr, self.decay, self.eps = list(params), lr, decay, epsilon
        self.ms = [torch.ones_like(p) for p in self.params]

    @torch.no_grad()
    def step(self, grads):
        for p, g, ms in zip(self.params, grads, self.ms):
            ms.mul_(self.decay).add_((1 - self.decay) * g * g)
            p.sub_(self.lr * g / torch.sqrt(ms + self.eps))


def train_step(kind, gen, disc, x, opt_g, opt_d, z=None):
    """One step of the example: both gradient lists from one forward, then the updates
    (WGAN: then the critic's weights clipped to +-0.01, wasserstein_gan.py:118-123)."""
    gen_loss, disc_loss = losses(kind, gen, disc, x, z)[:2]
    gl, dl = trainable(gen), trainable(disc)
    gg = torch.autograd.grad(gen_loss, gl)
    dg = torch.autograd.grad(disc_loss, dl)
    if kind == "dcgan":
        for p, g in zip(gl, gg):
            p.grad = g
        for p, g in zip(dl, dg):
            p.grad = g
        opt_g.step()
        opt_d.step()
    else:
        opt_g.step(gg)
        opt_d.step(dg)
        with torch.no_grad():
            for p in dl:
                p.clamp_(-0.01, 0.01)
    return float(gen_loss), float(disc_loss)


def optimizers(kind, gen, disc):
    if kind == "dcgan":
        return (torch.optim.Adam(trainable(gen), lr=2e-4, betas=(0.5, 0.999)),
                torch.optim.Adam(trainable(disc), lr=2e-4, betas=(0.5, 0.999)))
    return TFRMSProp(trainable(gen)), TFRMSProp(trainable(disc))


def params_from_golden(arrays, kind, role):
    """Trainable CUDA parameters in this module's layout from the arrays of
    tests/golden/ref_gan.npz (gan_oracle.params_from_golden gives the structure)."""
    import gan_oracle as GO
    p = GO.params_from_golden(arrays, kind, role)
    out = {}
    for k, v in p.items():
        if isinstance(v, dict):
            out[k] = {kk: torch.tensor(vv, device="cuda").requires_grad_(kk in ("gamma", "beta"))
                      for kk, vv in v.items()}
        else:
            out[k] = torch.tensor(v, device="cuda").requires_grad_(True)
    return out
