"""The semi-supervised VAE trained by adaptive importance sampling
(examples/semi_supervised_vae/vae_ssl_adaptive_is.py) on the GPU: the fused arm of
tests/ssl_ais_models.py (class_linear, LinearOnehotCategorical and LinearNormal) and the generic arm
(F.linear and the registry) replay the reference run of tests/golden/ref_ssl_ais.npz, and at the
example's shape (500 hidden units, z 100, K 10, 100 labeled + 100 unlabeled rows) both match the
float64 oracle of tests/ssl_ais_oracle.py, through one Adam step and a test batch."""
import os

import numpy as np
import pytest
import torch

import ssl_ais_models as SM
import ssl_ais_oracle as SA

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = ("labeled_lb", "unlabeled_lb", "labeled_q_cost", "unlabeled_q_cost", "classifier_cost",
        "acc")


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return t.detach().double().cpu()


def _u_for_classes(x, L, y):
    """Uniforms that draw the classes y from q(y | x) by the inverse CDF: the middle of each
    class's interval, from the float64 logits."""
    p = torch.softmax(SA.qy_logits(x, L), -1)
    cdf = torch.cumsum(p, -1)
    hi = cdf.gather(1, y.long().view(-1, 1)).squeeze(1)
    lo = hi - p.gather(1, y.long().view(-1, 1)).squeeze(1)
    return (0.5 * (lo + hi)).float()


def _check(out, want, grads, want_grads, rtol=2e-5, atol=1e-5, grtol=2e-3):
    for k in KEYS:
        w = want[k].detach().numpy() if isinstance(want[k], torch.Tensor) else want[k]
        np.testing.assert_allclose(N64(out[k]).numpy(), w, rtol=rtol, atol=atol, err_msg=k)
    for n in SA.NAMES:
        for what, g, w in zip(("W", "b"), grads[n], want_grads[n]):
            w = w.numpy() if isinstance(w, torch.Tensor) else w
            np.testing.assert_allclose(N64(g).numpy(), w, rtol=grtol,
                                       atol=grtol * 0.1 * max(1.0, float(np.abs(w).max())),
                                       err_msg="grad %s %s" % (what, n))


@pytest.mark.parametrize("fused", [True, False])
def test_reference_run_replays(zs, fused):
    g = np.load(os.path.join(GOLD, "ref_ssl_ais.npz"))
    P = {n: tuple(T(g[p + n]).requires_grad_(True) for p in ("W_", "b_")) for n in SA.NAMES}
    L = {n: tuple(torch.tensor(g[p + n], dtype=torch.float64) for p in ("W_", "b_"))
         for n in SA.NAMES}
    x_u64 = (torch.tensor(g["u_u"]) < torch.tensor(g["xp_u"])).double()
    u_y = T(_u_for_classes(x_u64, L, torch.tensor(g["y_u"])))
    out = SM.ais_step(zs, P, T(g["xp_l"]), T(g["y_l"]), T(g["xp_u"]), int(g["eps_l"].shape[0]),
                      fused, u_l=T(g["u_l"]), u_u=T(g["u_u"]), u_y=u_y, eps_l=T(g["eps_l"]),
                      eps_u=T(g["eps_u"]))
    assert torch.equal(out["y_u"].cpu(), torch.tensor(g["y_u"]).long())
    want_g = {n: (g["grad_W_" + n], g["grad_b_" + n]) for n in SA.NAMES}
    _check(out, {k: g[k] for k in KEYS}, SM.step_grads(out, P), want_g)
    x = T(g["test_x"])
    L64 = {n: tuple(t.clone() for t in L[n]) for n in SA.NAMES}
    t_u = T(_u_for_classes(x.double().cpu(), L64, torch.tensor(g["test_y_u"])))
    got = SM.test_batch(zs, P, x, T(g["test_y"]), int(g["eps_l"].shape[0]), fused, u_y=t_u,
                        eps_l=T(g["test_eps_l"]), eps_u=T(g["test_eps_u"]))
    for k in ("labeled_lb", "unlabeled_lb", "acc"):
        np.testing.assert_allclose(N64(got[k]).numpy(), g["test_" + k], rtol=2e-5, atol=1e-5,
                                   err_msg="test " + k)


@pytest.mark.parametrize("fused", [True, False])
def test_example_shape_against_float64(zs, fused):
    """500 hidden units, z 100, K 10, 100 labeled and 100 unlabeled rows of 784 pixels: the step's
    bounds, costs and both gradient lists against float64, then one Adam step and a test batch."""
    rng = np.random.default_rng(7)
    x_dim, z_dim, C, K, N = 784, 100, 10, 10, 100
    P = SM.init_params(rng, x_dim, z_dim, C)
    xp_l, xp_u = T(rng.random((N, x_dim)) * 0.5), T(rng.random((N, x_dim)) * 0.5)
    y_l = T(np.eye(C)[rng.integers(0, C, N)])
    noise = dict(u_l=T(rng.random((N, x_dim))), u_u=T(rng.random((N, x_dim))),
                 u_y=T(rng.random(N)), eps_l=T(rng.standard_normal((K, N, z_dim))),
                 eps_u=T(rng.standard_normal((K, N, z_dim))))
    out = SM.ais_step(zs, P, xp_l, y_l, xp_u, K, fused, **noise)
    grads = SM.step_grads(out, P)
    L = {n: tuple(N64(t).requires_grad_(True) for t in P[n]) for n in SA.NAMES}
    x_l64 = (N64(noise["u_l"]) < N64(xp_l)).double()
    x_u64 = (N64(noise["u_u"]) < N64(xp_u)).double()
    want = SA.ais_step(x_l64, N64(y_l), x_u64, N64(noise["eps_l"]), N64(noise["eps_u"]),
                       out["y_u"].cpu(), L)
    _check(out, want, grads, SA.step_grads(want, L), rtol=1e-4, atol=1e-3, grtol=5e-3)
    opt = SM.Adam(P)
    opt.step(grads)
    x_t = T(rng.random((N, x_dim)) < 0.3)
    y_t = T(np.eye(C)[rng.integers(0, C, N)])
    tnoise = dict(u_y=T(rng.random(N)), eps_l=T(rng.standard_normal((K, N, z_dim))),
                  eps_u=T(rng.standard_normal((K, N, z_dim))))
    got = SM.test_batch(zs, P, x_t, y_t, K, fused, **tnoise)
    L = {n: tuple(N64(t) for t in P[n]) for n in SA.NAMES}
    full = SM.ais_step(zs, P, x_t, y_t, x_t, K, fused, u_l=torch.zeros_like(x_t),
                       u_u=torch.zeros_like(x_t), **tnoise)
    want = SA.ais_step(N64(x_t), N64(y_t), N64(x_t), N64(tnoise["eps_l"]), N64(tnoise["eps_u"]),
                       full["y_u"].cpu(), L)
    for k in ("labeled_lb", "unlabeled_lb", "acc"):
        np.testing.assert_allclose(N64(got[k]).numpy(), want[k].detach().numpy(), rtol=1e-4,
                                   atol=1e-3, err_msg="test " + k)
