"""The class-conditioned dense layer (zs.fused.class_linear) and the semi-supervised VAE of
examples/semi_supervised_vae/vae_ssl.py on it: per-row and enumerated forward against float64,
bit equality of the enumerated layer with the per-row layer on the tiled input, gradients, NaN rows
for out-of-range classes, inference mode, the reference run of tests/golden/ref_ssl.npz replayed on
the fused and the generic path, and a training step at the example's shape against the float64
oracle of tests/ssl_oracle.py."""
import math
import os

import numpy as np
import pytest
import torch

import ssl_oracle as SS

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return t.detach().double().cpu()


def _layer(rng, J, K, C):
    W = T(rng.standard_normal((J, K)) / math.sqrt(K))
    Wc = T(rng.standard_normal((J, C)))
    b = T(0.5 * rng.standard_normal(J))
    return W, Wc, b


def _input(zs, rng, lead, K, kind):
    """Activation [*lead, K]: dense floats, or a LinearBernoulli sample (binary operand plane)."""
    if kind == "dense":
        return T(rng.standard_normal(lead + (K,)))
    h0 = T(rng.standard_normal(lead + (16,)))
    W0 = T(rng.standard_normal((K, 16)))
    return zs.fused.LinearBernoulli(h0, W0, dtype=torch.float32).sample()


def _want(h, W, Wc, b, y, relu):
    y64 = N64(h) @ N64(W).t() + N64(b) + N64(Wc).t()[y.long().cpu()]
    return torch.relu(y64) if relu else y64


CONFIGS = [("index", "dense", False), ("onehot", "binary", True), ("broadcast", "dense", True),
           ("index", "binary", False)]


@pytest.mark.parametrize("J", [20, 200, 500, 784])
@pytest.mark.parametrize("C", [2, 10, 37])
def test_per_row_forward_matches_float64(zs, J, C):
    rng = np.random.default_rng(J * 100 + C)
    K = 72
    for ykind, hkind, relu in CONFIGS:
        lead = (3, 70) if ykind == "broadcast" else (301,)
        h = _input(zs, rng, lead, K, hkind)
        W, Wc, b = _layer(rng, J, K, C)
        yi = T(rng.integers(0, C, lead[-1:]), torch.int64)
        y = torch.nn.functional.one_hot(yi, C).float() if ykind == "onehot" else yi
        out = zs.fused.class_linear(h, W, Wc, y, b=b, relu=relu)
        assert out.shape == lead + (J,)
        want = _want(h.reshape(-1, K), W, Wc, b, yi.repeat(int(np.prod(lead[:-1]))), relu)
        np.testing.assert_allclose(N64(out).reshape(-1, J).numpy(), want.numpy(), rtol=1e-5,
                                   atol=1e-4, err_msg="%s %s relu=%s" % (ykind, hkind, relu))


@pytest.mark.parametrize("hkind", ["dense", "binary"])
@pytest.mark.parametrize("R,J,C", [(100, 500, 10), (129, 200, 37), (7, 784, 2)])
def test_enumerated_is_bitwise_the_per_row_layer_on_the_tiled_input(zs, hkind, R, J, C):
    rng = np.random.default_rng(R + J + C)
    K = 100
    h = _input(zs, rng, (R,), K, hkind)
    W, Wc, b = _layer(rng, J, K, C)
    for relu in (False, True):
        enum = zs.fused.class_linear(h, W, Wc, None, b=b, relu=relu)
        assert enum.shape == (C, R, J)
        tiled = zs.fused.class_linear(h.detach().clone().repeat(C, 1), W, Wc,
                                      torch.arange(C, device="cuda").repeat_interleave(R),
                                      b=b, relu=relu)
        assert torch.equal(enum.reshape(C * R, J), tiled)


def _grads(out, params, gy):
    return torch.autograd.grad(out, params, gy)


def _close_grads(got, want, what):
    for name, a, w in zip(("h", "W", "W_class", "b"), got, want):
        w = w.numpy() if isinstance(w, torch.Tensor) else w
        np.testing.assert_allclose(N64(a).numpy(), w, rtol=2e-3,
                                   atol=2e-4 * max(1.0, float(np.abs(w).max())),
                                   err_msg="%s d%s" % (what, name))


@pytest.mark.parametrize("R,J,C,relu", [(301, 500, 10, True), (64, 200, 37, False),
                                        (130, 784, 2, True)])
def test_gradients_match_float64(zs, R, J, C, relu):
    rng = np.random.default_rng(R * J + C)
    K = 136
    h = T(rng.standard_normal((R, K))).requires_grad_(True)
    W, Wc, b = (t.requires_grad_(True) for t in _layer(rng, J, K, C))
    params = [h, W, Wc, b]
    p64 = [N64(p).requires_grad_(True) for p in params]
    # per row
    y = T(rng.integers(0, C, R), torch.int64)
    gy = T(rng.standard_normal((R, J)))
    out = zs.fused.class_linear(h, W, Wc, y, b=b, relu=relu)
    o64 = p64[0] @ p64[1].t() + p64[3] + p64[2].t()[y.cpu()]
    o64 = torch.relu(o64) if relu else o64
    _close_grads(_grads(out, params, gy), torch.autograd.grad(o64, p64, N64(gy)), "per-row")
    # enumerated: against float64 and against the per-row layer on the tiled input
    gy = T(rng.standard_normal((C, R, J)))
    out = zs.fused.class_linear(h, W, Wc, None, b=b, relu=relu)
    ge = _grads(out, params, gy)
    o64 = (p64[0] @ p64[1].t() + p64[3]).unsqueeze(0) + p64[2].t().unsqueeze(1)
    o64 = torch.relu(o64) if relu else o64
    _close_grads(ge, torch.autograd.grad(o64, p64, N64(gy)), "enumerated")
    ht = h.repeat(C, 1)
    tiled = zs.fused.class_linear(ht, W, Wc, torch.arange(C, device="cuda").repeat_interleave(R),
                                  b=b, relu=relu)
    gt = _grads(tiled, params, gy.reshape(C * R, J))
    _close_grads(ge, [N64(g) for g in gt], "enumerated vs tiled")


def test_gradients_of_a_binary_input_and_broadcast_classes(zs):
    rng = np.random.default_rng(5)
    K, J, C = 200, 500, 10
    h = _input(zs, rng, (4, 90), K, "binary")
    W, Wc, b = (t.requires_grad_(True) for t in _layer(rng, J, K, C))
    y = T(rng.integers(0, C, 90), torch.int64)
    gy = T(rng.standard_normal((4, 90, J)))
    out = zs.fused.class_linear(h, W, Wc, y, b=b, relu=True)
    got = torch.autograd.grad(out, [W, Wc, b], gy)
    p64 = [N64(p).requires_grad_(True) for p in (W, Wc, b)]
    o64 = torch.relu(N64(h) @ p64[0].t() + p64[2] + p64[1].t()[y.cpu()])
    want = torch.autograd.grad(o64, p64, N64(gy))
    for name, a, w in zip(("W", "W_class", "b"), got, want):
        np.testing.assert_allclose(N64(a).numpy(), w.numpy(), rtol=2e-3,
                                   atol=2e-4 * max(1.0, float(w.abs().max())), err_msg=name)


@pytest.mark.parametrize("relu", [False, True])
def test_out_of_range_class_gives_a_nan_row(zs, relu):
    rng = np.random.default_rng(11)
    R, K, J, C = 200, 64, 200, 10
    h = T(rng.standard_normal((R, K)))
    W, Wc, b = _layer(rng, J, K, C)
    y = T(rng.integers(0, C, R), torch.int64)
    good = zs.fused.class_linear(h, W, Wc, y, b=b, relu=relu)
    bad_rows = [3, 130, 199]
    y_bad = y.clone()
    y_bad[3], y_bad[130], y_bad[199] = C, -1, C + 1000
    out = zs.fused.class_linear(h, W, Wc, y_bad, b=b, relu=relu)
    assert torch.isnan(out[bad_rows]).all()
    keep = torch.ones(R, dtype=torch.bool, device="cuda")
    keep[bad_rows] = False
    assert torch.equal(out[keep], good[keep])


def test_inference_mode(zs):
    rng = np.random.default_rng(3)
    R, K, J, C = 150, 100, 500, 10
    h = T(rng.standard_normal((R, K)))
    W, Wc, b = _layer(rng, J, K, C)
    y = T(rng.integers(0, C, R), torch.int64)
    want = zs.fused.class_linear(h, W, Wc, y, b=b, relu=True)
    want_e = zs.fused.class_linear(h, W, Wc, None, b=b, relu=True)
    with torch.inference_mode():
        hi = h.clone()
        got = zs.fused.class_linear(hi, W, Wc, y, b=b, relu=True)
        got_e = zs.fused.class_linear(hi, W, Wc, None, b=b, relu=True)
        nxt = zs.fused.linear(got_e, T(rng.standard_normal((7, J))))
    assert torch.equal(got, want) and torch.equal(got_e, want_e)
    assert nxt.shape == (C, R, 7)


# ---- the semi-supervised VAE of vae_ssl.py on class_linear -------------------------------------
def fused_ssl_step(zs, x_l, y_l, x_u, eps_l, eps_u, P, beta=1200.0):
    """vae_ssl.py:86-141 on fused layers: the one-hot class of the encoder's first layer and of the
    decoder's first layer is gathered in the epilogue, and the unlabeled rows enumerate the classes
    from one product over x_u (class-major).  y_l: int class indices [N_l]; eps_u [K, C, N, z]
    class-major.  Returns the quantities of ssl_oracle.ssl_step, with lb_z [C, N]."""
    C = int(P["g_y"][0].shape[1])
    xd = int(x_l.shape[1])
    Wq, bq = P["q_h1"]
    Wx, Wy = Wq[:, :xd], Wq[:, xd:]
    b_dec = P["g_z"][1] + P["g_y"][1]

    def encoder(h1):
        h = zs.fused.linear(h1, *P["q_h2"], relu=True)
        return zs.fused.linear(h, *P["q_mean"]), zs.fused.linear(h, *P["q_logstd"])

    def elbo(h1, eps, y, x):
        mean, logstd = encoder(h1)
        z = mean + torch.exp(logstd) * eps
        log_q = SS.normal_lp(z, mean, logstd)
        h = zs.fused.class_linear(z, P["g_z"][0], P["g_y"][0], y, b=b_dec, relu=True)
        h = zs.fused.linear(h, *P["g_h"], relu=True)
        log_p = (SS.normal_lp(z, torch.zeros_like(z), torch.zeros_like(z)) - math.log(C)
                 + zs.fused.LinearBernoulli(h, *P["g_x"]).log_prob(x))
        return (log_p - log_q).mean(0)

    def classifier(x):
        h = zs.fused.linear(x, *P["c_h1"], relu=True)
        return zs.fused.linear(zs.fused.linear(h, *P["c_h2"], relu=True), *P["c_logits"])

    lab = elbo(zs.fused.class_linear(x_l, Wx, Wy, y_l, b=bq, relu=True), eps_l, y_l, x_l).mean()
    N = int(x_u.shape[0])
    y_u = torch.arange(C, device=x_u.device).view(C, 1).expand(C, N)
    lb_z = elbo(zs.fused.class_linear(x_u, Wx, Wy, None, b=bq, relu=True), eps_u, y_u, x_u)
    qy = torch.softmax(classifier(x_u), -1) + 1e-8
    qy = qy / qy.sum(1, keepdim=True)
    unl = (qy * (lb_z.t() - torch.log(qy))).sum(1).mean()
    logits_l = classifier(x_l)
    clf = -beta * torch.log_softmax(logits_l, -1).gather(1, y_l.view(-1, 1).long()).mean()
    acc = (logits_l.argmax(1) == y_l).float().mean()
    cost = -(lab + unl - clf) / 2.0
    return dict(labeled_lb=lab, lb_z=lb_z, unlabeled_lb=unl, classifier_cost=clf, cost=cost,
                acc=acc)


@pytest.mark.parametrize("fused", [True, False])
def test_reference_run_replays(zs, fused):
    """tests/golden/ref_ssl.npz: the reference's own elbo() and OnehotCategorical on its graph."""
    g = np.load(os.path.join(GOLD, "ref_ssl.npz"))
    P = {n: tuple(T(g[p + n]).requires_grad_(True) for p in ("W_", "b_")) for n in SS.NAMES}
    x_l, x_u, y_l = T(g["x_l"]), T(g["x_u"]), T(g["y_l"])
    C, N = int(y_l.shape[1]), int(x_u.shape[0])
    eps_u = T(g["eps_u"])
    if fused:
        K, zd = int(eps_u.shape[0]), int(eps_u.shape[2])
        eps_cm = eps_u.reshape(K, N, C, zd).permute(0, 2, 1, 3).contiguous()
        out = fused_ssl_step(zs, x_l, y_l.argmax(1), x_u, T(g["eps_l"]), eps_cm, P)
        out["lb_z"] = out["lb_z"].t()
    else:
        out = SS.ssl_step(x_l, y_l, x_u, T(g["eps_l"]), eps_u, P)
    for k in ("labeled_lb", "lb_z", "unlabeled_lb", "classifier_cost", "cost", "acc"):
        np.testing.assert_allclose(N64(out[k]).numpy(), g[k], rtol=2e-5, atol=1e-5, err_msg=k)
    params = [p for n in SS.NAMES for p in P[n]]
    grads = torch.autograd.grad(out["cost"], params)
    for n, gW, gb in zip(SS.NAMES, grads[0::2], grads[1::2]):
        for what, got in (("W_", gW), ("b_", gb)):
            want = g["grad_" + what + n].astype(np.float64)
            np.testing.assert_allclose(N64(got).numpy(), want, rtol=2e-3,
                                       atol=2e-4 * max(1.0, np.abs(want).max()),
                                       err_msg="grad " + what + n)


def test_training_step_at_the_example_shape_matches_the_oracle(zs):
    """vae_ssl.py's step at its own shape (100 labeled and 100 unlabeled rows, K = 10, z = 100,
    784 -> 500 -> 500 layers), one Adam update, against the float64 oracle on the GPU's eps."""
    rng = np.random.default_rng(2024)
    XD, ZD, C, K, N, H = 784, 100, 10, 10, 100, 500
    shapes = dict(g_z=(H, ZD), g_y=(H, C), g_h=(H, H), g_x=(XD, H), q_h1=(H, XD + C),
                  q_h2=(H, H), q_mean=(ZD, H), q_logstd=(ZD, H), c_h1=(H, XD), c_h2=(H, H),
                  c_logits=(C, H))
    P = {n: (T(rng.standard_normal(s) / math.sqrt(s[1])).requires_grad_(True),
             T(0.1 * rng.standard_normal(s[0])).requires_grad_(True))
         for n, s in shapes.items()}
    x_l = T(rng.random((N, XD)) < 0.3)
    x_u = T(rng.random((N, XD)) < 0.3)
    y_l = T(rng.integers(0, C, N), torch.int64)
    g = torch.Generator(device="cuda").manual_seed(7)
    eps_l = torch.randn(K, N, ZD, device="cuda", generator=g)
    eps_cm = torch.randn(K, C, N, ZD, device="cuda", generator=g)
    params = [p for n in SS.NAMES for p in P[n]]
    before = [N64(p) for p in params]
    out = fused_ssl_step(zs, x_l, y_l, x_u, eps_l, eps_cm, P)
    opt = torch.optim.Adam(params, lr=3e-4)
    opt.zero_grad()
    out["cost"].backward()
    grads = [p.grad.detach().clone() for p in params]
    opt.step()
    # the oracle on the same eps, in the reference's row order
    L = {n: tuple(before[2 * i + j].requires_grad_(True) for j in range(2))
         for i, n in enumerate(SS.NAMES)}
    eps_ref = N64(eps_cm).permute(0, 2, 1, 3).reshape(K, N * C, ZD)
    o = SS.ssl_step(N64(x_l), torch.nn.functional.one_hot(y_l.cpu(), C).double(), N64(x_u),
                    N64(eps_l), eps_ref, L)
    for k in ("labeled_lb", "unlabeled_lb", "classifier_cost", "cost", "acc"):
        np.testing.assert_allclose(N64(out[k]).numpy(), o[k].detach().numpy(), rtol=1e-4,
                                   err_msg=k)
    np.testing.assert_allclose(N64(out["lb_z"]).t().numpy(), o["lb_z"].detach().numpy(),
                               rtol=1e-4, atol=1e-3)
    want = torch.autograd.grad(o["cost"], [p for n in SS.NAMES for p in L[n]])
    # sums over 1e4 particle rows in float32: an absolute floor of 1e-3 of the largest entry
    for name, a, w in zip([n + s for n in SS.NAMES for s in ("/W", "/b")], grads, want):
        np.testing.assert_allclose(N64(a).numpy(), w.numpy(), rtol=2e-3,
                                   atol=1e-3 * max(1.0, float(w.abs().max())), err_msg=name)
    assert all(torch.isfinite(p).all() for p in params)
