"""GPU tests of zs.fused.LinearNormal, the Gaussian dense layer of the VAE examples
(bn.normal of two dense heads, examples/semi_supervised_vae/vae_ssl_adaptive_is.py:53-68): its draws
against the registry's sampler bit for bit, its heads, log-probabilities and gradients against
float64, repeatability, the cache of its own sample's log q, the max |z| it hands to the next dense
layer, and the fallback outside the fused domain."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

K_IN = 48
HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return torch.tensor(t.detach().cpu().numpy(), dtype=torch.float64)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _params(rng, D, K=K_IN, requires_grad=False):
    ps = [T(rng.standard_normal((D, K)) / np.sqrt(K)), T(0.3 * rng.standard_normal(D)),
          T(0.5 * rng.standard_normal((D, K)) / np.sqrt(K)), T(0.2 * rng.standard_normal(D))]
    for p in ps:
        p.requires_grad_(requires_grad)
    return ps


def _heads64(h, ps):
    h64 = N64(h)
    Wm, bm, Wl, bl = (N64(p) for p in ps)
    return h64 @ Wm.t() + bm, h64 @ Wl.t() + bl


def _lq64(z, mu, ls):
    d = z - mu
    return (-HALF_LOG_2PI - ls - 0.5 * torch.exp(-2 * ls) * d * d).sum(-1)


@pytest.mark.parametrize("D", [1, 3, 4, 40, 63, 64, 65, 100, 256])
@pytest.mark.parametrize("R", [1, 127, 129, 4096])
def test_sample_equals_the_registry(zs, D, R):
    """LinearNormal.sample == ops.reparam_normal(layer.mean, layer.logstd, n) bit for bit, from the
    same zs.random state or the same injected eps, for n in {None, 1, 3, 64}; the stored log q
    against float64."""
    rng = np.random.RandomState(D * 7 + R)
    h = T(rng.standard_normal((R, K_IN)))
    ps = _params(rng, D)
    mu64, ls64 = _heads64(h, ps)
    for n in (None, 1, 3, 64):
        S = 1 if n is None else n
        for inject in (False, True):
            eps = T(rng.standard_normal((S, R, D))) if inject else None
            layer = zs.fused.LinearNormal(h, *ps, group_ndims=1)
            zs.random.set_random_seed(99 + D + S)
            zs.random.set_counter(40)
            got = layer.sample(n, eps=eps)
            assert inject or zs.random.counter() == 41
            want = zs.ops.reparam_normal(layer.mean, layer.logstd, S, eps=eps,
                                         seed=zs.random.get_seed(), it=41)
            if n is None:
                want = want.squeeze(0)
            assert got.shape == want.shape and got.dtype == torch.float32
            assert torch.equal(got, want), (n, inject)
            lq = layer.log_prob(got)
            assert lq.shape == got.shape[:-1]
            want_lq = _lq64(N64(got), mu64, ls64)
            np.testing.assert_allclose(lq.cpu().numpy(), want_lq.numpy(), rtol=1e-5,
                                       atol=1e-5 * D)


@pytest.mark.parametrize("D", [3, 40, 100])
def test_heads_against_linear_and_float64(zs, D):
    """mean / logstd (one product over the packed heads) against zs.fused.linear of each head and
    against float64; leading batch axes are kept."""
    rng = np.random.RandomState(D)
    h = T(rng.standard_normal((5, 60, K_IN)))
    ps = _params(rng, D)
    layer = zs.fused.LinearNormal(h, *ps)
    mu64, ls64 = _heads64(h.reshape(-1, K_IN), ps)
    for got, sep, want in ((layer.mean, zs.fused.linear(h, ps[0], ps[1]), mu64),
                           (layer.logstd, zs.fused.linear(h, ps[2], ps[3]), ls64)):
        assert got.shape == (5, 60, D)
        np.testing.assert_allclose(got.reshape(-1, D).cpu().numpy(), want.numpy(), rtol=1e-5,
                                   atol=1e-6)
        np.testing.assert_allclose(got.cpu().numpy(), sep.cpu().numpy(), rtol=1e-5, atol=1e-6)
    assert layer.batch_shape == (5, 60, D) and layer.value_shape == ()


def _registry_eps(zs, S, shape, it):
    """The standard normals the layer drew for counter ``it``: the registry's draw at mean 0 and
    logstd 0 (eps * exp(0) + 0 = eps exactly)."""
    zero = torch.zeros(shape, dtype=torch.float32, device="cuda")
    return zs.ops.reparam_normal(zero, zero, S, seed=zs.random.get_seed(), it=it)


@pytest.mark.parametrize("reparam", [True, False])
@pytest.mark.parametrize("inject", [True, False])
@pytest.mark.parametrize("D,R,S", [(40, 300, 8), (65, 129, 3), (1, 64, 1), (256, 300, 2),
                                   (40, 9000, 2)])
def test_gradients_against_float64(zs, reparam, inject, D, R, S):
    """d/d(h, W_mean, b_mean, W_logstd, b_logstd) of a loss on z and log q against float64 autograd
    of the same graph (z = mu + exp(ls) eps, log q of z; without reparameterisation z is a
    constant and log q keeps its partials)."""
    rng = np.random.RandomState(D + R + S + 2 * reparam + inject)
    h = T(rng.standard_normal((R, K_IN))).requires_grad_(True)
    ps = _params(rng, D, requires_grad=True)
    cz = T(rng.standard_normal((S, R, D)))
    cq = T(rng.standard_normal((S, R)))
    eps = T(rng.standard_normal((S, R, D))) if inject else None
    zs.random.set_counter(7)
    layer = zs.fused.LinearNormal(h, *ps, group_ndims=1, is_reparameterized=reparam)
    z = layer.sample(S, eps=eps)
    lq = layer.log_prob(z)
    assert z.requires_grad == reparam
    loss = (cq * lq).sum() + ((cz * z).sum() if reparam else 0.)
    grads = torch.autograd.grad(loss, [h] + ps)
    e64 = N64(eps if inject else _registry_eps(zs, S, (R, D), 8))
    leaves = [N64(t).requires_grad_(True) for t in [h] + ps]
    h64, Wm, bm, Wl, bl = leaves
    mu, ls = h64 @ Wm.t() + bm, h64 @ Wl.t() + bl
    z64 = mu + torch.exp(ls) * e64
    if not reparam:
        z64 = z64.detach()
    loss64 = (N64(cq) * _lq64(z64, mu, ls)).sum() + ((N64(cz) * z64).sum() if reparam else 0.)
    want = torch.autograd.grad(loss64, leaves)
    for name, g, w in zip(("h", "W_mean", "b_mean", "W_logstd", "b_logstd"), grads, want):
        scale = float(w.abs().max())
        np.testing.assert_allclose(g.cpu().numpy(), w.numpy(), rtol=1e-4, atol=1e-5 * scale,
                                   err_msg=name)


def test_device_epoch_moving_before_the_backward_pass(zs):
    """With the device epoch of CUDA-graph replays registered, the draws follow it, and a bump
    between the forward and the backward pass does not change the gradients: the backward pass
    recomputes eps with the epoch the forward launch used."""
    rng = np.random.RandomState(21)
    h = T(rng.standard_normal((300, K_IN))).requires_grad_(True)
    ps = _params(rng, 40, requires_grad=True)
    outs = []
    zs.random.enable_device_epoch()
    try:
        for bump_between in (0, 5):
            ep = zs.random._epoch["tensor"]
            ep.zero_()
            zs.random.bump_device_epoch(17)
            zs.random.set_counter(60)
            layer = zs.fused.LinearNormal(h, *ps, group_ndims=1)
            z = layer.sample(4)
            lq = layer.log_prob(z)
            if bump_between:
                zs.random.bump_device_epoch(bump_between)
            grads = torch.autograd.grad((z * 0.7).sum() + lq.sum(), [h] + ps)
            outs.append([z] + list(grads))
    finally:
        zs.random.disable_device_epoch()
    want = zs.ops.reparam_normal(layer.mean, layer.logstd, 4, seed=zs.random.get_seed(),
                                 it=61 + 17)                  # the epoch added in the kernel
    assert torch.equal(outs[0][0], want.detach())
    for i, (a, b) in enumerate(zip(*outs)):
        if i in (3, 5):                                       # b_mean, b_logstd: float atomics
            torch.testing.assert_close(a, b, rtol=1e-6, atol=0.)
        else:
            assert torch.equal(a, b), i


def test_repeated_calls_are_bitwise_identical(zs):
    """Two identical calls give identical z, log q and gradients w.r.t. h and the weights (the
    draws are summed in a fixed order, with no atomics).  The bias gradients are the column sums
    of the operand split, which adds its tiles with float atomics: equal to rounding."""
    rng = np.random.RandomState(5)
    h = T(rng.standard_normal((2000, K_IN))).requires_grad_(True)
    ps = _params(rng, 100, requires_grad=True)
    outs = []
    for _ in range(2):
        zs.random.set_counter(3)
        layer = zs.fused.LinearNormal(h, *ps, group_ndims=1)
        z = layer.sample(16)
        lq = layer.log_prob(z)
        grads = torch.autograd.grad((z * 0.3).sum() + lq.sum(), [h] + ps)
        outs.append([z, lq] + list(grads))
    for i, (a, b) in enumerate(zip(*outs)):
        if i in (4, 6):                                       # b_mean, b_logstd
            torch.testing.assert_close(a, b, rtol=1e-6, atol=0.)
        else:
            assert torch.equal(a, b), i


def test_cache_follows_in_place_changes(zs):
    """log_prob of the layer's own sample returns the stored log q only while the sample, h and
    the parameters are unchanged; after an in-place change it is scored afresh, and the next draw
    reads the new h."""
    rng = np.random.RandomState(11)
    h = T(rng.standard_normal((300, K_IN)))
    ps = _params(rng, 40)
    layer = zs.fused.LinearNormal(h, *ps, group_ndims=1)
    z = layer.sample(4)
    stored = layer.log_prob(z)
    for t, f in ((h, 1.5), (ps[0], 0.5), (ps[3], 2.0), (z, 1.1)):
        t.mul_(f)
        mu64, ls64 = _heads64(h, ps)
        got = layer.log_prob(z)
        assert not torch.equal(got, stored)
        np.testing.assert_allclose(got.cpu().numpy(), _lq64(N64(z), mu64, ls64).numpy(),
                                   rtol=1e-5, atol=1e-3)
        stored = got
    zs.random.set_counter(20)
    z2 = layer.sample(2)
    want = zs.ops.reparam_normal(layer.mean, layer.logstd, 2, seed=zs.random.get_seed(), it=21)
    assert torch.equal(z2, want)
    h.add_(1.0)
    zs.random.set_counter(20)
    z3 = layer.sample(2)
    want = zs.ops.reparam_normal(layer.mean, layer.logstd, 2, seed=zs.random.get_seed(), it=21)
    assert torch.equal(z3, want) and not torch.equal(z3, z2)


def test_inference_mode(zs):
    """Under torch.inference_mode nothing is cached and the draws and scores are the registry's."""
    rng = np.random.RandomState(12)
    with torch.inference_mode():
        h = T(rng.standard_normal((200, K_IN)))
        ps = _params(rng, 40)
        layer = zs.fused.LinearNormal(h, *ps, group_ndims=1)
        zs.random.set_counter(30)
        z = layer.sample(3)
        want = zs.ops.reparam_normal(layer.mean, layer.logstd, 3, seed=zs.random.get_seed(), it=31)
        assert torch.equal(z, want)
        reg = zs.distributions.Normal(layer.mean, logstd=layer.logstd, group_ndims=1)
        np.testing.assert_allclose(layer.log_prob(z).cpu().numpy(),
                                   reg.log_prob(z).cpu().numpy(), rtol=1e-5, atol=1e-4)


def test_group_ndims(zs):
    """group_ndims 0 scores per feature (the registry on mean / logstd); 2 sums the row axis of the
    stored sums as well."""
    rng = np.random.RandomState(13)
    h = T(rng.standard_normal((50, K_IN)))
    ps = _params(rng, 10)
    for g in (0, 2):
        layer = zs.fused.LinearNormal(h, *ps, group_ndims=g)
        z = layer.sample(3)
        want = zs.distributions.Normal(layer.mean, logstd=layer.logstd, group_ndims=g).log_prob(z)
        got = layer.log_prob(z)
        assert got.shape == want.shape
        np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-5, atol=1e-4)


def test_amax_tag_feeds_the_next_linear(zs):
    """The sample carries max |z| for the next zs.fused.linear (the decoder's first layer), which
    consumes it instead of running its own max pass; its result stays exact to fp32."""
    rng = np.random.RandomState(14)
    h = T(rng.standard_normal((500, K_IN)))
    ps = _params(rng, 40)
    z = zs.fused.LinearNormal(h, *ps, group_ndims=1).sample(8)
    amax = z._zsb_amax
    assert float(amax[2]) == float(z.abs().max())             # the max, as its float bits
    W2 = T(rng.standard_normal((70, 40)) / np.sqrt(40))
    y = zs.fused.linear(z, W2)
    assert not hasattr(z, "_zsb_amax") and z._zsb_pl.scale is amax
    want = N64(z) @ N64(W2).t()
    np.testing.assert_allclose(y.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)


def test_fallback_outside_the_domain(zs):
    """D = 300 and float64 parameters run Normal(linear(h, ...), logstd=linear(h, ...)), drawing
    the registry's samples."""
    rng = np.random.RandomState(15)
    h = T(rng.standard_normal((100, K_IN)))
    for D, dtype in ((300, torch.float32), (20, torch.float64)):
        hh = h.to(dtype)
        ps = [p.to(dtype) for p in _params(rng, D)]
        layer = zs.fused.LinearNormal(hh, *ps, group_ndims=1)
        assert not layer._fused
        zs.random.set_counter(50)
        z = layer.sample(2)
        zs.random.set_counter(50)
        reg = zs.distributions.Normal(zs.fused.linear(hh, ps[0], ps[1]),
                                      logstd=zs.fused.linear(hh, ps[2], ps[3]), group_ndims=1)
        want = reg.sample(2)
        assert torch.equal(z, want)
        np.testing.assert_allclose(layer.log_prob(z).cpu().numpy(),
                                   reg.log_prob(z).cpu().numpy(), rtol=1e-6)
