"""The noisy, batch-normalised dense layer (zs.fused.noisy_bn_linear) and the variational-dropout
classifier of examples/bayesian_neural_nets/variational_dropout.py on it: the forward in both modes
against float64 across widths, row counts, particle broadcasting and ReLU, the moving-statistics
update, bitwise repeatability, gradients, inference mode, shape errors, the reference run of
tests/golden/ref_vardrop.npz replayed on the fused and the generic path, and the example's training
step and evaluation bound at its own shape against the float64 oracle of tests/vardrop_oracle.py."""
import math
import os

import numpy as np
import pytest
import torch

import vardrop_oracle as VD

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NET = [784, 100, 100, 100, 10]


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return t.detach().double().cpu()


def _layer(rng, lead, K, J, h_full):
    noise = T(1.0 + 0.5 * rng.standard_normal(lead + (K,)))
    h = T(rng.standard_normal((lead if h_full else lead[1:]) + (K,)))
    W = T(rng.standard_normal((J, K)) / math.sqrt(K))
    beta = T(0.5 * rng.standard_normal(J))
    mm = T(0.1 * rng.standard_normal(J))
    mv = T(0.5 + rng.random(J))
    return h, noise, W, beta, mm, mv


def _close(got, want, what, rtol=1e-4, atol=1e-4):
    want = want.detach().numpy() if isinstance(want, torch.Tensor) else want
    np.testing.assert_allclose(N64(got).numpy(), want, rtol=rtol,
                               atol=atol * max(1.0, float(np.abs(want).max())), err_msg=what)


@pytest.mark.parametrize("K", [784, 37, 30])
@pytest.mark.parametrize("J", [10, 100, 200])
@pytest.mark.parametrize("lead,h_full", [((3, 70), False), ((1, 130), False), ((2, 333), True),
                                         ((10, 100), False)])
def test_forward_matches_float64(zs, K, J, lead, h_full):
    rng = np.random.default_rng(K * 1000 + J + lead[1])
    h, noise, W, beta, mm, mv = _layer(rng, lead, K, J, h_full)
    for training in (True, False):
        for relu in (True, False):
            m, v = mm.clone(), mv.clone()
            out = zs.fused.noisy_bn_linear(h, noise, W, beta, m, v, training, relu=relu)
            assert out.shape == lead + (J,)
            want, wm, wv = VD.bn_layer(N64(h), N64(noise), N64(W), N64(beta), N64(mm), N64(mv),
                                       training, relu=relu)
            what = "training=%s relu=%s" % (training, relu)
            _close(out, want, what)
            _close(m, wm, what + " moving mean", rtol=1e-5, atol=1e-6)
            _close(v, wv, what + " moving variance", rtol=1e-5, atol=1e-6)
            if not training:
                assert torch.equal(m, mm) and torch.equal(v, mv)


def test_moving_statistics_over_two_training_calls(zs):
    rng = np.random.default_rng(2)
    K, J, lead = 120, 100, (4, 300)
    h, noise, W, beta, _, _ = _layer(rng, lead, K, J, False)
    m, v = T(np.zeros(J)), T(np.ones(J))
    wm, wv = torch.zeros(J, dtype=torch.float64), torch.ones(J, dtype=torch.float64)
    for call in range(2):
        noise = T(1.0 + 0.5 * rng.standard_normal(lead + (K,)))
        zs.fused.noisy_bn_linear(h, noise, W, beta, m, v, True)
        _, wm, wv = VD.bn_layer(N64(h), N64(noise), N64(W), N64(beta), wm, wv, True)
        _close(m, wm, "moving mean after call %d" % call, rtol=1e-5, atol=1e-7)
        _close(v, wv, "moving variance after call %d" % call, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("training", [True, False])
def test_two_identical_calls_are_bitwise_equal(zs, training):
    rng = np.random.default_rng(4)
    K, J, lead = 784, 100, (10, 1000)
    h, noise, W, beta, mm, mv = _layer(rng, lead, K, J, False)
    gy = T(rng.standard_normal(lead + (J,)))
    res = []
    for _ in range(2):
        ps = [t.clone().requires_grad_(True) for t in (h, noise, W, beta)]
        m, v = mm.clone(), mv.clone()
        out = zs.fused.noisy_bn_linear(*ps, m, v, training)
        res.append([out, m, v] + list(torch.autograd.grad(out, ps, gy)))
    for a, b in zip(*res):
        assert torch.equal(a, b)


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("K,J,lead,h_full,relu", [(784, 100, (3, 333), False, True),
                                                  (37, 200, (2, 150), True, False),
                                                  (30, 10, (1, 257), False, True)])
def test_gradients_match_float64(zs, training, K, J, lead, h_full, relu):
    rng = np.random.default_rng(K + J + lead[1])
    h, noise, W, beta, mm, mv = _layer(rng, lead, K, J, h_full)
    ps = [t.requires_grad_(True) for t in (h, noise, W, beta)]
    gy = T(rng.standard_normal(lead + (J,)))
    out = zs.fused.noisy_bn_linear(*ps, mm.clone(), mv.clone(), training, relu=relu)
    got = torch.autograd.grad(out, ps, gy)
    p64 = [N64(p).requires_grad_(True) for p in ps]
    o64, _, _ = VD.bn_layer(*p64, N64(mm), N64(mv), training, relu=relu)
    want = torch.autograd.grad(o64, p64, N64(gy))
    for name, a, w in zip(("h", "noise", "W", "beta"), got, want):
        assert a.shape == w.shape, name
        _close(a, w, "d" + name, rtol=1e-3, atol=1e-4)


def test_inference_mode_and_the_amax_tag(zs):
    rng = np.random.default_rng(3)
    K, J, lead = 100, 100, (5, 200)
    h, noise, W, beta, mm, mv = _layer(rng, lead, K, J, False)
    want = zs.fused.noisy_bn_linear(h, noise, W, beta, mm.clone(), mv.clone(), False)
    assert hasattr(want, "_zsb_amax")
    m, v = mm.clone(), mv.clone()
    want_t = zs.fused.noisy_bn_linear(h, noise, W, beta, m, v, True)
    W2 = T(rng.standard_normal((7, J)))
    with torch.inference_mode():
        got = zs.fused.noisy_bn_linear(h, noise, W, beta, mm.clone(), mv.clone(), False)
        mi, vi = mm.clone(), mv.clone()
        got_t = zs.fused.noisy_bn_linear(h, noise, W, beta, mi, vi, True)
        nxt = zs.fused.linear(got_t, W2)
    assert torch.equal(got, want) and torch.equal(got_t, want_t)
    assert torch.equal(mi, m) and torch.equal(vi, v)
    _close(nxt, N64(want_t) @ N64(W2).t(), "linear on the tagged output", rtol=1e-5, atol=1e-5)


def test_mismatched_shapes_raise_before_any_launch(zs):
    rng = np.random.default_rng(5)
    h, noise, W, beta, mm, mv = _layer(rng, (3, 10), 20, 8, False)
    f = zs.fused.noisy_bn_linear
    with pytest.raises(ValueError, match="suffix"):
        f(T(np.ones((4, 20))), noise, W, beta, mm, mv, True)
    with pytest.raises(ValueError, match="suffix"):
        f(T(np.ones((2, 3, 10, 20))), noise, W, beta, mm, mv, True)
    with pytest.raises(ValueError, match="W"):
        f(h, noise, W[:, :19], beta, mm, mv, True)
    with pytest.raises(ValueError, match="beta"):
        f(h, noise, W, beta[:7], mm, mv, True)
    with pytest.raises(ValueError, match="moving_mean"):
        f(h, noise, W, beta, mm[:7], mv, True)
    with pytest.raises(ValueError, match="moving_variance"):
        f(h, noise, W, beta, mm, mv.double(), True)


# ---- the classifier of variational_dropout.py ----------------------------------------------------
def fused_layer(zs):
    def layer(h, eps, W, beta, mm, mv, training):
        return zs.fused.noisy_bn_linear(h, eps, W, beta, mm, mv, training), mm, mv
    return layer


def generic_layer(h, eps, W, beta, mm, mv, training):
    """F.linear and a batch-norm restatement in float32, the moving statistics updated in place."""
    y, m, v = VD.bn_layer(h, eps, W, beta, mm, mv, training)
    with torch.no_grad():
        mm.copy_(m)
        mv.copy_(v)
    return y, mm, mv


@pytest.mark.parametrize("fused", [True, False])
def test_reference_run_replays(zs, fused):
    """tests/golden/ref_vardrop.npz: the reference's own elbo() on its graph, training then
    evaluation on the updated moving statistics."""
    g = np.load(os.path.join(GOLD, "ref_vardrop.npz"))
    L = 4
    Ws = [T(g["W_%d" % i]).requires_grad_(True) for i in range(L)]
    betas = [T(g["beta_%d" % i]).requires_grad_(True) for i in range(L)]
    alphas = [T(g["logit_alpha_%d" % i]).requires_grad_(True) for i in range(L)]
    mms = [torch.zeros(int(W.shape[0]), device="cuda") for W in Ws]
    mvs = [torch.ones(int(W.shape[0]), device="cuda") for W in Ws]
    layer = fused_layer(zs) if fused else generic_layer
    x, y = T(g["x"]), T(g["y"], torch.int64)
    out = VD.vardrop_run(x, y, [T(g["z_%d" % i]) for i in range(L)], Ws, betas, alphas, mms, mvs,
                         True, 60000, layer=layer)
    for k in ("bound", "cost", "acc", "logits"):
        _close(out[k], g[k].astype(np.float64), k, rtol=2e-5, atol=2e-5)
    for i in range(L):
        _close(mms[i], g["moving_mean_%d" % i].astype(np.float64), "moving mean", 1e-5, 1e-6)
        _close(mvs[i], g["moving_variance_%d" % i].astype(np.float64), "moving var", 1e-5, 1e-6)
    grads = torch.autograd.grad(out["cost"], Ws + betas + alphas)
    names = ["grad_W_%d" % i for i in range(L)] + ["grad_beta_%d" % i for i in range(L)] + \
        ["grad_logit_alpha_%d" % i for i in range(L)]
    for name, got in zip(names, grads):
        _close(got, g[name].astype(np.float64), name, rtol=2e-3, atol=2e-4)
    with torch.no_grad():
        ev = VD.vardrop_run(x, y, [T(g["eval_z_%d" % i]) for i in range(L)], Ws, betas, alphas,
                            mms, mvs, False, 60000, layer=layer)
    for k in ("bound", "acc", "logits"):
        _close(ev[k], g["eval_" + k].astype(np.float64), "eval " + k, rtol=2e-5, atol=2e-5)


def _example_params(rng):
    Ws = [T(rng.standard_normal((o, i)) / math.sqrt(i)).requires_grad_(True)
          for i, o in zip(NET[:-1], NET[1:])]
    betas = [T(0.1 * rng.standard_normal(o)).requires_grad_(True) for o in NET[1:]]
    alphas = [T(rng.standard_normal(i) - 1.0).requires_grad_(True) for i in NET[:-1]]
    return Ws, betas, alphas


def test_training_step_and_evaluation_at_the_example_shape_match_the_oracle(zs):
    """variational_dropout.py at its own shape: one training step (S = 10 particles x 1000 rows,
    Adam) and one evaluation bound (S = 100, 1e5 particle rows), against the float64 oracle on the
    same draws."""
    rng = np.random.default_rng(2025)
    n, L = 1000, 4
    Ws, betas, alphas = _example_params(rng)
    params = Ws + betas + alphas
    before = [p.detach().double() for p in params]
    x = T(rng.standard_normal((n, NET[0])))
    y = T(rng.integers(0, 10, n), torch.int64)
    gen = torch.Generator(device="cuda").manual_seed(3)
    z = [torch.randn(10, n, k, device="cuda", generator=gen) for k in NET[:-1]]
    mms = [torch.zeros(o, device="cuda") for o in NET[1:]]
    mvs = [torch.ones(o, device="cuda") for o in NET[1:]]
    out = VD.vardrop_run(x, y, z, Ws, betas, alphas, mms, mvs, True, 60000, layer=fused_layer(zs))
    opt = torch.optim.Adam(params, lr=1e-3, eps=1e-4)
    opt.zero_grad()
    out["cost"].backward()
    grads = [p.grad.detach().clone() for p in params]
    opt.step()
    # the oracle in float64 on the GPU, on the same draws
    p64 = [b.clone().requires_grad_(True) for b in before]
    D = lambda t: t.detach().double()                              # noqa: E731
    m64 = [torch.zeros(o, dtype=torch.float64, device="cuda") for o in NET[1:]]
    v64 = [torch.ones(o, dtype=torch.float64, device="cuda") for o in NET[1:]]
    o = VD.vardrop_run(D(x), y, [D(t) for t in z], p64[:L], p64[L:2 * L], p64[2 * L:], m64, v64,
                       True, 60000)
    for k in ("bound", "cost"):
        _close(out[k], N64(o[k]), k, rtol=1e-5, atol=1e-6)
    _close(out["logits"], N64(o["logits"]), "logits", rtol=1e-4, atol=1e-4)
    for i in range(L):
        _close(mms[i], N64(o["moving_mean"][i]), "moving mean %d" % i, rtol=1e-5, atol=1e-6)
        _close(mvs[i], N64(o["moving_variance"][i]), "moving var %d" % i, rtol=1e-5, atol=1e-6)
    want = torch.autograd.grad(o["cost"], p64)
    for i, (a, w) in enumerate(zip(grads, want)):
        _close(a, N64(w), "grad %d" % i, rtol=2e-3, atol=1e-3)
    assert all(torch.isfinite(p).all() for p in params)
    # evaluation at S = 100 on the updated parameters and moving statistics
    z = [torch.randn(100, n, k, device="cuda", generator=gen) for k in NET[:-1]]
    with torch.no_grad():
        ev = VD.vardrop_run(x, y, z, Ws, betas, alphas, mms, mvs, False, 60000,
                            layer=fused_layer(zs))
        o = VD.vardrop_run(D(x), y, [D(t) for t in z], [D(p) for p in Ws], [D(p) for p in betas],
                           [D(p) for p in alphas], [D(t) for t in mms], [D(t) for t in mvs],
                           False, 60000)
    _close(ev["bound"], N64(o["bound"]), "eval bound", rtol=1e-5, atol=1e-6)
    _close(ev["logits"], N64(o["logits"]), "eval logits", rtol=1e-4, atol=1e-4)
    agree = (ev["logits"].softmax(-1).mean(0).argmax(1) == o["logits"].softmax(-1).mean(0)
             .argmax(1)).double().mean()
    assert float(agree) >= 0.998
