"""GPU tests of the sigmoid belief net layers (examples/sigmoid_belief_nets): the Bernoulli-sampling
epilogue of LinearBernoulli.sample, log-probabilities of S given samples per logit row, the
two-product mainloop of 0/1 activations, and whole VIMCO / reweighted wake-sleep steps at the
example's shape against the float64 oracle (tests/sbn_oracle.py) evaluated on the GPU's samples."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sbn_oracle as SO

pytestmark = pytest.mark.gpu

# (rows, J, S): J below 32, not a multiple of 128, the MNIST width; rows not a multiple of 128
CASES = [(240, 20, 1), (240, 200, 3), (240, 784, 10), (1300, 20, 10), (1300, 200, 1),
         (1300, 784, 3)]
K_IN = 50


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return torch.tensor(t.detach().cpu().numpy(), dtype=torch.float64)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _weights(rng, J, K, scale=2.0):
    return (T(rng.standard_normal((J, K)) * scale / np.sqrt(K)), T(0.3 * rng.standard_normal(J)))


def _input(zs, rng, R, kind):
    """A dense float activation [R, K_IN], or a 0/1 sample [R, 200] of a fused layer (it carries
    its binary operand plane)."""
    x = T(rng.standard_normal((R, K_IN)))
    if kind == "dense":
        return x
    W, b = _weights(rng, 200, K_IN)
    h = zs.fused.LinearBernoulli(x, W, b, dtype=torch.float32).sample()
    assert h._zsb_pl.binary
    return h


@pytest.mark.parametrize("R,J,S", CASES)
@pytest.mark.parametrize("kind", ["dense", "binary"])
@pytest.mark.parametrize("inject", [False, True])
def test_sample_equals_sampling_the_logits(zs, R, J, S, kind, inject):
    """LinearBernoulli.sample == Bernoulli(linear(h, W, b)).sample() bit for bit from the same
    zs.random state (Philox) or the same injected uniforms."""
    rng = np.random.RandomState(R + J + S)
    h = _input(zs, rng, R, kind)
    W, b = _weights(rng, J, int(h.shape[-1]))
    n = None if S == 1 else S
    u = T(rng.random_sample(((S,) if n else ()) + (R, J))) if inject else None
    zs.random.set_random_seed(1234 + S)
    zs.random.set_counter(40)
    d = zs.fused.LinearBernoulli(h, W, b, dtype=torch.float32)
    got = d.sample(n, u=u)
    zs.random.set_counter(40)
    ref = zs.distributions.Bernoulli(zs.fused.linear(h, W, b), dtype=torch.float32)
    want = ref._sample(S, u=u) if inject else ref._sample(S)
    if n is None:
        want = want.squeeze(0)
    assert got.shape == want.shape and got.dtype == torch.float32
    assert torch.equal(got, want)
    assert 0.05 < float(got.mean()) < 0.95
    assert zs.random.counter() == 41


@pytest.mark.parametrize("kind", ["dense", "binary"])
def test_sample_int32_and_device_epoch(zs, kind):
    """dtype int32, and the device epoch that CUDA-graph replays add to the Philox counter."""
    rng = np.random.RandomState(3)
    h = _input(zs, rng, 300, kind)
    W, b = _weights(rng, 130, int(h.shape[-1]))
    zs.random.enable_device_epoch()
    try:
        zs.random.bump_device_epoch(17)
        zs.random.set_counter(5)
        got = zs.fused.LinearBernoulli(h, W, b).sample(4)
        zs.random.set_counter(5)
        want = zs.distributions.Bernoulli(zs.fused.linear(h, W, b)).sample(4)
    finally:
        zs.random.disable_device_epoch()
    assert got.dtype == torch.int32 and torch.equal(got, want)
    zs.random.set_counter(5)
    assert not torch.equal(zs.fused.LinearBernoulli(h, W, b).sample(4), got)


def test_sample_and_log_prob_under_inference_mode(zs):
    """Inference tensors carry no version counter: sample() still runs (nothing is cached on its
    result) and equals the sample drawn outside inference mode."""
    rng = np.random.RandomState(5)
    h = _input(zs, rng, 200, "dense")
    W, b = _weights(rng, 64, K_IN)
    zs.random.set_counter(9)
    want = zs.fused.LinearBernoulli(h, W, b, dtype=torch.float32).sample(2)
    with torch.inference_mode():
        zs.random.set_counter(9)
        d = zs.fused.LinearBernoulli(h, W, b, dtype=torch.float32)
        got = d.sample(2)
        assert getattr(got, "_zsb_pl", None) is None
        lq = d.log_prob(got)
        y = zs.fused.linear(got, _weights(rng, 30, 64)[0])
    assert torch.equal(got, want)
    assert lq.shape == (2, 200) and y.shape == (2, 200, 30)


@pytest.mark.parametrize("R,J,S", CASES)
@pytest.mark.parametrize("mode", ["own", "given", "binary_given"])
def test_log_prob_of_samples_and_gradients(zs, R, J, S, mode):
    """log q of the sampling launch (own sample: no second GEMM) and log_prob of S given rows per
    logit row, for a dense h or a 0/1 sample h (two-product mainloop), against
    Bernoulli(logits).log_prob and the float64 oracle; gradients w.r.t. h (dense), W and b."""
    rng = np.random.RandomState(R * 7 + J + S)
    if mode == "binary_given":
        h = _input(zs, rng, R, "binary")
    else:
        h = T(rng.standard_normal((R, K_IN))).requires_grad_(True)
    W, b = (t.requires_grad_(True) for t in _weights(rng, J, int(h.shape[-1])))
    d = zs.fused.LinearBernoulli(h, W, b, dtype=torch.float32)
    s = d.sample(S)
    given = s if mode == "own" else T(rng.random_sample((S, R, J)) < 0.4)
    lq = d.log_prob(given)
    assert tuple(lq.shape) == (S, R)
    gen = zs.distributions.Bernoulli(zs.fused.linear(h, W, b), group_ndims=1,
                                     dtype=torch.float32).log_prob(given)
    np.testing.assert_allclose(lq.detach().cpu().numpy(), gen.detach().cpu().numpy(),
                               rtol=1e-5, atol=1e-4)
    h64, W64, b64 = (N64(t).requires_grad_(True) for t in (h, W, b))
    want = SO.bern_lp(N64(given), SO.dense(h64, (W64, b64)))
    np.testing.assert_allclose(lq.detach().cpu().numpy(), want.detach().numpy(), rtol=1e-5,
                               atol=1e-4)
    w = rng.standard_normal((S, R))
    n = 3 if h.requires_grad else 2
    got = torch.autograd.grad((lq * T(w)).sum(), [W, b, h][:n])
    exp = torch.autograd.grad((want * torch.tensor(w)).sum(), [W64, b64, h64][:n])
    for g, e in zip(got, exp):
        e = e.numpy()
        assert np.max(np.abs(g.cpu().numpy() - e)) < 2e-4 * max(1.0, np.max(np.abs(e)))


@pytest.mark.parametrize("R,J", [(240, 128), (1300, 200), (1000, 20)])
def test_binary_mainloop_is_bitwise_the_three_product_path(zs, R, J):
    """Forward, epi 1 (log-prob), epi 2 and weight-gradient products on a tagged 0/1 sample (two
    wgmma per k-step) equal those on an untagged copy (three) bit for bit; the sample's width J
    is the contraction length, a multiple of 64 or not.  (The bias gradient does not involve h
    and is summed with float atomics, so it is not compared.)"""
    rng = np.random.RandomState(R + J)
    x = T(rng.standard_normal((R, K_IN)))
    s = zs.fused.LinearBernoulli(x, *_weights(rng, J, K_IN), dtype=torch.float32).sample()
    assert s._zsb_pl.binary and float(s.max()) == 1.0
    plain = s.clone()
    assert getattr(plain, "_zsb_pl", None) is None
    W1, b1 = (t.requires_grad_(True) for t in _weights(rng, 300, J))
    xo = T(rng.random_sample((R, 300)) < 0.3)
    gy = T(rng.standard_normal((R, 300)))
    out = []
    for h in (s, plain):
        y = zs.fused.linear(h, W1, b1)
        dW, = torch.autograd.grad((y * gy).sum(), [W1])
        lp = zs.fused.linear_bernoulli_log_prob(h, W1, b1, xo)
        dW2, = torch.autograd.grad((lp * gy[:, 0]).sum(), [W1])
        out.append((y, dW, lp, dW2))
    for a, c in zip(*out):
        assert torch.equal(a, c)


def _sbn_objectives(zs, x, q_layers, m_layers, N, K, H):
    """The samples, iw_objective and klpq objective of sbn_vimco.py / sbn_adaptive_is.py with
    fused layers."""
    def layer(bn, name, h, Wb, n_samples=None, dtype=torch.float32):
        return bn.stochastic(name, zs.fused.LinearBernoulli(h, Wb[0], Wb[1], dtype=dtype),
                             n_samples=n_samples)

    q = zs.BayesianNet()
    h1 = layer(q, "h1", x.to(torch.float32), q_layers[0], n_samples=K)
    h2 = layer(q, "h2", h1.tensor, q_layers[1])
    h3 = layer(q, "h3", h2.tensor, q_layers[2])

    def log_joint(obs):
        bn = zs.BayesianNet(observed=obs)
        z3 = bn.bernoulli("h3", torch.zeros(N, H, device="cuda"), group_ndims=1, n_samples=K,
                          dtype=torch.float32)
        z2 = layer(bn, "h2", z3.tensor, m_layers[0])
        z1 = layer(bn, "h1", z2.tensor, m_layers[1])
        layer(bn, "x", z1.tensor, m_layers[2], dtype=torch.int32)
        return bn.log_joint()

    latent = {n: [t.tensor, t.cond_log_p] for n, t in (("h1", h1), ("h2", h2), ("h3", h3))}
    lb = zs.variational.iw_objective(log_joint, {"x": x}, latent=latent, axis=0)
    kl = zs.variational.klpq(log_joint, {"x": x}, latent=latent, axis=0)
    return [t.tensor for t in (h1, h2, h3)], lb, kl


def _sbn_step(zs, x, q_layers, m_layers, N, K, H):
    """One VIMCO step and one reweighted wake-sleep step from the same draws (the zs.random state
    is rewound before each objective is built): the samples, the per-datum IW bound, the vimco()
    cost, the importance() cost and their gradients."""
    import warnings
    qp = [p for l in q_layers for p in l]
    mp = [p for l in m_layers for p in l]
    c0 = zs.random.counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        samples, lb, _ = _sbn_objectives(zs, x, q_layers, m_layers, N, K, H)
        bound = lb.tensor.detach()
        assert torch.equal(lb.sgvb().detach(), -bound)
        vimco = lb.vimco().mean()
        g_vimco = torch.autograd.grad(vimco, qp + mp)
        zs.random.set_counter(c0)
        s2, lb, _ = _sbn_objectives(zs, x, q_layers, m_layers, N, K, H)
        g_model = torch.autograd.grad(-lb.tensor.mean(), mp)
        zs.random.set_counter(c0)
        s3, _, kl = _sbn_objectives(zs, x, q_layers, m_layers, N, K, H)
        imp = kl.importance().mean()
        g_prop = torch.autograd.grad(imp, qp)
    for a, b, c in zip(samples, s2, s3):
        assert torch.equal(a, b) and torch.equal(a, c)
    return samples, bound, vimco, g_vimco, g_model, imp, g_prop


def test_vimco_and_rws_steps_at_the_example_shape(zs):
    """N = 24, K = 10 particles, [784, 200, 200, 200]: the bound, both costs and all gradients of
    one VIMCO step and one reweighted wake-sleep step against the float64 oracle on the GPU's own
    samples."""
    rng = np.random.RandomState(11)
    N, K, X, H = 24, 10, 784, 200
    x = T(rng.random_sample((N, X)) < 0.3, torch.int32)
    q_layers = [tuple(t.requires_grad_(True) for t in _weights(rng, H, d, 1.0)) for d in (X, H, H)]
    m_layers = [tuple(t.requires_grad_(True) for t in _weights(rng, d, H, 1.0)) for d in (H, H, X)]
    c0 = zs.random.counter()
    samples, bound, vimco, g_vimco, g_model, imp, g_prop = _sbn_step(zs, x, q_layers, m_layers,
                                                                     N, K, H)
    for s in samples:
        assert s.shape == (K, N, H) and s._zsb_pl.binary
    # the draws against the float64 logits, with the Philox uniforms of zsb_sample_bernoulli_i32
    # (the three layers take counters c0 + 1, c0 + 2, c0 + 3)
    h = x.cpu().numpy().astype(np.float64)
    for i, (s, (W, b)) in enumerate(zip(samples, q_layers)):
        l64 = h @ W.detach().cpu().numpy().astype(np.float64).T + b.detach().cpu().numpy()
        p = 1 / (1 + np.exp(-np.broadcast_to(l64, s.shape)))
        u = _philox_uniforms(zs.random.get_seed(), c0 + 1 + i, s.numel()).reshape(s.shape)
        far = np.abs(u - p) > 1e-5
        assert far.mean() > 0.99
        np.testing.assert_array_equal(s.cpu().numpy()[far], (u < p)[far].astype(np.float32))
        h = s.cpu().numpy().astype(np.float64)
    q64 = [tuple(N64(t).requires_grad_(True) for t in l) for l in q_layers]
    m64 = [tuple(N64(t).requires_grad_(True) for t in l) for l in m_layers]
    hs, x64 = [N64(s) for s in samples], N64(x)
    lq = SO.log_q(x64, hs, q64)
    lp = SO.log_joint(x64, hs, m64)
    qp = [p for l in q64 for p in l]
    mp = [p for l in m64 for p in l]
    b64 = SO.iw_bound(lp, lq)
    np.testing.assert_allclose(bound.detach().cpu().numpy(), b64.detach().numpy(), rtol=2e-5)
    v64 = SO.vimco_cost(lp, lq).mean()
    np.testing.assert_allclose(float(vimco), float(v64), rtol=2e-5)
    i64 = SO.importance_cost(lp, lq).mean()
    np.testing.assert_allclose(float(imp), float(i64), rtol=2e-5)
    exp = (torch.autograd.grad(v64, qp + mp, retain_graph=True)
           + torch.autograd.grad(-b64.mean(), mp, retain_graph=True)
           + torch.autograd.grad(i64, qp))
    for g, e in zip(tuple(g_vimco) + tuple(g_model) + tuple(g_prop), exp):
        np.testing.assert_allclose(g.cpu().numpy(), e.numpy(), rtol=2e-3, atol=2e-4)


def _philox_uniforms(seed, it, n):
    """The uniforms zsb_sample_bernoulli_i32 draws for elements 0 .. n-1 at (seed, iteration it),
    restated with oracle/philox.py: counter (i >> 2, i >> 34, it, stream 5), word i & 3."""
    from oracle import philox
    i = np.arange(n, dtype=np.uint64)
    ctr = np.stack([(i >> np.uint64(2)) & np.uint64(0xFFFFFFFF), i >> np.uint64(34),
                    np.full(n, it, np.uint64), np.full(n, 5, np.uint64)], -1).astype(np.uint32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    words = philox.philox4x32_10(ctr, key)
    return philox.u32_to_uniform(words[np.arange(n), (i & np.uint64(3)).astype(np.int64)])


REF_Q = ["q_h1", "q_h2", "q_h3"]
REF_M = ["m_h2", "m_h1", "m_x"]


def _ref_step(zs, g, fused, q, m, which):
    """One objective of the recorded reference run (tests/golden/ref_sbn.npz) with its injected
    uniforms, on the fused layers or on the generic path (F.linear + Bernoulli)."""
    import warnings
    x = T(g["x"], torch.int32)
    N, H = int(g["x"].shape[0]), int(g["W_q_h1"].shape[0])
    K = int(g["u_h1"].shape[0])

    def q_layer(h, Wb, n, u):
        if fused:
            d = zs.fused.LinearBernoulli(h, Wb[0], Wb[1], dtype=torch.float32)
            s = d.sample(n, u=T(u))
        else:
            d = zs.distributions.Bernoulli(F.linear(h.to(torch.float32), Wb[0], Wb[1]),
                                           group_ndims=1, dtype=torch.float32)
            s = d._sample(n or 1, u=T(u))
            s = s if n else s.squeeze(0)
        return s, d.log_prob(s)

    def layer(bn, name, h, Wb, dtype=torch.float32):
        if fused:
            return bn.stochastic(name, zs.fused.LinearBernoulli(h, Wb[0], Wb[1], dtype=dtype))
        return bn.bernoulli(name, F.linear(h, Wb[0], Wb[1]), group_ndims=1, dtype=dtype)

    s1, lq1 = q_layer(x.to(torch.float32), q[0], K, g["u_h1"])
    s2, lq2 = q_layer(s1, q[1], None, g["u_h2"])
    s3, lq3 = q_layer(s2, q[2], None, g["u_h3"])
    for s, n in zip((s1, s2, s3), ("h1", "h2", "h3")):
        np.testing.assert_array_equal(s.cpu().numpy(), g[n])

    def log_joint(obs):
        bn = zs.BayesianNet(observed=obs)
        z3 = bn.bernoulli("h3", torch.zeros(N, H, device="cuda"), group_ndims=1, n_samples=K,
                          dtype=torch.float32)
        z2 = layer(bn, "h2", z3.tensor, m[0])
        z1 = layer(bn, "h1", z2.tensor, m[1])
        layer(bn, "x", z1.tensor, m[2], dtype=torch.int32)
        return bn.log_joint()

    latent = {"h1": [s1, lq1], "h2": [s2, lq2], "h3": [s3, lq3]}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        if which == "klpq":
            return zs.variational.klpq(log_joint, {"x": x}, latent=latent, axis=0)
        return zs.variational.iw_objective(log_joint, {"x": x}, latent=latent, axis=0)


@pytest.mark.parametrize("fused", [True, False])
def test_reference_run_replays(zs, fused):
    """tests/golden/ref_sbn.npz, the reference's own vimco() and klpq(...).importance() on its
    Bernoulli nets, reproduced with its injected uniforms: samples exactly, bounds and costs at
    rtol 2e-5, gradients of all 12 variables at rtol 2e-3 / atol 2e-4."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_sbn.npz"))
    q = [(T(g["W_" + n]).requires_grad_(True), T(g["b_" + n]).requires_grad_(True)) for n in REF_Q]
    m = [(T(g["W_" + n]).requires_grad_(True), T(g["b_" + n]).requires_grad_(True)) for n in REF_M]
    qp = [p for l in q for p in l]
    mp = [p for l in m for p in l]

    def check(got, prefix, names):
        for (gW, gb), n in zip(zip(got[0::2], got[1::2]), names):
            np.testing.assert_allclose(gW.cpu().numpy(), g[prefix + "W_" + n], rtol=2e-3,
                                       atol=2e-4, err_msg=prefix + n)
            np.testing.assert_allclose(gb.cpu().numpy(), g[prefix + "b_" + n], rtol=2e-3,
                                       atol=2e-4, err_msg=prefix + n)

    lb = _ref_step(zs, g, fused, q, m, "iw")
    np.testing.assert_allclose(lb.tensor.detach().cpu().numpy(), g["iw_bound"], rtol=2e-5)
    cost = lb.vimco().mean()
    np.testing.assert_allclose(cost.item(), float(g["vimco_cost"]), rtol=2e-5)
    check(torch.autograd.grad(cost, qp + mp), "vimco_grad_", REF_Q + REF_M)
    lb = _ref_step(zs, g, fused, q, m, "iw")
    check(torch.autograd.grad(-lb.tensor.mean(), mp), "rws_grad_", REF_M)
    kl = _ref_step(zs, g, fused, q, m, "klpq")
    cost = kl.importance().mean()
    np.testing.assert_allclose(cost.item(), float(g["rws_klpq_cost"]), rtol=2e-5)
    check(torch.autograd.grad(cost, qp), "rws_grad_", REF_Q)
