"""ExpConcrete / Concrete on the kernels of csrc/concrete.cu against the torch composition the
classes run for every other input, and against float64.

Tolerances.  The sample from the same zs.random state (or the same injected u) follows the
composition's operations on the same fp32 values; the division by t is the IEEE quotient for
normal operands and only the softmax normaliser differs (a multiply by a refined reciprocal, one
ulp).  So y agrees to rtol 1e-5 with an absolute term of 4 ulp of the largest |(l + g) / t| of the
row, the size of the rounding both paths make in a.  The log-density and its gradients are checked
against float64 autograd of the reference's formula on the same fp32 inputs, with an absolute
bound of 2e-6 times the sum of the magnitudes that enter each value (the terms of sum(temp), C
LSE(temp) and sum(x)), which covers the fp32 rounding of C-term sums with margin; a wrong term is
O(1) of that scale."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

CS = [1, 2, 10, 31, 32, 33, 256, 1024]


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _ref_parts(given, logits, t, log_space):
    """float64 log-density terms (multivariate.py:800-812, 938-955) and their magnitude scale."""
    x = given if log_space else torch.log(given)
    temp = logits - t * x
    C = logits.shape[-1]
    lse = torch.logsumexp(temp, -1)
    lp = math.lgamma(C) + (C - 1) * torch.log(t) + temp.sum(-1) - C * lse
    if not log_space:
        lp = lp - x.sum(-1)
    scale = temp.abs().sum(-1) + C * lse.abs() + x.abs().sum(-1) + abs(math.lgamma(C)) + \
        (C - 1) * torch.log(t).abs() + 1.0
    return lp, scale


def _group(lp, n):
    return lp.sum(tuple(range(lp.dim() - n, lp.dim()))) if n else lp


def _check_lp_and_grads(zs, given, logits, t, log_space, gnd=0, gscale=1.0):
    D = zs.distributions
    cls = D.ExpConcrete if log_space else D.Concrete
    g32 = given.detach().clone().requires_grad_(True)
    l32 = logits.detach().clone().requires_grad_(True)
    t32 = t.detach().clone().requires_grad_(True)
    d = cls(t32, l32, group_ndims=gnd)
    assert d._fused(g32)
    lp = d.log_prob(g32)
    g64 = given.detach().double().requires_grad_(True)
    l64 = logits.detach().double().requires_grad_(True)
    t64 = t.detach().double().requires_grad_(True)
    ref, scale = _ref_parts(g64, l64, t64, log_space)
    ref = _group(ref, gnd)
    scale = _group(scale.detach(), gnd)
    assert lp.shape == ref.shape
    err = (lp.double() - ref).abs()
    assert bool((err <= 2e-6 * scale).all()), float((err / scale).max())
    w = torch.randn(lp.shape, device="cuda", dtype=torch.float64)
    got = torch.autograd.grad((lp.double() * w).sum(), [g32, l32, t32])
    want = torch.autograd.grad((ref * w).sum(), [g64, l64, t64])
    with torch.no_grad():
        # d/dt sums (C-1)/t against sum(w x) per row, terms that cancel: its fp32 rounding is
        # relative to the magnitudes summed, not to the result
        x = g64 if log_space else torch.log(g64)
        temp = l64 - t64 * x
        C = temp.shape[-1]
        wv = 1 - C * torch.softmax(temp, -1)
        gout = w.reshape(tuple(w.shape) + (1,) * gnd).expand(temp.shape[:-1])
        mag_t = (gout.abs() * ((C - 1) / t64 + (wv.abs() * x.abs()).sum(-1))).sum().item()
    for name, a, b in zip(("given", "logits", "temperature"), got, want):
        assert a.shape == b.shape, name
        tol = 2e-5 * gscale * (b.abs().max().item() + 1.0)
        if name == "temperature":
            tol = max(tol, 1e-5 * mag_t)
        e = (a.double() - b).abs().max().item()
        assert e <= tol, (name, e, tol)


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("log_space", [True, False])
def test_log_prob_and_gradients_vs_float64(zs, C, log_space):
    torch.manual_seed(C)
    S, B = 3, 5
    logits = torch.randn(B, C, device="cuda") * 2
    t = torch.tensor(0.7, device="cuda")
    d = (zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete)(t, logits)
    given = d.sample(S).detach()
    for gnd in (0, 1, 2):
        _check_lp_and_grads(zs, given, logits, t, log_space, gnd=gnd)


@pytest.mark.parametrize("log_space", [True, False])
def test_broadcasts(zs, log_space):
    torch.manual_seed(1)
    C = 10
    t = torch.tensor(1.3, device="cuda")
    cls = zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete
    # suffix: logits [4, C] under given [3, 4, C]; given [4, C] under logits [3, 4, C]
    logits = torch.randn(4, C, device="cuda")
    given = cls(t, logits).sample(3).detach()
    _check_lp_and_grads(zs, given, logits, t, log_space, gnd=1)
    logits3 = torch.randn(3, 4, C, device="cuda")
    _check_lp_and_grads(zs, given[0], logits3, t, log_space, gnd=2)
    # non-suffix: logits [2, 1, C] against given [2, 5, C] (expanded on the host)
    logits_ns = torch.randn(2, 1, C, device="cuda")
    given_ns = cls(t, logits_ns.expand(2, 5, C).contiguous()).sample().detach()
    _check_lp_and_grads(zs, given_ns, logits_ns, t, log_space, gnd=0)


@pytest.mark.parametrize("tval", [0.05, 0.5, 5.0])
@pytest.mark.parametrize("log_space", [True, False])
def test_extreme_parameters(zs, tval, log_space):
    torch.manual_seed(7)
    C = 33
    logits = (torch.rand(6, C, device="cuda") * 160 - 80)
    t = torch.tensor(tval, device="cuda")
    cls = zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete
    given = cls(t, logits).sample(2).detach()
    if not log_space:
        # near the corners of the simplex: components down to 1e-30
        corner = torch.full((2, 6, C), 1e-30, device="cuda")
        corner[..., 0] = 1.0
        given = torch.maximum(given, torch.tensor(1e-30, device="cuda"))
        given = torch.cat([given, corner], 0)
    _check_lp_and_grads(zs, given, logits, t, log_space, gnd=1, gscale=10.0)


def _composition(zs, cls, t, logits, n, u=None):
    d = cls(t, logits)
    return d._gumbel_logits(n, u), d


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("log_space", [True, False])
def test_sample_matches_composition(zs, C, log_space):
    torch.manual_seed(100 + C)
    cls = zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete
    logits = torch.randn(7, C, device="cuda") * 3
    t = torch.tensor(0.6, device="cuda")
    c0 = zs.random.counter()
    y = cls(t, logits).sample(5)
    zs.random.set_counter(c0)
    a, _ = _composition(zs, cls, t, logits, 5)
    want = torch.log_softmax(a, -1) if log_space else torch.softmax(a, -1)
    assert zs.random.counter() == c0 + 1
    amax = a.abs().amax(-1, keepdim=True)
    tol = 1e-5 * want.abs() + 4 * torch.finfo(torch.float32).eps * amax + 1e-7
    assert bool(((y - want).abs() <= tol).all()), float((y - want).abs().max())
    # injected uniforms, clamped at both ends like drawn ones
    u = torch.rand(5, 7, C, device="cuda")
    u[0, :, 0] = 0.0
    u[1, :, -1] = 1.0
    u[2, :, :] = torch.where(u[2] < 0.5, torch.tensor(1e-9, device="cuda"),
                             torch.tensor(1 - 1e-9, device="cuda"))
    y = cls(t, logits)._sample(5, u=u)
    a, _ = _composition(zs, cls, t, logits, 5, u=u)
    want = torch.log_softmax(a, -1) if log_space else torch.softmax(a, -1)
    amax = a.abs().amax(-1, keepdim=True)
    tol = 1e-5 * want.abs() + 4 * torch.finfo(torch.float32).eps * amax + 1e-7
    assert bool(torch.isfinite(y).all())
    assert bool(((y - want).abs() <= tol).all()), float((y - want).abs().max())


@pytest.mark.parametrize("C", [1, 10, 33, 1024])
@pytest.mark.parametrize("log_space", [True, False])
def test_sample_gradients_vs_float64(zs, C, log_space):
    torch.manual_seed(200 + C)
    cls = zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete
    logits = (torch.randn(4, C, device="cuda") * 2).requires_grad_(True)
    t = torch.tensor(0.8, device="cuda", requires_grad=True)
    u = torch.rand(6, 4, C, device="cuda")
    y = cls(t, logits)._sample(6, u=u)
    w = torch.randn(y.shape, device="cuda")
    got = torch.autograd.grad((y * w).sum(), [logits, t])
    l64 = logits.detach().double().requires_grad_(True)
    t64 = t.detach().double().requires_grad_(True)
    uc = u.double().clamp(1e-7, 1 - 1e-7)
    a = (l64 + (-torch.log(-torch.log(uc)))) / t64
    y64 = torch.log_softmax(a, -1) if log_space else torch.softmax(a, -1)
    want = torch.autograd.grad((y64 * w.double()).sum(), [l64, t64])
    for name, g, r in zip(("logits", "temperature"), got, want):
        e = (g.double() - r).abs().max().item()
        assert e <= 1e-4 * (r.abs().max().item() + 1.0), (name, e)


def test_wide_rows_take_the_composition(zs, monkeypatch):
    from zhusuan_b200 import ops
    calls = []
    for name in ("sample_concrete", "concrete_log_prob"):
        orig = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _o=orig, _n=name, **k: (calls.append(_n),
                                                                          _o(*a, **k))[1])
    t = torch.tensor(0.5, device="cuda")
    for C, fused in ((1024, True), (1025, False)):
        calls.clear()
        d = zs.distributions.ExpConcrete(t, torch.randn(3, C, device="cuda"))
        lp = d.log_prob(d.sample(2))
        assert bool(torch.isfinite(lp).all())
        assert (calls == ["sample_concrete", "concrete_log_prob"]) == fused, (C, calls)
        assert fused or not calls


@pytest.mark.parametrize("log_space", [True, False])
def test_identical_calls_identical_bits(zs, log_space):
    torch.manual_seed(5)
    cls = zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete
    logits = torch.randn(50, 20, 10, device="cuda")
    u = torch.rand(300, 50, 20, 10, device="cuda")
    outs = []
    for _ in range(2):
        l = logits.clone().requires_grad_(True)
        t = torch.tensor(0.4, device="cuda", requires_grad=True)
        d = cls(t, l, group_ndims=1)
        y = d._sample(300, u=u)
        lp = d.log_prob(y)
        g = torch.autograd.grad(lp.sum() + (y * y).sum(), [l, t])
        outs.append([y.detach(), lp.detach(), g[0], g[1]])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_reparameterization_flags(zs):
    logits = torch.randn(4, 6, device="cuda", requires_grad=True)
    t = torch.tensor(0.5, device="cuda", requires_grad=True)
    y = zs.distributions.ExpConcrete(t, logits, is_reparameterized=False).sample(3)
    assert not y.requires_grad
    # path derivative: log_prob's parameter gradients are stopped, the sample's path stays
    d = zs.distributions.ExpConcrete(t, logits, use_path_derivative=True)
    y = d.sample(3)
    gl, gt = torch.autograd.grad(d.log_prob(y).sum(), [logits, t], retain_graph=True)
    y2 = y.detach().requires_grad_(True)
    gy = torch.autograd.grad(d.log_prob(y2).sum(), [y2])[0]
    want = torch.autograd.grad((y * gy).sum(), [logits, t])
    assert torch.allclose(gl, want[0], rtol=1e-5, atol=1e-5)
    assert torch.allclose(gt, want[1], rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("log_space", [True, False])
def test_broadcast_logits_over_many_samples(zs, log_space):
    """Few logits rows under many samples, the backward's sample axis split across CTAs: the
    prior pattern (logits [20, 10] under [K, N, 20, 10]) with every gradient and with the given
    gradient alone, and a sample from one logits row."""
    torch.manual_seed(11)
    cls = zs.distributions.ExpConcrete if log_space else zs.distributions.Concrete
    logits = torch.randn(20, 10, device="cuda")
    t = torch.tensor(0.5, device="cuda")
    given = cls(t, torch.randn(300, 20, 10, device="cuda")).sample(10).detach()
    _check_lp_and_grads(zs, given, logits, t, log_space, gnd=2)
    g32 = given.clone().requires_grad_(True)
    gz = torch.autograd.grad(cls(t, logits, group_ndims=2).log_prob(g32).sum(), [g32])[0]
    g64 = given.double().requires_grad_(True)
    ref, _ = _ref_parts(g64, logits.double(), t.double(), log_space)
    want = torch.autograd.grad(ref.sum(), [g64])[0]
    assert (gz.double() - want).abs().max().item() <= 2e-5 * (want.abs().max().item() + 1.0)
    # one logits row, 20000 draws
    l1 = (torch.randn(7, device="cuda") * 2).requires_grad_(True)
    t1 = torch.tensor(0.8, device="cuda", requires_grad=True)
    u = torch.rand(20000, 7, device="cuda")
    y = cls(t1, l1)._sample(20000, u=u)
    w = torch.randn(y.shape, device="cuda")
    got = torch.autograd.grad((y * w).sum(), [l1, t1])
    l64 = l1.detach().double().requires_grad_(True)
    t64 = t1.detach().double().requires_grad_(True)
    a = (l64 - torch.log(-torch.log(u.double().clamp(1e-7, 1 - 1e-7)))) / t64
    y64 = torch.log_softmax(a, -1) if log_space else torch.softmax(a, -1)
    want = torch.autograd.grad((y64 * w.double()).sum(), [l64, t64])
    mag = ((y64.detach().exp() if log_space else y64.detach()) * w.double().abs()).sum() * 4 / 0.8
    for name, g, r in zip(("logits", "temperature"), got, want):
        e = (g.double() - r).abs().max().item()
        assert e <= 1e-5 * (r.abs().max().item() + mag.item() * (1 + a.abs().max().item())), \
            (name, e)


@pytest.mark.parametrize("c", [0, 1])
@pytest.mark.parametrize("p", ["exp_", "con_"])
def test_golden_replay(zs, p, c):
    """tests/golden/ref_concrete.npz, recorded from the reference's own classes: the sample from
    the recorded uniforms, log_prob at group_ndims 0 and 1 and its gradients w.r.t. given, logits
    and temperature, on the kernels."""
    import os
    import numpy as np
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                             "ref_concrete.npz"))
    cls = zs.distributions.ExpConcrete if p == "exp_" else zs.distributions.Concrete
    dev = lambda k: torch.tensor(g[p + k + "_%d" % c], device="cuda")  # noqa: E731
    logits, t, u = dev("logits"), dev("t"), dev("u")
    d = cls(t, logits)
    assert d._fused()
    y = d._sample(u.shape[0], u=u)
    np.testing.assert_allclose(y.cpu().numpy(), g[p + "sample_%d" % c], rtol=1e-5, atol=2e-6)
    for gnd in (0, 1):
        x = dev("sample").requires_grad_(True)
        l = logits.clone().requires_grad_(True)
        tt = t.clone().requires_grad_(True)
        lp = cls(tt, l, group_ndims=gnd).log_prob(x)
        np.testing.assert_allclose(lp.detach().cpu().numpy(), g[p + "lp%d_%d" % (gnd, c)],
                                   rtol=1e-5, atol=2e-4)
        w = torch.tensor(g[p + "w%d_%d" % (gnd, c)], device="cuda")
        grads = torch.autograd.grad((lp * w).sum(), [x, l, tt])
        for name, a in zip(("dgiven", "dlogits", "dt"), grads):
            rec = g[p + "%s%d_%d" % (name, gnd, c)]
            np.testing.assert_allclose(a.cpu().numpy(), rec, rtol=1e-4,
                                       atol=1e-4 * (np.abs(rec).max() + 1), err_msg=name)
