"""zs.inv_autoregressive_flow on the flow-stack kernels of csrc/iaf.cu, and the normalizing-flow VAE
of examples/normalizing_flows/vae_nf.py with two IAF stacks: the forward against float64 across
widths, flow counts, leading shapes and both updates, chained calls, gradients w.r.t. samples,
log_probs, m_w and s_w, exact zeros at the masked entries, bitwise repeatability, inference mode,
non-contiguous samples, empty rows, the generic path at d = 300, the fused path against
LinearAR.__call__, the reference run of tests/golden/ref_iaf.npz replayed, and the example's training
step and IS bound against the float64 oracle of tests/iaf_oracle.py."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import iaf_oracle as IAF
import nf_oracle as NF

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
UPDATES = ("normal", "gru")


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def D(t):
    return t.detach().double()


def _close(got, want, what, rtol, atol=None):
    """|got - want| <= rtol |want| + atol max|want| (atol defaults to rtol)."""
    got, want = D(got).cpu().numpy(), D(want).cpu().numpy()
    scale = max(1.0, float(np.abs(want).max())) if want.size else 1.0
    np.testing.assert_allclose(got, want, rtol=rtol, atol=(rtol if atol is None else atol) * scale,
                               err_msg=what)


def _ar(zs, rng, d, n, scale=None):
    """A LinearAR with m_w of std `scale` (default 0.3 / sqrt(d)) and s_w of 0.1 times that: far
    from the identity, while a stack of tens of flows keeps z and exp(t) within float32's
    comfortable range."""
    ar = zs.LinearAR(d, n)
    sc = (0.3 / math.sqrt(d)) if scale is None else scale
    with torch.no_grad():
        ar.m_w.copy_(T(rng.standard_normal((n, d, d)) * sc))
        ar.s_w.copy_(T(rng.standard_normal((n, d, d)) * sc * 0.1))
    return ar


def _inputs(rng, lead, d):
    return T(rng.standard_normal(lead + (d,))), T(rng.standard_normal(lead) * 3.0)


def _ref(z, lq, ar, u):
    return IAF.linear_iaf(D(z).cpu(), D(lq).cpu(), D(ar.m_w).cpu(), D(ar.s_w).cpu(), u)


@pytest.mark.parametrize("u", UPDATES)
@pytest.mark.parametrize("d", [1, 2, 7, 31, 32, 33, 40, 64, 100, 128, 255, 256])
@pytest.mark.parametrize("n", [0, 1, 2, 10, 37])
def test_forward_matches_float64(zs, d, n, u):
    for lead in [(1,), (129,), (3, 70)]:
        rng = np.random.default_rng(d * 1000 + n * 10 + len(lead))
        z, lq = _inputs(rng, lead, d)
        ar = _ar(zs, rng, d, n)
        got_z, got_lq = zs.inv_autoregressive_flow(z, None, lq, ar, n, update=u)
        assert got_z.shape == z.shape and got_lq.shape == lq.shape
        want_z, want_lq = _ref(z, lq, ar, u)
        what = "d %d, n %d, lead %s, %s" % (d, n, lead, u)
        _close(got_z, want_z, "z: " + what, 1e-5)
        _close(got_lq, want_lq, "log_q: " + what, 1e-5)


@pytest.mark.parametrize("u", UPDATES)
def test_two_chained_calls_match_float64(zs, u):
    rng = np.random.default_rng(12)
    z, lq = _inputs(rng, (5, 33), 40)
    a1, a2 = _ar(zs, rng, 40, 10), _ar(zs, rng, 40, 7)
    z1, l1 = zs.inv_autoregressive_flow(z, None, lq, a1, 10, update=u)
    z2, l2 = zs.inv_autoregressive_flow(z1, None, l1, a2, 7, update=u)
    wz, wl = _ref(z, lq, a1, u)
    wz, wl = IAF.linear_iaf(wz, wl, D(a2.m_w).cpu(), D(a2.s_w).cpu(), u)
    _close(z2, wz, "z", 1e-5)
    _close(l2, wl, "log_q", 1e-5)


def _grads(zs, z, lq, ar, n, u, gz, gl):
    s, l = z.clone().requires_grad_(True), lq.clone().requires_grad_(True)
    zo, lo = zs.inv_autoregressive_flow(s, None, l, ar, n, update=u)
    return [zo, lo] + list(torch.autograd.grad((zo, lo), [s, l, ar.m_w, ar.s_w], (gz, gl)))


# The backward sweep runs on at most 264 persistent CTAs (fewer when n * d^2 > 2^18: each keeps
# a slice of 2 n d^2 floats), each taking row tiles of 64, 32 or 16 rows (d <= 16, <= 64, larger)
# in turn and adding each tile's weight gradients to its slice: the 20000-, 40000-, 12000- and
# 9000-row cases give every CTA two or more tiles for each tile shape.
@pytest.mark.parametrize("u", UPDATES)
@pytest.mark.parametrize("d,n,lead", [(1, 3, (50,)), (7, 4, (3, 5)), (33, 10, (129,)),
                                      (40, 20, (2, 64)), (100, 7, (70,)), (256, 3, (33,)),
                                      (40, 10, (20000,)), (7, 4, (40000,)), (128, 5, (12000,)),
                                      (256, 2, (9000,))])
def test_gradients_match_float64(zs, d, n, lead, u):
    rng = np.random.default_rng(d + n + len(u))
    z, lq = _inputs(rng, lead, d)
    ar = _ar(zs, rng, d, n)
    gz, gl = T(rng.standard_normal(lead + (d,))), T(rng.standard_normal(lead))
    got = _grads(zs, z, lq, ar, n, u, gz, gl)[2:]
    p64 = [D(t).cpu().requires_grad_(True) for t in (z, lq, ar.m_w, ar.s_w)]
    want = torch.autograd.grad(IAF.linear_iaf(*p64, update=u), p64, (D(gz).cpu(), D(gl).cpu()))
    for name, a, w in zip(("samples", "log_probs", "m_w", "s_w"), got, want):
        assert a.shape == w.shape, name
        _close(a, w, "d %s (d %d, n %d, %s)" % (name, d, n, u), 1e-4)
    lower = torch.ones(d, d, dtype=torch.bool, device="cuda").tril()
    for a in got[2:]:
        assert torch.equal(a[:, lower], torch.zeros_like(a[:, lower]))


@pytest.mark.parametrize("u", UPDATES)
def test_two_identical_calls_are_bitwise_equal(zs, u):
    rng = np.random.default_rng(4)
    z, lq = _inputs(rng, (100, 128), 40)
    ar = _ar(zs, rng, 40, 20)
    gz, gl = T(rng.standard_normal((100, 128, 40))), T(rng.standard_normal((100, 128)))
    a = _grads(zs, z, lq, ar, 20, u, gz, gl)
    b = _grads(zs, z, lq, ar, 20, u, gz, gl)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_empty_rows(zs):
    rng = np.random.default_rng(6)
    ar = _ar(zs, rng, 40, 5)
    for lead in [(0,), (3, 0)]:
        z, lq = _inputs(rng, lead, 40)
        z.requires_grad_(True)
        lq.requires_grad_(True)
        zo, lo = zs.inv_autoregressive_flow(z, None, lq, ar, 5)
        assert zo.shape == lead + (40,) and lo.shape == lead
        g = torch.autograd.grad((zo, lo), [z, lq, ar.m_w, ar.s_w],
                                (torch.ones_like(zo), torch.ones_like(lo)))
        assert [t.shape for t in g] == [z.shape, lq.shape, ar.m_w.shape, ar.s_w.shape]
        for t in g[2:]:
            assert torch.equal(t, torch.zeros_like(t))


def test_nothing_is_kept_for_backward_without_a_gradient(zs):
    """Under inference_mode (and no_grad) the forward pass allocates its outputs only; with a
    gradient it also keeps every flow's input z, n * R * d floats."""
    rng = np.random.default_rng(7)
    R, d, n = 8192, 40, 10
    z, lq = _inputs(rng, (R,), d)
    z.requires_grad_(True)
    ar = _ar(zs, rng, d, n)
    out_bytes = 4 * R * (d + 1)

    def peak(ctx):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with ctx():
            zo, lo = zs.inv_autoregressive_flow(z, None, lq, ar, n)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, zo, lo
    for ctx in (torch.inference_mode, torch.no_grad):
        used, zo, lo = peak(ctx)
        assert zo.grad_fn is None and lo.grad_fn is None and not zo.requires_grad
        assert used <= out_bytes + (1 << 20), (ctx.__name__, used)
        del zo, lo
    used, zo, lo = peak(torch.enable_grad)
    assert zo.grad_fn is not None
    assert used >= out_bytes + 4 * n * R * d, used


@pytest.mark.parametrize("u", UPDATES)
def test_inference_mode_and_non_contiguous_samples(zs, u):
    rng = np.random.default_rng(5)
    z, lq = _inputs(rng, (64, 9), 40)
    ar = _ar(zs, rng, 40, 10)
    want_z, want_lq = zs.inv_autoregressive_flow(z, None, lq, ar, 10, update=u)
    with torch.inference_mode():
        got_z, got_lq = zs.inv_autoregressive_flow(z, None, lq, ar, 10, update=u)
    assert torch.equal(got_z, want_z) and torch.equal(got_lq, want_lq)
    zt, lqt = z.transpose(0, 1).contiguous().transpose(0, 1), lq.t().contiguous().t()
    assert not zt.is_contiguous() and not lqt.is_contiguous()
    ps = [zt.clone().requires_grad_(True), lqt.clone().requires_grad_(True)]
    nz, nlq = zs.inv_autoregressive_flow(ps[0], None, ps[1], ar, 10, update=u)
    assert torch.equal(nz, want_z) and torch.equal(nlq, want_lq)
    g = torch.autograd.grad(nz.sum() + nlq.sum(), ps + [ar.m_w, ar.s_w])
    ref = [z.clone().requires_grad_(True), lq.clone().requires_grad_(True)]
    rz, rlq = zs.inv_autoregressive_flow(ref[0], None, ref[1], ar, 10, update=u)
    for x, y in zip(g, torch.autograd.grad(rz.sum() + rlq.sum(), ref + [ar.m_w, ar.s_w])):
        assert torch.equal(x, y)


@pytest.mark.parametrize("u", UPDATES)
def test_wide_samples_take_the_generic_path(zs, u):
    """d = 300 is beyond the kernels; the call runs the reference's loop through LinearAR."""
    rng = np.random.default_rng(300)
    z, lq = _inputs(rng, (17,), 300)
    ar = _ar(zs, rng, 300, 3)
    s = z.clone().requires_grad_(True)
    zo, lo = zs.inv_autoregressive_flow(s, None, lq, ar, 3, update=u)
    wz, wl = _ref(z, lq, ar, u)
    _close(zo, wz, "z", 1e-4)
    _close(lo, wl, "log_q", 1e-4)
    g = torch.autograd.grad(zo.sum() + lo.sum(), [s, ar.m_w])
    p64 = [D(t).cpu().requires_grad_(True) for t in (z, lq, ar.m_w, ar.s_w)]
    wz, wl = IAF.linear_iaf(*p64, update=u)
    w = torch.autograd.grad(wz.sum() + wl.sum(), [p64[0], p64[2]])
    _close(g[0], w[0], "d samples", 1e-3)
    _close(g[1], w[1], "d m_w", 1e-3)


@pytest.mark.parametrize("u", UPDATES)
def test_fused_path_matches_the_linear_ar_callable(zs, u):
    """The same LinearAR, once as the fused stack and once through a plain callable that the
    function can only call (the generic path)."""
    rng = np.random.default_rng(21)
    z, lq = _inputs(rng, (4, 50), 40)
    ar = _ar(zs, rng, 40, 6)
    ins = [z.clone().requires_grad_(True), lq.clone().requires_grad_(True)]
    f = zs.inv_autoregressive_flow(ins[0], None, ins[1], ar, 6, update=u)
    ins2 = [z.clone().requires_grad_(True), lq.clone().requires_grad_(True)]
    r = zs.inv_autoregressive_flow(ins2[0], None, ins2[1], lambda *a: ar(*a), 6, update=u)
    _close(f[0], r[0], "z", 1e-5)
    _close(f[1], r[1], "log_q", 1e-5)
    gz, gl = T(rng.standard_normal((4, 50, 40))), T(rng.standard_normal((4, 50)))
    a = torch.autograd.grad(f, ins + [ar.m_w, ar.s_w], (gz, gl))
    b = torch.autograd.grad(r, ins2 + [ar.m_w, ar.s_w], (gz, gl))
    for name, x, y in zip(("samples", "log_probs", "m_w", "s_w"), a, b):
        _close(x, y, "d " + name, 1e-4)


@pytest.mark.parametrize("u", UPDATES)
def test_reference_flow_replays(zs, u):
    g = np.load(os.path.join(GOLD, "ref_iaf.npz"))
    ar = zs.LinearAR(7, 3)
    with torch.no_grad():
        ar.m_w.copy_(T(g[u + "/m_w"]))
        ar.s_w.copy_(T(g[u + "/s_w"]))
    s = T(g[u + "/samples"]).requires_grad_(True)
    l = T(g[u + "/log_probs"]).requires_grad_(True)
    z, lq = zs.inv_autoregressive_flow(s, None, l, ar, 3, update=u)
    _close(z, T(g[u + "/z"]), "z", 1e-5)
    _close(lq, T(g[u + "/log_q"]), "log_q", 1e-5)
    f = (z * T(g[u + "/cz"])).sum() + (lq * T(g[u + "/cl"])).sum()
    for k, got in zip(("samples", "log_probs", "m_w", "s_w"),
                      torch.autograd.grad(f, [s, l, ar.m_w, ar.s_w])):
        _close(got, T(g[u + "/grad_" + k]), "grad " + k, 1e-4)


# ---- vae_nf.py with two IAF stacks on zs ----------------------------------------------------
def example(zs, x, eps, q, p, flows):
    """vae_nf.py:19-85 with inv_autoregressive_flow in place of the planar stacks.  The dense layers
    are F.linear in fp32, so that a ReLU pre-activation near zero does not change sign between
    this run and the float64 oracle, and the comparison measures the flows.  Returns (elbo
    objective, IS estimate per row)."""
    lin = lambda h, W, b, relu=False: torch.relu(F.linear(h, W, b)) if relu else F.linear(h, W, b)  # noqa: E731,E501
    S, n, z_dim = eps.shape

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, z_dim, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        h = lin(lin(z, p[0], p[1], True), p[2], p[3], True)
        bn.bernoulli("x", F.linear(h, p[4], p[5]), group_ndims=1, dtype=torch.float32)
        return bn

    h = lin(lin(x, q[0], q[1], True), q[2], q[3], True)
    mean, logstd = lin(h, q[4], q[5]), lin(h, q[6], q[7])
    qz = mean + torch.exp(logstd) * eps
    log_qz = zs.distributions.Normal(mean, logstd=logstd, group_ndims=1).log_prob(qz)
    for ar in flows:
        qz, log_qz = zs.inv_autoregressive_flow(qz, None, log_qz, ar, ar.n_iters)
    model = build_gen(n, z_dim, S)
    lb = zs.variational.elbo(model, {"x": x}, latent={"z": [qz, log_qz]}, axis=0)
    return lb, lambda: zs.is_loglikelihood(model, {"x": x}, {"z": [qz, log_qz]}, axis=0)


def test_training_step_and_is_bound_at_the_example_shape_match_the_oracle(zs):
    """vae_nf.py's shape with IAF: one training step (128 rows, 1 particle, [784, 500, 500],
    z_dim 40, 2 x 10 fused flows, Adam) and an IS bound at 1000 particles, against float64."""
    rng = np.random.default_rng(2026)

    def dense(i, o):
        return [T(rng.standard_normal((o, i)) / math.sqrt(i)).requires_grad_(True),
                T(0.1 * rng.standard_normal(o)).requires_grad_(True)]
    q = dense(784, 500) + dense(500, 500) + dense(500, 40) + dense(500, 40)
    p = dense(40, 500) + dense(500, 500) + dense(500, 784)
    flows = [_ar(zs, rng, 40, 10, scale=0.05) for _ in range(2)]
    params = q + p + [t for ar in flows for t in (ar.m_w, ar.s_w)]
    before = [D(t) for t in params]
    x = T(rng.random((128, 784)) < 0.3)
    eps = T(rng.standard_normal((1, 128, 40)))
    lb, _ = example(zs, x, eps, q, p, flows)
    cost = lb.sgvb().mean()
    opt = torch.optim.Adam(params, lr=1e-3)
    opt.zero_grad()
    cost.backward()
    grads = [t.grad.detach().clone() for t in params]
    opt.step()
    p64 = [t.clone().requires_grad_(True) for t in before]
    fl64 = [tuple(p64[14 + 2 * c:16 + 2 * c]) for c in range(2)]
    bound64, cost64 = NF.bound_and_cost(IAF.vae_iaf(D(x), D(eps), p64[:8], p64[8:14], fl64))
    _close(lb.tensor.mean(), bound64, "bound", 1e-5)
    _close(cost, cost64, "cost", 1e-5)
    for i, (a, w) in enumerate(zip(grads, torch.autograd.grad(cost64, p64))):
        _close(a, w, "grad %d" % i, 2e-3, 1e-3)
    assert all(torch.isfinite(t).all() for t in params)
    x = T(rng.random((100, 784)) < 0.3)
    eps = T(rng.standard_normal((1000, 100, 40)))
    with torch.no_grad():
        _, is_ll = example(zs, x, eps, q, p, flows)
        got = is_ll().mean()
        P = [D(t) for t in params]
        want = NF.is_loglikelihood(IAF.vae_iaf(D(x), D(eps), P[:8], P[8:14],
                                               [tuple(P[14 + 2 * c:16 + 2 * c])
                                                for c in range(2)]))
    _close(got, want, "IS bound", 1e-5)
