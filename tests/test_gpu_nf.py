"""zs.planar_normalizing_flow on the flow-stack kernels of csrc/flows.cu, and the normalizing-flow
VAE of examples/normalizing_flows/vae_nf.py on it: the forward against float64 across widths, flow
counts and leading shapes, chained calls, gradients w.r.t. all five inputs, bitwise repeatability,
inference mode, non-contiguous samples, the reference run of tests/golden/ref_nf.npz replayed on the
fused and the F.linear layers, and the example's training step and IS bound at its own shape against
the float64 oracle of tests/nf_oracle.py."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import nf_oracle as NF

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


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


def _inputs(rng, lead, d, n, near_identity=False):
    """Random samples, log-probs and flow parameters.  ``near_identity``: aux_u = (log(e - 1) /
    w.w) w + 0.05 noise, so that u.w = softplus(w.aux_u) - 1 is near 0 and u is small; a stack of
    a thousand such flows stays well conditioned, where random parameters expand the gradients
    beyond what float32 can follow."""
    z = T(rng.standard_normal(lead + (d,)))
    lq = T(rng.standard_normal(lead) * 3.0)
    b = T(rng.standard_normal(n) * 0.5)
    w = rng.standard_normal((n, d)) * (1.5 / math.sqrt(d))
    if near_identity:
        u = w * (math.log(math.e - 1) / (w * w).sum(1, keepdims=True)) + \
            0.05 * rng.standard_normal((n, d)) / math.sqrt(d)
    else:
        u = rng.standard_normal((n, d)) / math.sqrt(d)
    return z, lq, b, T(u), T(w)


@pytest.mark.parametrize("d", [1, 2, 7, 31, 32, 33, 40, 100, 256, 1024])
@pytest.mark.parametrize("n", [0, 1, 10, 37])
def test_forward_matches_float64(zs, d, n):
    for lead in [(1,), (129,), (3, 70)]:
        rng = np.random.default_rng(d * 1000 + n * 10 + len(lead))
        z, lq, b, u, w = _inputs(rng, lead, d, n)
        got_z, got_lq = zs.planar_normalizing_flow(z, lq, n, b, u, w)
        assert got_z.shape == z.shape and got_lq.shape == lq.shape
        want_z, want_lq = NF.planar_flow(D(z), D(lq), D(b), D(u), D(w))
        what = "d %d, n %d, lead %s" % (d, n, lead)
        _close(got_z, want_z, "z: " + what, 1e-5)
        _close(got_lq, want_lq, "log_q: " + what, 1e-5)


def test_forward_at_the_is_shape(zs):
    """vae_nf.py's IS evaluation: 1000 particles x 400 rows at z_dim 40, two stacks of 10."""
    rng = np.random.default_rng(11)
    z, lq, b, u, w = _inputs(rng, (1000, 400), 40, 10)
    _, _, b2, u2, w2 = _inputs(rng, (1,), 40, 10)
    with torch.no_grad():
        z1, l1 = zs.planar_normalizing_flow(z, lq, 10, b, u, w)
        z1, l1 = zs.planar_normalizing_flow(z1, l1, 10, b2, u2, w2)
    wz, wl = NF.planar_flow(D(z), D(lq), D(b), D(u), D(w))
    wz, wl = NF.planar_flow(wz, wl, D(b2), D(u2), D(w2))
    _close(z1, wz, "z", 1e-5)
    _close(l1, wl, "log_q", 1e-5)


def test_two_chained_calls_match_float64(zs):
    rng = np.random.default_rng(12)
    z, lq, b, u, w = _inputs(rng, (5, 33), 40, 10)
    _, _, b2, u2, w2 = _inputs(rng, (1,), 40, 7)
    z1, l1 = zs.planar_normalizing_flow(z, lq, 10, b, u, w)
    z2, l2 = zs.planar_normalizing_flow(z1, l1, 7, b2, u2, w2)
    wz, wl = NF.planar_flow(*map(D, (z, lq, b, u, w)))
    wz, wl = NF.planar_flow(wz, wl, D(b2), D(u2), D(w2))
    _close(z2, wz, "z", 1e-5)
    _close(l2, wl, "log_q", 1e-5)


def _grads(zs, ins, n, gz, gl):
    ps = [t.clone().requires_grad_(True) for t in ins]
    z, lq = zs.planar_normalizing_flow(ps[0], ps[1], n, *ps[2:])
    return [z, lq] + list(torch.autograd.grad((z, lq), ps, (gz, gl)))


# The backward sweep runs on at most 264 CTAs (fewer at large n * d), each taking row tiles of
# 256 / L rows (L = 1, 8 or 32 lanes per row for d <= 8, <= 64, larger) in turn and adding each tile
# to its warps' partial sums: the 20000-, 70000-, 3000- and 2000-row cases give every CTA several
# tiles for each L.  n = 1100 exceeds the 1024 flows whose scalars fit in shared memory at once, so
# both kernels stage them in chunks, and the sweep restages them for every tile.
@pytest.mark.parametrize("d,n,lead", [(1, 3, (50,)), (7, 4, (3, 5)), (33, 10, (129,)),
                                      (40, 20, (2, 64)), (100, 37, (70,)), (256, 5, (33,)),
                                      (1024, 3, (9,)), (40, 10, (20000,)), (7, 4, (70000,)),
                                      (100, 5, (3000,)), (1024, 3, (2000,)), (7, 1100, (16000,))])
def test_gradients_match_float64(zs, d, n, lead):
    rng = np.random.default_rng(d + n)
    ins = _inputs(rng, lead, d, n, near_identity=n > 1000)
    gz, gl = T(rng.standard_normal(lead + (d,))), T(rng.standard_normal(lead))
    got = _grads(zs, ins, n, gz, gl)[2:]
    p64 = [D(t).requires_grad_(True) for t in ins]
    want = torch.autograd.grad(NF.planar_flow(*p64), p64, (D(gz), D(gl)))
    for name, a, w in zip(("samples", "log_probs", "b", "aux_u", "w"), got, want):
        assert a.shape == w.shape, name
        _close(a, w, "d %s (d %d, n %d)" % (name, d, n), 1e-4)


def test_two_identical_calls_are_bitwise_equal(zs):
    rng = np.random.default_rng(4)
    ins = _inputs(rng, (100, 128), 40, 20)
    gz, gl = T(rng.standard_normal((100, 128, 40))), T(rng.standard_normal((100, 128)))
    a, b = _grads(zs, ins, 20, gz, gl), _grads(zs, ins, 20, gz, gl)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_empty_rows(zs):
    rng = np.random.default_rng(6)
    for lead in [(0,), (3, 0)]:
        ins = [t.requires_grad_(True) for t in _inputs(rng, lead, 40, 5)]
        z, lq = zs.planar_normalizing_flow(ins[0], ins[1], 5, *ins[2:])
        assert z.shape == lead + (40,) and lq.shape == lead
        g = torch.autograd.grad((z, lq), ins, (torch.ones_like(z), torch.ones_like(lq)))
        assert [t.shape for t in g] == [t.shape for t in ins]
        for t in g[2:]:
            assert torch.equal(t, torch.zeros_like(t))


def test_nothing_is_kept_for_backward_without_a_gradient(zs):
    """Under inference_mode (and no_grad) the forward pass allocates its outputs only; with a
    gradient it also keeps every flow's input z, n * R * d floats."""
    rng = np.random.default_rng(7)
    R, d, n = 8192, 40, 10
    ins = [t.requires_grad_(True) for t in _inputs(rng, (R,), d, n)]
    out_bytes = 4 * R * (d + 1)

    def peak(ctx):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with ctx():
            z, lq = zs.planar_normalizing_flow(ins[0], ins[1], n, *ins[2:])
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, z, lq
    for ctx in (torch.inference_mode, torch.no_grad):
        used, z, lq = peak(ctx)
        assert z.grad_fn is None and lq.grad_fn is None and not z.requires_grad
        assert used <= out_bytes + (1 << 20), (ctx.__name__, used)
        del z, lq
    used, z, lq = peak(torch.enable_grad)
    assert z.grad_fn is not None
    assert used >= out_bytes + 4 * n * R * d, used


def test_inference_mode_and_non_contiguous_samples(zs):
    rng = np.random.default_rng(5)
    z, lq, b, u, w = _inputs(rng, (64, 9), 40, 10)
    want_z, want_lq = zs.planar_normalizing_flow(z, lq, 10, b, u, w)
    with torch.inference_mode():
        got_z, got_lq = zs.planar_normalizing_flow(z, lq, 10, b, u, w)
    assert torch.equal(got_z, want_z) and torch.equal(got_lq, want_lq)
    # samples [9, 64, 40] seen as [64, 9, 40]; log_probs transposed as well
    zt, lqt = z.transpose(0, 1).contiguous().transpose(0, 1), lq.t().contiguous().t()
    assert not zt.is_contiguous() and not lqt.is_contiguous()
    ps = [t.clone().requires_grad_(True) for t in (zt, lqt, b, u, w)]
    nz, nlq = zs.planar_normalizing_flow(ps[0], ps[1], 10, *ps[2:])
    assert torch.equal(nz, want_z) and torch.equal(nlq, want_lq)
    g = torch.autograd.grad(nz.sum() + nlq.sum(), ps)
    ref = [t.clone().requires_grad_(True) for t in (z, lq, b, u, w)]
    rz, rlq = zs.planar_normalizing_flow(ref[0], ref[1], 10, *ref[2:])
    for x, y in zip(g, torch.autograd.grad(rz.sum() + rlq.sum(), ref)):
        assert torch.equal(x, y)


def test_standalone_reference_flow_replays(zs):
    g = np.load(os.path.join(GOLD, "ref_nf.npz"))
    ins = [T(g["flow/" + k]).requires_grad_(True) for k in ("samples", "log_probs", "b", "aux_u",
                                                            "w")]
    z, lq = zs.planar_normalizing_flow(ins[0], ins[1], 4, *ins[2:])
    _close(z, T(g["flow/z"]), "z", 1e-5)
    _close(lq, T(g["flow/log_q"]), "log_q", 1e-5)
    f = (z * T(g["flow/cz"])).sum() + (lq * T(g["flow/cl"])).sum()
    for k, got in zip(("samples", "log_probs", "b", "aux_u", "w"), torch.autograd.grad(f, ins)):
        _close(got, T(g["flow/grad_" + k]), "grad " + k, 1e-4)


# ---- vae_nf.py on zs -------------------------------------------------------------------------
def layers(zs, fused):
    if fused:
        return lambda h, W, b, relu=False: zs.fused.linear(h, W, b, relu=relu)
    return lambda h, W, b, relu=False: torch.relu(F.linear(h, W, b)) if relu else F.linear(h, W, b)


def example(zs, x, eps, q, p, flows, fused):
    """vae_nf.py:19-85 on zs: the q-net, the flow stacks, and elbo / is_loglikelihood with
    latent={'z': [qz, log_qz]}.  Returns (elbo objective, IS estimate per row)."""
    lin = layers(zs, fused)
    S, n, z_dim = eps.shape

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, z_dim, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        h = lin(lin(z, p[0], p[1], True), p[2], p[3], True)
        if fused:
            bn.stochastic("x", zs.fused.LinearBernoulli(h, p[4], p[5], dtype=torch.float32))
        else:
            bn.bernoulli("x", F.linear(h, p[4], p[5]), group_ndims=1, dtype=torch.float32)
        return bn

    h = lin(lin(x, q[0], q[1], True), q[2], q[3], True)
    mean, logstd = lin(h, q[4], q[5]), lin(h, q[6], q[7])
    qz = mean + torch.exp(logstd) * eps
    log_qz = zs.distributions.Normal(mean, logstd=logstd, group_ndims=1).log_prob(qz)
    for b, u, w in flows:
        qz, log_qz = zs.planar_normalizing_flow(qz, log_qz, int(b.shape[0]), b, u, w)
    model = build_gen(n, z_dim, S)
    lb = zs.variational.elbo(model, {"x": x}, latent={"z": [qz, log_qz]}, axis=0)
    return lb, lambda: zs.is_loglikelihood(model, {"x": x}, {"z": [qz, log_qz]}, axis=0)


def _golden_params(g):
    q = [T(g["vae/q%d_%s" % (i, s)]).requires_grad_(True) for i in range(4) for s in "Wb"]
    p = [T(g["vae/p%d_%s" % (i, s)]).requires_grad_(True) for i in range(3) for s in "Wb"]
    flows = [tuple(T(g["vae/f%d_%s" % (c, s)]).requires_grad_(True) for s in ("b", "aux_u", "w"))
             for c in range(2)]
    return q, p, flows


@pytest.mark.parametrize("fused", [True, False])
def test_reference_vae_run_replays(zs, fused):
    """tests/golden/ref_nf.npz: the reference's elbo() and is_loglikelihood on vae_nf.py's graph."""
    g = np.load(os.path.join(GOLD, "ref_nf.npz"))
    q, p, flows = _golden_params(g)
    lb, _ = example(zs, T(g["vae/x"]), T(g["vae/eps"]), q, p, flows, fused)
    cost = lb.sgvb().mean()
    _close(lb.tensor.mean(), T(g["vae/bound"]), "bound", 2e-5)
    _close(cost, T(g["vae/cost"]), "cost", 2e-5)
    names = ["q%d_%s" % (i, s) for i in range(4) for s in "Wb"] + \
        ["p%d_%s" % (i, s) for i in range(3) for s in "Wb"] + \
        ["f%d_%s" % (c, s) for c in range(2) for s in ("b", "aux_u", "w")]
    wrt = q + p + [t for f in flows for t in f]
    for nm, got in zip(names, torch.autograd.grad(cost, wrt)):
        _close(got, T(g["vae/grad_" + nm]), "grad " + nm, 2e-3, 2e-4)
    with torch.no_grad():
        _, is_ll = example(zs, T(g["vae/is_x"]), T(g["vae/is_eps"]), q, p, flows, fused)
        _close(is_ll().mean(), T(g["vae/is_ll"]), "IS", 2e-5)


def _example_params(rng, zs, x_dim=784, h=500, z_dim=40, n_flows=10):
    def dense(i, o):
        return [T(rng.standard_normal((o, i)) / math.sqrt(i)).requires_grad_(True),
                T(0.1 * rng.standard_normal(o)).requires_grad_(True)]
    q = dense(x_dim, h) + dense(h, h) + dense(h, z_dim) + dense(h, z_dim)
    p = dense(z_dim, h) + dense(h, h) + dense(h, x_dim)
    gen = torch.Generator(device="cuda").manual_seed(int(rng.integers(1 << 30)))
    flows = [zs.planar_flow_parameters(z_dim, n_flows, generator=gen) for _ in range(2)]
    return q, p, flows


def test_training_step_and_is_bound_at_the_example_shape_match_the_oracle(zs):
    """vae_nf.py at its own shape: one training step (128 rows, 1 particle, [784, 500, 500],
    z_dim 40, 2 x 10 flows, Adam) and an IS bound at 1000 particles, against float64."""
    rng = np.random.default_rng(2026)
    q, p, flows = _example_params(rng, zs)
    params = q + p + [t for f in flows for t in f]
    before = [D(t) for t in params]
    x = T(rng.random((128, 784)) < 0.3)
    eps = T(rng.standard_normal((1, 128, 40)))
    lb, _ = example(zs, x, eps, q, p, flows, True)
    cost = lb.sgvb().mean()
    opt = torch.optim.Adam(params, lr=1e-3)
    opt.zero_grad()
    cost.backward()
    grads = [t.grad.detach().clone() for t in params]
    opt.step()
    p64 = [t.clone().requires_grad_(True) for t in before]
    fl64 = [tuple(p64[14 + 3 * c:17 + 3 * c]) for c in range(2)]
    bound64, cost64 = NF.bound_and_cost(NF.vae_nf(D(x), D(eps), p64[:8], p64[8:14], fl64))
    _close(lb.tensor.mean(), bound64, "bound", 1e-5)
    for i, (a, w) in enumerate(zip(grads, torch.autograd.grad(cost64, p64))):
        _close(a, w, "grad %d" % i, 2e-3, 1e-3)
    assert all(torch.isfinite(t).all() for t in params)
    # IS bound at 1000 particles on the updated parameters
    x = T(rng.random((100, 784)) < 0.3)
    eps = T(rng.standard_normal((1000, 100, 40)))
    with torch.no_grad():
        _, is_ll = example(zs, x, eps, q, p, flows, True)
        got = is_ll().mean()
        P = [D(t) for t in params]
        want = NF.is_loglikelihood(NF.vae_nf(D(x), D(eps), P[:8], P[8:14],
                                             [tuple(P[14 + 3 * c:17 + 3 * c]) for c in range(2)]))
    _close(got, want, "IS bound", 1e-5)
