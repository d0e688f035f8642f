"""tests/golden/ref_nf.npz (made by tests/golden/make_ref_nf_golden.py): the reference's own
planar_normalizing_flow alone, and vae_nf.py's bound, gradients and IS estimate on the reference's
BayesianNet, distributions, elbo() and is_loglikelihood.  The committed arrays must match their
digests, the float64 oracle of tests/nf_oracle.py must reproduce every recorded value, and
zs.planar_normalizing_flow must reject malformed inputs before any launch.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import nf_oracle as NF
import zhusuan_b200 as zs
from zhusuan_b200._lib import ZsbError

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_nf.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_nf_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_nf/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def D(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=torch.float64).requires_grad_(grad)


def _close(got, want, what, rtol, atol):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(got.detach().numpy(), want, rtol=rtol,
                               atol=atol * max(1.0, np.abs(want).max()), err_msg=what)


def test_oracle_reproduces_the_standalone_flow(g):
    ins = [D(g["flow/" + k], True) for k in ("samples", "log_probs", "b", "aux_u", "w")]
    z, lq = NF.planar_flow(*ins)
    _close(z, g["flow/z"], "z", 1e-5, 1e-6)
    _close(lq, g["flow/log_q"], "log_q", 1e-5, 1e-6)
    f = (z * D(g["flow/cz"])).sum() + (lq * D(g["flow/cl"])).sum()
    for k, got in zip(("samples", "log_probs", "b", "aux_u", "w"), torch.autograd.grad(f, ins)):
        _close(got, g["flow/grad_" + k], "grad " + k, 1e-4, 1e-5)


def _vae_params(g):
    q = [D(g["vae/q%d_%s" % (i, s)], True) for i in range(4) for s in "Wb"]
    p = [D(g["vae/p%d_%s" % (i, s)], True) for i in range(3) for s in "Wb"]
    flows = [tuple(D(g["vae/f%d_%s" % (c, s)], True) for s in ("b", "aux_u", "w"))
             for c in range(2)]
    return q, p, flows


def test_oracle_reproduces_the_vae_bound_gradients_and_is_estimate(g):
    q, p, flows = _vae_params(g)
    lw = NF.vae_nf(D(g["vae/x"]), D(g["vae/eps"]), q, p, flows)
    bound, cost = NF.bound_and_cost(lw)
    _close(bound, g["vae/bound"], "bound", 1e-5, 1e-6)
    _close(cost, g["vae/cost"], "cost", 1e-5, 1e-6)
    wrt = q + p + [t for f in flows for t in f]
    names = ["q%d_%s" % (i, s) for i in range(4) for s in "Wb"] + \
        ["p%d_%s" % (i, s) for i in range(3) for s in "Wb"] + \
        ["f%d_%s" % (c, s) for c in range(2) for s in ("b", "aux_u", "w")]
    for nm, got in zip(names, torch.autograd.grad(cost, wrt)):
        _close(got, g["vae/grad_" + nm], "grad " + nm, 2e-4, 2e-5)
    with torch.no_grad():
        ll = NF.is_loglikelihood(NF.vae_nf(D(g["vae/is_x"]), D(g["vae/is_eps"]), q, p, flows))
    _close(ll, g["vae/is_ll"], "IS", 1e-5, 1e-6)


def test_top_level_names():
    """transform.py:12-14 exports planar_normalizing_flow; zhusuan/__init__.py re-exports it."""
    assert callable(zs.planar_normalizing_flow) and callable(zs.planar_flow_parameters)


def test_flow_parameters_are_initialised_as_the_reference():
    gen = torch.Generator().manual_seed(7)
    b, u, w = zs.planar_flow_parameters(5, 3, device="cpu", generator=gen)
    assert b.shape == (3,) and u.shape == (3, 5) and w.shape == (3, 5)
    assert all(t.is_leaf and t.requires_grad and t.dtype == torch.float32 for t in (b, u, w))
    assert torch.equal(b, torch.zeros(3))
    # aux_u then w for each flow in turn, N(0, 0.005^2)
    want = torch.randn((3, 2, 5), generator=torch.Generator().manual_seed(7)) * 0.005
    assert torch.equal(u, want[:, 0]) and torch.equal(w, want[:, 1])


def test_malformed_inputs_raise_before_any_launch():
    f = zs.planar_normalizing_flow
    z, lq = torch.zeros(4, 3), torch.zeros(4)
    b, u, w = torch.zeros(2), torch.zeros(2, 3), torch.zeros(2, 3)
    with pytest.raises(ValueError, match="n_iters should be type 'int'"):
        f(z, lq, 2.0, b, u, w)
    with pytest.raises(ValueError, match="rank >= 2"):
        f(torch.zeros(3), torch.zeros(()), 2, b, u, w)
    with pytest.raises(ValueError, match="rank \\(N-1\\)"):
        f(z, torch.zeros(4, 1), 2, b, u, w)
    with pytest.raises(ValueError, match="same shape of \\(N-1\\) dims"):
        f(z, torch.zeros(5), 2, b, u, w)
    with pytest.raises(ValueError, match="b must be"):
        f(z, lq, 2, torch.zeros(3), u, w)
    with pytest.raises(ValueError, match="aux_u must be"):
        f(z, lq, 2, b, torch.zeros(2, 4), w)
    with pytest.raises(ValueError, match="w must be"):
        f(z, lq, 2, b, u, torch.zeros(3))
    with pytest.raises(ValueError, match="1 <= d <= 1024"):
        f(torch.zeros(2, 1025), torch.zeros(2), 1, torch.zeros(1), torch.zeros(1, 1025),
          torch.zeros(1, 1025))
    # well-formed host tensors reach the library, which has no CPU path
    with pytest.raises(ZsbError, match="no CPU fallback"):
        f(z, lq, 2, b, u, w)


def test_zero_flows_return_the_inputs():
    z, lq = torch.randn(4, 3), torch.randn(4)
    zz, ll = zs.planar_normalizing_flow(z, lq, 0, torch.zeros(0), torch.zeros(0, 3),
                                        torch.zeros(0, 3))
    assert zz is z and ll is lq
