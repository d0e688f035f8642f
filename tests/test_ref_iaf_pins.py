"""tests/golden/ref_iaf.npz (made by tests/golden/make_ref_iaf_golden.py): the reference's own
inv_autoregressive_flow with linear_ar, for both updates.  The committed arrays must match their
digests, the float64 oracle of tests/iaf_oracle.py and the generic (torch) path of
zs.inv_autoregressive_flow must reproduce every recorded value, the Jacobian check of the
reference's TestLinearIaf must hold, LinearAR must draw its weights in the reference's order, and
malformed inputs must raise before any launch.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import iaf_oracle as IAF
import zhusuan_b200 as zs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
UPDATES = ("normal", "gru")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_iaf.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_iaf_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_iaf/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def D(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=torch.float64).requires_grad_(grad)


def _close(got, want, what, rtol, atol):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(got.detach().double().numpy(), want, rtol=rtol,
                               atol=atol * max(1.0, np.abs(want).max()), err_msg=what)


def _check_against_golden(g, u, z, lq, ins):
    _close(z, g[u + "/z"], u + " z", 1e-5, 1e-6)
    _close(lq, g[u + "/log_q"], u + " log_q", 1e-5, 1e-6)
    f = (z * D(g[u + "/cz"]).to(z.dtype)).sum() + (lq * D(g[u + "/cl"]).to(lq.dtype)).sum()
    for k, got in zip(("samples", "log_probs", "m_w", "s_w"), torch.autograd.grad(f, ins)):
        _close(got, g[u + "/grad_" + k], u + " grad " + k, 1e-4, 1e-5)


@pytest.mark.parametrize("u", UPDATES)
def test_oracle_reproduces_the_reference(g, u):
    ins = [D(g[u + "/" + k], True) for k in ("samples", "log_probs", "m_w", "s_w")]
    z, lq = IAF.linear_iaf(*ins, update=u)
    _check_against_golden(g, u, z, lq, ins)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("u", UPDATES)
def test_generic_path_on_cpu_reproduces_the_reference(g, u, dtype):
    ar = zs.LinearAR(7, 3, device="cpu")
    with torch.no_grad():
        ar.m_w.copy_(torch.from_numpy(g[u + "/m_w"]))
        ar.s_w.copy_(torch.from_numpy(g[u + "/s_w"]))
    s = torch.tensor(g[u + "/samples"], dtype=dtype, requires_grad=True)
    l = torch.tensor(g[u + "/log_probs"], dtype=dtype, requires_grad=True)
    z, lq = zs.inv_autoregressive_flow(s, None, l, ar, 3, update=u)
    tol = 1e-5 if dtype == torch.float64 else 2e-5
    _close(z, g[u + "/z"], u + " z", tol, tol / 10)
    _close(lq, g[u + "/log_q"], u + " log_q", tol, tol / 10)
    if dtype == torch.float64:
        _check_against_golden(g, u, z, lq, [s, l, ar.m_w, ar.s_w])


@pytest.mark.parametrize("u", UPDATES)
def test_log_det_jacobian_of_one_flow(u):
    """TestLinearIaf.test_linear_iaf (tests/test_transform.py:51-75): for one flow on the 8-vector
    below, -log|det dz_1/dz_0| equals the change in log_q."""
    vz = torch.tensor([[0.1, -1.2, 1.0, -0.3, 1.2, 2, 10.0, -23.2]], dtype=torch.float64)
    ar = zs.LinearAR(8, 1, device="cpu", generator=torch.Generator().manual_seed(3))
    with torch.no_grad():                       # scale the N(0, 0.005^2) draws to matter
        ar.m_w.mul_(20)
        ar.s_w.mul_(20)

    def f(z0):
        return zs.inv_autoregressive_flow(z0, None, torch.zeros(1, dtype=torch.float64), ar, 1,
                                          update=u)[0][0]
    jac = torch.autograd.functional.jacobian(f, vz)[:, 0, :]
    _, n_log_det = zs.inv_autoregressive_flow(vz, None, torch.zeros(1, dtype=torch.float64), ar,
                                              1, update=u)
    want = -torch.linalg.slogdet(jac)[1]
    assert torch.allclose(n_log_det[0], want, rtol=1e-10, atol=1e-10), (n_log_det, want)
    assert abs(float(want)) > 1e-3


def test_linear_ar_is_initialised_as_the_reference():
    gen = torch.Generator().manual_seed(7)
    ar = zs.LinearAR(5, 3, device="cpu", generator=gen)
    assert ar.m_w.shape == (3, 5, 5) and ar.s_w.shape == (3, 5, 5)
    assert all(t.is_leaf and t.requires_grad and t.dtype == torch.float32
               for t in (ar.m_w, ar.s_w))
    # m_w then s_w for each flow in turn (transform.py:48-55), N(0, 0.005^2)
    want = torch.randn((3, 2, 5, 5), generator=torch.Generator().manual_seed(7)) * 0.005
    assert torch.equal(ar.m_w, want[:, 0]) and torch.equal(ar.s_w, want[:, 1])


def test_linear_ar_call_is_linear_ar():
    """__call__ restates linear_ar for one flow and ignores `hidden`."""
    ar = zs.LinearAR(4, 2, device="cpu", generator=torch.Generator().manual_seed(1))
    z = torch.randn(2, 3, 4)
    m, s = ar("iaf", 1, z, torch.randn(2, 3, 4))
    mask = torch.tensor([[float(i < j) for j in range(4)] for i in range(4)])
    assert torch.allclose(m, z @ (mask * ar.m_w[1]))
    assert torch.allclose(s, torch.exp(z @ (mask * ar.s_w[1])))


def test_malformed_inputs_raise_before_any_launch():
    f = zs.inv_autoregressive_flow
    ar = zs.LinearAR(3, 2, device="cpu")
    z, lq = torch.zeros(4, 3), torch.zeros(4)
    with pytest.raises(ValueError, match="n_iters should be type 'int'"):
        f(z, None, lq, ar, 2.0)
    with pytest.raises(ValueError, match="rank >= 2"):
        f(torch.zeros(3), None, torch.zeros(()), ar, 2)
    with pytest.raises(ValueError, match="rank \\(N-1\\)"):
        f(z, None, torch.zeros(4, 1), ar, 2)
    with pytest.raises(ValueError, match="same shape of \\(N-1\\) dims"):
        f(z, None, torch.zeros(5), ar, 2)
    with pytest.raises(ValueError, match="update should be 'normal' or 'gru'"):
        f(z, None, lq, ar, 2, update="lstm")
    with pytest.raises(ValueError, match="LinearAR is for d = 3 and 2 flows"):
        f(z, None, lq, ar, 3)
    with pytest.raises(ValueError, match="LinearAR is for d = 3 and 2 flows"):
        f(torch.zeros(4, 5), None, lq, ar, 2)
    meta = torch.device("meta")
    with pytest.raises(ValueError, match="log_probs is on"):
        f(z, None, torch.zeros(4, device=meta), ar, 2)
    with pytest.raises(ValueError, match="the LinearAR is on"):
        f(z.to(meta), None, lq.to(meta), ar, 2)


def test_zero_flows_return_the_inputs():
    z, lq = torch.randn(4, 3), torch.randn(4)
    zz, ll = zs.inv_autoregressive_flow(z, None, lq, zs.LinearAR(3, 0, device="cpu"), 0)
    assert zz is z and ll is lq


def test_top_level_names():
    """zs exposes the reference's inv_autoregressive_flow and a LinearAR for its linear_ar."""
    assert callable(zs.inv_autoregressive_flow) and isinstance(zs.LinearAR, type)
    assert "inv_autoregressive_flow" in zs.transform.__all__ and "LinearAR" in zs.transform.__all__
