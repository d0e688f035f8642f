"""tests/golden/ref_bnn_vi.npz (made by tests/golden/make_ref_bnn_vi_golden.py): the mean-field
variational BNN of bnn_vi.py on the reference's own BayesianNet / elbo / .sgvb().  The committed
arrays must match their digests, and the float64 oracle (oracle/models.py::BNN plus the y_logstd
gradient and per-point outputs of tests/bnn_oracle.py) must reproduce the lower bound, the cost,
the gradient of every variable and the prediction fetches.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest

from bnn_oracle import BNN

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F64 = np.float64


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_bnn_vi.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_bnn_vi_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_bnn_vi/" + k] = [str(a.dtype), list(a.shape),
                                  hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def oracle_elbo(g, x, y, eps):
    """(lower bound, {variable: d cost / d variable}) of elbo(...).sgvb() in float64: w = mu +
    exp(s) eps, L = mean_k [log p(w_k) - log q(w_k)], cost = -L.  Along the reparameterisation
    log q depends on s only through -s per weight, so dL/dmu = mean_k g_k and
    dL/ds = mean_k g_k exp(s) eps_k + 1."""
    mu = [g["var_w_mean_%d" % i].astype(F64) for i in range(2)]
    s = [g["var_w_logstd_%d" % i].astype(F64) for i in range(2)]
    eps = [e.astype(F64) for e in eps]
    w = [m[None] + np.exp(l)[None] * e for m, l, e in zip(mu, s, eps)]
    om = BNN(x, y, int(g["n_train"]), 0.0, 0.0, dtype=F64, y_logstd=F64(g["var_y_logstd"]))
    lp = om.logp(w)
    c = -0.5 * np.log(2 * np.pi)
    logq = sum((c - l[None] - 0.5 * e ** 2).sum((1, 2)) for l, e in zip(s, eps))
    gw = om.grad(w)
    grads = {"y_logstd": -om.grad_y_logstd(w).mean()}
    for i in range(2):
        grads["w_mean_%d" % i] = -gw[i].mean(0)
        grads["w_logstd_%d" % i] = -((gw[i] * np.exp(s[i])[None] * eps[i]).mean(0) + 1)
    return (lp - logq).mean(), grads, om, w


def test_oracle_reproduces_elbo_and_gradients(g):
    lb, grads, _, _ = oracle_elbo(g, g["x"], g["y"], [g["eps0"], g["eps1"]])
    np.testing.assert_allclose(lb, g["lower_bound"], rtol=2e-6)
    np.testing.assert_allclose(-lb, g["cost"], rtol=2e-6)
    for n, want in grads.items():
        ref = g["grad_" + n]
        np.testing.assert_allclose(want, ref, rtol=2e-5, atol=2e-5 * float(np.abs(ref).max()),
                                   err_msg=n)


def test_oracle_reproduces_prediction_fetches(g):
    _, _, om, w = oracle_elbo(g, g["x_test"], g["y_test"], [g["eps_ll0"], g["eps_ll1"]])
    ym, ll = om.predictive(w)
    np.testing.assert_allclose(ym, g["ll_y_mean"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ll, g["ll_log_py_xw"], rtol=1e-5, atol=1e-5)
    std = F64(g["std_y_train"])
    rmse = np.sqrt(((ym.mean(0) - g["y_test"]) ** 2).mean()) * std
    K = ll.shape[0]
    lme = np.log(np.exp(ll - ll.max(0)).mean(0)) + ll.max(0)
    np.testing.assert_allclose(rmse, g["ll_rmse"], rtol=1e-5)
    np.testing.assert_allclose(lme.mean() - np.log(std), g["ll_log_likelihood"], rtol=1e-5)
    assert K == 6
