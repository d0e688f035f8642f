"""tests/golden/ref_bnn_deep.npz (made by tests/golden/make_ref_bnn_deep_golden.py): Bayesian neural
nets with two and three hidden layers on the reference's own BayesianNet, SG-MCMC samplers and
elbo / .sgvb().  The committed arrays must match their digests, and the float64 oracle of
tests/bnn_deep_oracle.py (with oracle/sgmcmc.py for the samplers) must follow every SG-MCMC run
and reproduce the lower bound, the cost, every gradient and the prediction fetches.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest

from bnn_deep_oracle import DeepBNN
from oracle import sgmcmc as OS

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F64 = np.float64
NETS = ["h2", "h3"]
TAGS = ["sghmc", "sgld", "psgld", "sgnht_vec_2nd", "sgnht_vec_1st", "sgnht_scalar_2nd",
        "sgnht_scalar_1st"]


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_bnn_deep.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_bnn_deep_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_bnn_deep/" + k] = [str(a.dtype), list(a.shape),
                                    hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want
    assert sorted({k.split("/")[0] for k in g.files}) == NETS


def n_layers(g, net):
    return len(g[net + "/sizes"]) - 1


def golden_oracle(g, net, dtype=F64):
    L = n_layers(g, net)
    return DeepBNN(g[net + "/x"].astype(dtype), g[net + "/y"].astype(dtype),
                   int(g[net + "/n_train"]), [g[net + "/logstd%d" % i].astype(dtype)
                                              for i in range(L)], y_logstd=-0.95, dtype=dtype)


def config(g, net, tag):
    p = "%s/%s/cfg_" % (net, tag)
    return {k[len(p):]: g[k] for k in g.files if k.startswith(p)}


def oracle_sampler(g, net, tag, dtype=F64):
    cfg = config(g, net, tag)
    lr = float(cfg["learning_rate"])
    L = n_layers(g, net)
    if tag == "sgld":
        return OS.SGLD(lr, dtype=dtype)
    if tag == "psgld":
        return OS.PSGLD(lr, dtype=dtype)
    if tag == "sghmc":
        s = OS.SGHMC(lr, friction=float(cfg["friction"]),
                     variance_estimate=float(cfg["variance_estimate"]),
                     n_iter_resample_v=int(cfg["n_iter_resample_v"]),
                     second_order=bool(cfg["second_order"]), dtype=dtype)
    else:
        s = OS.SGNHT(lr, variance_extra=float(cfg["variance_extra"]),
                     tune_rate=float(cfg["tune_rate"]),
                     n_iter_resample_v=int(cfg["n_iter_resample_v"]),
                     second_order=bool(cfg["second_order"]),
                     use_vector_alpha=bool(cfg["use_vector_alpha"]), dtype=dtype)
    s.init_v([g["%s/v0_%d" % (net, i)].astype(dtype) for i in range(L)])
    return s


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("net", NETS)
def test_oracle_follows_reference_run(g, net, tag):
    om = golden_oracle(g, net)
    s = oracle_sampler(g, net, tag)
    L = n_layers(g, net)
    q = [g["%s/w%d_init" % (net, i)].astype(F64) for i in range(L)]
    p = "%s/%s/" % (net, tag)
    for t in range(g[p + "w0"].shape[0]):
        nz = [g[p + "noise%d" % k][t].astype(F64) for k in range(L)]
        rs = [g[p + "resample%d" % k][t].astype(F64) for k in range(L)]
        if isinstance(s, (OS.SGHMC, OS.SGNHT)):
            q, info = s.step(q, om.grad, rs, nz)
        else:
            q, info = s.step(q, om.grad, nz)
        for k in range(L):
            want = g[p + "w%d" % k][t]
            np.testing.assert_allclose(q[k], want, rtol=2e-4, atol=2e-5,
                                       err_msg="%s%s step %d w%d" % (p, tag, t, k))
            if "mean_k" in info and p + "mean_k%d" % k in g.files:
                mk = np.asarray(g[p + "mean_k%d" % k][t])
                np.testing.assert_allclose(info["mean_k"][k], mk, rtol=1e-3,
                                           atol=1e-3 * float(np.abs(mk).max()))
            if "alpha" in info:
                np.testing.assert_allclose(info["alpha"][k], g[p + "alpha%d" % k][t],
                                           rtol=1e-4, atol=1e-6)
        # tolerance of one step: continue from the reference's float32 state
        q = [g[p + "w%d" % k][t].astype(F64) for k in range(L)]


def oracle_elbo(g, net, x, y, eps):
    """(lower bound, {variable: d cost / d variable}, oracle, weights) of elbo(...).sgvb() in
    float64, as tests/test_ref_bnn_vi_pins.py derives it: w = mu + exp(s) eps,
    L = mean_k [log p(w_k) - log q(w_k)], cost = -L, dL/dmu = mean_k g_k and
    dL/ds = mean_k g_k exp(s) eps_k + 1."""
    p = net + "/vi/"
    L = n_layers(g, net)
    mu = [g[p + "var_w_mean_%d" % i].astype(F64) for i in range(L)]
    s = [g[p + "var_w_logstd_%d" % i].astype(F64) for i in range(L)]
    eps = [e.astype(F64) for e in eps]
    w = [m[None] + np.exp(l)[None] * e for m, l, e in zip(mu, s, eps)]
    om = DeepBNN(x, y, int(g[p + "n_train"]), [0.0] * L, y_logstd=F64(g[p + "var_y_logstd"]))
    lp = om.logp(w)
    c = -0.5 * np.log(2 * np.pi)
    logq = sum((c - l[None] - 0.5 * e ** 2).sum((1, 2)) for l, e in zip(s, eps))
    gw = om.grad(w)
    grads = {"y_logstd": -om.grad_y_logstd(w).mean()}
    for i in range(L):
        grads["w_mean_%d" % i] = -gw[i].mean(0)
        grads["w_logstd_%d" % i] = -((gw[i] * np.exp(s[i])[None] * eps[i]).mean(0) + 1)
    return (lp - logq).mean(), grads, om, w


@pytest.mark.parametrize("net", NETS)
def test_oracle_reproduces_elbo_and_gradients(g, net):
    p = net + "/vi/"
    L = n_layers(g, net)
    lb, grads, _, _ = oracle_elbo(g, net, g[p + "x"], g[p + "y"],
                                  [g[p + "eps%d" % i] for i in range(L)])
    np.testing.assert_allclose(lb, g[p + "lower_bound"], rtol=2e-6)
    np.testing.assert_allclose(-lb, g[p + "cost"], rtol=2e-6)
    assert sorted(grads) == sorted(k[len(p) + 5:] for k in g.files if k.startswith(p + "grad_"))
    for n, want in grads.items():
        ref = g[p + "grad_" + n]
        np.testing.assert_allclose(want, ref, rtol=2e-5, atol=2e-5 * float(np.abs(ref).max()),
                                   err_msg=n)


@pytest.mark.parametrize("net", NETS)
def test_oracle_reproduces_prediction_fetches(g, net):
    p = net + "/vi/"
    L = n_layers(g, net)
    _, _, om, w = oracle_elbo(g, net, g[p + "x_test"], g[p + "y_test"],
                              [g[p + "eps_ll%d" % i] for i in range(L)])
    ym, ll = om.predictive(w)
    np.testing.assert_allclose(ym, g[p + "ll_y_mean"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ll, g[p + "ll_log_py_xw"], rtol=1e-5, atol=1e-5)
    std = F64(g[p + "std_y_train"])
    np.testing.assert_allclose(np.sqrt(((ym.mean(0) - g[p + "y_test"]) ** 2).mean()) * std,
                               g[p + "ll_rmse"], rtol=1e-5)
    lme = np.log(np.exp(ll - ll.max(0)).mean(0)) + ll.max(0)
    np.testing.assert_allclose(lme.mean() - np.log(std), g[p + "ll_log_likelihood"], rtol=1e-5)
