"""tests/golden/ref_svgp.npz (made by make_ref_svgp_golden.py from the reference's own utils.py and
the svgp.py graph): its digests, the float64 oracle of tests/svgp_oracle.py against every recorded
value, the public names and the RBFKernel initialiser.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import svgp_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PARAMS = ["z_pos", "k_raw_scale", "noise_level", "z_mean", "z_cov_raw"]


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_svgp.npz"))


def T(a):
    return torch.tensor(np.asarray(a), dtype=torch.float64)


def test_digests(g):
    with open(os.path.join(GOLD, "ref_svgp_digests.json")) as f:
        want = json.load(f)
    assert sorted(want) == sorted("ref_svgp/" + k for k in g.files)
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        assert want["ref_svgp/" + k] == [str(a.dtype), list(a.shape),
                                         hashlib.sha256(a.tobytes()).hexdigest()], k


def _params(g, grad=False):
    return {k: T(g["param/" + k]).requires_grad_(grad) for k in PARAMS}


def test_oracle_bound_cost_and_gradients(g):
    p = _params(g, grad=True)
    obj = O.svgp_bound(p, T(g["x"]), T(g["y"]), float(g["n_train"]), T(g["train/eps_fz"]),
                       T(g["train/eps_fx"]))
    cost = -obj.mean()
    np.testing.assert_allclose(float(obj.mean()), float(g["train/bound"]), rtol=2e-5)
    np.testing.assert_allclose(float(cost), float(g["train/cost"]), rtol=2e-5)
    grads = torch.autograd.grad(cost, [p[k] for k in PARAMS])
    for k, gr in zip(PARAMS, grads):
        want = g["train/grad_" + k]
        np.testing.assert_allclose(gr.numpy(), want, rtol=2e-3,
                                   atol=2e-4 * max(1.0, float(np.abs(want).max())), err_msg=k)


def test_oracle_prediction_fetches(g):
    with torch.no_grad():
        ll, mse = O.svgp_predict(_params(g), T(g["x"]), T(g["y"]), float(g["std_y_train"]),
                                 T(g["pred/eps_fz"]), T(g["pred/eps_fx"]))
    np.testing.assert_allclose(float(ll), float(g["pred/log_likelihood"]), rtol=2e-5)
    np.testing.assert_allclose(float(mse), float(g["pred/pred_mse"]), rtol=2e-5)


def test_oracle_standalone_conditional(g):
    s = O.softplus(T(g["param/k_raw_scale"]))
    z, fz, x = T(g["param/z_pos"]), T(g["cond/fz"]), T(g["x"])
    mean, std = O.gp_conditional(z, fz, x, s)
    np.testing.assert_allclose(mean.numpy(), g["cond/mean"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(std.numpy(), g["cond/std"], rtol=1e-3, atol=1e-5)
    mean_c, tril = O.gp_conditional(z, fz, x, s, full_cov=True)
    np.testing.assert_allclose(mean_c.numpy(), g["cond/full_mean"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(tril.numpy(), g["cond/full_cov_tril"], rtol=1e-2, atol=1e-3)


def test_public_names_and_initialiser():
    import zhusuan_b200 as zs
    assert {"RBFKernel", "gp_conditional"} <= set(zs.fused.__all__)
    k = zs.fused.RBFKernel(4, device="cpu")
    assert k.k_raw_scale.is_leaf and k.k_raw_scale.requires_grad
    assert torch.equal(k.k_raw_scale, torch.zeros(4))         # tf.zeros_initializer (utils.py:15)
