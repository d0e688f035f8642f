"""tests/golden/ref_vardrop.npz (made by tests/golden/make_ref_vardrop_golden.py): a training-mode
and an evaluation-mode run of the variational-dropout classifier of variational_dropout.py on the
reference's own BayesianNet, distributions and elbo().  The committed arrays must match their
digests, and the float64 oracle of tests/vardrop_oracle.py must reproduce every recorded value.
CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import vardrop_oracle as VD

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
L, N_TRAIN = 4, 60000


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_vardrop.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_vardrop_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_vardrop/" + k] = [str(a.dtype), list(a.shape),
                                   hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def _params(g):
    T = lambda k: torch.tensor(g[k], dtype=torch.float64).requires_grad_(True)   # noqa: E731
    return ([T("W_%d" % i) for i in range(L)], [T("beta_%d" % i) for i in range(L)],
            [T("logit_alpha_%d" % i) for i in range(L)])


def test_oracle_reproduces_the_training_run(g):
    Ws, betas, alphas = _params(g)
    J = [int(W.shape[0]) for W in Ws]
    out = VD.vardrop_run(torch.tensor(g["x"], dtype=torch.float64), torch.tensor(g["y"]),
                         [torch.tensor(g["z_%d" % i], dtype=torch.float64) for i in range(L)],
                         Ws, betas, alphas, [torch.zeros(j, dtype=torch.float64) for j in J],
                         [torch.ones(j, dtype=torch.float64) for j in J], True, N_TRAIN)
    for k in ("bound", "cost", "acc", "logits"):
        np.testing.assert_allclose(out[k].detach().numpy(), g[k], rtol=2e-5, atol=2e-5, err_msg=k)
    assert (g["logits"] >= 0).all()                     # the ReLU on the logits layer
    for i in range(L):
        for k in ("moving_mean", "moving_variance"):
            np.testing.assert_allclose(out[k][i].detach().numpy(), g["%s_%d" % (k, i)],
                                       rtol=1e-5, atol=1e-6, err_msg="%s %d" % (k, i))
    grads = torch.autograd.grad(out["cost"], Ws + betas + alphas)
    names = ["grad_W_%d" % i for i in range(L)] + ["grad_beta_%d" % i for i in range(L)] + \
        ["grad_logit_alpha_%d" % i for i in range(L)]
    for name, got in zip(names, grads):
        want = g[name].astype(np.float64)
        np.testing.assert_allclose(got.numpy(), want, rtol=2e-4,
                                   atol=2e-5 * max(1.0, np.abs(want).max()), err_msg=name)


def test_oracle_reproduces_the_evaluation_run(g):
    Ws, betas, alphas = _params(g)
    T = lambda k: torch.tensor(g[k], dtype=torch.float64)          # noqa: E731
    out = VD.vardrop_run(T("x"), torch.tensor(g["y"]), [T("eval_z_%d" % i) for i in range(L)],
                         Ws, betas, alphas, [T("moving_mean_%d" % i) for i in range(L)],
                         [T("moving_variance_%d" % i) for i in range(L)], False, N_TRAIN)
    np.testing.assert_allclose(out["bound"].detach().numpy(), g["eval_bound"], rtol=2e-5)
    np.testing.assert_allclose(out["acc"].detach().numpy(), g["eval_acc"])
    np.testing.assert_allclose(out["logits"].detach().numpy(), g["eval_logits"], rtol=2e-5,
                               atol=2e-5)
