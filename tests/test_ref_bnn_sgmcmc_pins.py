"""tests/golden/ref_bnn_sgmcmc.npz (made by tests/golden/make_ref_bnn_sgmcmc_golden.py): config 4's
BNN run on the reference's own SGLD, PSGLD and SGNHT classes.  The committed arrays must match their
digests, and the float64 / float32 oracle (oracle/models.py::BNN + oracle/sgmcmc.py) must follow
every run.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import models as OM
from oracle import sgmcmc as OS

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TAGS = ["sgld", "psgld", "sgnht_vec_2nd", "sgnht_vec_1st", "sgnht_scalar_2nd", "sgnht_scalar_1st"]


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_bnn_sgmcmc.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_bnn_sgmcmc_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_bnn_sgmcmc/" + k] = [str(a.dtype), list(a.shape),
                                      hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want
    assert sorted({k.split("/")[0] for k in g.files if "/" in k}) == sorted(TAGS)


def oracle_sampler(g, tag, dtype):
    cfg = {k[len(tag) + 5:]: g[k] for k in g.files if k.startswith(tag + "/cfg_")}
    lr = float(cfg["learning_rate"])
    if tag == "sgld":
        return OS.SGLD(lr, dtype=dtype)
    if tag == "psgld":
        return OS.PSGLD(lr, dtype=dtype)
    s = OS.SGNHT(lr, variance_extra=float(cfg["variance_extra"]),
                 tune_rate=float(cfg["tune_rate"]),
                 n_iter_resample_v=int(cfg["n_iter_resample_v"]),
                 second_order=bool(cfg["second_order"]),
                 use_vector_alpha=bool(cfg["use_vector_alpha"]), dtype=dtype)
    s.init_v([g["v0_0"].astype(dtype), g["v0_1"].astype(dtype)])
    return s


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_follows_reference_run(g, tag):
    """Weights to float32 rounding of five steps; SGNHT's mean_k and alpha as well.  Re-draws of
    v happen at t = 0 and 3 for SGNHT (four draws in those steps, two otherwise)."""
    for dtype, tol in ((np.float32, 2e-5), (np.float64, 2e-5)):
        om = OM.BNN(g["x"].astype(dtype), g["y"].astype(dtype), int(g["n_train"]),
                    g["logstd0"].astype(dtype), g["logstd1"].astype(dtype), dtype=dtype)
        s = oracle_sampler(g, tag, dtype)
        q = [g["w0_init"].astype(dtype), g["w1_init"].astype(dtype)]
        for t in range(g[tag + "/w0"].shape[0]):
            nz = [g[tag + "/noise0"][t], g[tag + "/noise1"][t]]
            if isinstance(s, OS.SGNHT):
                rs = [g[tag + "/resample0"][t], g[tag + "/resample1"][t]]
                q, info = s.step(q, om.grad, rs, nz)
            else:
                q, info = s.step(q, om.grad, nz)
            for k in range(2):
                np.testing.assert_allclose(q[k], g[tag + "/w%d" % k][t], rtol=tol * 10, atol=tol,
                                           err_msg="%s step %d w%d" % (tag, t, k))
                if isinstance(s, OS.SGNHT):
                    mk = np.asarray(g[tag + "/mean_k%d" % k][t])
                    np.testing.assert_allclose(info["mean_k"][k], mk, rtol=1e-3,
                                               atol=1e-3 * float(np.abs(mk).max()))
                    np.testing.assert_allclose(info["alpha"][k], g[tag + "/alpha%d" % k][t],
                                               rtol=1e-4, atol=1e-6)
    want = [4, 2, 2, 4, 2] if tag.startswith("sgnht") else [2] * 5
    assert g[tag + "/n_used"].tolist() == want
