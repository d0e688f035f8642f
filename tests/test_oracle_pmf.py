"""CPU tests of the chunked PMF log-joint (pmf_hmc.py:19-31, 136-144): the NumPy oracle's
gradient, the oracle HMC run as ONE [K, n_chunks] iteration per sweep against the reference's own
chunk-by-chunk run (tests/golden/ref_pmf_hmc.npz), the fixture's digests, and the host-side input
checks and torch restatement of zs.fused.PMFLogJoint."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import hmc as OH
from pmf_oracle import PMF, make_corpus

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _problem(K=3, D=5, n_rows=12, n_cols=9, chunk=4, nnz=40, seed=0):
    rows, cols, r = make_corpus(n_rows, n_cols, nnz, seed, pad_rows=chunk)
    rng = np.random.RandomState(seed + 1)
    lat = (0.5 * rng.standard_normal((K, n_rows // chunk, chunk, D)))
    fixed = (0.5 * rng.standard_normal((K, n_cols, D)))
    return rows, cols, r, lat, fixed


def test_oracle_gradient_matches_finite_differences():
    rows, cols, r, lat, fixed = _problem()
    om = PMF(rows, cols, r, fixed, 12, 4, 0.8, 1.3, 0.3)
    g = om.grad([lat])[0]
    h = 1e-6
    it = np.nditer(lat, flags=["multi_index"])
    for _ in it:
        ix = it.multi_index
        e = np.zeros_like(lat)
        e[ix] = h
        fd = (om.logp([lat + e]) - om.logp([lat - e])) / (2 * h)
        # only chain (k, chunk of ix) depends on the element
        assert np.allclose(fd.sum(), g[ix], rtol=1e-6, atol=1e-6), ix
    np.testing.assert_allclose(g[:, -1], -lat[:, -1] / np.float32(0.8) ** 2, rtol=1e-6)  # padding


def _sweep_oracle(g, side, e, hmc):
    """One HMC iteration over ALL chunks of one factor, continuing from the reference's state."""
    cs = int(g["cfg_chunk"])
    K, D = int(g["cfg_K"]), int(g["cfg_D"])
    U = g["U"][e] if side == "v" else (g["U0"] if e == 0 else g["U"][e - 1])
    V = g["V0"] if e == 0 else g["V"][e - 1]        # the V-sweep follows the epoch's U-sweep
    if side == "u":
        rows, cols, lat, fixed, stds = g["rows"], g["cols"], U, V, ("alpha_u", "alpha_v")
    else:
        rows, cols, lat, fixed, stds = g["cols"], g["rows"], V, U, ("alpha_v", "alpha_u")
    n_lat = lat.shape[1]
    om = PMF(rows, cols, g["rating"], fixed, n_lat, cs, float(g["cfg_" + stds[0]]),
             float(g["cfg_" + stds[1]]), float(g["cfg_alpha_pred"]))
    q = lat.reshape(K, n_lat // cs, cs, D)
    noise_p = np.moveaxis(g[side + "_noise_p"][e], 0, 1)           # [chunk, K, ...] -> [K, chunk, ...]
    noise_u = g[side + "_noise_u"][e].T
    nq, info = hmc.step([q], om.logp, om.grad, [noise_p], noise_u)
    return nq[0].reshape(K, n_lat, D), info


def test_oracle_hmc_all_chunks_at_once_reproduces_reference_chunk_by_chunk():
    g = np.load(os.path.join(GOLD, "ref_pmf_hmc.npz"))
    n_acc = n = 0
    for e in range(int(g["cfg_epochs"])):
        for side in "uv":
            hmc = OH.HMC(step_size=float(g["cfg_step_size"]), n_leapfrogs=int(g["cfg_n_leapfrogs"]))
            q, info = _sweep_oracle(g, side, e, hmc)
            ref = lambda k: g[side + "_" + k][e].T                      # noqa: E731 [K, chunks]
            msg = "epoch %d sweep %s" % (e, side)
            np.testing.assert_allclose(info.orig_log_prob, ref("lp0"), rtol=2e-5, atol=1e-3,
                                       err_msg=msg)
            np.testing.assert_allclose(info.orig_hamiltonian, ref("h0"), rtol=2e-5, atol=1e-3,
                                       err_msg=msg)
            np.testing.assert_allclose(info.acceptance_rate, ref("acc"), rtol=1e-3, atol=1e-4,
                                       err_msg=msg)
            np.testing.assert_allclose(info.log_prob, ref("lp"), rtol=2e-5, atol=1e-3, err_msg=msg)
            live = ref("acc") > 1e-6
            np.testing.assert_allclose(info.hamiltonian[live], ref("h1")[live], rtol=2e-5,
                                       atol=1e-3, err_msg=msg)
            assert np.array_equal(info.if_accept, ref("noise_u") < ref("acc")), msg
            np.testing.assert_allclose(q, g[side.upper()][e], rtol=1e-4, atol=1e-5, err_msg=msg)
            n_acc += int(info.if_accept.sum())
            n += info.if_accept.size
    assert 0 < n_acc < n                 # the fixture has accepted and rejected proposals


def test_committed_pmf_fixture_is_what_the_reference_code_produced():
    digests = json.load(open(os.path.join(GOLD, "ref_pmf_digests.json")))
    assert sorted({k.split("/")[0] for k in digests}) == ["ref_pmf_hmc"]
    g = np.load(os.path.join(GOLD, "ref_pmf_hmc.npz"))
    assert sorted(k.split("/")[1] for k in digests) == sorted(g.files)
    for key, (dtype, shape, sha) in digests.items():
        a = np.ascontiguousarray(g[key.split("/")[1]])
        assert (str(a.dtype), list(a.shape)) == (dtype, shape), key
        assert hashlib.sha256(a.tobytes()).hexdigest() == sha, key


def test_pmf_fixture_covers_padding_and_long_rows():
    g = np.load(os.path.join(GOLD, "ref_pmf_hmc.npz"))
    deg = np.bincount(g["rows"], minlength=int(g["cfg_n_users"]))
    assert deg[-1] == 0 and deg.max() >= 3 * np.median(deg[deg > 0])


def _lj(**kw):
    import zhusuan_b200 as zs
    rows, cols, r, lat, fixed = _problem()
    args = dict(rows=rows, cols=cols, ratings=r, fixed=torch.tensor(fixed, dtype=torch.float32),
                n_rows=12, chunk_size=4, std=0.8, fixed_std=1.3, rating_std=0.3)
    args.update(kw)
    return zs.fused.PMFLogJoint(**args)


@pytest.mark.parametrize("bad", [
    dict(rows=np.array([0, 1, 12])), dict(rows=np.array([-1, 0, 1])),
    dict(cols=np.array([0, 9, 1])), dict(n_rows=10), dict(n_rows=0), dict(chunk_size=0),
    dict(fixed=torch.zeros(3, 9, 6)[..., :5]), dict(fixed=torch.zeros(9, 5)),
    dict(fixed=torch.zeros(3, 9, 5, dtype=torch.float64)), dict(fixed=torch.zeros(3, 9, 129)),
    dict(fixed=torch.zeros(3, 9, 0)), dict(ratings=np.zeros(5)), dict(cols=np.zeros(4, np.int64)),
    dict(rating_std=0.0), dict(std=-1.0), dict(ratings=np.full(3, np.nan)),
    dict(rows=np.zeros((3, 1), np.int64)),
])
def test_pmf_logjoint_rejects_bad_input(bad):
    rows, cols, r = np.array([0, 1, 2]), np.array([0, 1, 2]), np.zeros(3, np.float32)
    kw = dict(rows=rows, cols=cols, ratings=r)
    kw.update(bad)
    with pytest.raises(ValueError):
        _lj(**kw)


def test_pmf_logjoint_checks_latent_and_fixed_shapes():
    lj = _lj()
    for shape in ((3, 3, 4, 6), (2, 3, 4, 5), (3, 12, 5)):
        with pytest.raises(ValueError):
            lj.logp([torch.zeros(shape)])
        with pytest.raises(ValueError):
            lj.grad([torch.zeros(shape)])
    with pytest.raises(ValueError):
        lj.set_fixed(torch.zeros(3, 10, 5))
    lj.set_fixed(torch.zeros(3, 3, 3, 5))          # [K, col_chunks, col_chunk, D] is accepted


def test_pmf_csr_and_neighbour_lists():
    rows, cols, r, lat, fixed = _problem()
    lj = _lj()
    rp = lj.row_ptr.numpy()
    assert rp[0] == 0 and rp[-1] == rows.size and np.all(np.diff(rp) == np.bincount(rows, minlength=12))
    for i in range(12):                       # stable: a row's ratings keep their input order
        sel = np.nonzero(rows == i)[0]
        np.testing.assert_array_equal(lj.col_idx.numpy()[rp[i]:rp[i + 1]], cols[sel])
        np.testing.assert_array_equal(lj.rating.numpy()[rp[i]:rp[i + 1]], r[sel])
    nbp, nbi = lj.nbr_ptr.numpy(), lj.nbr_idx.numpy()
    for c in range(3):
        want = np.unique(cols[rows // 4 == c])
        np.testing.assert_array_equal(nbi[nbp[c]:nbp[c + 1]], want)
    assert nbp[3] == nbp[2]                   # the padding chunk has no neighbours


def test_pmf_torch_restatement_matches_oracle():
    rows, cols, r, lat, fixed = _problem()
    om = PMF(rows, cols, r, fixed, 12, 4, 0.8, 1.3, 0.3)
    lj = _lj(fixed=torch.tensor(fixed, dtype=torch.float32))
    lj.fixed = torch.tensor(fixed)                # float64 for the comparison
    x = torch.tensor(lat, requires_grad=True)
    lp = lj({"u": x})
    np.testing.assert_allclose(lp.detach().numpy(), om.logp([lat]), rtol=1e-6)
    lp.sum().backward()
    np.testing.assert_allclose(x.grad.numpy(), om.grad([lat])[0], rtol=1e-6, atol=1e-7)
