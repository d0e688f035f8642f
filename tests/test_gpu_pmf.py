"""GPU tests of zs.fused.PMFLogJoint (csrc/pmf.cu): the chunked log-joint of the Bayesian PMF
example (pmf_hmc.py:19-31, 136-144) against the float64 oracle, determinism, HMC on the provider
against the oracle HMC, against the reference's own chunk-by-chunk run (ref_pmf_hmc.npz), and
against the same model written on zs.BayesianNet on the generic autograd path; C ABI checks."""
import os

import numpy as np
import pytest
import torch

from oracle import hmc as OH
from pmf_oracle import PMF, make_corpus

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _case(D, K, chunk, n_chunks=4, n_cols=700, nnz=2000, heavy=500, seed=0):
    """Zipf-like degrees, the last chunk without any rating (padding), one row with `heavy`
    ratings (longer than the 32-rating tile of a warp and the 128 of a block)."""
    n_rows = chunk * n_chunks
    rows, cols, r = make_corpus(n_rows, n_cols, nnz, seed + D, pad_rows=chunk, heavy_row=0,
                                heavy_n=heavy)
    rng = np.random.RandomState(seed + 7 * D)
    s = 1.0 / np.sqrt(D)
    lat = (s * rng.standard_normal((K, n_chunks, chunk, D))).astype(np.float32)
    fixed = (s * rng.standard_normal((K, n_cols, D))).astype(np.float32)
    return rows, cols, r, lat, fixed, n_rows


@pytest.mark.parametrize("D,K,chunk", [(1, 3, 50), (7, 5, 1), (30, 8, 50), (30, 3, 1),
                                       (64, 3, 50), (128, 2, 50)])
def test_pmf_kernel_matches_oracle(zs, D, K, chunk):
    rows, cols, r, lat, fixed, n_rows = _case(D, K, chunk, n_chunks=4 if chunk > 1 else 60)
    assert np.bincount(rows).max() > 128 and not np.any(rows >= n_rows - chunk)
    om = PMF(rows, cols, r, fixed, n_rows, chunk, 1.0, 0.7, 0.05)
    lj = zs.fused.PMFLogJoint(rows, cols, r, fixed=T(fixed), n_rows=n_rows, chunk_size=chunk,
                              std=1.0, fixed_std=0.7, rating_std=0.05, name="u")
    lp, g = N(lj.logp([T(lat)])), N(lj.grad([T(lat)])[0])
    ref_lp, ref_g = om.logp([lat]), om.grad([lat])[0]
    assert lp.shape == ref_lp.shape == (K, n_rows // chunk)
    np.testing.assert_allclose(lp, ref_lp, rtol=2e-5, atol=1e-3)
    np.testing.assert_allclose(g, ref_g, rtol=2e-4, atol=2e-4 * np.abs(ref_g).max())
    np.testing.assert_allclose(N(lj({"u": T(lat)})), ref_lp, rtol=5e-5, atol=5e-3)


def test_pmf_kernel_is_deterministic(zs):
    rows, cols, r, lat, fixed, n_rows = _case(30, 8, 50, n_chunks=6, nnz=20000)
    lj = zs.fused.PMFLogJoint(rows, cols, r, fixed=T(fixed), n_rows=n_rows, chunk_size=50,
                              std=1.0, fixed_std=1.0, rating_std=0.05)
    x = T(lat)
    a, b = N(lj.logp([x])), N(lj.logp([x]))
    ga, gb = N(lj.grad([x])[0]), N(lj.grad([x])[0])
    assert a.tobytes() == b.tobytes() and ga.tobytes() == gb.tobytes()


def test_pmf_provider_hmc_matches_oracle(zs):
    rows, cols, r, lat, fixed, n_rows = _case(30, 4, 10, n_chunks=5, n_cols=300, nnz=600,
                                              heavy=150)
    K, nc, cs, D = lat.shape
    om = PMF(rows, cols, r, fixed, n_rows, cs, 1.0, 1.0, 0.05, dtype=np.float32)
    lj = zs.fused.PMFLogJoint(rows, cols, r, fixed=T(fixed), n_rows=n_rows, chunk_size=cs,
                              std=1.0, fixed_std=1.0, rating_std=0.05)
    u = T(lat)
    h = zs.HMC(step_size=0.01, n_leapfrogs=10)
    op, info = h.sample(lj, {}, {"u": u})
    assert h._provider is lj and tuple(info.acceptance_rate.shape) == (K, nc)
    oh = OH.HMC(step_size=0.01, n_leapfrogs=10)
    oq = [lat]
    rng = np.random.RandomState(3)
    n_acc = 0
    for i in range(4):
        npz = rng.standard_normal(lat.shape).astype(np.float32)
        nu = rng.random_sample((K, nc)).astype(np.float32)
        oq, oi = oh.step(oq, om.logp, om.grad, [npz], nu)
        op(noise={"p": {"u": T(npz)}, "u": T(nu)})
        np.testing.assert_allclose(N(info.acceptance_rate), oi.acceptance_rate, rtol=2e-3,
                                   atol=2e-4)
        np.testing.assert_allclose(N(info.orig_log_prob), oi.orig_log_prob, rtol=2e-5, atol=2e-3)
        near = np.abs(nu - oi.acceptance_rate) < 1e-3
        np.testing.assert_allclose(N(u)[~near], oq[0][~near], rtol=1e-3, atol=1e-4)
        oq = [N(u)]                        # continue from the same state
        n_acc += int(oi.if_accept.sum())
    assert 0 < n_acc


def test_pmf_provider_hmc_follows_reference_run(zs):
    """ref_pmf_hmc.npz was recorded chunk by chunk, one HMC call per chunk, by the reference's own
    BayesianNet / Normal / HMC; here each sweep is ONE call over all chunks, the two samplers read
    each other's latent in place, and every chunk's slice follows the reference."""
    g = np.load(os.path.join(GOLD, "ref_pmf_hmc.npz"))
    K, D, cs = int(g["cfg_K"]), int(g["cfg_D"]), int(g["cfg_chunk"])
    N_, M_ = int(g["cfg_n_users"]), int(g["cfg_n_movies"])
    U, V = T(g["U0"]), T(g["V0"])
    u, v = U.view(K, N_ // cs, cs, D), V.view(K, M_ // cs, cs, D)
    kw = dict(chunk_size=cs, rating_std=float(g["cfg_alpha_pred"]))
    lj_u = zs.fused.PMFLogJoint(g["rows"], g["cols"], g["rating"], fixed=v, n_rows=N_,
                                std=float(g["cfg_alpha_u"]), fixed_std=float(g["cfg_alpha_v"]),
                                name="u", **kw)
    lj_v = zs.fused.PMFLogJoint(g["cols"], g["rows"], g["rating"], fixed=u, n_rows=M_,
                                std=float(g["cfg_alpha_v"]), fixed_std=float(g["cfg_alpha_u"]),
                                name="v", **kw)
    hk = dict(step_size=float(g["cfg_step_size"]), n_leapfrogs=int(g["cfg_n_leapfrogs"]))
    op_u, info_u = zs.HMC(**hk).sample(lj_u, {}, {"u": u})
    op_v, info_v = zs.HMC(**hk).sample(lj_v, {}, {"v": v})
    for e in range(int(g["cfg_epochs"])):
        for side, op, info, X in (("u", op_u, info_u, U), ("v", op_v, info_v, V)):
            ref = lambda k: g[side + "_" + k][e].T                      # noqa: E731 [K, chunks]
            op(noise={"p": {side: T(np.moveaxis(g[side + "_noise_p"][e], 0, 1))},
                      "u": T(ref("noise_u"))})
            msg = "epoch %d sweep %s" % (e, side)
            np.testing.assert_allclose(N(info.orig_log_prob), ref("lp0"), rtol=2e-5, atol=2e-3,
                                       err_msg=msg)
            np.testing.assert_allclose(N(info.acceptance_rate), ref("acc"), rtol=3e-3, atol=3e-4,
                                       err_msg=msg)
            near = np.abs(ref("noise_u") - ref("acc")) < 2e-3                # [K, chunks]
            far = ~np.repeat(near, cs, axis=1)                               # [K, rows]
            want = g[side.upper()][e]
            np.testing.assert_allclose(N(X)[far], want[far], rtol=1e-3, atol=2e-4, err_msg=msg)
            X.copy_(T(want))                 # continue from the reference's state


def _generic_model(zs, rows, cols, r, fixed, n_rows, cs):
    """The example's model (pmf_hmc.py:19-31, 136-144) written on zs.BayesianNet with torch gathers,
    evaluated chunk by chunk as the example does and stacked to [K, n_chunks]."""
    @zs.meta_bayesian_net(scope="pmf")
    def pmf(n, m, D, K, su, sv):
        bn = zs.BayesianNet()
        uu = bn.normal("u", torch.zeros(n, D, device="cuda"), std=1.0, n_samples=K, group_ndims=1)
        vv = bn.normal("v", torch.zeros(m, D, device="cuda"), std=1.0, n_samples=K, group_ndims=1)
        logits = (uu.tensor[:, su] * vv.tensor[:, sv]).sum(2)
        bn.normal("r", torch.sigmoid(logits), std=0.05)
        return bn

    chunks = []
    for c in range(n_rows // cs):
        sel = np.nonzero(rows // cs == c)[0]
        nbr = np.unique(cols[sel])
        sv = np.searchsorted(nbr, cols[sel])
        chunks.append((torch.tensor(nbr, device="cuda"), torch.tensor(rows[sel] - c * cs,
                       device="cuda"), torch.tensor(sv, device="cuda"), T(r[sel]), len(nbr)))

    def log_joint(obs):
        u = obs["u"]
        K, D = int(u.shape[0]), int(u.shape[-1])
        out = []
        for c, (nbr, su, sv, rc, m) in enumerate(chunks):
            model = pmf(cs, m, D, K, su, sv)
            model.log_joint = lambda bn: sum(x.sum(-1) for x in bn.cond_log_prob(["u", "v"])) + \
                bn.cond_log_prob("r").sum(-1)
            out.append(model.observe(u=u[:, c], v=fixed[:, nbr], r=rc).log_joint())
        return torch.stack(out, 1)
    return log_joint


def test_pmf_provider_matches_generic_autograd_path(zs):
    rows, cols, r, lat, fixed, n_rows = _case(7, 3, 5, n_chunks=3, n_cols=40, nnz=60, heavy=30)
    n_rows -= 5                              # drop the padding chunk: every chunk has ratings
    lat = lat[:, :2]
    lj = zs.fused.PMFLogJoint(rows, cols, r, fixed=T(fixed), n_rows=n_rows, chunk_size=5,
                              std=1.0, fixed_std=1.0, rating_std=0.05)
    generic = _generic_model(zs, rows, cols, r, T(fixed), n_rows, 5)
    x = T(lat).requires_grad_(True)
    lp = generic({"u": x})
    lp.sum().backward()
    np.testing.assert_allclose(N(lp), N(lj.logp([x.detach()])), rtol=2e-5, atol=1e-3)
    gp = N(lj.grad([x.detach()])[0])
    np.testing.assert_allclose(N(x.grad), gp, rtol=2e-4, atol=2e-4 * np.abs(gp).max())
    q_f, q_g = T(lat), T(lat)
    op_f, inf_f = zs.HMC(step_size=0.03, n_leapfrogs=5).sample(lj, {}, {"u": q_f})
    op_g, inf_g = zs.HMC(step_size=0.03, n_leapfrogs=5).sample(generic, {}, {"u": q_g})
    assert inf_g is not None and op_g._hmc._provider is None
    rng = np.random.RandomState(5)
    for i in range(3):
        npz = T(rng.standard_normal(lat.shape))
        nu = rng.random_sample(lat.shape[:2])
        op_f(noise={"p": {"u": npz}, "u": T(nu)})
        op_g(noise={"p": {"u": npz}, "u": T(nu)})
        acc_f, acc_g = N(inf_f.acceptance_rate), N(inf_g.acceptance_rate)
        np.testing.assert_allclose(acc_f, acc_g, rtol=2e-3, atol=2e-4)
        near = np.abs(nu - acc_g) < 1e-3
        assert np.array_equal((nu < acc_f)[~near], (nu < acc_g)[~near])
        np.testing.assert_allclose(N(q_f)[~near], N(q_g)[~near], rtol=1e-3, atol=1e-4)
        q_f.copy_(q_g)


def test_pmf_c_abi_rejects_bad_arguments(zs):
    from zhusuan_b200._lib import lib, ptr, stream
    rows, cols, r, lat, fixed, n_rows = _case(7, 2, 5, n_chunks=2, n_cols=20, nnz=30, heavy=0)
    lj = zs.fused.PMFLogJoint(rows, cols, r, fixed=T(fixed), n_rows=n_rows, chunk_size=5)
    x, lp = T(lat), torch.empty(2, 2, device="cuda")
    g, work = torch.empty_like(x), torch.empty(2, n_rows, device="cuda")
    dll = lib.load()

    def call(D=7, lat_p=ptr(x), fixed_p=ptr(lj.fixed), row_ptr=ptr(lj.row_ptr), lp_p=ptr(lp),
             g_p=ptr(g), work_p=ptr(work), nbr=ptr(lj.nbr_ptr), chunk=5):
        return dll.zsb_pmf_logjoint_f32(lat_p, fixed_p, row_ptr, ptr(lj.col_idx), ptr(lj.rating),
                                        nbr, ptr(lj.nbr_idx), 0.0, 0.0, 0.0, lp_p, g_p, work_p,
                                        2, n_rows, 20, D, chunk, stream())
    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(D=0), dict(D=129), dict(lat_p=None), dict(fixed_p=None), dict(row_ptr=None),
                dict(lp_p=None, g_p=None), dict(work_p=None), dict(nbr=None), dict(chunk=3)):
        assert call(**bad) == -1, bad
        assert "zsb_pmf_logjoint_f32" in lib.last_error()
    call(D=129)
    assert "D = 129" in lib.last_error()
    assert call(lp_p=None, work_p=None, nbr=None) == 0       # gradient only needs no workspace
    torch.cuda.synchronize()
