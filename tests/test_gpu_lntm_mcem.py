"""The logistic-normal topic model trained by Monte-Carlo EM and scored by AIS
(examples/topic_models/lntm_mcem.py) on the sparse kernels of csrc/lntm.cu:

* the E-step log-joint and its gradient for any 1 <= K <= 128, on a subset of the corpus' documents
  and at an AIS temperature, against the float64 oracle of tests/lntm_mcem_oracle.py;
* the M-step's log p(x | eta, beta) and its beta gradient (``LNTMLogJoint.cond_log_px``) against
  the same oracle, bit-identical across repeated calls;
* ``zs.AIS`` on the tempered provider, step for step against the reference's AIS run
  (tests/golden/ref_lntm_mcem.npz), and against the generic route under the same noise;
* one training epoch of tests/lntm_mcem_models.py, both arms, against the reference's run.
"""
import collections
import os

import numpy as np
import pytest
import torch

import lntm_mcem_oracle as LO
from oracle import evaluation as OE
from oracle import hmc as OH

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


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_lntm_mcem.npz"))


def _corpus(rng, n_docs, V, K):
    x = rng.poisson(0.05, (n_docs, V)).astype(np.float32)
    x[:, :4] += rng.integers(1, 4, (n_docs, 4))           # words shared by every document
    x[2] = 0                                              # an empty (padding) document
    beta = rng.standard_normal((K, V)).astype(np.float32)
    mean = (0.3 * rng.standard_normal(K)).astype(np.float32)
    logstd = (0.2 * rng.standard_normal(K)).astype(np.float32)
    return x, beta, mean, logstd


def _close_grad(got, want):
    np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-4 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("K", [1, 7, 20, 100, 127, 128])
def test_estep_any_topic_count_subset_and_temperature(zs, K):
    rng = np.random.Generator(np.random.PCG64(K))
    V, n_docs, C = 300, 9, 70
    x, beta, mean, logstd = _corpus(rng, n_docs, V, K)
    lj = zs.fused.LNTMLogJoint(T(x), T(beta), T(mean), T(logstd))
    Kp = 16 * -(-K // 16)
    assert tuple(lj.phi_t.shape) == (V, Kp) and not lj.phi_t[:, K:].any()
    for ids in (None, [7, 2, 4, 0]):
        lj.set_docs(None if ids is None else T(ids, torch.int64))
        B = n_docs if ids is None else len(ids)
        eta = rng.standard_normal((C, B, K)).astype(np.float32)
        om = LO.LNTM(x, beta, mean, logstd, doc_ids=ids)
        lp, gr = lj.logp([T(eta)]), lj.grad([T(eta)])[0]
        np.testing.assert_allclose(N(lp), om.logp([eta]), rtol=2e-5, atol=1e-3)
        _close_grad(N(gr), om.grad([eta])[0])
        for t in (0.0, 0.37, 1.0):
            prov = lj.tempered(T(t))
            lp_t, gr_t = prov.logp([T(eta)]), prov.grad([T(eta)])[0]
            np.testing.assert_allclose(N(lp_t), om.logp_t([eta], t), rtol=2e-5, atol=1e-3)
            _close_grad(N(gr_t), om.grad_t([eta], t)[0])
            if t == 1.0:
                assert torch.equal(lp_t, lp) and torch.equal(gr_t, gr)
        np.testing.assert_allclose(N(lj({"eta": T(eta)})), om.logp([eta]), rtol=5e-5, atol=5e-3)


def test_estep_rejects_more_than_128_topics(zs):
    rng = np.random.Generator(np.random.PCG64(5))
    x, beta, mean, logstd = _corpus(rng, 4, 50, 129)
    lj = zs.fused.LNTMLogJoint(T(x), T(beta), T(mean), T(logstd))
    assert not hasattr(lj, "_zsb_fused")                  # HMC differentiates the dense form
    with pytest.raises(ValueError, match="n_topics"):
        lj.logp([T(np.zeros((1, 4, 129)))])
    from zhusuan_b200._lib import ZsbError, lib, ptr, stream
    eta, phi_t = T(np.zeros((1, 4, 129))), T(np.zeros((50, 144)))
    with pytest.raises(ZsbError, match="n_topics"):
        lib.call("zsb_lntm_logjoint_f32", ptr(eta), ptr(lj.eta_mean), ptr(lj.eta_logstd),
                 ptr(phi_t), ptr(lj.doc_ptr), ptr(lj.word_idx), ptr(lj.word_cnt), None, None,
                 ptr(T(np.zeros((1, 4)))), None, 1, 4, 129, stream())
    np.testing.assert_allclose(N(lj.cond_log_px(eta, T(beta))),
                               LO.LNTM(x, beta, mean, logstd).log_px(np.zeros((1, 4, 129))),
                               rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize("C,K", [(1, 100), (3, 20), (70, 20), (3, 128)])
def test_mstep_value_and_beta_gradient(zs, C, K):
    rng = np.random.Generator(np.random.PCG64(100 * C + K))
    V, n_docs = 400, 11
    x, beta, mean, logstd = _corpus(rng, n_docs, V, K)
    lj = zs.fused.LNTMLogJoint(T(x), T(beta), T(mean), T(logstd))
    for ids in (None, [9, 2, 5, 0, 10]):
        lj.set_docs(None if ids is None else T(ids, torch.int64))
        B = n_docs if ids is None else len(ids)
        eta = rng.standard_normal((C, B, K)).astype(np.float32)
        gup = rng.standard_normal((C, B)).astype(np.float32)
        om = LO.LNTM(x, beta, mean, logstd, doc_ids=ids)
        outs = []
        for _ in range(2):
            b = T(beta).requires_grad_(True)
            lp = lj.cond_log_px(T(eta), b)
            db, = torch.autograd.grad((lp * T(gup)).sum(), [b])
            outs.append((lp.detach(), db))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        lp, db = outs[0]
        np.testing.assert_allclose(N(lp), om.log_px(eta), rtol=2e-5, atol=1e-3)
        _close_grad(N(db), om.beta_grad(eta, gup))
        # float64 takes the dense restatement
        b64 = T(beta, torch.float64).requires_grad_(True)
        lp64 = lj.cond_log_px(T(eta, torch.float64), b64)
        db64, = torch.autograd.grad((lp64 * T(gup, torch.float64)).sum(), [b64])
        np.testing.assert_allclose(N(lp64), om.log_px(eta), rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(N(db64), om.beta_grad(eta, gup), rtol=1e-8, atol=1e-10)


def _eta_prior(zs, mean, logstd, n_chains, n_docs):
    @zs.meta_bayesian_net()
    def eta_prior():
        bn = zs.BayesianNet()
        bn.normal("eta", mean.unsqueeze(0).expand(n_docs, -1), logstd=logstd, n_samples=n_chains,
                  group_ndims=1)
        return bn
    return eta_prior()


def _run_ais(zs, g, fused):
    x_test, init = g["x_test"], g["ais_init"]
    n_chains, n_test, K = init.shape[1:]
    n_t = g["ais_schedule"].shape[0] - 1
    n_adapt = g["ais_noise_u"].shape[0] - n_t
    mean, logstd = T(g["Eta_mean"]), T(g["Eta_logstd"])
    lj = zs.fused.LNTMLogJoint(T(x_test), T(g["beta"][-1]), mean, logstd)
    eta = torch.zeros(n_chains, n_test, K, device="cuda")
    hmc = zs.HMC(step_size=0.01, n_leapfrogs=3, adapt_step_size=True, target_acceptance_rate=0.6)
    ais = zs.AIS(lj if fused else (lambda obs: lj(obs)), _eta_prior(zs, mean, logstd, n_chains,
                                                                     n_test),
                 hmc, observed={}, latent={"eta": eta}, n_temperatures=n_t, n_adapt=n_adapt)
    assert (hmc._provider is not None) == fused
    accs, op = [], ais.sample_op

    def sample_op(**kw):
        op(**kw)
        accs.append(N(ais.hmc_info.acceptance_rate))
    ais.sample_op = sample_op
    bound = ais.run(noise=lambda k: {"p": {"eta": T(g["ais_noise_p"][k])},
                                     "u": T(g["ais_noise_u"][k])},
                    init=[[T(init[0])], [T(init[1])]])
    return ais, bound, eta, accs


def test_ais_fused_route_follows_reference_run(zs, g):
    ais, bound, eta, accs = _run_ais(zs, g, fused=True)
    # the float64 oracle's acceptance rates locate knife-edge uniforms
    m = LO.LNTM(g["x_test"], g["beta"][-1], g["Eta_mean"], g["Eta_logstd"])
    hmc = OH.HMC(step_size=0.01, n_leapfrogs=3, adapt_step_size=True, target_acceptance_rate=0.6)
    ref_accs, step = [], hmc.step

    def oracle_step(*a):
        q, info = step(*a)
        ref_accs.append(info.acceptance_rate)
        return q, info
    hmc.step = oracle_step
    n_t = g["ais_schedule"].shape[0] - 1
    oa = OE.AIS(lambda q: m.log_prior(q[0]), lambda q: m.grad_t(q, 0.0), m.logp, m.grad, hmc,
                n_temperatures=n_t, n_adapt=g["ais_noise_u"].shape[0] - n_t, dtype=np.float64)
    oa.run([[g["ais_init"][0]], [g["ais_init"][1]]],
           lambda k: ([g["ais_noise_p"][k]], g["ais_noise_u"][k]), adapt_flags=(True, False))
    for k, (a, ra) in enumerate(zip(accs, ref_accs)):
        u = g["ais_noise_u"][k]
        np.testing.assert_allclose(a, ra, rtol=2e-3, atol=2e-4)
        far = np.abs(u - ra) > 2e-3
        np.testing.assert_array_equal((a > u)[far], (ra > u)[far])
    np.testing.assert_allclose(N(ais.log_weights), g["ais_log_weights"], rtol=2e-4, atol=2e-3)
    assert abs(bound - float(g["ais_bound"])) < 2e-3
    np.testing.assert_allclose(N(eta), g["ais_eta_final"], rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(N(ais._schedule), g["ais_schedule"], rtol=1e-6, atol=1e-7)


def test_ais_fused_and_generic_routes_reach_the_same_bound(zs, g):
    _, fused, eta_f, _ = _run_ais(zs, g, fused=True)
    _, generic, eta_g, _ = _run_ais(zs, g, fused=False)
    assert abs(fused - generic) < 2e-3
    np.testing.assert_allclose(N(eta_f), N(eta_g), rtol=1e-3, atol=2e-4)


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
def test_training_epoch_replays_reference_run(zs, g, fused):
    import lntm_mcem_models as LM
    C, B = g["noise_u"].shape[1:]
    e_steps = g["acc"].shape[0] // (g["x_train"].shape[0] // B)
    model = LM.MCEM(zs, g["x_train"], T(g["beta0"]), n_chains=C, batch_size=B, fused=fused,
                    num_e_steps=e_steps, step_size=0.05, n_leapfrogs=3)
    assert (model.hmc._provider is model.lj) == fused
    rec = collections.defaultdict(list)

    def noise(t, j):
        i = t * e_steps + j
        return {"p": {"eta": T(g["noise_p"][i])}, "u": T(g["noise_u"][i])}
    perplexity = model.run_epoch(perm=T(g["perm"], torch.int64), noise=noise, record=rec)
    for i in range(g["acc"].shape[0]):
        np.testing.assert_allclose(N(rec["acc"][i]), g["acc"][i], rtol=3e-3, atol=3e-4)
        np.testing.assert_allclose(float(rec["step_size"][i]), g["step_size"][i], rtol=3e-4)
        np.testing.assert_allclose(N(rec["eta"][i]), g["eta"][i], rtol=1e-3, atol=2e-4)
    for t in range(g["log_px"].shape[0]):
        np.testing.assert_allclose(float(rec["log_px"][t]), g["log_px"][t], rtol=2e-5)
        want = g["grad_beta"][t]
        np.testing.assert_allclose(N(rec["grad_beta"][t]), want, rtol=2e-3,
                                   atol=2e-4 * np.abs(want).max())
        np.testing.assert_allclose(N(rec["beta"][t]), g["beta"][t], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(N(model.Eta), g["Eta"], rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(N(model.lj.eta_mean), g["Eta_mean"], rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(N(model.lj.eta_logstd), g["Eta_logstd"], rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(float(perplexity), g["perplexity"], rtol=2e-5)
    n_t = g["ais_schedule"].shape[0] - 1
    ais, bound = model.ais(g["x_test"], n_chains=g["ais_init"].shape[1], n_temperatures=n_t,
                           n_adapt=g["ais_noise_u"].shape[0] - n_t, n_leapfrogs=3,
                           noise=lambda k: {"p": {"eta": T(g["ais_noise_p"][k])},
                                            "u": T(g["ais_noise_u"][k])},
                           init=[[T(g["ais_init"][0])], [T(g["ais_init"][1])]])
    assert abs(bound - float(g["ais_bound"])) < 5e-3
