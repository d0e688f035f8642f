"""tests/golden/ref_lntm_mcem.npz: one epoch of the logistic-normal topic model trained by
Monte-Carlo EM (examples/topic_models/lntm_mcem.py) and a short AIS evaluation of it, on THE
REFERENCE'S OWN BayesianNet, Normal, UnnormalizedMultinomial, HMC, tf.gradients and AIS, executed on
the NumPy TensorFlow stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_lntm_mcem_golden.py  ->  ref_lntm_mcem.npz,
                                                          ref_lntm_mcem_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.

The graph is the example's (the lntm meta-net, :33-48; the E-step with e_obj, :97-105; the M-step
objective, :106-114; AIS with the eta prior as proposal, :116-142) at small shapes: 6 training
documents zero-padded to 8 (:71-74), batches of 4, V = 30, K = 20 topics (not a multiple of 16),
2 chains, 2 E-steps of 3 leapfrog steps each, one epoch (:148-194).  beta starts from non-zero
random values rather than zeros.  The stand-in has no AdamOptimizer, so the M-step takes
tf.gradients of -log_joint_beta w.r.t. beta and applies TF's Adam formula in float32 here.  The
shuffle permutation and every HMC draw are injected.

The AIS run uses the trained beta and the updated eta prior: 3 chains over 3 test documents,
5 temperatures after 2 adaptation iterations, HMC with 3 leapfrog steps.  Its two prior draws are
injected as standard normals and recorded as eta (noise * exp(logstd) + mean, float32).
"""
import copy
import importlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import make_ref_ssl_golden as ssl_golden  # noqa: E402  (digests)

V, K, C, B, N_TRAIN, N_TEST = 30, 20, 2, 4, 6, 3
E_STEPS, LEAPFROGS, STEP_SIZE, TARGET = 2, 3, 0.05, 0.6
LOG_DELTA, LR0, T0, EPOCH = 10.0, 1.0, 10, 1
AIS_CHAINS, AIS_T, AIS_ADAPT, AIS_STEP = 3, 5, 2, 0.01
ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-8


def run_reference(seed=4242):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, hmc_mod, _ = mrg.load_reference()
    fw = importlib.import_module("zhusuan.framework")
    stub = types.ModuleType("zhusuan.variational")      # evaluation.py imports it for
    stub.ImportanceWeightedObjective = None              # is_loglikelihood only
    sys.modules["zhusuan.variational"] = stub
    ev = importlib.import_module("zhusuan.evaluation")
    assert os.path.realpath(ev.__file__).startswith(os.path.realpath(mrg.REF))
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()

    @fw.meta_bayesian_net(scope="lntm")
    def lntm(n_chains, n_docs, n_topics, n_vocab, eta_mean, eta_logstd):
        bn = fw.BayesianNet()
        eta_mean = tf.tile(tf.expand_dims(eta_mean, 0), [n_docs, 1])
        eta = bn.normal("eta", eta_mean, logstd=eta_logstd, n_samples=n_chains, group_ndims=1)
        theta = tf.nn.softmax(eta)
        beta = bn.normal("beta", tf.zeros([n_topics, n_vocab]), logstd=LOG_DELTA, group_ndims=1)
        phi = tf.nn.softmax(beta)
        doc_word = tf.matmul(tf.reshape(theta, [-1, n_topics]), phi)
        doc_word = tf.reshape(doc_word, [n_chains, n_docs, n_vocab])
        bn.unnormalized_multinomial("x", tf.log(doc_word), normalize_logits=False,
                                    dtype=tf.float32)
        return bn

    def e_obj(bn):
        return bn.cond_log_prob("eta") + bn.cond_log_prob("x")

    def log_prior(bn):
        return bn.cond_log_prob("eta")

    # corpus: Poisson counts with a few repeated words, a test split, zero padding to the batch
    x_all = rng.poisson(0.4, (N_TRAIN + N_TEST, V)).astype(np.float32)
    x_all[:, :3] += rng.integers(0, 3, (N_TRAIN + N_TEST, 3)).astype(np.float32)
    x_train, x_test = x_all[:N_TRAIN], x_all[N_TRAIN:]
    rem = B - x_train.shape[0] % B
    if rem < B:
        x_train = np.vstack((x_train, np.zeros((rem, V), np.float32)))
    n_rows = x_train.shape[0]
    iters = n_rows // B
    beta0 = (0.3 * rng.standard_normal((K, V))).astype(np.float32)
    perm = rng.permutation(n_rows)

    x = tf.placeholder(tf.float32, shape=[B, V], name="x")
    eta_mean = tf.placeholder(tf.float32, shape=[K], name="eta_mean")
    eta_logstd = tf.placeholder(tf.float32, shape=[K], name="eta_logstd")
    eta = tf.Variable(np.zeros((C, B, K), np.float32), name="eta")
    beta = tf.Variable(beta0, name="beta")
    hmc = hmc_mod.HMC(step_size=STEP_SIZE, n_leapfrogs=LEAPFROGS, adapt_step_size=True,
                      target_acceptance_rate=TARGET)
    model = lntm(C, B, K, V, eta_mean, eta_logstd)
    model.log_joint = e_obj
    sample_op, hmc_info = hmc.sample(model, observed={"x": x, "beta": beta}, latent={"eta": eta})
    bn = model.observe(eta=eta, x=x, beta=beta)
    log_p_beta, log_px = bn.cond_log_prob(["beta", "x"])
    log_p_beta = tf.reduce_sum(log_p_beta)
    log_px = tf.reduce_sum(tf.reduce_mean(log_px, axis=0))
    log_joint_beta = log_p_beta + log_px
    grad_beta = tf.gradients(-log_joint_beta, [beta])[0]

    sess = tf.Session()
    Eta = np.zeros((C, n_rows, K), np.float32)
    Eta_mean = np.zeros(K, np.float32)
    Eta_logstd = np.zeros(K, np.float32)
    m = np.zeros((K, V), np.float32)
    v = np.zeros((K, V), np.float32)
    lr = np.float32(LR0 * (T0 / (T0 + EPOCH)) ** 2)
    X = x_train[perm, :]
    Eta = Eta[:, perm, :]
    rec = {k: [] for k in ("noise_p", "noise_u", "eta", "acc", "step_size", "lp", "lp0",
                           "log_px", "grad_beta", "beta")}
    for t in range(iters):
        x_batch = X[t * B:(t + 1) * B]
        eta.load(Eta[:, t * B:(t + 1) * B, :])
        feed = {x: x_batch, eta_mean: Eta_mean, eta_logstd: Eta_logstd}
        for j in range(E_STEPS):
            npz = rng.standard_normal((C, B, K)).astype(np.float32)
            nu = rng.random((C, B)).astype(np.float32)
            tf.set_noise(normal=[npz], uniform=[nu])
            with np.errstate(all="ignore"):
                _, new_eta, info = sess.run([sample_op, hmc_info.samples["eta"], hmc_info],
                                            feed_dict=feed)
            rec["noise_p"].append(npz); rec["noise_u"].append(nu)
            rec["eta"].append(np.array(new_eta)); rec["acc"].append(info.acceptance_rate)
            rec["step_size"].append(np.float32(info.updated_step_size))
            rec["lp"].append(info.log_prob); rec["lp0"].append(info.orig_log_prob)
            if j + 1 == E_STEPS:
                Eta[:, t * B:(t + 1) * B, :] = new_eta
        g, ll = sess.run([grad_beta, log_px], feed_dict=feed)
        g = np.asarray(g, np.float32)
        # tf.train.AdamOptimizer(lr).minimize: TF's update in float32
        step = t + 1
        m = (ADAM_B1 * m + (1 - ADAM_B1) * g).astype(np.float32)
        v = (ADAM_B2 * v + (1 - ADAM_B2) * g * g).astype(np.float32)
        lr_t = np.float32(lr * np.sqrt(1 - ADAM_B2 ** step) / (1 - ADAM_B1 ** step))
        new_beta = (np.array(beta.value) - lr_t * m / (np.sqrt(v) + np.float32(ADAM_EPS)))
        beta.load(new_beta.astype(np.float32))
        rec["log_px"].append(np.float32(ll)); rec["grad_beta"].append(g)
        rec["beta"].append(np.array(beta.value))
    Eta_mean = np.mean(Eta, axis=(0, 1))
    Eta_logstd = np.log(np.std(Eta, axis=(0, 1)) + 1e-6)
    perplexity = np.exp(-np.sum(rec["log_px"]) / np.sum(X))

    # AIS on the test documents (:116-142, :208-219)
    _x = tf.placeholder(tf.float32, shape=[N_TEST, V], name="x")
    _eta = tf.Variable(np.zeros((AIS_CHAINS, N_TEST, K), np.float32), name="eta")
    _model = lntm(AIS_CHAINS, N_TEST, K, V, eta_mean, eta_logstd)
    _model.log_joint = e_obj
    proposal_model = copy.copy(_model)
    proposal_model.log_joint = log_prior
    _hmc = hmc_mod.HMC(step_size=AIS_STEP, n_leapfrogs=LEAPFROGS, adapt_step_size=True,
                       target_acceptance_rate=TARGET)
    ais = ev.AIS(_model, proposal_model, _hmc, observed={"x": _x, "beta": beta},
                 latent={"eta": _eta}, n_temperatures=AIS_T, n_adapt=AIS_ADAPT)
    shape = (AIS_CHAINS, N_TEST, K)
    init_noise = [rng.standard_normal(shape).astype(np.float32) for _ in range(2)]
    noises = [(rng.standard_normal(shape).astype(np.float32),
               rng.random(shape[:2]).astype(np.float32)) for _ in range(AIS_ADAPT + AIS_T)]
    normal = ([init_noise[0]] + [n[0] for n in noises[:AIS_ADAPT]] + [init_noise[1]]
              + [n[0] for n in noises[AIS_ADAPT:]])
    tf.set_noise(normal=normal, uniform=[n[1] for n in noises])
    captured = {}
    orig = ais._get_lower_bound
    ais._get_lower_bound = lambda lw: captured.setdefault("lw", np.array(lw)) is None or orig(lw)
    with np.errstate(all="ignore"):
        bound = ais.run(sess, feed_dict={_x: x_test, eta_mean: Eta_mean.astype(np.float32),
                                         eta_logstd: Eta_logstd.astype(np.float32)})
    assert not tf._NOISE["normal"] and not tf._NOISE["uniform"]
    std = np.exp(Eta_logstd.astype(np.float32))
    init = np.stack([(n * std + Eta_mean.astype(np.float32)).astype(np.float32)
                     for n in init_noise])

    out = {k: np.stack(val) for k, val in rec.items()}
    out.update(x_train=x_train, x_test=x_test, perm=perm.astype(np.int64), beta0=beta0,
               lr=lr, Eta=Eta[:, np.argsort(perm), :], Eta_mean=Eta_mean.astype(np.float32),
               Eta_logstd=Eta_logstd.astype(np.float32), perplexity=np.float64(perplexity),
               ais_init=init, ais_noise_p=np.stack([n[0] for n in noises]),
               ais_noise_u=np.stack([n[1] for n in noises]),
               ais_log_weights=captured["lw"].astype(np.float32), ais_bound=np.float64(bound),
               ais_eta_final=np.array(_eta.value),
               ais_schedule=np.array([ais._get_schedule_t(t) for t in range(AIS_T + 1)]))
    return out


def main():
    out = run_reference()
    np.savez_compressed(os.path.join(HERE, "ref_lntm_mcem.npz"), **out)
    with open(os.path.join(HERE, "ref_lntm_mcem_digests.json"), "w") as f:
        json.dump(ssl_golden.digests("ref_lntm_mcem", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("log_px %s, perplexity %.6g, acc mean %.3f, AIS bound %.6g"
          % (np.round(out["log_px"], 4).tolist(), out["perplexity"], out["acc"].mean(),
             out["ais_bound"]))


if __name__ == "__main__":
    main()
