"""tests/golden/ref_ssl_ais.npz: one training step and one test batch of the semi-supervised VAE
trained by adaptive importance sampling (examples/semi_supervised_vae/vae_ssl_adaptive_is.py) on
THE REFERENCE'S OWN BayesianNet, Normal, OnehotCategorical, klpq and
importance_weighted_objective, executed on the NumPy TensorFlow stand-in of oracle/tf_shim (TEST
INFRASTRUCTURE).

    python tests/golden/make_ref_ssl_ais_golden.py  ->  ref_ssl_ais.npz, ref_ssl_ais_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  The graph follows the example's structure (build_gen,
qz_xy, qy_x and the two proposals, :19-68; the objectives and costs, :75-146) with 64-unit hidden
layers in place of 500, at x_dim = 30, z_dim = 8, C = 10 classes, K = 3 particles, 4 labeled and 3
unlabeled rows, beta = 1200.  Every tf.layers.dense kernel and bias is loaded with non-zero random
values on a grid of 2^-9.  All noise is injected: the uniforms that binarise x (tf.random_uniform),
the normals of both z draws, and the unlabeled class draw.  The stand-in lacks tf.random.categorical
(OnehotCategorical._sample, multivariate.py:522-540); it is installed here as an op that returns the
injected class indices, together with the ops make_ref_ssl_golden.py installs.  The stand-in itself
is unchanged for every other fixture.

The test batch is the same graph fed pre-binarised x (the example feeds the binarised tensors
directly at test time) with its own noise.

Recorded (kernels stored as W = kernel^T, [units, fan_in], the layout of zs.fused.linear): the
inputs, the noise, labeled_lb, unlabeled_lb, labeled_q_cost, unlabeled_q_cost, classifier_cost and
acc of the step and of the test batch (test_*), and grad_W_<layer> / grad_b_<layer>: model_cost
w.r.t. the model's layers and proposal_cost w.r.t. qy_x's and qz_xy's (:148-156).
"""
import importlib
import itertools
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import make_ref_ssl_golden as ssl_golden  # noqa: E402

X_DIM, Z_DIM, C, K, N_L, N_U, H = 30, 8, 10, 3, 4, 3, 64
BETA = 1200.0
MODEL = ["g_z", "g_y", "g_h", "g_x"]
ENCODER = ["q_h1", "q_h2", "q_mean", "q_logstd"]
CLASSIFIER = ["c_h1", "c_h2", "c_logits"]
_DRAWS = []


def _install_categorical(tf):
    def categorical(logits, num_samples, dtype=None, seed=None, name=None):
        lg = tf.convert_to_tensor(logits)

        def f(c):
            rows = np.shape(c.eval(lg))[0]
            n = int(c.eval(num_samples)) if isinstance(num_samples, tf.Tensor) else int(num_samples)
            if tf._is_peek(c):                          # shape inference: no draw is consumed
                return np.zeros((rows, n), np.int64)
            a = np.asarray(_DRAWS.pop(0), np.int64)
            assert a.shape == (rows, n), a.shape
            return a
        return tf.Tensor(f, inputs=(lg,), op="random_categorical", dtype=np.int64)
    tf.random.categorical = staticmethod(categorical)


def run_reference(seed=2037):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    ssl_golden._install_ops(tf)
    _install_categorical(tf)
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    dist = importlib.import_module("zhusuan.distributions")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)

    @fw.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, x_dim, n_class, z_dim, n_particles):             # :19-33
        bn = fw.BayesianNet()
        z = bn.normal("z", tf.zeros([n, z_dim]), std=1., group_ndims=1, n_samples=n_particles)
        h_from_z = tf.layers.dense(z, H)
        y = bn.onehot_categorical("y", tf.zeros([n, n_class]))
        h_from_y = tf.layers.dense(tf.cast(y, tf.float32), H)
        h = tf.nn.relu(h_from_z + h_from_y)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        bn.bernoulli("x", tf.layers.dense(h, x_dim), group_ndims=1)
        return bn

    @fw.reuse_variables(scope="qz_xy")
    def qz_xy(x, y, z_dim):                                            # :36-43
        h = tf.layers.dense(tf.cast(tf.concat([x, y], -1), tf.float32), H, activation=tf.nn.relu)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        return tf.layers.dense(h, z_dim), tf.layers.dense(h, z_dim)

    @fw.reuse_variables(scope="qy_x")
    def qy_x(x, n_class):                                              # :46-51
        h = tf.layers.dense(tf.cast(x, tf.float32), H, activation=tf.nn.relu)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        return tf.layers.dense(h, n_class)

    def labeled_proposal(x, y, z_dim, n_particles):                    # :53-58
        bn = fw.BayesianNet()
        z_mean, z_logstd = qz_xy(x, y, z_dim)
        bn.normal("z", z_mean, logstd=z_logstd, n_samples=n_particles, group_ndims=1,
                  is_reparameterized=False)
        return bn

    def unlabeled_proposal(x, n_class, z_dim, n_particles):            # :61-68
        bn = fw.BayesianNet()
        y = bn.onehot_categorical("y", qy_x(x, n_class))
        z_mean, z_logstd = qz_xy(x, y, z_dim)
        bn.normal("z", z_mean, logstd=z_logstd, group_ndims=1, is_reparameterized=False,
                  n_samples=n_particles)
        return bn

    model = build_gen(1, X_DIM, C, Z_DIM, K)      # one model for the step and the test batch

    def graph(x_l, y_l, x_u):                                          # :75-146
        proposal = labeled_proposal(x_l, y_l, Z_DIM, K)
        lab_q = tf.reduce_mean(var.klpq(model, observed={"x": x_l, "y": y_l},
                                        variational=proposal, axis=0).importance())
        lab_lb = tf.reduce_mean(var.importance_weighted_objective(
            model, observed={"x": x_l, "y": y_l}, variational=proposal, axis=0))
        proposal = unlabeled_proposal(x_u, C, Z_DIM, K)
        unl_q = tf.reduce_mean(var.klpq(model, observed={"x": x_u}, variational=proposal,
                                        axis=0).importance())
        unl_lb = tf.reduce_mean(var.importance_weighted_objective(
            model, observed={"x": x_u}, variational=proposal, axis=0))
        logits_l = qy_x(x_l, C)
        pred_y = tf.argmax(tf.nn.softmax(logits_l), 1)
        acc = tf.reduce_sum(tf.cast(tf.equal(pred_y, tf.argmax(y_l, 1)), tf.float32) /
                            tf.cast(tf.shape(x_l)[0], tf.float32))
        clf = -BETA * tf.reduce_mean(dist.OnehotCategorical(logits_l).log_prob(y_l))
        return [lab_lb, unl_lb, lab_q, unl_q, clf, acc]

    out = {}
    xp_l = rng.random((N_L, X_DIM)).astype(np.float32)
    xp_u = rng.random((N_U, X_DIM)).astype(np.float32)
    y_l_np = np.eye(C, dtype=np.int32)[rng.integers(0, C, N_L)]
    xp_l_ph, xp_u_ph = tf.constant(xp_l), tf.constant(xp_u)
    x_l = tf.cast(tf.less(tf.random_uniform(tf.shape(xp_l_ph)), xp_l_ph), tf.int32)
    x_u = tf.cast(tf.less(tf.random_uniform(tf.shape(xp_u_ph)), xp_u_ph), tf.int32)
    y_l = tf.constant(y_l_np)
    fetches = graph(x_l, y_l, x_u)
    model_cost = -fetches[0] - fetches[1]
    proposal_cost = fetches[2] + fetches[3] + fetches[4]

    all_vars = tf.trainable_variables()
    names = ENCODER + MODEL + CLASSIFIER                              # creation order
    assert len(all_vars) == 2 * len(names), len(all_vars)
    fans = dict(g_z=(Z_DIM, H), g_y=(C, H), g_h=(H, H), g_x=(H, X_DIM), q_h1=(X_DIM + C, H),
                q_h2=(H, H), q_mean=(H, Z_DIM), q_logstd=(H, Z_DIM), c_h1=(X_DIM, H),
                c_h2=(H, H), c_logits=(H, C))
    by_name = {}
    for i, name in enumerate(names):
        kern, bias = all_vars[2 * i], all_vars[2 * i + 1]
        fan_in, units = np.shape(kern.value)
        assert (fan_in, units) == fans[name], (name, fan_in, units)
        kv = (np.round(rng.standard_normal((fan_in, units)) * 1.2 / np.sqrt(fan_in) * 512)
              / 512).astype(np.float32)
        kv[kv == 0] = 1.0 / 512
        bv = (np.round(0.3 * rng.standard_normal(units) * 512) / 512).astype(np.float32)
        bv[bv == 0] = 1.0 / 512
        kern.load(kv)
        bias.load(bv)
        out["W_" + name] = np.ascontiguousarray(kv.T)
        out["b_" + name] = bv
        by_name[name] = (kern, bias)
    model_vars = [v for n in MODEL for v in by_name[n]]
    prop_names = CLASSIFIER + ENCODER
    prop_vars = [v for n in prop_names for v in by_name[n]]
    grads = tf.gradients(model_cost, model_vars) + tf.gradients(proposal_cost, prop_vars)

    def run(fetch, uniforms, normals, draws):
        sess = tf.Session()
        for uo in itertools.permutations(uniforms):
            for no in itertools.permutations(normals):
                tf.set_noise(normal=list(no), uniform=list(uo))
                _DRAWS[:] = [d[:, None] for d in draws]
                try:
                    r = sess.run(fetch)
                except AssertionError:                  # a draw of the wrong shape
                    continue
                assert not tf._NOISE["normal"] and not tf._NOISE["uniform"] and not _DRAWS
                return r, no
        raise AssertionError("no order of the injected draws fits")

    u_l = rng.random((N_L, X_DIM)).astype(np.float32)
    u_u = rng.random((N_U, X_DIM)).astype(np.float32)
    eps_l = rng.standard_normal((K, N_L, Z_DIM)).astype(np.float32)
    eps_u = rng.standard_normal((K, N_U, Z_DIM)).astype(np.float32)
    y_u = rng.integers(0, C, N_U).astype(np.int64)
    r, order = run(fetches + grads, (u_l, u_u), (eps_l, eps_u), [y_u])
    l_first = order[0] is eps_l                       # the order the two z draws are evaluated in
    keys = ["labeled_lb", "unlabeled_lb", "labeled_q_cost", "unlabeled_q_cost",
            "classifier_cost", "acc"]
    out.update(xp_l=xp_l, xp_u=xp_u, y_l=y_l_np, u_l=u_l, u_u=u_u, eps_l=eps_l, eps_u=eps_u,
               y_u=y_u.astype(np.int32))
    for k, v in zip(keys, r):
        out[k] = np.asarray(v, np.float32)
    gs = r[len(keys):]
    for i, name in enumerate(MODEL + prop_names):
        out["grad_W_" + name] = np.ascontiguousarray(np.asarray(gs[2 * i], np.float32).T)
        out["grad_b_" + name] = np.asarray(gs[2 * i + 1], np.float32)

    # the test batch: pre-binarised x fed to the same graph, as the example feeds it
    tx = (rng.random((N_U, X_DIM)) < 0.4).astype(np.int32)
    ty = np.eye(C, dtype=np.int32)[rng.integers(0, C, N_U)]
    t_eps_l = rng.standard_normal((K, N_U, Z_DIM)).astype(np.float32)
    t_eps_u = rng.standard_normal((K, N_U, Z_DIM)).astype(np.float32)
    t_y_u = rng.integers(0, C, N_U).astype(np.int64)
    test = graph(tf.constant(tx), tf.constant(ty), tf.constant(tx))
    # both z draws have one shape here: they are handed out in the order the step evaluated them
    assert len(tf.trainable_variables()) == len(all_vars)   # no variable is created again
    r, _ = run([test[0], test[1], test[5]], (),
               (t_eps_l, t_eps_u) if l_first else (t_eps_u, t_eps_l), [t_y_u])
    out.update(test_x=tx, test_y=ty, test_eps_l=t_eps_l, test_eps_u=t_eps_u,
               test_y_u=t_y_u.astype(np.int32))
    for k, v in zip(["test_labeled_lb", "test_unlabeled_lb", "test_acc"], r):
        out[k] = np.asarray(v, np.float32)
    return out


def main():
    out = run_reference()
    np.savez_compressed(os.path.join(HERE, "ref_ssl_ais.npz"), **out)
    with open(os.path.join(HERE, "ref_ssl_ais_digests.json"), "w") as f:
        json.dump(ssl_golden.digests("ref_ssl_ais", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print(" ".join("%s %.6g" % (k, out[k]) for k in (
        "labeled_lb", "unlabeled_lb", "labeled_q_cost", "unlabeled_q_cost", "classifier_cost",
        "acc", "test_labeled_lb", "test_unlabeled_lb", "test_acc")))


if __name__ == "__main__":
    main()
