"""tests/golden/ref_bnn_vi.npz: the mean-field variational BNN of
examples/bayesian_neural_nets/bnn_vi.py on THE REFERENCE'S OWN BayesianNet, Normal, elbo and
.sgvb() (zhusuan/framework, zhusuan/variational), executed on the NumPy TensorFlow stand-in of
oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_bnn_vi_golden.py  ->  ref_bnn_vi.npz, ref_bnn_vi_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  The model is bnn_vi.py:18-50 (build_bnn,
build_mean_field_variational, y_logstd a learned variable) with its log_joint override (83-86) at
layer sizes [13, 20, 1], 10 particles, a minibatch of 10 rows and n_train = 455.  Every variable
(w_mean_*, w_logstd_*, y_logstd) is loaded with non-zero random values, so ReLUs and signs are
exercised; the variational draws eps are injected and stored.  Recorded: the lower bound, the
cost (.sgvb()) and tf.gradients of the cost w.r.t. every variable; then the prediction /
log-likelihood fetches of bnn_vi.py:98-103 on a 12-row test set at ll_samples = 6.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

N_IN, H, K, B, N_TRAIN = 13, 20, 10, 10, 455
K_LL, B_TEST, STD_Y_TRAIN = 6, 12, 1.7


def run_reference_bnn_vi(seed=515):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    utils = importlib.import_module("zhusuan.utils")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()

    @fw.meta_bayesian_net(scope="bnn", reuse_variables=True)
    def build_bnn(x, layer_sizes, n_particles):                    # bnn_vi.py:18-35
        bn = fw.BayesianNet()
        h = tf.tile(x[None, ...], [n_particles, 1, 1])
        for i, (n_in, n_out) in enumerate(zip(layer_sizes[:-1], layer_sizes[1:])):
            w = bn.normal("w" + str(i), tf.zeros([n_out, n_in + 1]), std=1.,
                          group_ndims=2, n_samples=n_particles)
            h = tf.concat([h, tf.ones(tf.shape(h)[:-1])[..., None]], -1)
            h = tf.einsum("imk,ijk->ijm", w, h) / tf.sqrt(
                tf.cast(tf.shape(h)[2], tf.float32))
            if i < len(layer_sizes) - 2:
                h = tf.nn.relu(h)
        y_mean = bn.deterministic("y_mean", tf.squeeze(h, 2))
        y_logstd = tf.get_variable("y_logstd", shape=[],
                                   initializer=tf.constant_initializer(0.))
        bn.normal("y", y_mean, logstd=y_logstd)
        return bn

    @fw.reuse_variables(scope="variational")
    def build_mean_field_variational(layer_sizes, n_particles):    # bnn_vi.py:38-50
        bn = fw.BayesianNet()
        for i, (n_in, n_out) in enumerate(zip(layer_sizes[:-1], layer_sizes[1:])):
            w_mean = tf.get_variable(
                "w_mean_" + str(i), shape=[n_out, n_in + 1],
                initializer=tf.constant_initializer(0.))
            w_logstd = tf.get_variable(
                "w_logstd_" + str(i), shape=[n_out, n_in + 1],
                initializer=tf.constant_initializer(0.))
            bn.normal("w" + str(i), w_mean, logstd=w_logstd,
                      n_samples=n_particles, group_ndims=2)
        return bn

    layer_sizes = [N_IN, H, 1]
    w_names = ["w0", "w1"]
    x_np = rng.standard_normal((B, N_IN)).astype(np.float32)
    y_np = rng.standard_normal(B).astype(np.float32)
    xt_np = rng.standard_normal((B_TEST, N_IN)).astype(np.float32)
    yt_np = rng.standard_normal(B_TEST).astype(np.float32)
    x, y = tf.constant(x_np), tf.constant(y_np)
    model = build_bnn(x, layer_sizes, K)
    variational = build_mean_field_variational(layer_sizes, K)

    def log_joint(bn):                                             # bnn_vi.py:83-86
        log_pws = bn.cond_log_prob(w_names)
        log_py_xw = bn.cond_log_prob('y')
        return tf.add_n(log_pws) + tf.reduce_mean(log_py_xw, 1) * N_TRAIN
    model.log_joint = log_joint
    lower_bound = var.elbo(model, {'y': y}, variational=variational, axis=0)
    cost = lower_bound.sgvb()
    lb_tensor = lower_bound.tensor
    _ = lower_bound.bn                             # builds the model: creates y_logstd
    all_vars = tf.trainable_variables()
    names = [v.name.split("/")[-1].split(":")[0] for v in all_vars]
    assert sorted(names) == sorted(["w_mean_0", "w_logstd_0", "w_mean_1", "w_logstd_1",
                                    "y_logstd"]), names
    out = dict(x=x_np, y=y_np, x_test=xt_np, y_test=yt_np, n_train=np.int32(N_TRAIN),
               std_y_train=np.float32(STD_Y_TRAIN))
    for n, v in zip(names, all_vars):
        shape = np.shape(v.value)
        if n.startswith("w_mean"):
            val = rng.uniform(-1.5, 1.5, shape)
        elif n.startswith("w_logstd"):
            val = rng.uniform(-2.0, -0.5, shape)
        else:
            val = np.float32(-0.3)
        val = np.asarray(val, np.float32)
        v.load(val)
        out["var_" + n] = val
    eps = [rng.standard_normal((K, H, N_IN + 1)).astype(np.float32),
           rng.standard_normal((K, 1, H + 1)).astype(np.float32)]
    out.update(eps0=eps[0], eps1=eps[1])
    sess = tf.Session()
    tf.set_noise(normal=list(eps))
    r = sess.run([lb_tensor, cost] + tf.gradients(cost, all_vars))
    assert not tf._NOISE["normal"]
    out.update(lower_bound=np.asarray(r[0], np.float32), cost=np.asarray(r[1], np.float32))
    for n, g in zip(names, r[2:]):
        out["grad_" + n] = np.asarray(g, np.float32)

    # ---- prediction: rmse & log likelihood (bnn_vi.py:98-103) at ll_samples particles
    xt, yt = tf.constant(xt_np), tf.constant(yt_np)
    model_t = build_bnn(xt, layer_sizes, K_LL)
    model_t.log_joint = log_joint
    variational_t = build_mean_field_variational(layer_sizes, K_LL)
    lb_t = var.elbo(model_t, {'y': yt}, variational=variational_t, axis=0)
    y_mean = lb_t.bn["y_mean"]
    y_pred = tf.reduce_mean(y_mean, 0)
    rmse = tf.sqrt(tf.reduce_mean((y_pred - yt) ** 2)) * STD_Y_TRAIN
    log_py_xw = lb_t.bn.cond_log_prob("y")
    log_likelihood = tf.reduce_mean(utils.log_mean_exp(log_py_xw, 0)) - tf.log(STD_Y_TRAIN)
    _ = lb_t.tensor
    # the stand-in's reuse_variables templates own their variables: give the test graph's
    # copies the same values
    for v in tf.trainable_variables()[len(all_vars):]:
        v.load(out["var_" + v.name.split("/")[-1].split(":")[0]])
    eps_ll = [rng.standard_normal((K_LL, H, N_IN + 1)).astype(np.float32),
              rng.standard_normal((K_LL, 1, H + 1)).astype(np.float32)]
    out.update(eps_ll0=eps_ll[0], eps_ll1=eps_ll[1])
    tf.set_noise(normal=[eps_ll[1], eps_ll[0]])    # y_mean evaluates the w1 draw first
    r = sess.run([y_mean, log_py_xw, rmse, log_likelihood])
    assert not tf._NOISE["normal"]
    out.update(ll_y_mean=np.asarray(r[0], np.float32), ll_log_py_xw=np.asarray(r[1], np.float32),
               ll_rmse=np.float32(r[2]), ll_log_likelihood=np.float32(r[3]))
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_bnn_vi()
    np.savez_compressed(os.path.join(HERE, "ref_bnn_vi.npz"), **out)
    with open(os.path.join(HERE, "ref_bnn_vi_digests.json"), "w") as f:
        json.dump(digests("ref_bnn_vi", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("lower bound %.6g, cost %.6g, rmse %.6g, test ll %.6g"
          % (out["lower_bound"], out["cost"], out["ll_rmse"], out["ll_log_likelihood"]))


if __name__ == "__main__":
    main()
