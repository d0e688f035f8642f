"""tests/golden/ref_ssl.npz: one training step of the semi-supervised VAE (M2) of
examples/semi_supervised_vae/vae_ssl.py on THE REFERENCE'S OWN BayesianNet, Normal, Bernoulli,
OnehotCategorical and elbo(), executed on the NumPy TensorFlow stand-in of oracle/tf_shim (TEST
INFRASTRUCTURE).

    python tests/golden/make_ref_ssl_golden.py  ->  ref_ssl.npz, ref_ssl_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  build_gen, qz_xy and qy_x are vae_ssl.py:19-54 with
64-unit hidden layers in place of the example's 500, at x_dim = 30, z_dim = 8, C = 10 classes,
K = 3 particles, 4 labeled and 3 unlabeled rows of pre-binarised x.  The width keeps the committed
fixture small (every gradient is recorded in full); the example's own widths are checked on the
GPU against tests/ssl_oracle.py, which this fixture pins.  Every tf.layers.dense kernel and bias is loaded with
non-zero random values on a grid of 2^-9; the normal noise of both z draws ([K, 4, z] labeled,
[K, 30, z] for the unlabeled rows tiled as vae_ssl.py:108-116 tiles them, row n C + c) is
injected.  The model is built with n = 1: its prior parameters are zeros, which broadcast to the labeled and to the tiled
unlabeled rows alike (the example feeds one `n` to both, the "n not match" of its TODO).

The stand-in lacks three ops this graph uses: tf.eye, tf.argmax and
tf.nn.softmax_cross_entropy_with_logits (OnehotCategorical.log_prob, multivariate.py:542-559).  They
are installed onto it here, with TF 1.x semantics (no gradient reaches the labels of the cross
entropy), so the stand-in itself is unchanged for every other fixture.

Recorded (kernels stored as W = kernel^T, [units, fan_in], the layout of zs.fused.linear):
  labeled_lb, lb_z [N, C] (reference order), unlabeled_lb, classifier_cost (beta = 1200), cost,
  acc, and tf.gradients(cost) w.r.t. all 22 variables as grad_W_<layer> / grad_b_<layer>.
"""
import hashlib
import importlib
import itertools
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

X_DIM, Z_DIM, C, K, N_L, N_U, H = 30, 8, 10, 3, 4, 3, 64
BETA = 1200.0
MODEL = ["g_z", "g_y", "g_h", "g_x"]
ENCODER = ["q_h1", "q_h2", "q_mean", "q_logstd"]
CLASSIFIER = ["c_h1", "c_h2", "c_logits"]


def _install_ops(tf):
    """tf.eye, tf.argmax and tf.nn.softmax_cross_entropy_with_logits on the stand-in."""
    def eye(num_rows, num_columns=None, batch_shape=None, dtype=np.float32, name=None):
        return tf.constant(np.eye(int(num_rows), None if num_columns is None
                                  else int(num_columns), dtype=dtype))

    def argmax(input, axis=None, name=None, dimension=None, output_type=np.int64):  # noqa: A002
        ax = dimension if axis is None else axis
        ax = 0 if ax is None else ax
        t = tf.convert_to_tensor(input)
        return tf.Tensor(lambda c: np.argmax(c.eval(t), axis=ax).astype(output_type),
                         inputs=(t,), op="argmax", dtype=output_type)

    def softmax_cross_entropy_with_logits(_sentinel=None, labels=None, logits=None, dim=-1,
                                          name=None):
        z, x = tf.convert_to_tensor(labels), tf.convert_to_tensor(logits)

        def f(c):
            xv, zv = np.asarray(c.eval(x)), np.asarray(c.eval(z))
            m = np.max(xv, axis=dim, keepdims=True)
            lsm = xv - m - np.log(np.exp(xv - m).sum(axis=dim, keepdims=True))
            return (-(zv * lsm).sum(axis=dim)).astype(xv.dtype)
        out = tf.Tensor(f, inputs=(z, x), op="softmax_xent", dtype=x._dtype)
        out.vjp = lambda g: [None, tf.expand_dims(g, dim) * (
            tf.nn.softmax(x, axis=dim) * tf.reduce_sum(z, axis=dim, keepdims=True) - z)]
        return out
    tf.eye, tf.argmax = eye, argmax
    tf.nn.softmax_cross_entropy_with_logits = staticmethod(softmax_cross_entropy_with_logits)


def run_reference_ssl(seed=2036):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    _install_ops(tf)
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    dist = importlib.import_module("zhusuan.distributions")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)

    @fw.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, x_dim, n_class, z_dim, n_particles):            # vae_ssl.py:19-33
        bn = fw.BayesianNet()
        z = bn.normal("z", tf.zeros([n, z_dim]), std=1., group_ndims=1, n_samples=n_particles)
        h_from_z = tf.layers.dense(z, H)
        y = bn.onehot_categorical("y", tf.zeros([n, n_class]))
        h_from_y = tf.layers.dense(tf.cast(y, tf.float32), H)
        h = tf.nn.relu(h_from_z + h_from_y)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        bn.bernoulli("x", tf.layers.dense(h, x_dim), group_ndims=1)
        return bn

    @fw.reuse_variables(scope="variational")
    def qz_xy(x, y, z_dim, n_particles):                               # vae_ssl.py:36-46
        bn = fw.BayesianNet()
        h = tf.layers.dense(tf.cast(tf.concat([x, y], -1), tf.float32), H, activation=tf.nn.relu)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        bn.normal("z", tf.layers.dense(h, z_dim), logstd=tf.layers.dense(h, z_dim),
                  group_ndims=1, n_samples=n_particles)
        return bn

    @fw.reuse_variables("classifier")
    def qy_x(x, n_class):                                              # vae_ssl.py:49-54
        h = tf.layers.dense(tf.cast(x, tf.float32), H, activation=tf.nn.relu)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        return tf.layers.dense(h, n_class)

    x_l_np = (rng.random((N_L, X_DIM)) < 0.4).astype(np.int32)
    y_l_np = np.eye(C, dtype=np.int32)[rng.integers(0, C, N_L)]
    x_u_np = (rng.random((N_U, X_DIM)) < 0.4).astype(np.int32)
    x_l, y_l, x_u = tf.constant(x_l_np), tf.constant(y_l_np), tf.constant(x_u_np)

    # labeled, vae_ssl.py:86-96
    model = build_gen(1, X_DIM, C, Z_DIM, K)
    variational = qz_xy(x_l, y_l, Z_DIM, K)
    lb_l_obj = var.elbo(model, observed={"x": x_l, "y": y_l}, variational=variational, axis=0)
    labeled_lb = tf.reduce_mean(lb_l_obj.tensor)
    _ = lb_l_obj.bn                                   # builds the model's layers
    # unlabeled, vae_ssl.py:100-124
    y_diag = tf.eye(C, dtype=tf.int32)
    y_u = tf.reshape(tf.tile(y_diag[None, ...], [N_U, 1, 1]), [-1, C])
    x_ut = tf.reshape(tf.tile(x_u[:, None, ...], [1, C, 1]), [-1, X_DIM])
    variational_u = qz_xy(x_ut, y_u, Z_DIM, K)
    lb_z_obj = var.elbo(model, observed={"x": x_ut, "y": y_u}, variational=variational_u,
                        axis=0)
    lb_z = tf.reshape(lb_z_obj.tensor, [-1, C])
    qy_logits_u = qy_x(x_u, C)
    qy_u = tf.nn.softmax(qy_logits_u) + 1e-8
    qy_u /= tf.reduce_sum(qy_u, 1, keepdims=True)
    log_qy_u = tf.log(qy_u)
    unlabeled_lb = tf.reduce_mean(tf.reduce_sum(qy_u * (lb_z - log_qy_u), 1))
    # classifier, vae_ssl.py:126-136
    qy_logits_l = qy_x(x_l, C)
    qy_l = tf.nn.softmax(qy_logits_l)
    pred_y = tf.argmax(qy_l, 1)
    acc = tf.reduce_sum(tf.cast(tf.equal(pred_y, tf.argmax(y_l, 1)), tf.float32) /
                        tf.cast(tf.shape(x_l)[0], tf.float32))
    log_qy_x = dist.OnehotCategorical(qy_logits_l).log_prob(y_l)
    classifier_cost = -BETA * tf.reduce_mean(log_qy_x)
    cost = -(labeled_lb + unlabeled_lb - classifier_cost) / 2.

    all_vars = tf.trainable_variables()
    names = ENCODER + MODEL + CLASSIFIER              # creation order
    assert len(all_vars) == 2 * len(names), len(all_vars)
    fans = dict(g_z=(Z_DIM, H), g_y=(C, H), g_h=(H, H), g_x=(H, X_DIM), q_h1=(X_DIM + C, H),
                q_h2=(H, H), q_mean=(H, Z_DIM), q_logstd=(H, Z_DIM), c_h1=(X_DIM, H),
                c_h2=(H, H), c_logits=(H, C))
    out = dict(x_l=x_l_np, y_l=y_l_np, x_u=x_u_np)
    for i, name in enumerate(names):
        kern, bias = all_vars[2 * i], all_vars[2 * i + 1]
        fan_in, units = np.shape(kern.value)
        assert (fan_in, units) == fans[name], (name, fan_in, units)
        # on a grid of 2^-9 (exact in float32, and the fixture compresses to a fraction)
        kv = (np.round(rng.standard_normal((fan_in, units)) * 1.2 / np.sqrt(fan_in) * 512)
              / 512).astype(np.float32)
        kv[kv == 0] = 1.0 / 512
        bv = (np.round(0.3 * rng.standard_normal(units) * 512) / 512).astype(np.float32)
        bv[bv == 0] = 1.0 / 512
        kern.load(kv)
        bias.load(bv)
        out["W_" + name] = np.ascontiguousarray(kv.T)
        out["b_" + name] = bv
    eps_l = rng.standard_normal((K, N_L, Z_DIM)).astype(np.float32)
    eps_u = rng.standard_normal((K, N_U * C, Z_DIM)).astype(np.float32)
    out.update(eps_l=eps_l, eps_u=eps_u)

    sess = tf.Session()
    fetches = [labeled_lb, lb_z, unlabeled_lb, classifier_cost, cost, acc]
    grads = tf.gradients(cost, all_vars)
    r = None
    for order in itertools.permutations((eps_l, eps_u)):
        tf.set_noise(normal=list(order))
        try:
            r = sess.run(fetches + grads)
        except AssertionError:                         # a draw of the wrong shape
            continue
        assert not tf._NOISE["normal"]
        break
    assert r is not None, "no order of the injected draws fits"
    for k, v in zip(["labeled_lb", "lb_z", "unlabeled_lb", "classifier_cost", "cost", "acc"], r):
        out[k] = np.asarray(v, np.float32)
    for name, gW, gb in zip(names, r[6::2], r[7::2]):
        out["grad_W_" + name] = np.ascontiguousarray(np.asarray(gW, np.float32).T)
        out["grad_b_" + name] = np.asarray(gb, np.float32)
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_ssl()
    np.savez_compressed(os.path.join(HERE, "ref_ssl.npz"), **out)
    with open(os.path.join(HERE, "ref_ssl_digests.json"), "w") as f:
        json.dump(digests("ref_ssl", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("labeled %.6g, unlabeled %.6g, classifier cost %.6g, cost %.6g, acc %.3g"
          % (out["labeled_lb"], out["unlabeled_lb"], out["classifier_cost"], out["cost"],
             out["acc"]))


if __name__ == "__main__":
    main()
