"""tests/golden/ref_vardrop.npz: one training-mode run and one evaluation-mode run of the
variational-dropout classifier of examples/bayesian_neural_nets/variational_dropout.py on THE
REFERENCE'S OWN BayesianNet, Normal, Categorical and elbo(), executed on the NumPy TensorFlow
stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_vardrop_golden.py  ->  ref_vardrop.npz, ref_vardrop_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  var_dropout and q are variational_dropout.py:19-50
at widths [30, 20, 20, 20, 10] in place of [784, 100, 100, 100, 10], with S = 3 particles over
n = 5 rows in training and S = 4 in evaluation, and N_TRAIN = 60000 as in the example.  Every
weight, beta and logit_alpha is loaded with non-zero random values on a grid of 2^-9; the
standard-normal draws of q's reparameterised eps are injected.

The stand-in lacks the ops of tf.contrib.layers and two more that this graph uses; they are
installed onto it here with TF 1.x semantics, so the stand-in itself is unchanged for every other
fixture:
  * tf.contrib.layers.fully_connected: no bias when a normalizer_fn is given, then the normalizer,
    then activation_fn, whose default is tf.nn.relu;
  * tf.contrib.layers.batch_norm for a rank-3 input (the non-fused path): center=True (beta),
    scale=False, epsilon=1e-3, decay=0.999.  Training: tf.nn.moments over every axis but the last
    (population variance, the mean under stop_gradient in the variance), normalisation with those
    batch moments, and -- updates_collections=None -- the moving averages updated in place,
    m -= (m - batch) * (1 - decay), no zero-debiasing.  Evaluation: the moving statistics.
    tf.nn.batch_normalization's form x * inv + (beta - mean * inv), inv = rsqrt(var + eps).
  * tf.nn.sparse_softmax_cross_entropy_with_logits (Categorical.log_prob) and tf.argmax;
  * tf.variable_scope with name prefixes for tf.get_variable (q's per-layer logit_alpha).
The updated moving statistics are fetched as the values the in-place update assigns.

Recorded (W_i stored as the kernel transposed, [n_out, n_in], the layout of zs.fused):
  x, y, W_i, beta_i, logit_alpha_i, z_i (the injected draws of layer i, [S, n, n_in]);
  bound (tf.reduce_mean(lower_bound) / N_TRAIN), cost (mean(sgvb()) / N_TRAIN), acc, logits
  [S, n, 10], grad_W_i / grad_beta_i / grad_logit_alpha_i = tf.gradients(cost), and
  moving_mean_i / moving_variance_i after the run;
  eval_z_i, eval_bound, eval_acc and eval_logits: is_training=False on those moving statistics.
"""
import contextlib
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

NET = [30, 20, 20, 20, 10]
S, S_EVAL, N, N_TRAIN = 3, 4, 5, 60000
DECAY, EPS = 0.999, 1e-3


def _install_ops(tf):
    scopes = []
    base_get_variable = tf.get_variable

    @contextlib.contextmanager
    def variable_scope(name, *a, **k):
        scopes.append(str(name))
        try:
            yield name
        finally:
            scopes.pop()

    latest = {}                     # full name -> the variable the latest graph build uses

    def get_variable(name, *a, **k):
        full = "/".join(scopes + [name])
        v = latest[full] = base_get_variable(full, *a, **k)
        return v

    def argmax(input, axis=None, name=None, dimension=None, output_type=np.int64):  # noqa: A002
        ax = dimension if axis is None else axis
        ax = 0 if ax is None else ax
        t = tf.convert_to_tensor(input)
        return tf.Tensor(lambda c: np.argmax(c.eval(t), axis=ax).astype(output_type),
                         inputs=(t,), op="argmax", dtype=output_type)

    def sparse_softmax_cross_entropy_with_logits(_sentinel=None, labels=None, logits=None,
                                                 name=None):
        z, x = tf.convert_to_tensor(labels), tf.convert_to_tensor(logits)

        def f(c):
            xv, zv = np.asarray(c.eval(x)), np.asarray(c.eval(z))
            m = np.max(xv, axis=-1, keepdims=True)
            lsm = xv - m - np.log(np.exp(xv - m).sum(axis=-1, keepdims=True))
            return (-np.take_along_axis(lsm, zv[..., None].astype(np.int64), -1)[..., 0]) \
                .astype(xv.dtype)
        out = tf.Tensor(f, inputs=(z, x), op="sparse_softmax_xent", dtype=x._dtype)
        out.vjp = lambda g: [None, tf.expand_dims(g, -1) * (
            tf.nn.softmax(x) - tf.one_hot(z, tf.shape(x)[-1]))]
        return out

    base_tile = tf.tile

    def tile(a, multiples, name=None):
        a = tf.convert_to_tensor(a)
        out = base_tile(a, multiples)

        def vjp(g):
            def f(c):
                gv, av = np.asarray(c.eval(g)), np.asarray(c.eval(a))
                m = [int(v) for v in np.asarray(c.eval(multiples) if isinstance(multiples, tf.Tensor)
                                                else multiples)]
                shp = [d for mi, di in zip(m, av.shape) for d in (mi, di)]
                return gv.reshape(shp).sum(axis=tuple(range(0, 2 * len(m), 2))).astype(gv.dtype)
            return [tf.Tensor(f, inputs=(g, a), op="tile_grad", dtype=a._dtype)]
        out.vjp = vjp
        return out

    moving = []                                 # (moving_mean, new value, moving_var, new value)

    def batch_norm(inputs, decay=0.999, center=True, scale=False, epsilon=0.001,
                   is_training=True, updates_collections=None, scope=None, **kw):
        assert center and not scale and updates_collections is None
        x = tf.convert_to_tensor(inputs)
        J = int(x.get_shape().as_list()[-1])
        beta = get_variable(scope + "/BatchNorm/beta", [J])
        mm = get_variable(scope + "/BatchNorm/moving_mean", [J], trainable=False)
        mv = get_variable(scope + "/BatchNorm/moving_variance", [J],
                          initializer=tf.constant_initializer(1.0), trainable=False)
        if is_training:
            axes = [0, 1]
            mean = tf.reduce_mean(x, axes, keepdims=True)
            var = tf.reduce_mean(tf.square(x - tf.stop_gradient(mean)), axes, keepdims=True)
            mean, var = tf.reshape(mean, [J]), tf.reshape(var, [J])
            d = np.float32(1.0 - decay)
            moving.append((mm, mm - (mm - mean) * d, mv, mv - (mv - var) * d))
        else:
            mean, var = mm, mv
        inv = 1.0 / tf.sqrt(var + np.float32(epsilon))
        return x * inv + (beta - mean * inv)

    def fully_connected(inputs, num_outputs, activation_fn=tf.nn.relu, normalizer_fn=None,
                        normalizer_params=None, scope=None, **kw):
        store = tf._TEMPLATES[-1] if tf._TEMPLATES else tf._DEFAULT_STORE
        k = store.setdefault("fc_count", 0)
        store["fc_count"] = k + 1
        key = scope or ("fully_connected" if k == 0 else "fully_connected_%d" % k)
        x = tf.convert_to_tensor(inputs)
        W = get_variable(key + "/weights", [int(x.get_shape().as_list()[-1]), num_outputs])
        y = tf._dense_matmul(x, W)
        if normalizer_fn is not None:
            y = normalizer_fn(y, scope=key, **(normalizer_params or {}))
        else:
            y = y + get_variable(key + "/biases", [num_outputs])
        return activation_fn(y) if activation_fn is not None else y

    tf.variable_scope, tf.get_variable, tf.argmax = variable_scope, get_variable, argmax
    tf.tile = tile
    tf.nn.sparse_softmax_cross_entropy_with_logits = staticmethod(
        sparse_softmax_cross_entropy_with_logits)
    layers = type("layers", (object,), {"fully_connected": staticmethod(fully_connected),
                                        "batch_norm": staticmethod(batch_norm)})
    tf.contrib.layers = layers
    return moving, latest


def run_reference_vardrop(seed=2040):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    moving, latest = _install_ops(tf)
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    layers = tf.contrib.layers
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)
    L = len(NET) - 1

    @fw.meta_bayesian_net(scope="model", reuse_variables=True)
    def var_dropout(x, n, net_size, n_particles, is_training):       # variational_dropout.py:19-37
        tf._TEMPLATES[-1]["fc_count"] = 0
        normalizer_params = {'is_training': is_training, 'updates_collections': None}
        bn = fw.BayesianNet()
        h = x
        for i, [n_in, n_out] in enumerate(zip(net_size[:-1], net_size[1:])):
            eps_mean = tf.ones([n, n_in])
            eps = bn.normal('layer' + str(i) + '/eps', eps_mean, std=1.,
                            n_samples=n_particles, group_ndims=1)
            h = layers.fully_connected(h * eps, n_out, normalizer_fn=layers.batch_norm,
                                       normalizer_params=normalizer_params)
            if i < len(net_size) - 2:
                h = tf.nn.relu(h)
        bn.categorical('y', h)
        bn.deterministic('y_logit', h)
        return bn

    @fw.reuse_variables(scope="variational")
    def q(n, net_size, n_particles):                                   # variational_dropout.py:40-50
        bn = fw.BayesianNet()
        stds = []
        for i, [n_in, n_out] in enumerate(zip(net_size[:-1], net_size[1:])):
            with tf.variable_scope('layer' + str(i)):
                logit_alpha = tf.get_variable('logit_alpha', [n_in])
            std = tf.sqrt(tf.nn.sigmoid(logit_alpha) + 1e-10)
            std = tf.tile(tf.expand_dims(std, 0), [n, 1])
            bn.normal('layer' + str(i) + '/eps', 1., std=std, n_samples=n_particles,
                      group_ndims=1)
            stds.append(std)
        return bn, stds

    x_np = (np.round(rng.standard_normal((N, NET[0])) * 512) / 512).astype(np.float32)
    y_np = rng.integers(0, NET[-1], N).astype(np.int32)
    e_names = ['layer' + str(i) + '/eps' for i in range(L)]

    def graph(n_particles, is_training):                                # :86-114
        del moving[:]
        x, y = tf.constant(x_np), tf.constant(y_np)
        x_obs = tf.tile(tf.expand_dims(x, 0), [n_particles, 1, 1])
        y_obs = tf.tile(tf.expand_dims(y, 0), [n_particles, 1])
        model = var_dropout(x_obs, N, NET, n_particles, is_training)
        variational, stds = q(N, NET, n_particles)

        def log_joint(bn):
            log_pe = bn.cond_log_prob(e_names)
            log_py_xe = bn.cond_log_prob('y')
            return tf.add_n(log_pe) + log_py_xe * N_TRAIN
        model.log_joint = log_joint
        lower_bound = var.elbo(model, {'y': y_obs}, variational=variational, axis=0)
        y_logit = lower_bound.bn["y_logit"]
        h_pred = tf.reduce_mean(tf.nn.softmax(y_logit), 0)
        y_pred = tf.argmax(h_pred, 1, output_type=np.int32)
        acc = tf.reduce_mean(tf.cast(tf.equal(y_pred, y), tf.float32))
        cost = tf.reduce_mean(lower_bound.sgvb()) / N_TRAIN
        bound = tf.reduce_mean(lower_bound) / N_TRAIN
        eps = [variational[nm].tensor for nm in e_names]
        return dict(bound=bound, cost=cost, acc=acc, logits=y_logit, eps=eps, stds=stds)

    def run(fetches, n_particles):
        """Session.run with injected draws; returns the results and the draws in layer order."""
        zs_ = [rng.standard_normal((n_particles, N, n_in)).astype(np.float32)
               for n_in in NET[:-1]]
        tf.set_noise(normal=list(zs_))
        r = tf.Session().run(fetches)
        assert not tf._NOISE["normal"]
        return r, zs_

    tr = graph(S, True)
    n_moving = len(moving)
    assert n_moving == L, "the model graph was built %d times" % (n_moving // L)
    model_vars = dict(latest)
    out = dict(x=x_np, y=y_np)
    Ws, betas, alphas = [], [], []
    for i in range(L):
        key = "fully_connected" if i == 0 else "fully_connected_%d" % i
        W = model_vars[key + "/weights"]
        beta = model_vars[key + "/BatchNorm/beta"]
        la = model_vars["layer%d/logit_alpha" % i]
        n_in, n_out = NET[i], NET[i + 1]
        wv = (np.round(rng.standard_normal((n_in, n_out)) / np.sqrt(n_in) * 512) / 512)
        wv[wv == 0] = 1.0 / 512
        bv = np.round(0.3 * rng.standard_normal(n_out) * 512) / 512
        bv[bv == 0] = 1.0 / 512
        av = np.round((rng.standard_normal(n_in) - 1.0) * 512) / 512
        W.load(wv.astype(np.float32))
        beta.load(bv.astype(np.float32))
        la.load(av.astype(np.float32))
        Ws.append(W), betas.append(beta), alphas.append(la)
        out["W_%d" % i] = np.ascontiguousarray(wv.T.astype(np.float32))
        out["beta_%d" % i] = bv.astype(np.float32)
        out["logit_alpha_%d" % i] = av.astype(np.float32)
    grads = tf.gradients(tr["cost"], Ws + betas + alphas)
    new_stats = [m[1] for m in moving] + [m[3] for m in moving]
    fetch = [tr["bound"], tr["cost"], tr["acc"], tr["logits"]] + tr["eps"] + tr["stds"] + \
        grads + new_stats
    r, zs_ = run(fetch, S)
    out.update(bound=np.float32(r[0]), cost=np.float32(r[1]), acc=np.float32(r[2]),
               logits=np.asarray(r[3], np.float32))
    eps_v, std_v = r[4:4 + L], r[4 + L:4 + 2 * L]
    rest = r[4 + 2 * L:]
    for i in range(L):
        # the draw each layer took, found from its eps = 1 + std * z
        errs = [np.abs(eps_v[i] - (1.0 + std_v[i] * z)).max() if z.shape == eps_v[i].shape
                else np.inf for z in zs_]
        k = int(np.argmin(errs))
        assert errs[k] < 1e-5, errs
        out["z_%d" % i] = zs_[k]
        out["grad_W_%d" % i] = np.ascontiguousarray(np.asarray(rest[i], np.float32).T)
        out["grad_beta_%d" % i] = np.asarray(rest[L + i], np.float32)
        out["grad_logit_alpha_%d" % i] = np.asarray(rest[2 * L + i], np.float32)
        out["moving_mean_%d" % i] = np.asarray(rest[3 * L + i], np.float32)
        out["moving_variance_%d" % i] = np.asarray(rest[4 * L + i], np.float32)
    # evaluation on the updated moving statistics (a second build of the templates here makes
    # variables of its own: every value is loaded into them by name)
    ev = graph(S_EVAL, False)
    for i in range(L):
        key = "fully_connected" if i == 0 else "fully_connected_%d" % i
        latest[key + "/weights"].load(out["W_%d" % i].T)
        latest[key + "/BatchNorm/beta"].load(out["beta_%d" % i])
        latest[key + "/BatchNorm/moving_mean"].load(out["moving_mean_%d" % i])
        latest[key + "/BatchNorm/moving_variance"].load(out["moving_variance_%d" % i])
        latest["layer%d/logit_alpha" % i].load(out["logit_alpha_%d" % i])
    r, zs_ = run([ev["bound"], ev["acc"], ev["logits"]] + ev["eps"] + ev["stds"], S_EVAL)
    out.update(eval_bound=np.float32(r[0]), eval_acc=np.float32(r[1]),
               eval_logits=np.asarray(r[2], np.float32))
    r = r[:2] + r[3:]
    for i in range(L):
        errs = [np.abs(r[2 + i] - (1.0 + r[2 + L + i] * z)).max() if z.shape == r[2 + i].shape
                else np.inf for z in zs_]
        k = int(np.argmin(errs))
        assert errs[k] < 1e-5, errs
        out["eval_z_%d" % i] = zs_[k]
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_vardrop()
    np.savez_compressed(os.path.join(HERE, "ref_vardrop.npz"), **out)
    with open(os.path.join(HERE, "ref_vardrop_digests.json"), "w") as f:
        json.dump(digests("ref_vardrop", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("bound %.6g, cost %.6g, acc %.3g, eval bound %.6g, eval acc %.3g"
          % (out["bound"], out["cost"], out["acc"], out["eval_bound"], out["eval_acc"]))


if __name__ == "__main__":
    main()
