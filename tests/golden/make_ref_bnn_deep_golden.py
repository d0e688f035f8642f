"""tests/golden/ref_bnn_deep.npz: the Bayesian neural nets of examples/bayesian_neural_nets with
two and three hidden layers, on THE REFERENCE'S OWN BayesianNet, SGHMC / SGLD / PSGLD / SGNHT
(zhusuan/sgmcmc.py) and elbo / .sgvb() (zhusuan/variational), executed on the NumPy TensorFlow
stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_bnn_deep_golden.py  ->  ref_bnn_deep.npz, ref_bnn_deep_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  Two nets, layer sizes NETS below: build_bnn of
bnn_sgmcmc.py:19-35 / bnn_vi.py:18-35 (as oracle/tf_shim/make_ref_golden.py restates it, the loop
over layer_sizes) with the log-joint override (bnn_sgmcmc.py:74-77, bnn_vi.py:83-86).  For each net:
  * SG-MCMC, every array prefixed "<net>/<tag>/": four steps of SGHMC (the example's sampler, second
    order) and SGNHT (vector and scalar thermostat, first and second order) with v re-drawn at
    t = 0 and 2, and of SGLD and PSGLD, from the same initial weights, every draw injected and
    stored;
  * VI, prefixed "<net>/vi/": one elbo(...).sgvb() with tf.gradients of the cost w.r.t. every
    variational variable and y_logstd, then the prediction fetches of bnn_vi.py:98-103 on a test
    set.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# net tag -> (layer sizes, particles, rows, n_train)
NETS = {"h2": ([4, 20, 20, 1], 4, 15, 300), "h3": ([3, 6, 5, 4, 1], 5, 11, 200)}
_SGNHT = dict(learning_rate=1e-4, variance_extra=0.05, tune_rate=10., n_iter_resample_v=2)
CONFIGS = {
    "sghmc": ("SGHMC", dict(learning_rate=1e-4, friction=0.2, variance_estimate=0.01,
                            n_iter_resample_v=2, second_order=True)),
    "sgld": ("SGLD", dict(learning_rate=1e-4)),
    "psgld": ("PSGLD", dict(learning_rate=1e-4)),
    "sgnht_vec_2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=True)),
    "sgnht_vec_1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=True)),
    "sgnht_scalar_2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=False)),
    "sgnht_scalar_1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=False)),
}
STEPS = 4


def _reference():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, sg = mrg.load_reference()
    return tf, sg, importlib.import_module("zhusuan.framework")


def _build_bnn(tf, fw, scope):
    @fw.meta_bayesian_net(scope=scope, reuse_variables=True)
    def build_bnn(x, layer_sizes, logstds, n_particles, y_logstd):     # bnn_sgmcmc.py:19-35
        bn = fw.BayesianNet()
        h = tf.tile(x[None, ...], [n_particles, 1, 1])
        for i, (n_i, n_o) in enumerate(zip(layer_sizes[:-1], layer_sizes[1:])):
            w = bn.normal("w" + str(i), tf.zeros([n_o, n_i + 1]), logstd=logstds[i],
                          group_ndims=2, n_samples=n_particles)
            h = tf.concat([h, tf.ones(tf.shape(h)[:-1])[..., None]], -1)
            h = tf.einsum("imk,ijk->ijm", w, h) / tf.sqrt(tf.cast(tf.shape(h)[2], tf.float32))
            if i < len(layer_sizes) - 2:
                h = tf.nn.relu(h)
        y_mean = bn.deterministic("y_mean", tf.squeeze(h, 2))
        bn.normal("y", y_mean, logstd=y_logstd)
        return bn
    return build_bnn


def _log_joint(tf, w_names, n_train):
    def log_joint(bn):                                                  # bnn_sgmcmc.py:74-77
        log_pws = bn.cond_log_prob(w_names)
        log_py_xw = bn.cond_log_prob('y')
        return tf.add_n(log_pws) + tf.reduce_mean(log_py_xw, 1) * n_train
    return log_joint


def run_sgmcmc(net, rng):
    sizes, C, B, n_train = NETS[net]
    tf, sg, fw = _reference()
    tf.reset_default_graph()
    L = len(sizes) - 1
    names = ["w%d" % i for i in range(L)]
    x_np = rng.standard_normal((B, sizes[0])).astype(np.float32)
    y_np = rng.standard_normal(B).astype(np.float32)
    ls_np = [(0.1 * rng.standard_normal((sizes[i + 1], sizes[i] + 1))).astype(np.float32)
             for i in range(L)]
    w_init = [rng.uniform(-1, 1, (C, sizes[i + 1], sizes[i] + 1)).astype(np.float32)
              for i in range(L)]
    wv = [tf.Variable(w, name=n) for w, n in zip(w_init, names)]
    model = _build_bnn(tf, fw, "bnn_" + net)(tf.constant(x_np), sizes,
                                             [tf.constant(a) for a in ls_np], C, -0.95)
    model.log_joint = _log_joint(tf, names, n_train)
    observed = {"y": tf.constant(y_np)}
    latent = dict(zip(names, wv))
    out = dict(x=x_np, y=y_np, n_train=np.int32(n_train), sizes=np.int32(sizes))
    for i in range(L):
        out.update({"logstd%d" % i: ls_np[i], "w%d_init" % i: w_init[i]})
    v0 = [rng.standard_normal(w.shape).astype(np.float32) for w in w_init]
    out.update({"v0_%d" % i: v for i, v in enumerate(v0)})
    sess = tf.Session()
    for tag, (cls, kw) in CONFIGS.items():
        for w, init in zip(wv, w_init):
            w.load(init)
        tf.set_noise(normal=list(v0) * 2)          # initial momenta (sgmcmc.py:320-324, 450-452)
        s = getattr(sg, cls)(**kw)
        sample_op, info = s.sample(model, observed=observed, latent=latent)
        tf.set_noise()
        out.update({tag + "/cfg_" + k: np.float32(v) for k, v in kw.items()})
        rec = {}
        for t in range(STEPS):
            rs = [rng.standard_normal(w.shape).astype(np.float32) for w in w_init]
            nz = [rng.standard_normal(w.shape).astype(np.float32) for w in w_init]
            redraw = cls != "SGLD" and cls != "PSGLD" and t % kw["n_iter_resample_v"] == 0
            # consumption order inside a run (latents in dictionary order): the re-draws of v,
            # then the update noise; the first-order update builds each latent's new v in turn
            if not redraw:
                rs = [np.zeros_like(w) for w in w_init]
                feed = nz
            elif kw["second_order"]:
                feed = rs + nz
            else:
                feed = [a for pair in zip(rs, nz) for a in pair]
            tf.set_noise(normal=list(feed))
            _, r = sess.run([sample_op, info])
            assert not tf._NOISE["normal"], (net, tag, t)
            row = {"n_used": np.int32(len(feed))}
            for k, n in enumerate(names):
                row["w%d" % k] = np.array(latent[n].value)
                row["noise%d" % k] = nz[k]
                row["resample%d" % k] = rs[k]
                if hasattr(r, "mean_k"):
                    row["mean_k%d" % k] = np.asarray(r.mean_k[n], np.float32)
                if hasattr(r, "alpha"):
                    row["alpha%d" % k] = np.asarray(r.alpha[n], np.float32)
            for k, v in row.items():
                rec.setdefault(k, []).append(v)
        out.update({tag + "/" + k: np.stack(v) for k, v in rec.items()})
    return out


def run_vi(net, rng, B_TEST=12, K_LL=6, STD_Y_TRAIN=1.7):
    sizes, K, B, n_train = NETS[net]
    tf, _, fw = _reference()
    var = importlib.import_module("zhusuan.variational")
    utils = importlib.import_module("zhusuan.utils")
    tf.reset_default_graph()
    L = len(sizes) - 1
    names = ["w%d" % i for i in range(L)]

    @fw.meta_bayesian_net(scope="bnn", reuse_variables=True)
    def build_bnn(x, layer_sizes, n_particles):                         # bnn_vi.py:18-35
        bn = fw.BayesianNet()
        h = tf.tile(x[None, ...], [n_particles, 1, 1])
        for i, (n_in, n_out) in enumerate(zip(layer_sizes[:-1], layer_sizes[1:])):
            w = bn.normal("w" + str(i), tf.zeros([n_out, n_in + 1]), std=1.,
                          group_ndims=2, n_samples=n_particles)
            h = tf.concat([h, tf.ones(tf.shape(h)[:-1])[..., None]], -1)
            h = tf.einsum("imk,ijk->ijm", w, h) / tf.sqrt(tf.cast(tf.shape(h)[2], tf.float32))
            if i < len(layer_sizes) - 2:
                h = tf.nn.relu(h)
        y_mean = bn.deterministic("y_mean", tf.squeeze(h, 2))
        y_logstd = tf.get_variable("y_logstd", shape=[],
                                   initializer=tf.constant_initializer(0.))
        bn.normal("y", y_mean, logstd=y_logstd)
        return bn

    @fw.reuse_variables(scope="variational")
    def build_mean_field_variational(layer_sizes, n_particles):         # bnn_vi.py:38-50
        bn = fw.BayesianNet()
        for i, (n_in, n_out) in enumerate(zip(layer_sizes[:-1], layer_sizes[1:])):
            w_mean = tf.get_variable("w_mean_" + str(i), shape=[n_out, n_in + 1],
                                     initializer=tf.constant_initializer(0.))
            w_logstd = tf.get_variable("w_logstd_" + str(i), shape=[n_out, n_in + 1],
                                       initializer=tf.constant_initializer(0.))
            bn.normal("w" + str(i), w_mean, logstd=w_logstd, n_samples=n_particles,
                      group_ndims=2)
        return bn

    x_np = rng.standard_normal((B, sizes[0])).astype(np.float32)
    y_np = rng.standard_normal(B).astype(np.float32)
    xt_np = rng.standard_normal((B_TEST, sizes[0])).astype(np.float32)
    yt_np = rng.standard_normal(B_TEST).astype(np.float32)
    model = build_bnn(tf.constant(x_np), sizes, K)
    variational = build_mean_field_variational(sizes, K)
    log_joint = _log_joint(tf, names, n_train)                         # bnn_vi.py:83-86
    model.log_joint = log_joint
    lower_bound = var.elbo(model, {'y': tf.constant(y_np)}, variational=variational, axis=0)
    cost = lower_bound.sgvb()
    lb_tensor = lower_bound.tensor
    _ = lower_bound.bn
    all_vars = tf.trainable_variables()
    vnames = [v.name.split("/")[-1].split(":")[0] for v in all_vars]
    out = dict(x=x_np, y=y_np, x_test=xt_np, y_test=yt_np, n_train=np.int32(n_train),
               std_y_train=np.float32(STD_Y_TRAIN), sizes=np.int32(sizes))
    for n, v in zip(vnames, all_vars):
        shape = np.shape(v.value)
        if n.startswith("w_mean"):
            val = rng.uniform(-1.0, 1.0, shape)
        elif n.startswith("w_logstd"):
            val = rng.uniform(-2.0, -0.5, shape)
        else:
            val = -0.3
        val = np.asarray(val, np.float32)
        v.load(val)
        out["var_" + n] = val
    shapes = [(sizes[i + 1], sizes[i] + 1) for i in range(L)]
    eps = [rng.standard_normal((K,) + s).astype(np.float32) for s in shapes]
    out.update({"eps%d" % i: e for i, e in enumerate(eps)})
    sess = tf.Session()
    tf.set_noise(normal=list(eps))
    r = sess.run([lb_tensor, cost] + tf.gradients(cost, all_vars))
    assert not tf._NOISE["normal"]
    out.update(lower_bound=np.asarray(r[0], np.float32), cost=np.asarray(r[1], np.float32))
    for n, gr in zip(vnames, r[2:]):
        out["grad_" + n] = np.asarray(gr, np.float32)

    # ---- prediction: rmse & log likelihood (bnn_vi.py:98-103) at ll_samples particles
    xt, yt = tf.constant(xt_np), tf.constant(yt_np)
    model_t = build_bnn(xt, sizes, K_LL)
    model_t.log_joint = log_joint
    lb_t = var.elbo(model_t, {'y': yt}, variational=build_mean_field_variational(sizes, K_LL),
                    axis=0)
    y_mean = lb_t.bn["y_mean"]
    rmse = tf.sqrt(tf.reduce_mean((tf.reduce_mean(y_mean, 0) - yt) ** 2)) * STD_Y_TRAIN
    log_py_xw = lb_t.bn.cond_log_prob("y")
    log_likelihood = tf.reduce_mean(utils.log_mean_exp(log_py_xw, 0)) - tf.log(STD_Y_TRAIN)
    _ = lb_t.tensor
    for v in tf.trainable_variables()[len(all_vars):]:
        v.load(out["var_" + v.name.split("/")[-1].split(":")[0]])
    eps_ll = [rng.standard_normal((K_LL,) + s).astype(np.float32) for s in shapes]
    out.update({"eps_ll%d" % i: e for i, e in enumerate(eps_ll)})
    # y_mean evaluates the einsum's weight before its input: the last layer's draw first
    tf.set_noise(normal=eps_ll[::-1])
    r = sess.run([y_mean, log_py_xw, rmse, log_likelihood])
    assert not tf._NOISE["normal"]
    out.update(ll_y_mean=np.asarray(r[0], np.float32), ll_log_py_xw=np.asarray(r[1], np.float32),
               ll_rmse=np.float32(r[2]), ll_log_likelihood=np.float32(r[3]))
    return out


def run_reference_bnn_deep(seed=919):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = {}
    for net in NETS:
        out.update({net + "/" + k: v for k, v in run_sgmcmc(net, rng).items()})
        out.update({net + "/vi/" + k: v for k, v in run_vi(net, rng).items()})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_bnn_deep()
    np.savez_compressed(os.path.join(HERE, "ref_bnn_deep.npz"), **out)
    with open(os.path.join(HERE, "ref_bnn_deep_digests.json"), "w") as f:
        json.dump(digests("ref_bnn_deep", out), f, indent=1, sort_keys=True)
        f.write("\n")
    for net in NETS:
        print(net, "lower bound %.6g" % out[net + "/vi/lower_bound"],
              {tag: out["%s/%s/n_used" % (net, tag)].tolist() for tag in CONFIGS})


if __name__ == "__main__":
    main()
