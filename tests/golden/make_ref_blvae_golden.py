"""tests/golden/ref_blvae.npz: one training step and one evaluation of the Bernoulli-latent VAE of
examples/variational_autoencoders/bernoulli_latent_vae.py on THE REFERENCE'S OWN BayesianNet,
Bernoulli, elbo().reinforce(baseline=cx) and is_loglikelihood, executed on the NumPy TensorFlow
stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_blvae_golden.py  ->  ref_blvae.npz, ref_blvae_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  build_gen, build_q_net and baseline_net are
bernoulli_latent_vae.py:18-55 restated line for line at widths x_dim 30, hidden 20 (500 in the
example), z_dim 6 and a baseline hidden width of 8 (100), with S = 3 particles over n = 5 rows in
training and S = 4 in evaluation.  Every weight, bias, gamma and beta is loaded with non-zero
values on a grid of 2^-9; the data x_input sits on that grid in [0, 1].  The uniforms of the
dynamic binarisation (:72-73) and of the z draws are injected.

The stand-in lacks tf.layers.batch_normalization; it is installed onto it here with the semantics
of TF 1.x's non-fused path (the only one for inputs that are not 4-D), so the stand-in itself is
unchanged for every other fixture: center=True (beta, zeros), scale=True (gamma, ones),
momentum=0.99, epsilon=1e-3, moving_mean zeros and moving_variance ones.  Training: tf.nn.moments
over every axis but the last (population variance, the mean under stop_gradient in the variance);
the update op moves each moving statistic by m -= (m - batch) * (1 - momentum), no zero-debiasing.
Evaluation: the moving statistics.  Output: tf.nn.batch_normalization's form x * inv + (beta -
mean * inv) with inv = gamma / sqrt(var + eps).

The reference builds the decoder twice per step (for the bound and for the unfetched
is_loglikelihood, :89-90), and TF runs the update ops of both builds (:93-95).  The fixture records
the moving statistics after ONE update per layer, from the training graph's own build: the
semantics zs.fused.bn_linear implements (one update per training call of a layer).

Recorded (W stored as the kernel transposed, [n_out, n_in], the layout of zs.fused; names
q0, q1 (encoder batch-norm layers), qz (z logits), p0, p1 (decoder batch-norm layers), px (x
logits), c0, c1 (baseline net)):
  x_input, u_x (binarisation uniforms), x (the binarised data), u_z [S, n, z_dim];
  W_*, b_* (the dense biases of qz, px, c0, c1), gamma_* and beta_* (q0, q1, p0, p1);
  bound (tf.reduce_mean(lower_bound)), cost (tf.reduce_mean(cost + baseline_cost)),
  baseline_cost [n], z [S, n, z_dim], grad_* of every variable (tf.gradients(cost)),
  rf_moving_mean (REINFORCE's moving_mean after the step, zero-debiased from 0), and
  moving_mean_* / moving_variance_* after the step;
  eval_u_z [S_EVAL, n, z_dim], eval_z, eval_bound and eval_is_ll: is_training=False on those
  moving statistics, the same x.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

X_DIM, H_DIM, Z_DIM, C_DIM = 30, 20, 6, 8
S, S_EVAL, N = 3, 4, 5
MOMENTUM, EPS = 0.99, 1e-3
BN_NAMES = {"q_net": ("q0", "q1"), "gen": ("p0", "p1")}
DENSE_NAMES = {"q_net": ("q0", "q1", "qz"), "gen": ("p0", "p1", "px"), "baseline": ("c0", "c1")}


def _install_ops(tf):
    """tf.layers.batch_normalization (non-fused) on the stand-in; returns the registries of the
    dense and batch-norm variables per variable store, and the list of update values."""
    dense_vars, bn_vars, updates = {}, {}, []
    base_dense = tf.layers.dense

    def store():
        return tf._TEMPLATES[-1] if tf._TEMPLATES else tf._DEFAULT_STORE

    def dense(inputs, units, *a, **k):
        s = store()
        key = "dense" if s["count"] == 0 else "dense_%d" % s["count"]
        new = key not in s["vars"]
        y = base_dense(inputs, units, *a, **k)
        if new:
            dense_vars.setdefault(id(s), []).append(s["vars"][key])
        return y

    def batch_normalization(inputs, axis=-1, momentum=0.99, epsilon=1e-3, center=True,
                            scale=True, training=False, **kw):
        assert center and scale and axis == -1
        s = store()
        x = tf.convert_to_tensor(inputs)
        J = int(x.get_shape().as_list()[-1])
        key = "bn:after_dense_%d" % s["count"]         # the dense layer it follows
        if key not in s["vars"]:
            gamma = tf.Variable(np.ones(J, np.float32), name="gamma")
            beta = tf.Variable(np.zeros(J, np.float32), name="beta")
            mm = tf.Variable(np.zeros(J, np.float32), name="moving_mean", trainable=False)
            mv = tf.Variable(np.ones(J, np.float32), name="moving_variance", trainable=False)
            tf._TRAINABLE.extend([gamma, beta])
            s["vars"][key] = (gamma, beta, mm, mv)
            bn_vars.setdefault(id(s), []).append(s["vars"][key])
        gamma, beta, mm, mv = s["vars"][key]
        if training:
            axes = list(range(len(x.get_shape().as_list()) - 1))
            mean = tf.reduce_mean(x, axes, keepdims=True)
            var = tf.reduce_mean(tf.square(x - tf.stop_gradient(mean)), axes, keepdims=True)
            mean, var = tf.reshape(mean, [J]), tf.reshape(var, [J])
            d = np.float32(1.0 - momentum)
            updates.append((id(s), mm, mm - (mm - mean) * d, mv, mv - (mv - var) * d))
        else:
            mean, var = mm, mv
        inv = gamma / tf.sqrt(var + np.float32(epsilon))
        return x * inv + (beta - mean * inv)

    tf.layers.dense = staticmethod(dense)
    tf.layers.batch_normalization = staticmethod(batch_normalization)
    return dense_vars, bn_vars, updates


def _grid(rng, shape, scale, shift=0.0):
    v = np.round((rng.standard_normal(shape) * scale + shift) * 512) / 512
    v[v == 0] = 1.0 / 512
    return v.astype(np.float32)


def run_reference_blvae(seed=4242):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    dense_vars, bn_vars, updates = _install_ops(tf)
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    ev = importlib.import_module("zhusuan.evaluation")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)

    @fw.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, x_dim, z_dim, n_particles, is_training):          # :18-33
        bn = fw.BayesianNet()
        z_logits = tf.zeros([n, z_dim])
        z = bn.bernoulli("z", z_logits, group_ndims=1, n_samples=n_particles,
                         dtype=tf.float32)
        h = tf.layers.dense(z, H_DIM, use_bias=False)
        h = tf.layers.batch_normalization(h, training=is_training)
        h = tf.nn.relu(h)
        h = tf.layers.dense(h, H_DIM, use_bias=False)
        h = tf.layers.batch_normalization(h, training=is_training)
        h = tf.nn.relu(h)
        x_logits = tf.layers.dense(h, x_dim)
        bn.bernoulli("x", x_logits, group_ndims=1)
        return bn

    @fw.reuse_variables(scope="q_net")
    def build_q_net(x, z_dim, n_particles, is_training):                # :36-48
        bn = fw.BayesianNet()
        h = tf.layers.dense(tf.cast(x, tf.float32), H_DIM, use_bias=False)
        h = tf.layers.batch_normalization(h, training=is_training)
        h = tf.nn.relu(h)
        h = tf.layers.dense(h, H_DIM, use_bias=False)
        h = tf.layers.batch_normalization(h, training=is_training)
        h = tf.nn.relu(h)
        z_logits = tf.layers.dense(h, z_dim)
        bn.bernoulli("z", z_logits, group_ndims=1, n_samples=n_particles,
                     dtype=tf.float32)
        return bn

    def baseline_net(x):                                                # :51-55
        lc_x = tf.layers.dense(tf.cast(x, tf.float32), C_DIM, activation=tf.nn.relu)
        lc_x = tf.layers.dense(lc_x, 1)
        lc_x = tf.squeeze(lc_x, -1)
        return lc_x

    x_input_np = (np.round(rng.random((N, X_DIM)) ** 2 * 512) / 512).astype(np.float32)
    u_x = rng.random((N, X_DIM)).astype(np.float32)

    def graph(n_particles, is_training):                                # :70-90
        del updates[:]
        x_input = tf.constant(x_input_np)
        x = tf.cast(tf.less(tf.random_uniform(tf.shape(x_input)), x_input), tf.int32)
        model = build_gen(N, X_DIM, Z_DIM, n_particles, is_training)
        variational = build_q_net(x, Z_DIM, n_particles, is_training)
        out = dict(x=x, z=variational["z"].tensor)
        lower_bound = var.elbo(model, {"x": x}, variational=variational, axis=0)
        if is_training:
            cx = tf.expand_dims(baseline_net(x), 0)
            cost, baseline_cost = lower_bound.reinforce(baseline=cx)
            out.update(cost=tf.reduce_mean(cost + baseline_cost), baseline_cost=baseline_cost)
        out["bound"] = tf.reduce_mean(lower_bound)
        if not is_training:
            out["is_ll"] = tf.reduce_mean(
                ev.is_loglikelihood(model, {"x": x}, proposal=variational, axis=0))
        return out

    def stores():
        """id(store) -> role, told apart by the first dense layer's shape."""
        roles = {}
        for sid, vs in dense_vars.items():
            shp = vs[0][0].value.shape
            roles[sid] = {(X_DIM, H_DIM): "q_net", (Z_DIM, H_DIM): "gen",
                          (X_DIM, C_DIM): "baseline"}[shp]
        return roles

    tr = graph(S, True)
    roles = stores()
    # build order: the bound's model and the reinforce graph each touch the generator once
    assert sorted(roles.values()) == ["baseline", "gen", "q_net"], roles
    out = dict(x_input=x_input_np, u_x=u_x)
    params, names = [], []
    for sid, role in sorted(roles.items(), key=lambda kv: kv[1]):
        for nm, (kern, bias) in zip(DENSE_NAMES[role], dense_vars[sid]):
            fan_in, units = kern.value.shape
            wv = _grid(rng, (fan_in, units), 1.0 / np.sqrt(fan_in))
            kern.load(wv)
            out["W_" + nm] = np.ascontiguousarray(wv.T)
            params.append(kern)
            names.append("W_" + nm)
            if nm not in ("q0", "q1", "p0", "p1"):
                bv = _grid(rng, units, 0.3)
                bias.load(bv)
                out["b_" + nm] = bv
                params.append(bias)
                names.append("b_" + nm)
        for nm, (gamma, beta, _, _) in zip(BN_NAMES.get(role, ()), bn_vars.get(sid, [])):
            J = gamma.value.shape[0]
            gv, bv = _grid(rng, J, 0.3, 1.0), _grid(rng, J, 0.3)
            gamma.load(gv)
            beta.load(bv)
            out["gamma_" + nm], out["beta_" + nm] = gv, bv
            params += [gamma, beta]
            names += ["gamma_" + nm, "beta_" + nm]
    # one update per layer: the training graph's first build of each batch-norm layer
    first = {}
    for u in updates:
        first.setdefault(id(u[1]), u)
    assert len(first) == 4, len(first)
    grads = tf.gradients(tr["cost"], params)
    u_z = rng.random((S, N, Z_DIM)).astype(np.float32)
    bn_list = []
    for sid, role in sorted(roles.items(), key=lambda kv: kv[1]):
        for nm, v in zip(BN_NAMES.get(role, ()), bn_vars.get(sid, [])):
            bn_list.append((nm, first[id(v[2])]))
    fetch = [tr["bound"], tr["cost"], tr["baseline_cost"], tr["x"], tr["z"]] + grads + \
        [u[2] for _, u in bn_list] + [u[4] for _, u in bn_list]
    tf.set_noise(uniform=[u_z, u_x])          # evaluation order: the z draw first
    r = tf.Session().run(fetch)
    assert not tf._NOISE["uniform"]
    mm = tf.get_variable("moving_mean")
    out.update(u_z=u_z, bound=np.float32(r[0]), cost=np.float32(r[1]),
               baseline_cost=np.asarray(r[2], np.float32), x=np.asarray(r[3], np.int32),
               z=np.asarray(r[4], np.float32), rf_moving_mean=np.float32(mm.value))
    assert (out["x"] == (u_x < x_input_np)).all()
    g = r[5:5 + len(params)]
    for nm, gv in zip(names, g):
        gv = np.asarray(gv, np.float32)
        out["grad_" + nm] = np.ascontiguousarray(gv.T) if nm.startswith("W_") else gv
    rest = r[5 + len(params):]
    L = len(bn_list)
    for i, (nm, u) in enumerate(bn_list):
        out["moving_mean_" + nm] = np.asarray(rest[i], np.float32)
        out["moving_variance_" + nm] = np.asarray(rest[L + i], np.float32)
        u[1].load(out["moving_mean_" + nm])
        u[3].load(out["moving_variance_" + nm])
    # evaluation on the updated moving statistics.  build_q_net's template is made once and
    # reuses its variables; each call of build_gen makes a MetaBayesianNet with a template of its
    # own, so every value of the training graph's generator is loaded into the new one
    evg = graph(S_EVAL, False)
    gen_old = [sid for sid, role in roles.items() if role == "gen"][0]
    gen_new = [sid for sid in dense_vars if sid not in roles]
    assert len(gen_new) == 1
    for old_v, new_v in zip(dense_vars[gen_old] + bn_vars[gen_old],
                            dense_vars[gen_new[0]] + bn_vars[gen_new[0]]):
        for a, b in zip(old_v, new_v):
            b.load(np.array(a.value))
    eval_u_z = rng.random((S_EVAL, N, Z_DIM)).astype(np.float32)
    tf.set_noise(uniform=[eval_u_z, u_x])
    r = tf.Session().run([evg["bound"], evg["is_ll"], evg["x"], evg["z"]])
    assert not tf._NOISE["uniform"]
    assert (np.asarray(r[2]) == out["x"]).all()
    out.update(eval_u_z=eval_u_z, eval_bound=np.float32(r[0]), eval_is_ll=np.float32(r[1]),
               eval_z=np.asarray(r[3], np.float32))
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_blvae()
    np.savez_compressed(os.path.join(HERE, "ref_blvae.npz"), **out)
    with open(os.path.join(HERE, "ref_blvae_digests.json"), "w") as f:
        json.dump(digests("ref_blvae", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("bound %.6g, cost %.6g, moving mean %.6g, eval bound %.6g, eval IS ll %.6g"
          % (out["bound"], out["cost"], out["rf_moving_mean"], out["eval_bound"],
             out["eval_is_ll"]))


if __name__ == "__main__":
    main()
