"""tests/golden/ref_nf.npz: the reference's own planar_normalizing_flow (zhusuan/transform.py), alone
and inside the normalizing-flow VAE of examples/normalizing_flows/vae_nf.py on THE REFERENCE'S OWN
BayesianNet, Normal, Bernoulli, elbo() and is_loglikelihood, executed on the NumPy TensorFlow
stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_nf_golden.py  ->  ref_nf.npz, ref_nf_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  Every draw is injected with tf.set_noise: the flow
parameters' initialisers (tf.random_normal(stddev=0.005), fed values whose product with 0.005 has
std 0.5 on a grid of 2^-9, so the flows are far from the identity), q's eps and the uniforms that
binarise x.  The dense layers are the stand-in's Glorot-uniform draws; their biases and every flow's
param_b are then loaded with non-zero values on a grid of 2^-9.

The stand-in lacks three things transform.py uses; they are installed onto it here with TF 1.x
semantics, so the stand-in itself is unchanged for every other fixture:
  * tf.tanh, with its gradient;
  * tf.assert_equal;
  * the gradient of tf.matmul with transpose_a / transpose_b (u = aux_u + w / (w^T w) ...).
tf.Variable is wrapped to record the variables transform.py creates, in creation order.

Recorded:
  flow/*: the standalone flow, d = 7, n_iters = 4, samples [3, 5, 7], log_probs [3, 5]; outputs z
    and log_q, and tf.gradients of sum(z * cz) + sum(log_q * cl) w.r.t. samples, log_probs and
    every param_b ([4]), aux_u and para_w ([4, 7], row k = flow k).
  vae/*: vae_nf.py at x_dim 30, hidden 20, z_dim 6, two calls of 3 flows; 2 particles over 5 rows
    for the bound, cost and the gradient of the cost w.r.t. every variable; the IS estimate at 4
    particles.  Dense weights are stored [out, in] (the kernel transposed); flow parameters of call
    c as f{c}_b [3], f{c}_aux_u and f{c}_w [3, 6].  x_* are the binarised inputs each run drew.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

X_DIM, H, Z_DIM, N_FLOWS, N, S, S_IS = 30, 20, 6, 3, 5, 2, 4


def _install_ops(tf):
    created = []
    base_variable = tf.Variable

    class Variable(base_variable):
        def __init__(self, *a, **k):
            base_variable.__init__(self, *a, **k)
            created.append(self)

    def tanh(a, name=None):
        a = tf.convert_to_tensor(a)
        out = tf._unary(lambda x: np.tanh(x).astype(np.asarray(x).dtype, copy=False), a, "tanh")
        out.vjp = lambda g: [g * (1.0 - out * out)]
        return out

    def assert_equal(x, y, message=None, data=None, summarize=None, name=None):
        return tf._assert(lambda xv, yv: np.array_equal(xv, np.asarray(yv)), "equal")(
            x, y, message=message)

    base_matmul = tf.matmul

    def matmul(a, b, transpose_a=False, transpose_b=False, name=None):
        a, b = tf.convert_to_tensor(a), tf.convert_to_tensor(b)
        out = base_matmul(a, b, transpose_a=transpose_a, transpose_b=transpose_b)
        if transpose_a or transpose_b:
            sw = lambda x: np.swapaxes(x, -1, -2)                       # noqa: E731

            def vjp(g):
                def da(c):                 # d op(a) = g op(b)^T
                    gv, bv = np.asarray(c.eval(g)), np.asarray(c.eval(b))
                    r = np.matmul(gv, sw(sw(bv) if transpose_b else bv))
                    return sw(r) if transpose_a else r

                def db(c):                 # d op(b) = op(a)^T g
                    gv, av = np.asarray(c.eval(g)), np.asarray(c.eval(a))
                    r = np.matmul(sw(sw(av) if transpose_a else av), gv)
                    return sw(r) if transpose_b else r
                return [tf.Tensor(da, inputs=(g, a, b), op="matmul_da", dtype=a._dtype),
                        tf.Tensor(db, inputs=(g, a, b), op="matmul_db", dtype=b._dtype)]
            out.vjp = vjp
        return out

    tf.Variable, tf.tanh, tf.assert_equal, tf.matmul = Variable, tanh, assert_equal, matmul
    return created


def _grid(rng, shape, std):
    v = np.round(std * rng.standard_normal(shape) * 512) / 512
    v[v == 0] = 1.0 / 512
    return v.astype(np.float32)


def _init_draws(rng, n, d):
    """Noise for n flows' initialisers (aux_u then para_w, [d, 1] each), scaled by 1 / 0.005."""
    return [(_grid(rng, (d, 1), 0.5) / np.float32(0.005)).astype(np.float32)
            for _ in range(2 * n)]


def _flow_params(tf, created, n, rng):
    """Load param_b and return the stacked (b, aux_u, w) values of the flows in `created`."""
    assert len(created) == 3 * n, len(created)
    bs, us, ws = created[0::3], created[1::3], created[2::3]
    for v in bs:
        v.load(_grid(rng, (1,), 0.5))
    return (np.concatenate([v.value for v in bs]).astype(np.float32),
            np.stack([v.value[:, 0] for v in us]).astype(np.float32),
            np.stack([v.value[:, 0] for v in ws]).astype(np.float32)), bs, us, ws


def run_reference_nf(seed=4141):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    created = _install_ops(tf)
    tr = importlib.import_module("zhusuan.transform")
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    ev = importlib.import_module("zhusuan.evaluation")
    rng = np.random.Generator(np.random.PCG64(seed))
    out = {}

    # ---- the standalone flow ------------------------------------------------------------------
    tf.reset_default_graph()
    d, n = 7, 4
    z0 = _grid(rng, (3, 5, d), 1.0)
    lq0 = _grid(rng, (3, 5), 2.0)
    cz, cl = _grid(rng, (3, 5, d), 1.0), _grid(rng, (3, 5), 1.0)
    samples, log_probs = tf.constant(z0), tf.constant(lq0)
    tf.set_noise(normal=_init_draws(rng, n, d))
    z, lq = tr.planar_normalizing_flow(samples, log_probs, n_iters=n)
    assert not tf._NOISE["normal"]
    (b, u, w), bs, us, ws = _flow_params(tf, created, n, rng)
    f = tf.reduce_sum(z * tf.constant(cz)) + tf.reduce_sum(lq * tf.constant(cl))
    grads = tf.gradients(f, [samples, log_probs] + bs + us + ws)
    r = tf.Session().run([z, lq] + grads)
    out.update({"flow/samples": z0, "flow/log_probs": lq0, "flow/cz": cz, "flow/cl": cl,
                "flow/b": b, "flow/aux_u": u, "flow/w": w,
                "flow/z": np.asarray(r[0], np.float32), "flow/log_q": np.asarray(r[1], np.float32),
                "flow/grad_samples": np.asarray(r[2], np.float32),
                "flow/grad_log_probs": np.asarray(r[3], np.float32),
                "flow/grad_b": np.concatenate([np.asarray(g, np.float32) for g in r[4:4 + n]]),
                "flow/grad_aux_u": np.stack([np.asarray(g, np.float32)[:, 0]
                                             for g in r[4 + n:4 + 2 * n]]),
                "flow/grad_w": np.stack([np.asarray(g, np.float32)[:, 0]
                                         for g in r[4 + 2 * n:4 + 3 * n]])})

    # ---- vae_nf.py at small widths ------------------------------------------------------------
    del created[:]
    tf.reset_default_graph()
    tf.set_init_rng(rng)

    @fw.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, x_dim, z_dim, n_particles):                     # vae_nf.py:19-28
        bn = fw.BayesianNet()
        z_mean = tf.zeros([n, z_dim])
        z = bn.normal("z", z_mean, std=1., group_ndims=1, n_samples=n_particles)
        h = tf.layers.dense(z, H, activation=tf.nn.relu)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        x_logits = tf.layers.dense(h, x_dim)
        bn.bernoulli("x", x_logits, group_ndims=1)
        return bn

    @fw.reuse_variables(scope="q_net")
    def build_q_net(x, z_dim, n_particles):                          # vae_nf.py:31-40
        bn = fw.BayesianNet()
        h = tf.layers.dense(tf.cast(x, tf.float32), H, activation=tf.nn.relu)
        h = tf.layers.dense(h, H, activation=tf.nn.relu)
        z_mean = tf.layers.dense(h, z_dim)
        z_logstd = tf.layers.dense(h, z_dim)
        bn.normal("z", z_mean, logstd=z_logstd, group_ndims=1, n_samples=n_particles)
        return bn

    x_input_np = rng.random((N, X_DIM)).astype(np.float32)
    n_particles = tf.placeholder(np.int32, shape=[], name="n_particles")   # vae_nf.py:60-71
    x_input = tf.constant(x_input_np)
    x = tf.cast(tf.less(tf.random_uniform(tf.shape(x_input)), x_input), np.int32)
    model = build_gen(N, X_DIM, Z_DIM, n_particles)
    q_net = build_q_net(x, Z_DIM, n_particles)
    qz_samples, log_qz = q_net.query('z', outputs=True, local_log_prob=True)
    tf.set_noise(normal=_init_draws(rng, 2 * N_FLOWS, Z_DIM))
    n0 = len(created)                                   # the q-net's dense variables
    qz_samples, log_qz = tr.planar_normalizing_flow(qz_samples, log_qz, n_iters=N_FLOWS)
    flows1 = created[n0:]
    qz_samples, log_qz = tr.planar_normalizing_flow(qz_samples, log_qz, n_iters=N_FLOWS)
    flows2 = created[n0 + len(flows1):]
    assert not tf._NOISE["normal"]
    lower_bound = var.elbo(model, observed={"x": x}, latent={"z": [qz_samples, log_qz]}, axis=0)
    cost = tf.reduce_mean(lower_bound.sgvb())
    lower_bound = tf.reduce_mean(lower_bound)
    is_log_likelihood = tf.reduce_mean(
        ev.is_loglikelihood(model, {'x': x}, {'z': [qz_samples, log_qz]}, axis=0))

    dense = tf.trainable_variables()
    names = ["q%d" % i for i in range(4)] + ["p%d" % i for i in range(3)]
    assert [v.value.shape for v in dense] == [
        (X_DIM, H), (H,), (H, H), (H,), (H, Z_DIM), (Z_DIM,), (H, Z_DIM), (Z_DIM,),
        (Z_DIM, H), (H,), (H, H), (H,), (H, X_DIM), (X_DIM,)], [v.value.shape for v in dense]
    for i, nm in enumerate(names):
        kern, bias = dense[2 * i], dense[2 * i + 1]
        bias.load(_grid(rng, bias.value.shape, 0.3))
        out["vae/%s_W" % nm] = np.ascontiguousarray(kern.value.T)
        out["vae/%s_b" % nm] = np.array(bias.value)
    flow_vars = []
    for c, fl in enumerate((flows1, flows2)):
        (b, u, w), bs, us, ws = _flow_params(tf, fl, N_FLOWS, rng)
        out.update({"vae/f%d_b" % c: b, "vae/f%d_aux_u" % c: u, "vae/f%d_w" % c: w})
        flow_vars.append((bs, us, ws))
    out["vae/x_input"] = x_input_np
    sess = tf.Session()

    def run(fetches, n_part):
        eps = rng.standard_normal((n_part, N, Z_DIM)).astype(np.float32)
        ub = rng.random((N, X_DIM)).astype(np.float32)
        tf.set_noise(normal=[eps], uniform=[ub])
        r = sess.run([x] + fetches, feed_dict={n_particles: n_part})
        assert not tf._NOISE["normal"] and not tf._NOISE["uniform"]
        return r[1:], eps, np.asarray(r[0], np.int32)

    wrt = dense + [v for bs, us, ws in flow_vars for v in bs + us + ws]
    r, eps, xb = run([lower_bound, cost] + tf.gradients(cost, wrt), S)
    out.update({"vae/eps": eps, "vae/x": xb, "vae/bound": np.float32(r[0]),
                "vae/cost": np.float32(r[1])})
    g = r[2:]
    for i, nm in enumerate(names):
        out["vae/grad_%s_W" % nm] = np.ascontiguousarray(np.asarray(g[2 * i], np.float32).T)
        out["vae/grad_%s_b" % nm] = np.asarray(g[2 * i + 1], np.float32)
    g = g[len(dense):]
    for c in range(2):
        gc, g = g[:3 * N_FLOWS], g[3 * N_FLOWS:]
        out["vae/grad_f%d_b" % c] = np.concatenate([np.asarray(t, np.float32)
                                                    for t in gc[:N_FLOWS]])
        out["vae/grad_f%d_aux_u" % c] = np.stack([np.asarray(t, np.float32)[:, 0]
                                                  for t in gc[N_FLOWS:2 * N_FLOWS]])
        out["vae/grad_f%d_w" % c] = np.stack([np.asarray(t, np.float32)[:, 0]
                                              for t in gc[2 * N_FLOWS:]])
    r, eps, xb = run([is_log_likelihood], S_IS)
    out.update({"vae/is_eps": eps, "vae/is_x": xb, "vae/is_ll": np.float32(r[0])})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_nf()
    np.savez_compressed(os.path.join(HERE, "ref_nf.npz"), **out)
    with open(os.path.join(HERE, "ref_nf_digests.json"), "w") as f:
        json.dump(digests("ref_nf", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("flow log_q[0, :3] %s; vae bound %.6g, cost %.6g, IS %.6g"
          % (out["flow/log_q"][0, :3], out["vae/bound"], out["vae/cost"], out["vae/is_ll"]))


if __name__ == "__main__":
    main()
