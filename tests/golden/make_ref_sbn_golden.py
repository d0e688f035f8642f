"""tests/golden/ref_sbn.npz: the sigmoid belief nets of examples/sigmoid_belief_nets/sbn_vimco.py
and sbn_adaptive_is.py on THE REFERENCE'S OWN BayesianNet, Bernoulli, importance_weighted_objective
(.vimco()) and klpq (.importance()), executed on the NumPy TensorFlow stand-in of oracle/tf_shim
(TEST INFRASTRUCTURE).

    python tests/golden/make_ref_sbn_golden.py  ->  ref_sbn.npz, ref_sbn_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  The nets are build_sbn / build_q_net of
sbn_vimco.py:19-44 (build_proposal of sbn_adaptive_is.py is the same net under another scope) at
x_dim = 50, h_dim = 20, N = 6 rows and K = 5 particles.  Every tf.layers.dense kernel and bias is
loaded with non-zero random values.  The uniforms of the three proposal draws are injected; any u
within 1e-3 of sigmoid(l), with l the float64 logits computed layer by layer on the drawn samples, is
re-drawn, so no float32 path can flip a sample.

Recorded (kernels stored as W = kernel^T, [units, fan_in], the layout of zs.fused.LinearBernoulli):
  sbn_vimco.py:        the per-datum IW bound, the vimco() cost (reduce_mean) and tf.gradients of
                       that cost w.r.t. all 12 variables;
  sbn_adaptive_is.py:  tf.gradients of -mean(IW bound) w.r.t. the 6 model variables, the
                       klpq(...).importance() cost (reduce_mean) and its gradients w.r.t. the 6
                       proposal variables.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

X_DIM, H_DIM, N, K = 50, 20, 6, 5
Q_NAMES = ["q_h1", "q_h2", "q_h3"]          # proposal layers: x -> h1 -> h2 -> h3
M_NAMES = ["m_h2", "m_h1", "m_x"]           # model layers: h3 -> h2 -> h1 -> x


def _sigmoid64(l):
    return 1.0 / (1.0 + np.exp(-l))


def _draw(rng, logits64, shape):
    """Uniforms of one Bernoulli draw, none within 1e-3 of sigmoid(l)."""
    p = _sigmoid64(np.broadcast_to(logits64, shape))
    u = rng.random(shape)
    bad = np.abs(u - p) < 1e-3
    while bad.any():
        u[bad] = rng.random(int(bad.sum()))
        bad = np.abs(u - p) < 1e-3
    return u.astype(np.float32)


def run_reference_sbn(seed=2024):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)

    @fw.meta_bayesian_net(scope="sbn", reuse_variables=True)
    def build_sbn(n, x_dim, h_dim, n_particles):                  # sbn_vimco.py:19-31
        bn = fw.BayesianNet()
        h3_logits = tf.zeros([n, h_dim])
        h3 = bn.bernoulli("h3", h3_logits, group_ndims=1, n_samples=n_particles,
                          dtype=tf.float32)
        h2_logits = tf.layers.dense(h3, h_dim)
        h2 = bn.bernoulli("h2", h2_logits, group_ndims=1, dtype=tf.float32)
        h1_logits = tf.layers.dense(h2, h_dim)
        h1 = bn.bernoulli("h1", h1_logits, group_ndims=1, dtype=tf.float32)
        x_logits = tf.layers.dense(h1, x_dim)
        bn.bernoulli("x", x_logits, group_ndims=1)
        return bn

    @fw.reuse_variables(scope="q_net")
    def build_q_net(x, h_dim, n_particles):                         # sbn_vimco.py:34-44
        bn = fw.BayesianNet()
        h1_logits = tf.layers.dense(tf.cast(x, tf.float32), h_dim)
        h1 = bn.bernoulli("h1", h1_logits, group_ndims=1,
                          n_samples=n_particles, dtype=tf.float32)
        h2_logits = tf.layers.dense(h1, h_dim)
        h2 = bn.bernoulli("h2", h2_logits, group_ndims=1, dtype=tf.float32)
        h3_logits = tf.layers.dense(h2, h_dim)
        bn.bernoulli("h3", h3_logits, group_ndims=1, dtype=tf.float32)
        return bn

    x_np = (rng.random((N, X_DIM)) < 0.3).astype(np.int32)
    x = tf.constant(x_np)
    model = build_sbn(N, X_DIM, H_DIM, K)
    variational = build_q_net(x, H_DIM, K)
    q_vars = tf.trainable_variables()                 # the q-net layers, built first
    lower_bound = var.importance_weighted_objective(model, observed={"x": x},
                                                    variational=variational, axis=0)
    vimco_cost = tf.reduce_mean(lower_bound.vimco())               # sbn_vimco.py:72-75
    lb_tensor = lower_bound.tensor
    _ = lower_bound.bn                                # builds the model's layers
    all_vars = tf.trainable_variables()
    m_vars = all_vars[len(q_vars):]
    assert len(q_vars) == 6 and len(m_vars) == 6, (len(q_vars), len(m_vars))
    # sbn_adaptive_is.py:70-83 on the same nets
    iw_mean = tf.reduce_mean(lb_tensor)
    klpq_cost = tf.reduce_mean(var.klpq(model, observed={"x": x}, variational=variational,
                                        axis=0).importance())

    out = dict(x=x_np)
    layers64 = {}
    for names, vs in ((Q_NAMES, q_vars), (M_NAMES, m_vars)):
        for i, name in enumerate(names):
            kern, bias = vs[2 * i], vs[2 * i + 1]
            fan_in, units = np.shape(kern.value)
            kv = (rng.standard_normal((fan_in, units)) * 1.5 / np.sqrt(fan_in)).astype(np.float32)
            bv = (0.5 * rng.standard_normal(units)).astype(np.float32)
            kern.load(kv)
            bias.load(bv)
            out["W_" + name] = np.ascontiguousarray(kv.T)
            out["b_" + name] = bv
            layers64[name] = (kv.astype(np.float64), bv.astype(np.float64))

    # uniforms of the proposal's draws, chosen on float64 logits layer by layer
    def dense64(h, name):
        kv, bv = layers64[name]
        return h.astype(np.float64) @ kv + bv
    l1 = dense64(x_np, "q_h1")
    u1 = _draw(rng, l1, (K, N, H_DIM))
    h1 = (u1 < _sigmoid64(l1)).astype(np.float32)
    l2 = dense64(h1, "q_h2")
    u2 = _draw(rng, l2, (1, K, N, H_DIM))
    h2 = (u2[0] < _sigmoid64(l2)).astype(np.float32)
    l3 = dense64(h2, "q_h3")
    u3 = _draw(rng, l3, (1, K, N, H_DIM))
    h3 = (u3[0] < _sigmoid64(l3)).astype(np.float32)
    out.update(u_h1=u1, u_h2=u2, u_h3=u3, h1=h1, h2=h2, h3=h3)

    sess = tf.Session()
    qh = [variational.get(n).tensor for n in ("h1", "h2", "h3")]

    def run(fetches):
        """Session.run with the three injected draws.  The stand-in hands uniforms out in the
        order its random ops execute, which follows the graph's evaluation order, so each order
        is tried and the one whose samples reproduce h1, h2, h3 is kept."""
        import itertools
        for order in itertools.permutations((u1, u2, u3)):
            tf.set_noise(uniform=list(order))
            try:
                r = sess.run(list(fetches) + qh)
            except AssertionError:                     # a draw of the wrong shape
                continue
            if not tf._NOISE["uniform"] and all(
                    np.array_equal(np.asarray(g, np.float32), w)
                    for g, w in zip(r[-3:], (h1, h2, h3))):
                return r[:-3]
        raise RuntimeError("no order of the injected draws reproduces the samples")

    r = run([lb_tensor, vimco_cost] + tf.gradients(vimco_cost, all_vars))
    out.update(iw_bound=np.asarray(r[0], np.float32), vimco_cost=np.float32(r[1]))
    for name, g in zip(Q_NAMES + M_NAMES, zip(r[2::2], r[3::2])):
        out["vimco_grad_W_" + name] = np.ascontiguousarray(np.asarray(g[0], np.float32).T)
        out["vimco_grad_b_" + name] = np.asarray(g[1], np.float32)

    r = run([klpq_cost] + tf.gradients(-iw_mean, m_vars) + tf.gradients(klpq_cost, q_vars))
    out["rws_klpq_cost"] = np.float32(r[0])
    gm, gq = r[1:7], r[7:13]
    for name, g in zip(M_NAMES, zip(gm[0::2], gm[1::2])):
        out["rws_grad_W_" + name] = np.ascontiguousarray(np.asarray(g[0], np.float32).T)
        out["rws_grad_b_" + name] = np.asarray(g[1], np.float32)
    for name, g in zip(Q_NAMES, zip(gq[0::2], gq[1::2])):
        out["rws_grad_W_" + name] = np.ascontiguousarray(np.asarray(g[0], np.float32).T)
        out["rws_grad_b_" + name] = np.asarray(g[1], np.float32)
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_sbn()
    np.savez_compressed(os.path.join(HERE, "ref_sbn.npz"), **out)
    with open(os.path.join(HERE, "ref_sbn_digests.json"), "w") as f:
        json.dump(digests("ref_sbn", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("mean IW bound %.6g, vimco cost %.6g, klpq cost %.6g"
          % (out["iw_bound"].mean(), out["vimco_cost"], out["rws_klpq_cost"]))


if __name__ == "__main__":
    main()
