"""tests/golden/ref_concrete.npz: samples, log-densities and their gradients from THE REFERENCE'S
OWN ExpConcrete and Concrete (zhusuan/distributions/multivariate.py:683-958), executed on the NumPy
TensorFlow stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_concrete_golden.py  ->  ref_concrete.npz, ref_concrete_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.

The stand-in lacks tf.reduce_logsumexp and tf.nn.log_softmax; they are installed onto it here,
composed from its own max / exp / sum / log ops (so tf.gradients differentiates them), and the
stand-in itself is unchanged for every other fixture.  The uniforms of _sample come through
tf.set_noise: open_interval_standard_uniform (utils.py:311-324) reads its minval from
dtype.as_numpy_dtype, which the stand-in's dtypes lack, and the stand-in's tf.random_uniform
ignores minval and maxval; so multivariate.py's name for it is bound to the stand-in's
tf.random_uniform(shape, dtype=dtype), which hands out the same injected array.

For each class (prefix exp_ / con_) and each case, with logits [B, C] on a grid of 2^-7, a
temperature t and injected uniforms u [S, B, C] in [0.01, 0.99]:
  <p>logits_<c>, <p>t_<c>, <p>u_<c>;
  <p>sample_<c> [S, B, C]: dist.sample(S);
  <p>lp<g>_<c>: dist.log_prob(sample) at group_ndims g = 0 ([S, B]) and 1 ([S]), the sample axis
    broadcast against the logits;
  <p>dgiven<g>_<c>, <p>dlogits<g>_<c>, <p>dt<g>_<c>: tf.gradients(reduce_sum(lp * w), [given,
    logits, t]) with the weights <p>w<g>_<c> of lp's shape.
Cases: c = 0: B = 4, C = 6, S = 3, t = 0.6; c = 1: B = 2, C = 33, S = 2, t = 1.7.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CASES = [(4, 6, 3, 0.6), (2, 33, 2, 1.7)]


def _install_ops(tf):
    def reduce_logsumexp(a, axis=None, keepdims=False, name=None):
        m = tf.stop_gradient(tf.reduce_max(a, axis, keepdims=True))
        s = tf.log(tf.reduce_sum(tf.exp(a - m), axis, keepdims=True)) + m
        return s if keepdims else tf.reduce_sum(s, axis)

    def log_softmax(logits, axis=-1, name=None):
        return logits - reduce_logsumexp(logits, axis, keepdims=True)

    tf.reduce_logsumexp = reduce_logsumexp
    tf.nn.log_softmax = staticmethod(log_softmax)


def run_reference_concrete(seed=777):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    _install_ops(tf)
    dist = importlib.import_module("zhusuan.distributions.multivariate")
    dist.open_interval_standard_uniform = lambda shape, dtype: tf.random_uniform(shape, dtype=dtype)
    rng = np.random.Generator(np.random.PCG64(seed))
    out = {}
    for c, (B, C, S, tval) in enumerate(CASES):
        logits_np = (np.round(rng.standard_normal((B, C)) * 2 * 128) / 128).astype(np.float32)
        t_np = np.float32(tval)
        for p, cls in (("exp_", dist.ExpConcrete), ("con_", dist.Concrete)):
            u = rng.uniform(0.01, 0.99, (S, B, C)).astype(np.float32)
            tf.reset_default_graph()
            logits = tf.constant(logits_np)
            t = tf.constant(t_np)
            d0 = cls(t, logits, group_ndims=0)
            tf.set_noise(uniform=[u])
            sample = tf.Session().run(d0.sample(S))
            out.update({p + "logits_%d" % c: logits_np, p + "t_%d" % c: t_np,
                        p + "u_%d" % c: u, p + "sample_%d" % c: np.asarray(sample, np.float32)})
            for g in (0, 1):
                d = cls(t, logits, group_ndims=g)
                given = tf.constant(np.asarray(sample, np.float32))
                lp = d.log_prob(given)
                w = rng.standard_normal((S, B) if g == 0 else (S,)).astype(np.float32)
                grads = tf.gradients(tf.reduce_sum(lp * tf.constant(w)), [given, logits, t])
                r = tf.Session().run([lp] + list(grads))
                out.update({p + "lp%d_%d" % (g, c): np.asarray(r[0], np.float32),
                            p + "w%d_%d" % (g, c): w,
                            p + "dgiven%d_%d" % (g, c): np.asarray(r[1], np.float32),
                            p + "dlogits%d_%d" % (g, c): np.asarray(r[2], np.float32),
                            p + "dt%d_%d" % (g, c): np.float32(r[3])})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_concrete()
    np.savez_compressed(os.path.join(HERE, "ref_concrete.npz"), **out)
    with open(os.path.join(HERE, "ref_concrete_digests.json"), "w") as f:
        json.dump(digests("ref_concrete", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("exp lp %s, con lp %s" % (out["exp_lp0_0"][0, :2], out["con_lp0_0"][0, :2]))


if __name__ == "__main__":
    main()
