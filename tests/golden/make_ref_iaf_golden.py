"""tests/golden/ref_iaf.npz: the reference's own inv_autoregressive_flow with its own linear_ar
(zhusuan/transform.py:17-67, :200-282), executed on the NumPy TensorFlow stand-in of oracle/tf_shim
(TEST INFRASTRUCTURE).

    python tests/golden/make_ref_iaf_golden.py  ->  ref_iaf.npz, ref_iaf_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  The initialisers' draws (tf.random_normal(stddev=0.005)
of m_w and s_w, in creation order) are injected with tf.set_noise, fed values whose product with
0.005 has std 0.4 on a grid of 2^-9, so the flows are far from the identity.

The stand-in lacks two things transform.py uses; they are installed onto it here with TF 1.x
semantics, so the stand-in itself is unchanged for every other fixture:
  * tf.reverse, with its gradient (the reversed upstream gradient);
  * tf.assert_equal.
tf.Variable is wrapped to record the variables linear_ar creates, in creation order.

Recorded, for update in ("normal", "gru") under the key prefix "<update>/": d = 7, n_iters = 3,
samples [3, 5, 7], log_probs [3, 5]; the outputs z and log_q, and tf.gradients of
sum(z * cz) + sum(log_q * cl) w.r.t. samples, log_probs and every m_w and s_w (stacked [3, 7, 7],
row k = flow k; the variables themselves, so zero at i >= j).
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

D, N_FLOWS, LEAD = 7, 3, (3, 5)


def _install_ops(tf):
    created = []
    base_variable = tf.Variable

    class Variable(base_variable):
        def __init__(self, *a, **k):
            base_variable.__init__(self, *a, **k)
            created.append(self)

    def reverse(a, axis, name=None):
        a = tf.convert_to_tensor(a)
        ax = tuple(int(x) for x in axis)
        return tf._unary(lambda x: np.flip(x, ax).copy(), a, "reverse",
                         lambda g: [reverse(g, axis)])

    def assert_equal(x, y, message=None, data=None, summarize=None, name=None):
        return tf._assert(lambda xv, yv: np.array_equal(xv, np.asarray(yv)), "equal")(
            x, y, message=message)

    tf.Variable, tf.reverse, tf.assert_equal = Variable, reverse, assert_equal
    return created


def _grid(rng, shape, std):
    v = np.round(std * rng.standard_normal(shape) * 512) / 512
    v[v == 0] = 1.0 / 512
    return v.astype(np.float32)


def _init_draws(rng, n, d):
    """Noise for n flows' initialisers (m_w then s_w, [d, d] each), scaled by 1 / 0.005."""
    return [(_grid(rng, (d, d), 0.4) / np.float32(0.005)).astype(np.float32)
            for _ in range(2 * n)]


def run_reference_iaf(seed=5151):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    created = _install_ops(tf)
    tr = importlib.import_module("zhusuan.transform")
    rng = np.random.Generator(np.random.PCG64(seed))
    out = {}
    for update in ("normal", "gru"):
        del created[:]
        tf.reset_default_graph()
        z0 = _grid(rng, LEAD + (D,), 1.0)
        lq0 = _grid(rng, LEAD, 2.0)
        cz, cl = _grid(rng, LEAD + (D,), 1.0), _grid(rng, LEAD, 1.0)
        samples, log_probs = tf.constant(z0), tf.constant(lq0)
        tf.set_noise(normal=_init_draws(rng, N_FLOWS, D))
        z, lq = tr.inv_autoregressive_flow(samples, None, log_probs, tr.linear_ar,
                                           n_iters=N_FLOWS, update=update)
        assert len(created) == 2 * N_FLOWS, len(created)
        mws, sws = created[0::2], created[1::2]
        f = tf.reduce_sum(z * tf.constant(cz)) + tf.reduce_sum(lq * tf.constant(cl))
        grads = tf.gradients(f, [samples, log_probs] + mws + sws)
        r = tf.Session().run([z, lq] + grads)
        assert not tf._NOISE["normal"]
        n = N_FLOWS
        p = update + "/"
        out.update({p + "samples": z0, p + "log_probs": lq0, p + "cz": cz, p + "cl": cl,
                    p + "m_w": np.stack([np.asarray(v.value, np.float32) for v in mws]),
                    p + "s_w": np.stack([np.asarray(v.value, np.float32) for v in sws]),
                    p + "z": np.asarray(r[0], np.float32),
                    p + "log_q": np.asarray(r[1], np.float32),
                    p + "grad_samples": np.asarray(r[2], np.float32),
                    p + "grad_log_probs": np.asarray(r[3], np.float32),
                    p + "grad_m_w": np.stack([np.asarray(g, np.float32) for g in r[4:4 + n]]),
                    p + "grad_s_w": np.stack([np.asarray(g, np.float32)
                                              for g in r[4 + n:4 + 2 * n]])})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_iaf()
    np.savez_compressed(os.path.join(HERE, "ref_iaf.npz"), **out)
    with open(os.path.join(HERE, "ref_iaf_digests.json"), "w") as f:
        json.dump(digests("ref_iaf", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("normal log_q[0, :3] %s; gru log_q[0, :3] %s"
          % (out["normal/log_q"][0, :3], out["gru/log_q"][0, :3]))


if __name__ == "__main__":
    main()
