"""tests/golden/ref_bnn_sgmcmc.npz: config 4's BNN run with THE REFERENCE'S OWN SGLD, PSGLD and SGNHT
(zhusuan/sgmcmc.py:170-257, 374-523) through the NumPy TensorFlow stand-in of oracle/tf_shim
(TEST INFRASTRUCTURE).

    python tests/golden/make_ref_bnn_sgmcmc_golden.py  ->  ref_bnn_sgmcmc.npz,
                                                          ref_bnn_sgmcmc_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  The model, data, prior scales and initial weights
are those of oracle/tf_shim/make_ref_golden.py::run_reference_bnn_sghmc (bnn_sgmcmc.py:19-35 with
its log_joint override 74-77): that function is run up to its sampler's sample() call, where the
reference's model and latent variables are taken over.  Each sampler then runs five steps from the
same initial weights with every draw injected and stored: SGLD, PSGLD, and SGNHT with vector and
scalar thermostat in first and second order, re-drawing v at t = 0 and t = 3.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

_SGNHT = dict(learning_rate=1e-4, variance_extra=0.05, tune_rate=10., n_iter_resample_v=3)
# fixture prefix -> (reference class, constructor keywords)
CONFIGS = {
    "sgld": ("SGLD", dict(learning_rate=1e-4)),
    "psgld": ("PSGLD", dict(learning_rate=1e-4)),
    "sgnht_vec_2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=True)),
    "sgnht_vec_1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=True)),
    "sgnht_scalar_2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=False)),
    "sgnht_scalar_1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=False)),
}
STEPS = 5


class _Taken(Exception):
    pass


def reference_bnn_problem(seed=707):
    """Run make_ref_golden.run_reference_bnn_sghmc until its SGHMC.sample() call and return the
    stand-in module, the reference's sgmcmc module, the model, observed and latent it passes,
    and the data / prior constants it built (recorded from tf.constant)."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    load = mrg.load_reference
    got = {}

    def load_and_intercept():
        tf, hmc, sg = load()
        real_constant = tf.constant
        consts = []

        def constant(value, *a, **k):
            consts.append(np.array(value))
            return real_constant(value, *a, **k)

        class TakeOver(object):
            def __init__(self, **kw):
                pass

            def sample(self, meta_bn, observed, latent):
                tf.constant = real_constant
                got.update(tf=tf, sg=sg, model=meta_bn, observed=observed, latent=latent,
                           consts=consts)
                raise _Taken()
        tf.constant = constant
        return tf, hmc, type("sgmcmc", (), {"SGHMC": TakeOver})
    mrg.load_reference = load_and_intercept
    try:
        mrg.run_reference_bnn_sghmc(seed)
    except _Taken:
        pass
    finally:
        mrg.load_reference = load
    return got


def run_reference_bnn_sgmcmc(seed=707):
    p = reference_bnn_problem(seed)
    tf, sg, model, observed, latent = p["tf"], p["sg"], p["model"], p["observed"], p["latent"]
    names = sorted(latent)
    w_init = [np.array(latent[n].value) for n in names]
    C, H, in1 = w_init[0].shape
    sess = tf.Session()
    y = np.asarray(sess.run(observed["y"]), np.float32)

    def first(shape):
        return next(c for c in p["consts"] if c.shape == shape).astype(np.float32)
    lj = model.log_joint
    n_train = dict(zip(lj.__code__.co_freevars, (c.cell_contents for c in lj.__closure__)))[
        "n_train"]
    out = dict(x=first((y.shape[0], in1 - 1)), y=y, logstd0=first((H, in1)),
               logstd1=first((1, H + 1)), w0_init=w_init[0], w1_init=w_init[1],
               n_train=np.int32(n_train))
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    v0 = [rng.standard_normal(w.shape).astype(np.float32) for w in w_init]
    out.update(v0_0=v0[0], v0_1=v0[1])
    for tag, (cls, kw) in CONFIGS.items():
        for n, w in zip(names, w_init):
            latent[n].load(w)
        tf.set_noise(normal=list(v0))          # SGNHT's initial momenta (sgmcmc.py:450-452)
        s = getattr(sg, cls)(**kw)
        sample_op, info = s.sample(model, observed=observed, latent=latent)
        tf.set_noise()
        out.update({tag + "/cfg_" + k: np.float32(v) for k, v in kw.items()})
        rec = {}
        for t in range(STEPS):
            pool = [rng.standard_normal(w_init[k % 2].shape).astype(np.float32)
                    for k in range(4)]
            rs, nz = pool[:2], pool[2:]
            redraw = cls == "SGNHT" and t % kw["n_iter_resample_v"] == 0    # sgmcmc.py:470-478
            # consumption order inside a run (latents in dictionary order, sgmcmc.py:105-107):
            # the re-draws of v, then the update noise; the first-order update builds each
            # latent's new v in turn, so there it is re-draw and noise of w0, then of w1
            if not redraw:
                rs = [np.zeros_like(pool[0]), np.zeros_like(pool[1])]
                feed = nz
            elif kw["second_order"]:
                feed = rs + nz
            else:
                feed = [rs[0], nz[0], rs[1], nz[1]]
            tf.set_noise(normal=list(feed))
            _, r = sess.run([sample_op, info])
            assert not tf._NOISE["normal"]
            row = {"n_used": np.int32(len(feed))}
            for k, n in enumerate(names):
                row["w%d" % k] = np.array(latent[n].value)
                row["noise%d" % k] = nz[k]
                row["resample%d" % k] = rs[k]
                if cls == "SGNHT":
                    row["mean_k%d" % k] = np.asarray(r.mean_k[n], np.float32)
                    row["alpha%d" % k] = np.asarray(r.alpha[n], np.float32)
            for k, v in row.items():
                rec.setdefault(k, []).append(v)
        out.update({tag + "/" + k: np.stack(v) for k, v in rec.items()})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_bnn_sgmcmc()
    np.savez_compressed(os.path.join(HERE, "ref_bnn_sgmcmc.npz"), **out)
    with open(os.path.join(HERE, "ref_bnn_sgmcmc_digests.json"), "w") as f:
        json.dump(digests("ref_bnn_sgmcmc", out), f, indent=1, sort_keys=True)
        f.write("\n")
    for tag in CONFIGS:
        print(tag, "draws per step", out[tag + "/n_used"].tolist())


if __name__ == "__main__":
    main()
