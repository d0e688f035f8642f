"""tests/golden/ref_pmf_hmc.npz: the Bayesian PMF example run on THE REFERENCE'S OWN BayesianNet,
Normal and HMC, through the NumPy TensorFlow stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_pmf_golden.py     ->  ref_pmf_hmc.npz, ref_pmf_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  The model is pmf_hmc.py:19-31 with its log_joint
override (136-144), adaptation off (122-125), and the example's loop (176-209): every epoch samples
the user factor ONE CHUNK AT A TIME, sequentially, with the movie factor gathered over the chunk's
neighbour set (select_from_corpus, 34-60), then the movie factor chunk by chunk the same way.
Every momentum and acceptance draw is injected and stored.  The stand-in has no tf.gather; it is
added here, with its vector-Jacobian product (a scatter-add), for this run only.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

CFG = dict(K=3, D=7, chunk=5, n_users=15, n_movies=10, epochs=3, step_size=0.06, n_leapfrogs=10,
           alpha_u=1.0, alpha_v=1.0, alpha_pred=0.05, seed=2024)


def _add_gather(tf):
    def gather(params, indices, axis=0, name=None):
        p, ix = tf.convert_to_tensor(params), tf.convert_to_tensor(indices)
        ax = int(axis)
        idx = lambda c: np.asarray(c.eval(ix), np.int64)                     # noqa: E731
        out = tf.Tensor(lambda c: np.take(c.eval(p), idx(c), axis=ax), inputs=(p, ix),
                        op="gather", dtype=p._dtype)

        def vjp(g):
            def fn(c):
                res = np.zeros_like(np.asarray(c.eval(p)))
                np.add.at(res, (slice(None),) * ax + (idx(c),), np.asarray(c.eval(g)))
                return res
            return [tf.Tensor(fn, inputs=(g, p, ix), op="gather_grad", dtype=p._dtype), None]
        out.vjp = vjp
        return out
    tf.gather = gather


def make_corpus(rng, n_users, n_movies):
    """A few ratings per user; user 0 rates every movie, the last user and movie have none."""
    pairs = {(0, j) for j in range(n_movies - 1)}
    for i in range(1, n_users - 1):
        for j in rng.choice(n_movies - 1, size=rng.randint(1, 4), replace=False):
            pairs.add((i, int(j)))
    pairs = sorted(pairs)
    order = rng.permutation(len(pairs))
    rows = np.array([pairs[o][0] for o in order], np.int64)
    cols = np.array([pairs[o][1] for o in order], np.int64)
    score = rng.randint(1, 6, rows.size).astype(np.float32)
    return rows, cols, score


def select_from_corpus(l, r, u_v, u_v_score):                # pmf_hmc.py:34-60
    sv, tr = [], []
    for i in range(r - l):
        if l + i in u_v:
            sv = sv + u_v[l + i]
            tr = tr + u_v_score[l + i]
    sv = sorted(set(sv))
    idx = {s: k for k, s in enumerate(sv)}
    ssu, ssv = [], []
    for i in range(r - l):
        if l + i in u_v:
            ssu += [i] * len(u_v[l + i])
            ssv += [idx[j] for j in u_v[l + i]]
    return len(sv), np.array(sv, np.int32), np.array(tr, np.float32), ssu, ssv


def run_reference_pmf_hmc(cfg=CFG):
    sys.path.insert(0, ROOT)
    from oracle.tf_shim.make_ref_golden import load_reference
    tf, hmc_mod, _ = load_reference()
    _add_gather(tf)
    fw = importlib.import_module("zhusuan.framework")
    tf.reset_default_graph()
    rng = np.random.RandomState(cfg["seed"])
    K, D, cs = cfg["K"], cfg["D"], cfg["chunk"]
    N, M = cfg["n_users"], cfg["n_movies"]
    rows, cols, score = make_corpus(rng, N, M)
    user_movie, user_score, movie_user, movie_score = {}, {}, {}, {}
    for i, j, s in zip(rows.tolist(), cols.tolist(), score.tolist()):
        user_movie.setdefault(i, []).append(j)
        user_score.setdefault(i, []).append(s)
        movie_user.setdefault(j, []).append(i)
        movie_score.setdefault(j, []).append(s)

    @fw.meta_bayesian_net(scope="pmf", reuse_variables=True)
    def pmf(n, m, D, n_particles, select_u, select_v, alpha_u, alpha_v, alpha_pred):
        bn = fw.BayesianNet()
        u = bn.normal("u", tf.zeros(shape=[n, D]), std=alpha_u, n_samples=n_particles,
                      group_ndims=1)
        v = bn.normal("v", tf.zeros(shape=[m, D]), std=alpha_v, n_samples=n_particles,
                      group_ndims=1)
        gather_u = tf.gather(u, select_u, axis=1)
        gather_v = tf.gather(v, select_v, axis=1)
        r_logits = tf.reduce_sum(gather_u * gather_v, axis=2)
        bn.deterministic("r_pred", tf.sigmoid(r_logits))
        bn.normal("r", tf.sigmoid(r_logits), std=alpha_pred)
        return bn

    U0 = (0.1 * rng.standard_normal((K, N, D))).astype(np.float32)
    V0 = (0.1 * rng.standard_normal((K, M, D))).astype(np.float32)
    U, V = tf.Variable(U0.copy(), name="U"), tf.Variable(V0.copy(), name="V")
    cand_u = tf.Variable(np.zeros((K, cs, D), np.float32), name="cand_u")
    cand_v = tf.Variable(np.zeros((K, cs, D), np.float32), name="cand_v")

    def log_joint(bn):                                         # pmf_hmc.py:136-142
        log_pu, log_pv = bn.cond_log_prob(['u', 'v'])
        log_pr = bn.cond_log_prob('r')
        return (tf.reduce_sum(log_pu, axis=-1) + tf.reduce_sum(log_pv, axis=-1)
                + tf.reduce_sum(log_pr, axis=-1))

    def chunk_sampler(side, c):
        """The graph of one sess.run(sample_u_op / sample_v_op) of pmf_hmc.py:187-192, 203-208:
        the stand-in cannot infer static shapes through unfed placeholders, so the chunk's sizes
        and selections are constants of a graph built per chunk; with adaptation off an HMC
        carries no state from one run to the next."""
        l, r = c * cs, (c + 1) * cs
        if side == "u":
            nv, sv, tr, ssu, ssv = select_from_corpus(l, r, user_movie, user_score)
            n_, m_, obs = cs, nv, {"v": tf.gather(V, tf.constant(sv), axis=1)}
        else:
            nu, su, tr, ssv, ssu = select_from_corpus(l, r, movie_user, movie_score)
            n_, m_, obs = nu, cs, {"u": tf.gather(U, tf.constant(su), axis=1)}
        model = pmf(n_, m_, D, K, tf.constant(np.array(ssu, np.int32)),
                    tf.constant(np.array(ssv, np.int32)), cfg["alpha_u"], cfg["alpha_v"],
                    cfg["alpha_pred"])
        model.log_joint = log_joint
        obs["r"] = (tf.constant(tr) - 1.0) / 4.0
        hmc = hmc_mod.HMC(step_size=cfg["step_size"], n_leapfrogs=cfg["n_leapfrogs"],
                          adapt_step_size=None, target_acceptance_rate=0.9)
        return hmc.sample(model, obs, {side: cand_u if side == "u" else cand_v})
    sess = tf.Session()
    keys = ("noise_p", "noise_u", "acc", "lp0", "lp", "h0", "h1")
    rec = {s + "_" + k: [] for s in "uv" for k in keys}
    rec["U"], rec["V"] = [], []
    for epoch in range(cfg["epochs"]):
        for side, n_lat, cand, var in (("u", N, cand_u, U), ("v", M, cand_v, V)):
            ep = {k: [] for k in keys}
            for c in range(n_lat // cs):
                l, r = c * cs, (c + 1) * cs
                op, info = chunk_sampler(side, c)
                whole = np.array(var.value)
                cand.load(whole[:, l:r])                        # trans_cand_U / trans_cand_V
                p = rng.standard_normal((K, cs, D)).astype(np.float32)
                u01 = rng.random_sample(K).astype(np.float32)
                tf.set_noise(normal=[p], uniform=[u01])
                with np.errstate(all="ignore"):
                    _, res = sess.run([op, info])
                assert not tf._NOISE["normal"] and not tf._NOISE["uniform"]
                whole[:, l:r] = np.array(cand.value)            # trans_us_cand / trans_vs_cand
                var.load(whole)
                for k, x in zip(keys, (p, u01, res.acceptance_rate, res.orig_log_prob,
                                       res.log_prob, res.orig_hamiltonian, res.hamiltonian)):
                    ep[k].append(np.asarray(x, np.float32))
            for k in keys:
                rec[side + "_" + k].append(np.stack(ep[k]))
            rec[side.upper()].append(np.array(var.value))
    out = {k: np.stack(v) for k, v in rec.items()}
    out.update(rows=rows, cols=cols, rating=((score - 1.0) / 4.0).astype(np.float32), U0=U0, V0=V0,
               **{"cfg_" + k: np.float32(v) for k, v in cfg.items()})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_pmf_hmc()
    np.savez_compressed(os.path.join(HERE, "ref_pmf_hmc.npz"), **out)
    with open(os.path.join(HERE, "ref_pmf_digests.json"), "w") as f:
        json.dump(digests("ref_pmf_hmc", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("ref_pmf_hmc acc mean per epoch: u", np.round(out["u_acc"].mean((1, 2)), 3).tolist(),
          "v", np.round(out["v_acc"].mean((1, 2)), 3).tolist(),
          "accepted", int((out["u_noise_u"] < out["u_acc"]).sum() +
                          (out["v_noise_u"] < out["v_acc"]).sum()),
          "of", out["u_acc"].size + out["v_acc"].size)


if __name__ == "__main__":
    main()
