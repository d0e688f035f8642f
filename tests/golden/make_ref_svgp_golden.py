"""tests/golden/ref_svgp.npz: the reference's own RBFKernel and gp_conditional
(examples/gaussian_process/utils.py, imported unmodified) inside the sparse variational GP of
examples/gaussian_process/svgp.py, on THE REFERENCE'S OWN BayesianNet, MultivariateNormalCholesky,
Normal, elbo() and log_mean_exp, executed on the NumPy TensorFlow stand-in of oracle/tf_shim (TEST
INFRASTRUCTURE).

    python tests/golden/make_ref_svgp_golden.py  ->  ref_svgp.npz, ref_svgp_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.  Every draw is injected with tf.set_noise: the
variational fz's normals ([K, M, 1], multivariate.py:157) and the variational fx's normals
([1, K, B], univariate.py:166-167).  z_pos, z_mean, z_cov_raw, noise_level and k_log_scale are loaded
with non-trivial values on a grid of 2^-9 (z_cov_raw near 0.6 I, so the variational factor is well
conditioned, and z_pos spread so that Kzz is).

The stand-in lacks these ops; they are installed onto it here with TF 1.x semantics, so the stand-in
itself is unchanged for every other fixture:
  * tf.cholesky and tf.matrix_triangular_solve, with their gradients;
  * tf.eye, tf.matrix_band_part, tf.matrix_set_diag, tf.matrix_diag_part, tf.matrix_transpose;
  * tf.random_uniform_initializer, tf.nn.softplus (with its gradient), tf.assert_equal;
  * the gradient of tf.tile (MultivariateNormalCholesky._sample tiles mean and cov_tril),
    the gradient of tf.pow (utils.py:85-86 squares with **), get_variable with a Tensor
    initializer (svgp.py:79-80) and
    TensorShape.assert_is_compatible_with (multivariate.py:92).

Recorded (M = 7 inducing points, d = 3, B = 11 rows, K = 4 particles, n_train = 50):
  train/*: the bound, the sgvb cost and the cost's gradient w.r.t. every variable (z_pos,
    k_log_scale, noise_level, z_mean, z_cov_raw), with the draws eps_fz [K, M] and eps_fx [K, B];
  pred/*: log_likelihood and pred_mse of svgp.py:143-150 at 6 particles, with their draws;
  cond/*: a standalone gp_conditional(z, fz, x, ., kernel): mean and std for full_cov=False, and
    mean and the Cholesky factor of the covariance (particle 0 of the tiled factor) for
    full_cov=True.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np
import scipy.linalg as sla

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

M, D, B, K, N_TRAIN, K_PRED = 7, 3, 11, 4, 50, 6


def _tril(a):
    return np.tril(a)


def _install_ops(tf):
    T = tf.Tensor
    sw = lambda x: np.swapaxes(x, -1, -2)                               # noqa: E731

    def cholesky(a, name=None):
        a = tf.convert_to_tensor(a)
        out = tf._unary(lambda x: np.linalg.cholesky(x).astype(np.asarray(x).dtype), a,
                        "cholesky")

        def vjp(g):                     # Murray (2016): A_bar = sym(L^-T Phi(L^T L_bar) L^-1)
            def f(c):
                L, gL = np.asarray(c.eval(out)), np.asarray(c.eval(g))
                P = np.tril(sw(L) @ gL)
                P = P - 0.5 * np.eye(L.shape[-1], dtype=L.dtype) * P
                Li = np.linalg.inv(L)
                S = sw(Li) @ P @ Li
                return (0.5 * (S + sw(S))).astype(L.dtype)
            return [T(f, inputs=(g, out), op="cholesky_grad", dtype=a._dtype)]
        out.vjp = vjp
        return out

    def _solve(A, b, lower, adjoint):
        A, b = np.asarray(A), np.asarray(b)
        batch = np.broadcast_shapes(A.shape[:-2], b.shape[:-2])
        A, b = np.broadcast_to(A, batch + A.shape[-2:]), np.broadcast_to(b, batch + b.shape[-2:])
        out = np.empty(b.shape, b.dtype)
        for idx in np.ndindex(*b.shape[:-2]):
            out[idx] = sla.solve_triangular(A[idx], b[idx], lower=lower,
                                            trans="T" if adjoint else "N")
        return out

    def matrix_triangular_solve(matrix, rhs, lower=True, adjoint=False, name=None):
        matrix, rhs = tf.convert_to_tensor(matrix), tf.convert_to_tensor(rhs)
        out = T(lambda c: _solve(c.eval(matrix), c.eval(rhs), lower, adjoint),
                inputs=(matrix, rhs), op="matrix_triangular_solve", dtype=rhs._dtype)

        def vjp(g):                     # rhs_bar = A^-T g;  A_bar = -band(rhs_bar X^T)
            def grhs(c):
                return _solve(c.eval(matrix), c.eval(g), lower, not adjoint)

            def gmat(c):
                gb, X = grhs(c), np.asarray(c.eval(out))
                gA = -(X @ sw(gb)) if adjoint else -(gb @ sw(X))
                gA = np.tril(gA) if lower else np.triu(gA)
                shape = np.shape(c.eval(matrix))
                while gA.ndim > len(shape):
                    gA = gA.sum(0)
                return gA.astype(X.dtype)
            return [T(gmat, inputs=(g, matrix, out), op="mts_dA", dtype=matrix._dtype),
                    T(grhs, inputs=(g, matrix), op="mts_db", dtype=rhs._dtype)]
        out.vjp = vjp
        return out

    def eye(num_rows, num_columns=None, batch_shape=None, dtype=np.float32, name=None):
        return tf.constant(np.eye(int(num_rows), dtype=dtype))

    def matrix_band_part(a, num_lower, num_upper, name=None):
        assert (num_lower, num_upper) == (-1, 0), "only the lower triangle is needed"
        return tf._unary(_tril, a, "band_part", lambda g: [tf._unary(_tril, g, "band_part")])

    def matrix_diag_part(a, name=None):
        a = tf.convert_to_tensor(a)

        def vjp(g):
            return [tf._unary(lambda gv: gv[..., None] * np.eye(gv.shape[-1], dtype=gv.dtype),
                              g, "matrix_diag")]
        return tf._unary(lambda x: np.diagonal(x, axis1=-2, axis2=-1).copy(), a, "diag_part", vjp)

    def matrix_set_diag(a, diagonal, name=None):
        a, diagonal = tf.convert_to_tensor(a), tf.convert_to_tensor(diagonal)

        def f(c):
            x = np.array(c.eval(a))
            i = np.arange(x.shape[-1])
            x[..., i, i] = c.eval(diagonal)
            return x

        def vjp(g):
            def ga(c):
                gv = np.array(c.eval(g))
                i = np.arange(gv.shape[-1])
                gv[..., i, i] = 0
                return gv
            return [T(ga, inputs=(g,), op="set_diag_ga", dtype=a._dtype),
                    tf._unary(lambda gv: np.diagonal(gv, axis1=-2, axis2=-1).copy(), g,
                              "set_diag_gd")]
        return T(f, inputs=(a, diagonal), op="set_diag", vjp=vjp, dtype=a._dtype)

    def matrix_transpose(a, name=None):
        return tf._unary(sw, a, "matrix_transpose", lambda g: [tf._unary(sw, g, "mt")])

    def random_uniform_initializer(minval=0, maxval=None, seed=None, dtype=np.float32):
        init = np.random.Generator(np.random.PCG64(0))            # replaced by loaded values
        return lambda shape=(): init.uniform(minval, maxval, tuple(shape)).astype(dtype)

    def softplus(a, name=None):
        a = tf.convert_to_tensor(a)
        f = lambda x: (np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))).astype(  # noqa: E731
            np.asarray(x).dtype)
        return tf._unary(f, a, "softplus", lambda g: [g * tf.sigmoid(a)])

    def assert_equal(x, y, message=None, data=None, summarize=None, name=None):
        return tf._assert(lambda xv, yv: np.array_equal(xv, np.asarray(yv)), "equal")(
            x, y, message=message)

    base_tile = tf.tile

    def tile(a, multiples, name=None):
        a = tf.convert_to_tensor(a)
        out = base_tile(a, multiples)

        def vjp(g):
            def f(c):
                gv, av = np.asarray(c.eval(g)), np.asarray(c.eval(a))
                m = [int(v) for v in np.asarray(c.eval(multiples) if isinstance(multiples, T)
                                                else multiples)]
                shp = [d for mi, di in zip(m, av.shape) for d in (mi, di)]
                return gv.reshape(shp).sum(axis=tuple(range(0, 2 * len(m), 2))).astype(gv.dtype)
            return [T(f, inputs=(g, a), op="tile_grad", dtype=a._dtype)]
        out.vjp = vjp
        return out

    base_get_variable = tf.get_variable

    def get_variable(name, shape=None, dtype=None, initializer=None, **kw):
        if isinstance(initializer, T):
            initializer = np.asarray(tf.Session().run(initializer))
        return base_get_variable(name, shape=shape, dtype=dtype, initializer=initializer, **kw)

    base_pow = tf.pow

    def pow_(a, b, name=None):          # d a^b / d a = b a^(b-1); the exponents here are constants
        out = base_pow(a, b)
        a_t, b_t = out.inputs
        out.vjp = lambda g: [tf._unbroadcast(g * b_t * base_pow(a_t, b_t - 1.0), a_t), None]
        return out

    def assert_is_compatible_with(self, other):
        if not self.is_compatible_with(other):
            raise ValueError("Shapes %s and %s are incompatible" % (self, other))

    tf.TensorShape.assert_is_compatible_with = assert_is_compatible_with
    tf.cholesky, tf.matrix_triangular_solve, tf.eye = cholesky, matrix_triangular_solve, eye
    tf.matrix_band_part, tf.matrix_diag_part = matrix_band_part, matrix_diag_part
    tf.matrix_set_diag, tf.matrix_transpose = matrix_set_diag, matrix_transpose
    tf.random_uniform_initializer, tf.nn.softplus = random_uniform_initializer, softplus
    tf.assert_equal, tf.tile, tf.get_variable = assert_equal, tile, get_variable
    tf.pow = pow_


def _grid(rng, shape, std, mean=0.0):
    v = np.round((mean + std * rng.standard_normal(shape)) * 512) / 512
    return v.astype(np.float32)


def run_reference_svgp(seed=5150):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    _install_ops(tf)
    ref = os.environ.get("ZHUSUAN_REFERENCE", "/root/reference")
    if ref not in sys.path:
        sys.path.insert(0, ref)
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    zdist = importlib.import_module("zhusuan.distributions")
    zutils = importlib.import_module("zhusuan.utils")
    zs = sys.modules["zhusuan"]
    for mod in (fw, var, zutils):
        for k in getattr(mod, "__all__", []):
            setattr(zs, k, getattr(mod, k))
    zs.distributions, zs.variational = zdist, var
    for m in [k for k in sys.modules if k.startswith("examples")]:
        del sys.modules[m]
    gpu = importlib.import_module("examples.gaussian_process.utils")
    assert os.path.realpath(gpu.__file__).startswith(os.path.realpath(ref))
    RBFKernel, gp_conditional = gpu.RBFKernel, gpu.gp_conditional
    rng = np.random.Generator(np.random.PCG64(seed))
    out = {}

    @fw.meta_bayesian_net(scope='model', reuse_variables=True)
    def build_model(kernel, z_pos, x, n_particles, full_cov=False):        # svgp.py:49-72
        bn = fw.BayesianNet()
        Kzz_chol = tf.cholesky(kernel(z_pos, z_pos))
        fz = bn.multivariate_normal_cholesky(
            'fz', tf.zeros([M], dtype=np.float32), Kzz_chol, n_samples=n_particles)
        fx_given_fz = bn.stochastic(
            'fx', gp_conditional(z_pos, fz, x, full_cov, kernel, Kzz_chol))
        noise_level = tf.get_variable('noise_level', shape=[], dtype=np.float32,
                                      initializer=tf.constant_initializer(0.05))
        noise_level = tf.nn.softplus(noise_level)
        bn.normal('y', mean=fx_given_fz, std=noise_level, group_ndims=1)
        return bn

    def build_variational(kernel, z_pos, x, n_particles):                   # svgp.py:75-87
        bn = fw.BayesianNet()
        z_mean = tf.get_variable('z/mean', [M], np.float32, tf.zeros_initializer())
        z_cov_raw = tf.get_variable('z/cov_raw', initializer=tf.eye(M, dtype=np.float32))
        z_cov_tril = tf.matrix_set_diag(
            tf.matrix_band_part(z_cov_raw, -1, 0),
            tf.nn.softplus(tf.matrix_diag_part(z_cov_raw)))
        fz = bn.multivariate_normal_cholesky('fz', z_mean, z_cov_tril, n_samples=n_particles)
        bn.stochastic('fx', gp_conditional(z_pos, fz, x, False, kernel))
        return bn

    x = _grid(rng, (B, D), 1.0)
    y = _grid(rng, (B,), 1.0)
    std_y_train = np.float32(1.75)
    vals = {
        "k_log_scale_rbf_kernel": _grid(rng, (D,), 0.5),
        "z/pos": (np.round(rng.uniform(-1.5, 1.5, (M, D)) * 512) / 512).astype(np.float32),
        "noise_level": np.float32(-0.75),
        "z/mean": _grid(rng, (M,), 0.5),
        "z/cov_raw": (np.tril(_grid(rng, (M, M), 0.1), -1)
                      + np.diag(_grid(rng, (M,), 0.1, -0.5))).astype(np.float32),
    }
    out.update({"x": x, "y": y, "n_train": np.float32(N_TRAIN), "std_y_train": std_y_train})

    def graph(n_particles):
        """svgp.py:110-150 with n_particles a Python int: the stand-in takes static shapes from an
        evaluation, where a placeholder particle count would read as 0."""
        tf.reset_default_graph()
        kernel = RBFKernel(D)
        x_ph = tf.placeholder(np.float32, [B, D], 'x')
        y_ph = tf.placeholder(np.float32, [B], 'y')
        z_pos = tf.get_variable('z/pos', [M, D], np.float32,
                                initializer=tf.random_uniform_initializer(-1, 1))
        batch_size = tf.cast(tf.shape(x_ph)[0], np.float32)
        model = build_model(kernel, z_pos, x_ph, n_particles)
        variational = build_variational(kernel, z_pos, x_ph, n_particles)

        def log_joint(bn):
            prior, log_py_given_fx = bn.cond_log_prob(['fz', 'y'])
            return prior + log_py_given_fx / batch_size * N_TRAIN

        model.log_joint = log_joint
        [var_fz, var_fx] = variational.query(['fz', 'fx'], outputs=True, local_log_prob=True)
        var_fx = (var_fx[0], tf.zeros_like(var_fx[1]))
        lower_bound = var.elbo(model, observed={'y': y_ph},
                               latent={'fz': var_fz, 'fx': var_fx}, axis=0)
        cost = tf.reduce_mean(lower_bound.sgvb())
        lower_bound = tf.reduce_mean(lower_bound)
        model = model.observe(fx=var_fx[0], y=y_ph)
        log_likelihood = model.cond_log_prob('y')
        log_likelihood = zutils.log_mean_exp(log_likelihood, 0) / batch_size - \
            tf.log(std_y_train)
        y_pred_mean = tf.reduce_mean(model['y'].distribution.mean, axis=0)
        pred_mse = tf.reduce_mean((y_pred_mean - y_ph) ** 2) * std_y_train ** 2
        names = {v.name: v for v in tf.trainable_variables()}
        assert sorted(names) == sorted(vals), sorted(names)
        wrt = []
        for nm, v in vals.items():
            names[nm].load(np.asarray(v, np.float32))
            wrt.append((nm.replace("/", "_").replace("k_log_scale_rbf_kernel", "k_raw_scale"),
                        names[nm]))
        return kernel, z_pos, wrt, (lower_bound, cost, log_likelihood, pred_mse), {x_ph: x,
                                                                                 y_ph: y}

    def run(fetches, feed, n_part, fx_first=False):
        """fx_first: the fetches evaluate the fx draw before the fz draw it depends on (the
        stand-in hands out injected arrays in evaluation order)."""
        eps_fz = rng.standard_normal((n_part, M, 1)).astype(np.float32)
        eps_fx = rng.standard_normal((1, n_part, B)).astype(np.float32)
        tf.set_noise(normal=[eps_fx, eps_fz] if fx_first else [eps_fz, eps_fx])
        r = tf.Session().run(fetches, feed_dict=feed)
        assert not tf._NOISE["normal"]
        return r, eps_fz[..., 0], eps_fx[0]

    _, _, wrt, (lower_bound, cost, _, _), feed = graph(K)
    for key, v in wrt:
        out["param/" + key] = np.asarray(v.value, np.float32)
    r, efz, efx = run([lower_bound, cost] + tf.gradients(cost, [v for _, v in wrt]), feed, K)
    out.update({"train/eps_fz": efz, "train/eps_fx": efx, "train/bound": np.float32(r[0]),
                "train/cost": np.float32(r[1])})
    for (key, _), g in zip(wrt, r[2:]):
        out["train/grad_" + key] = np.asarray(g, np.float32)
    kernel, z_pos, _, (_, _, log_likelihood, pred_mse), feed = graph(K_PRED)
    r, efz, efx = run([log_likelihood, pred_mse], feed, K_PRED, fx_first=True)
    out.update({"pred/eps_fz": efz, "pred/eps_fx": efx,
                "pred/log_likelihood": np.float32(r[0]), "pred/pred_mse": np.float32(r[1])})
    sess = tf.Session()

    # a standalone gp_conditional on the loaded kernel and inducing points
    fz = _grid(rng, (K, M), 1.0)
    d = gp_conditional(z_pos, tf.constant(fz), tf.constant(x), False, kernel)
    mean, std = sess.run([d.mean, d.std])
    dc = gp_conditional(z_pos, tf.constant(fz), tf.constant(x), True, kernel)
    mean_c, tril_c = sess.run([dc.mean, dc.cov_tril])
    out.update({"cond/fz": fz, "cond/mean": np.asarray(mean, np.float32),
                "cond/std": np.asarray(std, np.float32),
                "cond/full_mean": np.asarray(mean_c, np.float32),
                "cond/full_cov_tril": np.asarray(tril_c[0], np.float32)})
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_svgp()
    np.savez_compressed(os.path.join(HERE, "ref_svgp.npz"), **out)
    with open(os.path.join(HERE, "ref_svgp_digests.json"), "w") as f:
        json.dump(digests("ref_svgp", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("bound %.6g, cost %.6g, log_likelihood %.6g, pred_mse %.6g"
          % (out["train/bound"], out["train/cost"], out["pred/log_likelihood"],
             out["pred/pred_mse"]))


if __name__ == "__main__":
    main()
