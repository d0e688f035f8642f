"""tests/golden/ref_gan.npz: one training step of the DCGAN and the Wasserstein GAN of
examples/generative_adversarial_nets (dcgan.py, wasserstein_gan.py) at small widths on THE
REFERENCE'S OWN BayesianNet (the z prior bn.uniform("z", -1, 1), drawn through tf.random_uniform
with the uniforms injected by tf.set_noise) and reuse_variables, executed on the NumPy TensorFlow
stand-in of oracle/tf_shim (TEST INFRASTRUCTURE).

    python tests/golden/make_ref_gan_golden.py  ->  ref_gan.npz, ref_gan_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.

The example modules import examples.utils (datasets, multi_gpu flags), which the stand-in cannot
load, so `generator`, `discriminator` and the loss graph of `build_tower_graph` are restated below
with line citations, on the reference's framework.  The stand-in lacks the layers they use; they are
installed onto it here, in NumPy, with their gradients, straight from TensorFlow's definitions:
  * tf.layers.conv2d(x, Cout, k, strides, padding, use_bias, activation), kernel [k, k, Cin, Cout]:
    Ho = ceil(H / s) (SAME) or ceil((H - k + 1) / s) (VALID); SAME pads pad_total = max((Ho - 1) s
    + k - H, 0) rows, pad_total // 2 of them before;
  * tf.layers.conv2d_transpose(x, Cout, k, strides, padding, use_bias, activation), kernel
    [k, k, Cout, Cin]: the adjoint of that convolution from the output grid, whose size is
    conv_utils.deconv_output_length: H s (SAME), H s + max(k - s, 0) (VALID);
  * tf.layers.batch_normalization(x, training, scale) with TF 1.x's defaults (momentum 0.99,
    epsilon 1e-3, moving mean 0 and variance 1).  A 2-D input takes the non-fused path (as in
    make_ref_blvae_golden.py): the population variance normalises and updates.  A 4-D input takes
    `BatchNormalization._fused_batch_norm` (tensorflow/python/layers/normalization.py, via
    keras/layers/normalization.py in TF 1.13), as read here (TensorFlow is not installed where
    this runs): fused_batch_norm normalises with the population variance over N*H*W and returns the
    Bessel-corrected variance R / (R - 1) var (the CPU kernel uses the factor 1 at R = 1);
    `_bessels_correction_test_only` defaults to True, so that corrected variance is NOT scaled back
    and it is what the moving variance moves towards: m -= (m - batch) * (1 - momentum).
The stand-in itself is unchanged for every other fixture.  This shares no code with
tests/gan_oracle.py (F.pad + F.conv2d, F.conv_transpose2d + crop) nor with zs.fused.

Widths: DCGAN ngf = ndf = 2 on 3 images of 32x32x3; WGAN ngf = 3, ndf = 2 on 3 images of 28x28x1;
z_dim 40.  Weights are Glorot-uniform draws rounded to a grid of 2^-8, gamma / beta / biases are
loaded with values on a grid of 2^-9, images are on a grid of 2^-8.

Recorded per model m in (dcgan, wgan): m/x, m/u (the uniforms of z), m/z, every parameter as
m/gen/<name>, m/disc/<name> (kernels in the tf.layers layouts, dense kernels stored [out, in]);
m/gen_loss and m/disc_loss (WGAN's w_distance = -disc_loss); tf.gradients of gen_loss w.r.t. the
generator's trainable variables and of disc_loss w.r.t. the discriminator's, those of more than
GRAD_PROJ_MIN entries as projections onto PROJ_K fixed vectors (`proj_vectors`); the moving
statistics after the step (the generator's layers move once; each discriminator layer twice, on
the real batch and then on the fake batch -- TF runs the two update ops in an unspecified order,
this is the order the fused port uses); and m/x_eval, the evaluation-mode generator on those
statistics for a second draw m/u_eval.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

N, Z_DIM = 3, 40
MOMENTUM, EPS = 0.99, 1e-3
GRAD_PROJ_MIN, PROJ_K, PROJ_SEED = 300, 8, 20261018


def proj_vectors(index, size):
    """The fixed vectors gradient `index` (of `size` entries) is projected onto: [PROJ_K, size]."""
    return np.random.default_rng([PROJ_SEED, index]).standard_normal((PROJ_K, size))


# ---- k x k convolution in NumPy ------------------------------------------------------------------

def out_size(big, k, s, padding):
    return -(-big // s) if padding == "same" else -(-(big - k + 1) // s)


def _pad_before(big, small, k, s, padding):
    return max((small - 1) * s + k - big, 0) // 2 if padding == "same" else 0


def _padded(x, small_hw, k, s, padding):
    """x zero-padded to the rows and columns the taps of small_hw reach (x cut where none does)."""
    N_, H, W_, C = x.shape
    Ho, Wo = small_hw
    pt, pl = _pad_before(H, Ho, k, s, padding), _pad_before(W_, Wo, k, s, padding)
    xp = np.zeros((N_, (Ho - 1) * s + k, (Wo - 1) * s + k, C))
    hh, ww = min(H, xp.shape[1] - pt), min(W_, xp.shape[2] - pl)
    xp[:, pt:pt + hh, pl:pl + ww] = x[:, :hh, :ww]
    return xp, pt, pl, hh, ww


def np_conv(x, w, s, padding):
    """y[n, i, j] = sum_{kh, kw} x[n, s i + kh - pt, s j + kw - pl] . w[kh, kw] (x zero outside)."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    k = w.shape[0]
    Ho, Wo = out_size(x.shape[1], k, s, padding), out_size(x.shape[2], k, s, padding)
    xp = _padded(x, (Ho, Wo), k, s, padding)[0]
    y = np.zeros((x.shape[0], Ho, Wo, w.shape[3]))
    for kh in range(k):
        for kw in range(k):
            y += xp[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s] @ w[kh, kw]
    return y


def np_conv_adjoint(g, w, s, padding, big_hw):
    """The adjoint of np_conv(., w, s, padding) from big_hw [H, W, Cin] to g's [Ho, Wo, Cout]."""
    g, w = np.asarray(g, np.float64), np.asarray(w, np.float64)
    k = w.shape[0]
    N_, Ho, Wo, _ = g.shape
    H, W_ = big_hw
    pt, pl = _pad_before(H, Ho, k, s, padding), _pad_before(W_, Wo, k, s, padding)
    xp = np.zeros((N_, (Ho - 1) * s + k, (Wo - 1) * s + k, w.shape[2]))
    for kh in range(k):
        for kw in range(k):
            xp[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s] += g @ w[kh, kw].T
    out = np.zeros((N_, H, W_, w.shape[2]))
    hh, ww = min(H, xp.shape[1] - pt), min(W_, xp.shape[2] - pl)
    out[:, :hh, :ww] = xp[:, pt:pt + hh, pl:pl + ww]
    return out


def np_conv_wgrad(x, g, s, padding, k):
    """d <np_conv(x, w, s, padding), g> / d w: [k, k, Cin, Cout]."""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    Ho, Wo = g.shape[1], g.shape[2]
    xp = _padded(x, (Ho, Wo), k, s, padding)[0]
    dw = np.zeros((k, k, x.shape[3], g.shape[3]))
    for kh in range(k):
        for kw in range(k):
            xs = xp[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s]
            dw[kh, kw] = np.einsum("nijc,nijd->cd", xs, g)
    return dw


def _install_ops(tf, bn_calls):
    """tf.layers.conv2d, conv2d_transpose and batch_normalization on the stand-in.  bn_calls
    collects, per training call of a batch-norm layer, (moving_mean, moving_variance, batch mean,
    the variance the moving variance moves towards)."""
    f32 = lambda a: np.asarray(a, np.float32)                          # noqa: E731

    def store():
        return tf._TEMPLATES[-1] if tf._TEMPLATES else tf._DEFAULT_STORE

    def _int(v):
        return v if isinstance(v, int) else v[0]

    def _kernel(key, shape, fan_in, fan_out):
        s = store()
        if key not in s["vars"]:
            limit = np.sqrt(6.0 / (fan_in + fan_out))                   # glorot_uniform
            w0 = tf._INIT["rng"].uniform(-limit, limit, shape).astype(np.float32)
            kern = tf.Variable(w0, name=key + "/kernel")
            bias = tf.Variable(np.zeros(shape[-2] if "transpose" in key else shape[-1],
                                        np.float32), name=key + "/bias")
            s["vars"][key] = (kern, bias)
            tf._TRAINABLE.append(kern)
        return s["vars"][key]

    def _key(kind):
        s = store()
        k = s["count"]
        s["count"] += 1
        return kind if k == 0 else "%s_%d" % (kind, k)

    def conv2d(inputs, filters, kernel_size, strides=(1, 1), padding="valid", activation=None,
               use_bias=True, name=None, **kw):
        k, s, pad = _int(kernel_size), _int(strides), padding.lower()
        x = tf.convert_to_tensor(inputs)
        cin = int(x.get_shape().as_list()[-1])
        key = name or _key("conv2d")
        kern, bias = _kernel(key, (k, k, cin, filters), k * k * cin, k * k * filters)
        if use_bias and all(bias is not v for v in tf._TRAINABLE):
            tf._TRAINABLE.append(bias)
        out = tf.Tensor(lambda c: f32(np_conv(c.eval(x), c.eval(kern), s, pad)),
                        inputs=(x, kern), op="conv2d", dtype=np.float32)

        def vjp(g):
            dx = tf.Tensor(lambda c: f32(np_conv_adjoint(c.eval(g), c.eval(kern), s, pad,
                                                         np.shape(c.eval(x))[1:3])),
                           inputs=(g, kern, x), op="conv2d_dx", dtype=np.float32)
            dw = tf.Tensor(lambda c: f32(np_conv_wgrad(c.eval(x), c.eval(g), s, pad, k)),
                           inputs=(x, g), op="conv2d_dw", dtype=np.float32)
            return [dx, dw]
        out.vjp = vjp
        y = out + bias if use_bias else out
        return activation(y) if activation is not None else y

    def conv2d_transpose(inputs, filters, kernel_size, strides=(1, 1), padding="valid",
                         activation=None, use_bias=True, name=None, **kw):
        k, s, pad = _int(kernel_size), _int(strides), padding.lower()
        x = tf.convert_to_tensor(inputs)
        cin = int(x.get_shape().as_list()[-1])
        key = name or _key("conv2d_transpose")
        kern, bias = _kernel(key, (k, k, filters, cin), k * k * filters, k * k * cin)
        if use_bias and all(bias is not v for v in tf._TRAINABLE):
            tf._TRAINABLE.append(bias)
        grow = 0 if pad == "same" else max(k - s, 0)

        def big(c):
            h, w_ = np.shape(c.eval(x))[1:3]
            return (h * s + grow, w_ * s + grow)
        out = tf.Tensor(lambda c: f32(np_conv_adjoint(c.eval(x), c.eval(kern), s, pad, big(c))),
                        inputs=(x, kern), op="conv2d_transpose", dtype=np.float32)

        def vjp(g):
            dx = tf.Tensor(lambda c: f32(np_conv(c.eval(g), c.eval(kern), s, pad)),
                           inputs=(g, kern), op="conv2d_transpose_dx", dtype=np.float32)
            dw = tf.Tensor(lambda c: f32(np_conv_wgrad(c.eval(g), c.eval(x), s, pad, k)),
                           inputs=(g, x), op="conv2d_transpose_dw", dtype=np.float32)
            return [dx, dw]
        out.vjp = vjp
        y = out + bias if use_bias else out
        return activation(y) if activation is not None else y

    def batch_normalization(inputs, axis=-1, momentum=MOMENTUM, epsilon=EPS, center=True,
                            scale=True, training=False, **kw):
        assert center and axis == -1
        s = store()
        x = tf.convert_to_tensor(inputs)
        shp = x.get_shape().as_list()
        J = int(shp[-1])
        key = "bn:after_%d" % s["count"]            # the layer it follows
        if key not in s["vars"]:
            gamma = tf.Variable(np.ones(J, np.float32), name="gamma") if scale else None
            beta = tf.Variable(np.zeros(J, np.float32), name="beta")
            mm = tf.Variable(np.zeros(J, np.float32), name="moving_mean", trainable=False)
            mv = tf.Variable(np.ones(J, np.float32), name="moving_variance", trainable=False)
            tf._TRAINABLE.extend(([gamma] if scale else []) + [beta])
            s["vars"][key] = (gamma, beta, mm, mv)
        gamma, beta, mm, mv = s["vars"][key]
        if training:
            axes = list(range(len(shp) - 1))
            mean = tf.reduce_mean(x, axes, keepdims=True)
            var = tf.reduce_mean(tf.square(x - tf.stop_gradient(mean)), axes, keepdims=True)
            mean, var = tf.reshape(mean, [J]), tf.reshape(var, [J])
            if len(shp) == 4:                        # fused path: Bessel-corrected update
                def bessel(c):
                    R = int(np.prod(np.shape(c.eval(x))[:3]))
                    return f32(c.eval(var) * (np.float32(R) / np.float32(max(R - 1, 1))))
                var_mv = tf.Tensor(bessel, inputs=(var, x), op="bessel", dtype=np.float32)
            else:
                var_mv = var
            bn_calls.append((mm, mv, mean, var_mv))
        else:
            mean, var = mm, mv
        inv = 1.0 / tf.sqrt(var + np.float32(epsilon))
        if gamma is not None:
            inv = inv * gamma
        return x * inv + (beta - mean * inv)

    tf.layers.conv2d = staticmethod(conv2d)
    tf.layers.conv2d_transpose = staticmethod(conv2d_transpose)
    tf.layers.batch_normalization = staticmethod(batch_normalization)


def _grid(rng, shape, scale, shift=0.0, step=512):
    v = np.round((rng.standard_normal(shape) * scale + shift) * step) / step
    return v.astype(np.float32)


WIDTHS = {"dcgan": dict(ngf=2, ndf=2, hwc=(32, 32, 3)), "wgan": dict(ngf=3, ndf=2, hwc=(28, 28, 1))}


def run_reference_gan(kind, seed):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    bn_calls = []
    _install_ops(tf, bn_calls)
    fw = importlib.import_module("zhusuan.framework")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)
    ngf, ndf, hwc = WIDTHS[kind]["ngf"], WIDTHS[kind]["ndf"], WIDTHS[kind]["hwc"]

    if kind == "dcgan":
        @fw.reuse_variables(scope="gen")
        def generator(n, z_dim, is_training, ngf=64):                   # dcgan.py:20-40
            bn = fw.BayesianNet()
            z_min = -tf.ones([n, z_dim])
            z_max = tf.ones([n, z_dim])
            z = bn.uniform("z", z_min, z_max)
            lx_z = tf.layers.dense(z, ngf * 8 * 4 * 4, use_bias=False)
            lx_z = tf.layers.batch_normalization(lx_z, training=is_training)
            lx_z = tf.nn.relu(lx_z)
            lx_z = tf.reshape(lx_z, [-1, 4, 4, ngf * 8])
            lx_z = tf.layers.conv2d_transpose(lx_z, ngf * 4, 5, strides=(2, 2),
                                              padding="same", use_bias=False)
            lx_z = tf.layers.batch_normalization(lx_z, training=is_training)
            lx_z = tf.nn.relu(lx_z)
            lx_z = tf.layers.conv2d_transpose(lx_z, ngf * 2, 5, strides=(2, 2),
                                              padding="same", use_bias=False)
            lx_z = tf.layers.batch_normalization(lx_z, training=is_training)
            lx_z = tf.nn.relu(lx_z)
            x = tf.layers.conv2d_transpose(lx_z, 3, 5, strides=(2, 2),
                                           padding="same", activation=tf.sigmoid)
            return x, z

        @fw.reuse_variables(scope="disc")
        def discriminator(x, is_training, ndf=32):                      # dcgan.py:43-60
            lc_x = tf.layers.conv2d(x, ndf * 2, 5, strides=(2, 2),
                                    padding="same", use_bias=False)
            lc_x = tf.layers.batch_normalization(lc_x, training=is_training)
            lc_x = tf.nn.relu(lc_x)
            lc_x = tf.layers.conv2d(lc_x, ndf * 4, 5, strides=(2, 2),
                                    padding='same', use_bias=False)
            lc_x = tf.layers.batch_normalization(lc_x, training=is_training)
            lc_x = tf.nn.relu(lc_x)
            lc_x = tf.layers.conv2d(lc_x, ndf * 8, 5, strides=(2, 2),
                                    padding='same', use_bias=False)
            lc_x = tf.layers.batch_normalization(lc_x, training=is_training)
            lc_x = tf.nn.relu(lc_x)
            lc_x = tf.reshape(lc_x, [-1, ndf * 8 * 4 * 4])
            class_logits = tf.layers.dense(lc_x, 1)
            return class_logits
    else:
        @fw.reuse_variables(scope="gen")
        def generator(n, z_dim, is_training, ngf=32):           # wasserstein_gan.py:20-43
            bn = fw.BayesianNet()
            z_min = -tf.ones([n, z_dim])
            z_max = tf.ones([n, z_dim])
            z = bn.uniform("z", z_min, z_max)
            lx_z = tf.reshape(z, [-1, 1, 1, z_dim])
            lx_z = tf.layers.conv2d_transpose(lx_z, ngf * 4, 3, use_bias=False)
            lx_z = tf.layers.batch_normalization(lx_z, training=is_training,
                                                 scale=False)
            lx_z = tf.nn.relu(lx_z)
            lx_z = tf.layers.conv2d_transpose(lx_z, ngf * 2, 5, use_bias=False)
            lx_z = tf.layers.batch_normalization(lx_z, training=is_training,
                                                 scale=False)
            lx_z = tf.nn.relu(lx_z)
            lx_z = tf.layers.conv2d_transpose(lx_z, ngf, 5, strides=(2, 2),
                                              padding="same", use_bias=False)
            lx_z = tf.layers.batch_normalization(lx_z, training=is_training,
                                                 scale=False)
            lx_z = tf.nn.relu(lx_z)
            x = tf.layers.conv2d_transpose(
                lx_z, 1, 5, strides=(2, 2), padding="same", activation=tf.sigmoid)
            return x, z

        @fw.reuse_variables(scope="disc")
        def discriminator(x, is_training, ndf=16):              # wasserstein_gan.py:46-62
            lc_x = tf.layers.conv2d(x, ndf, 5, strides=(2, 2), padding='same',
                                    use_bias=False)
            lc_x = tf.layers.batch_normalization(lc_x, training=is_training,
                                                 scale=False)
            lc_x = tf.nn.relu(lc_x)
            lc_x = tf.layers.conv2d(lc_x, ndf * 2, 5, strides=(2, 2), padding='same',
                                    use_bias=False)
            lc_x = tf.layers.batch_normalization(lc_x, training=is_training,
                                                 scale=False)
            lc_x = tf.nn.relu(lc_x)
            lc_x = tf.layers.conv2d(lc_x, ndf * 4, 5, use_bias=False)
            lc_x = tf.layers.batch_normalization(lc_x, training=is_training,
                                                 scale=False)
            lc_x = tf.nn.relu(lc_x)
            lc_x = tf.reshape(lc_x, [-1, ndf * 4 * 3 * 3])
            critic = tf.layers.dense(lc_x, 1)
            return critic

    x_np = (np.round(rng.random((N,) + hwc) * 256) / 256).astype(np.float32)
    x = tf.constant(x_np)
    n_trainable = len(tf._TRAINABLE)
    if kind == "dcgan":                                                 # dcgan.py:79-100
        x_gen, z = generator(N, Z_DIM, True, ngf=ngf)
        x_class_logits = discriminator(x, True, ndf=ndf)
        x_gen_class_logits = discriminator(x_gen, True, ndf=ndf)
        gen_loss = tf.reduce_mean(
            tf.nn.sigmoid_cross_entropy_with_logits(
                labels=tf.ones_like(x_gen_class_logits),
                logits=x_gen_class_logits))
        disc_loss = (
            tf.reduce_mean(
                tf.nn.sigmoid_cross_entropy_with_logits(
                    labels=tf.ones_like(x_class_logits),
                    logits=x_class_logits)) +
            tf.reduce_mean(
                tf.nn.sigmoid_cross_entropy_with_logits(
                    labels=tf.zeros_like(x_gen_class_logits),
                    logits=x_gen_class_logits))) / 2.
    else:                                                       # wasserstein_gan.py:82-96
        x_critic = discriminator(x, True, ndf=ndf)
        x_gen, z = generator(N, Z_DIM, True, ngf=ngf)
        x_gen_critic = discriminator(x_gen, True, ndf=ndf)
        gen_loss = -tf.reduce_mean(x_gen_critic)
        disc_loss = -tf.reduce_mean(x_critic - x_gen_critic)

    # the two variable lists, told apart by scope (tf.trainable_variables(scope=...)); the stand-in's
    # dense layer makes a bias even with use_bias=False, which tf.layers does not: dropped here
    trainable = [v for v in tf._TRAINABLE[n_trainable:]
                 if not (kind == "dcgan" and v.name.startswith("dense/bias") and
                         id(v) in _store_var_ids(generator))]
    gen_ids = _store_var_ids(generator)
    gen_vars = [v for v in trainable if id(v) in gen_ids]
    disc_vars = [v for v in trainable if id(v) not in gen_ids]
    out = {kind + "/x": x_np}
    names = {}
    for role, vs in (("gen", gen_vars), ("disc", disc_vars)):
        for i, v in enumerate(vs):
            nm = "%s/%s/%d_%s" % (kind, role, i, v.name.split("/")[-1].split(":")[0])
            if v.value.ndim == 1:
                shift = 1.0 if "gamma" in nm else 0.0
                v.load(_grid(rng, v.value.shape, 0.3, shift))
            else:
                v.load((np.round(v.value * 256) / 256).astype(np.float32))
            val = v.value.T if v.value.ndim == 2 else v.value              # dense: [out, in]
            out[nm] = np.ascontiguousarray(val, np.float32)
            names[id(v)] = nm
    u = rng.random((N, Z_DIM)).astype(np.float32)
    grads_g = tf.gradients(gen_loss, gen_vars)
    grads_d = tf.gradients(disc_loss, disc_vars)
    calls = list(bn_calls)
    fetch = [gen_loss, disc_loss, z, x_gen] + grads_g + grads_d + \
        [c[2] for c in calls] + [c[3] for c in calls]
    tf.set_noise(uniform=[u[None]])          # Uniform draws [1, n, z_dim], then squeezes
    r = tf.Session().run(fetch)
    assert not tf._NOISE["uniform"]
    out.update({kind + "/u": u, kind + "/z": np.asarray(r[2], np.float32),
                kind + "/gen_loss": np.float32(r[0]), kind + "/disc_loss": np.float32(r[1]),
                kind + "/x_gen": np.asarray(r[3], np.float32)})
    ng = len(grads_g) + len(grads_d)
    for k, (v, g) in enumerate(zip(gen_vars + disc_vars, r[4:4 + ng])):
        g = np.asarray(g, np.float64)
        g = g.T if g.ndim == 2 else g
        nm = names[id(v)]
        if g.size > GRAD_PROJ_MIN:
            out[nm.replace("/gen/", "/grad_proj_gen/").replace("/disc/", "/grad_proj_disc/")] = \
                (proj_vectors(k, g.size) @ g.ravel()).astype(np.float32)
        else:
            out[nm.replace("/gen/", "/grad_gen/").replace("/disc/", "/grad_disc/")] = \
                np.ascontiguousarray(g, np.float32)
    # moving statistics: each training call of a layer, in build order (for the discriminator the
    # real batch's call comes first in both examples' graphs), applied in that order
    means, vars_ = r[4 + ng:4 + ng + len(calls)], r[4 + ng + len(calls):]
    moved = {}
    d = np.float32(1.0 - MOMENTUM)
    for (mm, mv, _, _), bm, bv in zip(calls, means, vars_):
        m0, v0 = moved.get(id(mm), (mm.value.copy(), mv.value.copy()))
        moved[id(mm)] = (m0 - (m0 - np.float32(bm)) * d, v0 - (v0 - np.float32(bv)) * d)
    order = []
    for mm, mv, _, _ in calls:
        if all(mm is not o[0] for o in order):
            order.append((mm, mv))
    counts = {"gen": 0, "disc": 0}
    for mm, mv in order:
        role = "gen" if id(mm) in gen_ids else "disc"
        n_calls = sum(1 for c in calls if c[0] is mm)
        assert n_calls == (1 if role == "gen" else 2), (role, n_calls)
        m1, v1 = moved[id(mm)]
        out["%s/moving_mean_%s%d" % (kind, role, counts[role])] = np.asarray(m1, np.float32)
        out["%s/moving_variance_%s%d" % (kind, role, counts[role])] = np.asarray(v1, np.float32)
        mm.load(np.asarray(m1, np.float32))
        mv.load(np.asarray(v1, np.float32))
        counts[role] += 1
    # evaluation-mode generator on the moved statistics (dcgan.py:113, eval_x_gen)
    x_eval, _ = generator(N, Z_DIM, False, ngf=ngf)
    u_eval = rng.random((N, Z_DIM)).astype(np.float32)
    tf.set_noise(uniform=[u_eval[None]])
    out[kind + "/x_eval"] = np.asarray(tf.Session().run(x_eval), np.float32)
    out[kind + "/u_eval"] = u_eval
    return out


def _store_var_ids(template):
    """ids of the variables a reuse_variables template (the stand-in's make_template) created."""
    ids = set()
    for vs in template.store["vars"].values():
        for v in (vs if isinstance(vs, tuple) else (vs,)):
            if v is not None:
                ids.add(id(v))
    return ids


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = {}
    out.update(run_reference_gan("dcgan", 1357))
    out.update(run_reference_gan("wgan", 2468))
    np.savez_compressed(os.path.join(HERE, "ref_gan.npz"), **out)
    with open(os.path.join(HERE, "ref_gan_digests.json"), "w") as f:
        json.dump(digests("ref_gan", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("dcgan gen %.6g disc %.6g, wgan gen %.6g disc %.6g, %d arrays"
          % (out["dcgan/gen_loss"], out["dcgan/disc_loss"], out["wgan/gen_loss"],
             out["wgan/disc_loss"], len(out)))


if __name__ == "__main__":
    main()
