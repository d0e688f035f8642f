"""tests/golden/ref_vae_conv.npz: the convolutional VAE of
examples/variational_autoencoders/vae_conv.py at small widths on THE REFERENCE'S OWN BayesianNet,
Normal, Bernoulli and elbo().sgvb(), executed on the NumPy TensorFlow stand-in of oracle/tf_shim
(TEST INFRASTRUCTURE).

    python tests/golden/make_ref_vae_conv_golden.py  ->  ref_vae_conv.npz, ref_vae_conv_digests.json

It writes only these two files.  It needs the reference checkout (ZHUSUAN_REFERENCE, default
/root/reference); the outputs are committed.

examples/utils cannot be imported on the stand-in (it pulls in tf.contrib.layers' initialisers and
arg scopes), so build_gen, build_q_net and the two resnet blocks (vae_conv.py:20-93) and the
conv2d_transpose helper (examples/utils/utils.py:74-113) are restated below with line citations.
The stand-in lacks the convolution ops; they are installed onto it here, in NumPy, straight from
TensorFlow's SAME definition (Ho = ceil(H / s), pad_total = max((Ho - 1) s + 3 - H, 0),
pad_before = pad_total // 2), with their gradients:
  * tf.layers.conv2d(x, Cout, 3, strides, padding="same", activation), kernel [3, 3, Cin, Cout];
  * tf.nn.conv2d_transpose(x, w, output_shape, strides, padding="SAME"), w [3, 3, Cout, Cin], the
    adjoint of the convolution from output_shape to x's shape;
  * tf.nn.bias_add and tf.layers.flatten.
`tf.get_variable` / `tf.variable_scope` and `tf.sigmoid` come from the stand-in.  The stand-in
itself is unchanged for every other fixture.  This shares no code with tests/vae_conv_oracle.py
(F.pad + F.conv2d, F.conv_transpose2d + crop) nor with zs.fused.

Widths: nf = 2, z_dim = 4, 3 images, 1 particle; q's eps is injected with tf.set_noise.  Weights
are Glorot-uniform draws rounded to a grid of 2^-8, biases are loaded with non-zero values on a
grid of 2^-9.

Recorded: x, eps, every parameter (conv kernels [3, 3, Cin, Cout], transposed-conv weights
[3, 3, Cout, Cin], dense kernels stored [out, in]) as q{i} / p{i} in the order the networks read
them, except those of more than PROJ_MIN entries, which are `seeded_param` draws; bound
(tf.reduce_mean of the elbo), cost (tf.reduce_mean of sgvb()), x_mean [1, 3, 784]; and
tf.gradients of the cost w.r.t. every parameter.  Gradients of more than GRAD_PROJ_MIN entries
are stored as their projections onto 8 fixed vectors (`proj_vectors`), so the file stays small.
"""
import hashlib
import importlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

NF, Z_DIM, N, S, X_DIM = 2, 4, 3, 1, 784
PROJ_MIN, GRAD_PROJ_MIN, PROJ_K, PROJ_SEED = 2000, 300, 8, 20261017


def seeded_param(name, shape):
    """A parameter of more than PROJ_MIN entries is not stored: it is this seeded draw (uniform on
    Glorot's range for a dense kernel stored [out, in], on a grid of 2^-8), which a replay
    regenerates from its name and shape."""
    tag = (1000 if name[0] == "q" else 2000) + int(name[1:])
    limit = np.sqrt(6.0 / (shape[0] + shape[1]))
    v = np.random.default_rng([PROJ_SEED, tag]).uniform(-limit, limit, shape)
    return (np.round(v * 256) / 256).astype(np.float32)


def proj_vectors(index, size):
    """The fixed vectors gradient `index` (of `size` entries) is projected onto: [PROJ_K, size]."""
    return np.random.default_rng([PROJ_SEED, index]).standard_normal((PROJ_K, size))


# ---- SAME 3x3 convolution in NumPy -----------------------------------------------------------------

def _pads(big, small, s):
    total = max((small - 1) * s + 3 - big, 0)
    return total // 2


def np_conv(x, w, s):
    """y[n, i, j] = sum_{kh, kw} x[n, s i + kh - pt, s j + kw - pl] . w[kh, kw] (x zero outside)."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    N_, H, W_, _ = x.shape
    Ho, Wo = -(-H // s), -(-W_ // s)
    pt, pl = _pads(H, Ho, s), _pads(W_, Wo, s)
    xp = np.zeros((N_, (Ho - 1) * s + 3, (Wo - 1) * s + 3, x.shape[3]))
    hh, ww = min(H, xp.shape[1] - pt), min(W_, xp.shape[2] - pl)
    xp[:, pt:pt + hh, pl:pl + ww] = x[:, :hh, :ww]
    y = np.zeros((N_, Ho, Wo, w.shape[3]))
    for kh in range(3):
        for kw in range(3):
            y += xp[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s] @ w[kh, kw]
    return y


def np_conv_adjoint(g, w, s, big_hw):
    """The adjoint of np_conv(., w, s) from [H, W, Cin] (big_hw) to g's [Ho, Wo, Cout]."""
    g, w = np.asarray(g, np.float64), np.asarray(w, np.float64)
    N_, Ho, Wo, _ = g.shape
    H, W_ = big_hw
    pt, pl = _pads(H, Ho, s), _pads(W_, Wo, s)
    xp = np.zeros((N_, (Ho - 1) * s + 3, (Wo - 1) * s + 3, w.shape[2]))
    for kh in range(3):
        for kw in range(3):
            xp[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s] += g @ w[kh, kw].T
    out = np.zeros((N_, H, W_, w.shape[2]))
    hh, ww = min(H, xp.shape[1] - pt), min(W_, xp.shape[2] - pl)
    out[:, :hh, :ww] = xp[:, pt:pt + hh, pl:pl + ww]
    return out


def np_conv_wgrad(x, g, s):
    """d <np_conv(x, w, s), g> / d w: [3, 3, Cin, Cout]."""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    N_, H, W_, _ = x.shape
    Ho, Wo = g.shape[1], g.shape[2]
    pt, pl = _pads(H, Ho, s), _pads(W_, Wo, s)
    xp = np.zeros((N_, (Ho - 1) * s + 3, (Wo - 1) * s + 3, x.shape[3]))
    hh, ww = min(H, xp.shape[1] - pt), min(W_, xp.shape[2] - pl)
    xp[:, pt:pt + hh, pl:pl + ww] = x[:, :hh, :ww]
    dw = np.zeros((3, 3, x.shape[3], g.shape[3]))
    for kh in range(3):
        for kw in range(3):
            xs = xp[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s]
            dw[kh, kw] = np.einsum("nijc,nijd->cd", xs, g)
    return dw


def _install_ops(tf, created):
    f32 = lambda a: np.asarray(a, np.float32)                          # noqa: E731

    def conv_op(x, w, s):
        out = tf.Tensor(lambda c: f32(np_conv(c.eval(x), c.eval(w), s)), inputs=(x, w),
                        op="conv2d", dtype=np.float32)

        def vjp(g):
            dx = tf.Tensor(lambda c: f32(np_conv_adjoint(c.eval(g), c.eval(w), s,
                                                         np.shape(c.eval(x))[1:3])),
                           inputs=(g, w, x), op="conv2d_dx", dtype=np.float32)
            dw = tf.Tensor(lambda c: f32(np_conv_wgrad(c.eval(x), c.eval(g), s)),
                           inputs=(x, g), op="conv2d_dw", dtype=np.float32)
            return [dx, dw]
        out.vjp = vjp
        return out

    def conv2d(inputs, filters, kernel_size, strides=(1, 1), padding="valid", activation=None,
               use_bias=True, name=None, **kw):
        assert kernel_size in (3, (3, 3)) and padding.lower() == "same"
        s = strides if isinstance(strides, int) else strides[0]
        store = tf._TEMPLATES[-1] if tf._TEMPLATES else tf._DEFAULT_STORE
        k = store["count"]
        store["count"] += 1
        key = name or "conv2d_%d" % k
        inputs = tf.convert_to_tensor(inputs)
        if key not in store["vars"]:
            cin = int(inputs.get_shape().as_list()[-1])
            limit = np.sqrt(6.0 / (9 * cin + 9 * filters))               # glorot_uniform
            w0 = tf._INIT["rng"].uniform(-limit, limit, (3, 3, cin, filters)).astype(np.float32)
            kern = tf.Variable(w0, name=key + "/kernel")
            bias = tf.Variable(np.zeros(filters, np.float32), name=key + "/bias")
            store["vars"][key] = (kern, bias)
            tf._TRAINABLE.extend([kern, bias])
            created.extend([kern, bias])
        kern, bias = store["vars"][key]
        y = conv_op(inputs, kern, s)
        if use_bias:
            y = y + bias
        return activation(y) if activation is not None else y

    def conv2d_transpose(value, filter, output_shape, strides, padding="SAME", name=None, **kw):
        assert padding == "SAME"
        s = strides[1]
        x, w = tf.convert_to_tensor(value), tf.convert_to_tensor(filter)

        def big_hw(c):
            return tuple(int(c.eval(v)) if isinstance(v, tf.Tensor) else int(v)
                         for v in output_shape[1:3])
        out = tf.Tensor(lambda c: f32(np_conv_adjoint(c.eval(x), c.eval(w), s, big_hw(c))),
                        inputs=(x, w), op="conv2d_transpose", dtype=np.float32)

        def vjp(g):
            dx = tf.Tensor(lambda c: f32(np_conv(c.eval(g), c.eval(w), s)), inputs=(g, w),
                           op="conv2d_transpose_dx", dtype=np.float32)
            dw = tf.Tensor(lambda c: f32(np_conv_wgrad(c.eval(g), c.eval(x), s)),
                           inputs=(g, x), op="conv2d_transpose_dw", dtype=np.float32)
            return [dx, dw]
        out.vjp = vjp
        return out

    def flatten(inputs, name=None):
        a = tf.convert_to_tensor(inputs)
        return tf.Tensor(lambda c: np.reshape(c.eval(a), (np.shape(c.eval(a))[0], -1)),
                         inputs=(a,), op="flatten", vjp=lambda g: [tf.reshape(g, tf.shape(a))],
                         dtype=a._dtype)

    tf.layers.conv2d = staticmethod(conv2d)
    tf.layers.flatten = staticmethod(flatten)
    tf.nn.conv2d_transpose = staticmethod(conv2d_transpose)
    tf.nn.bias_add = staticmethod(lambda value, bias, name=None: value + bias)


def _grid(rng, shape, std):
    v = np.round(std * rng.standard_normal(shape) * 512) / 512
    v[v == 0] = 1.0 / 512
    return v.astype(np.float32)


def run_reference_vae_conv(seed=2718):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.tf_shim import make_ref_golden as mrg
    tf, _, _ = mrg.load_reference()
    created = []
    _install_ops(tf, created)
    fw = importlib.import_module("zhusuan.framework")
    var = importlib.import_module("zhusuan.variational")
    rng = np.random.Generator(np.random.PCG64(seed))
    tf.reset_default_graph()
    tf.set_init_rng(rng)

    def conv2d_transpose(inputs, out_shape, kernel_size=(5, 5), stride=(1, 1),
                         activation_fn=tf.nn.relu):                 # utils.py:74-113
        batchsize = tf.shape(inputs)[0]
        in_channels = int(inputs.get_shape()[-1])
        output_shape = [batchsize, out_shape[0], out_shape[1], out_shape[2]]
        filter_shape = [kernel_size[0], kernel_size[1], out_shape[2], in_channels]
        store = tf._TEMPLATES[-1] if tf._TEMPLATES else tf._DEFAULT_STORE
        scope = "Conv2d_transpose_%d" % store["count"]            # variable_scope's default name
        store["count"] += 1
        fan_in, fan_out = 9 * in_channels, 9 * out_shape[2]
        limit = np.sqrt(6.0 / (fan_in + fan_out))                   # xavier_initializer()
        w = tf.get_variable(scope + "/weights", filter_shape, initializer=lambda shape: rng.uniform(
            -limit, limit, shape).astype(np.float32))
        outputs = tf.nn.conv2d_transpose(inputs, w, output_shape=output_shape,
                                         strides=[1, stride[0], stride[1], 1])
        biases = tf.get_variable(scope + "/biases", [out_shape[2]],
                                 initializer=tf.constant_initializer(0.0))
        outputs = tf.nn.bias_add(outputs, biases)
        if activation_fn is not None:
            outputs = activation_fn(outputs)
        return outputs

    def deconv_resnet_block(input_, out_shape, resize=False):       # vae_conv.py:20-36
        if not resize:
            lx_z = conv2d_transpose(input_, out_shape, kernel_size=(3, 3), stride=(1, 1))
            lx_z = conv2d_transpose(lx_z, out_shape, kernel_size=(3, 3), stride=(1, 1),
                                    activation_fn=None)
            lx_z += input_
        else:
            lx_z = conv2d_transpose(input_, input_.get_shape().as_list()[1:],
                                    kernel_size=(3, 3), stride=(1, 1))
            lx_z = conv2d_transpose(lx_z, out_shape, kernel_size=(3, 3), stride=(2, 2),
                                    activation_fn=None)
            residual = conv2d_transpose(input_, out_shape, kernel_size=(3, 3), stride=(2, 2),
                                        activation_fn=None)
            lx_z += residual
        lx_z = tf.nn.relu(lx_z)
        return lx_z

    def conv_resnet_block(input_, out_channel, resize=False):       # vae_conv.py:39-53
        if not resize:
            lz_x = tf.layers.conv2d(input_, out_channel, 3, padding="same",
                                    activation=tf.nn.relu)
            lz_x = tf.layers.conv2d(lz_x, out_channel, 3, padding="same")
            lz_x += input_
        else:
            lz_x = tf.layers.conv2d(input_, out_channel, 3, strides=(2, 2), padding="same",
                                    activation=tf.nn.relu)
            lz_x = tf.layers.conv2d(lz_x, out_channel, 3, padding="same")
            residual = tf.layers.conv2d(input_, out_channel, 3, strides=(2, 2), padding="same")
            lz_x += residual
        lz_x = tf.nn.relu(lz_x)
        return lz_x

    @fw.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, x_dim, z_dim, n_particles, nf=16):             # vae_conv.py:56-73
        bn = fw.BayesianNet()
        z_mean = tf.zeros([n, z_dim])
        z = bn.normal("z", z_mean, std=1., group_ndims=1, n_samples=n_particles)
        lx_z = tf.layers.dense(z, 7 * 7 * nf * 2, activation=tf.nn.relu)
        lx_z = tf.reshape(lx_z, [-1, 7, 7, nf * 2])
        lx_z = deconv_resnet_block(lx_z, [7, 7, nf * 2])
        lx_z = deconv_resnet_block(lx_z, [14, 14, nf * 2], resize=True)
        lx_z = deconv_resnet_block(lx_z, [14, 14, nf * 2])
        lx_z = deconv_resnet_block(lx_z, [28, 28, nf], resize=True)
        lx_z = deconv_resnet_block(lx_z, [28, 28, nf])
        lx_z = conv2d_transpose(lx_z, [28, 28, 1], kernel_size=(3, 3), stride=(1, 1),
                                activation_fn=None)
        x_logits = tf.reshape(lx_z, [n_particles, -1, x_dim])
        bn.deterministic("x_mean", tf.sigmoid(x_logits))
        bn.bernoulli("x", x_logits, group_ndims=1)
        return bn

    @fw.reuse_variables(scope="q_net")
    def build_q_net(x, z_dim, n_particles, nf=16):                  # vae_conv.py:76-93
        bn = fw.BayesianNet()
        lz_x = 2 * tf.cast(x, tf.float32) - 1
        lz_x = tf.reshape(lz_x, [-1, 28, 28, 1])
        lz_x = tf.layers.conv2d(lz_x, nf, 3, padding="same", activation=tf.nn.relu)
        lz_x = conv_resnet_block(lz_x, nf)
        lz_x = conv_resnet_block(lz_x, nf * 2, resize=True)
        lz_x = conv_resnet_block(lz_x, nf * 2)
        lz_x = conv_resnet_block(lz_x, nf * 2, resize=True)
        lz_x = conv_resnet_block(lz_x, nf * 2)
        lz_x = tf.layers.flatten(lz_x)
        lz_x = tf.layers.dense(lz_x, 500, activation=tf.nn.relu)
        z_mean = tf.layers.dense(lz_x, z_dim)
        z_logstd = tf.layers.dense(lz_x, z_dim)
        bn.normal("z", z_mean, logstd=z_logstd, group_ndims=1, n_samples=n_particles)
        return bn

    x_np = (rng.random((N, X_DIM)) < 0.4).astype(np.int32)
    x = tf.constant(x_np)
    n_particles = S             # vae_conv.py feeds 1 through a placeholder (vae_conv.py:147-150)
    model = build_gen(N, X_DIM, Z_DIM, n_particles, nf=NF)           # vae_conv.py:104-114
    variational = build_q_net(x, Z_DIM, n_particles, nf=NF)
    q_vars = list(tf.trainable_variables())
    lower_bound = var.elbo(model, {"x": x}, variational=variational, axis=0)
    cost = tf.reduce_mean(lower_bound.sgvb())
    lower_bound = tf.reduce_mean(lower_bound)
    qz = variational.outputs("z")
    x_mean = model.observe(x=x, z=qz)["x_mean"]
    p_vars = [v for v in tf.trainable_variables() if all(v is not u for u in q_vars)]

    out = {"x": x_np.astype(np.uint8)}
    params = []
    for tag, vs in (("q", q_vars), ("p", p_vars)):
        for i, v in enumerate(vs):
            name = "%s%d" % (tag, i)
            if v.value.ndim == 1:
                v.load(_grid(rng, v.value.shape, 0.3))
            elif v.value.size > PROJ_MIN:                               # dense kernel [in, out]
                v.load(np.ascontiguousarray(seeded_param(name, v.value.shape[::-1]).T))
            else:                       # the Glorot draw on a grid of 2^-8: a small, exact file
                v.load((np.round(v.value * 256) / 256).astype(np.float32))
            if v.value.size <= PROJ_MIN:
                val = v.value.T if v.value.ndim == 2 else v.value       # dense: [out, in]
                out[name] = np.ascontiguousarray(val, np.float32)
            params.append((name, v))

    eps = rng.standard_normal((S, N, Z_DIM)).astype(np.float32)
    tf.set_noise(normal=[eps])
    sess = tf.Session()
    r = sess.run([lower_bound, cost, x_mean] + tf.gradients(cost, [v for _, v in params]),
                 feed_dict={})
    assert not tf._NOISE["normal"]
    out.update({"eps": eps, "bound": np.float32(r[0]), "cost": np.float32(r[1]),
                "x_mean": np.asarray(r[2], np.float32)})
    for k, ((name, v), g) in enumerate(zip(params, r[3:])):
        g = np.asarray(g, np.float64)
        g = g.T if g.ndim == 2 else g
        if g.size > GRAD_PROJ_MIN:
            out["grad_proj_" + name] = (proj_vectors(k, g.size) @ g.ravel()).astype(np.float32)
        else:
            out["grad_" + name] = np.ascontiguousarray(g, np.float32)
    return out


def digests(name, out):
    res = {}
    for k in sorted(out):
        a = np.ascontiguousarray(out[k])
        res[name + "/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    return res


def main():
    out = run_reference_vae_conv()
    np.savez_compressed(os.path.join(HERE, "ref_vae_conv.npz"), **out)
    with open(os.path.join(HERE, "ref_vae_conv_digests.json"), "w") as f:
        json.dump(digests("ref_vae_conv", out), f, indent=1, sort_keys=True)
        f.write("\n")
    print("bound %.6g, cost %.6g, %d arrays" % (out["bound"], out["cost"], len(out)))


if __name__ == "__main__":
    main()
