"""CPU pins of the convolutional VAE port (examples/variational_autoencoders/vae_conv.py):
tests/golden/ref_vae_conv.npz (made by tests/golden/make_ref_vae_conv_golden.py from the
reference's own BayesianNet and elbo().sgvb() on the NumPy TF stand-in) matches its digests and is
reproduced by the float64 oracle of tests/vae_conv_oracle.py; the oracle's SAME padding rule on the
worked 4x4 example; the adjoint identity between its conv2d and conv2d_transpose in float64 over
even and odd sizes at both strides; the example's shapes; and the new public names."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import vae_conv_oracle as VC

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden():
    """(npz, generator module, q, p) of the fixture: parameters as float64 arrays in the oracle's
    order; the ones too large to store are regenerated from their seed."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "make_ref_vae_conv_golden", os.path.join(GOLD, "make_ref_vae_conv_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(os.path.join(GOLD, "ref_vae_conv.npz"))
    qs, ps = VC.param_shapes(mk.NF, mk.Z_DIM)
    params = []
    for tag, shapes in (("q", qs), ("p", ps)):
        vals = []
        for i, shp in enumerate(shapes):
            name = "%s%d" % (tag, i)
            a = g[name] if name in g.files else mk.seeded_param(name, shp)
            assert tuple(a.shape) == tuple(shp), (name, a.shape, shp)
            vals.append(np.asarray(a, np.float64))
        params.append(vals)
    return g, mk, params[0], params[1]


def golden_grad_checks(g, mk, grads, close):
    """Compare gradients (q then p, the oracle's layouts) with the fixture's recorded values or
    projections; `close(got, want, what)` on NumPy float64 arrays."""
    qs, ps = VC.param_shapes(mk.NF, mk.Z_DIM)
    names = ["q%d" % i for i in range(len(qs))] + ["p%d" % i for i in range(len(ps))]
    assert len(grads) == len(names)
    for k, (name, got) in enumerate(zip(names, grads)):
        got = np.asarray(got, np.float64)
        if "grad_" + name in g.files:
            close(got, g["grad_" + name], "grad " + name)
        else:
            close(mk.proj_vectors(k, got.size) @ got.ravel(), g["grad_proj_" + name],
                  "projected grad " + name)


def _close(got, want, what, rtol, atol):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=rtol,
                               atol=atol * max(1.0, np.abs(want).max()), err_msg=what)


def test_fixture_matches_digests():
    g = np.load(os.path.join(GOLD, "ref_vae_conv.npz"))
    with open(os.path.join(GOLD, "ref_vae_conv_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_vae_conv/" + k] = [str(a.dtype), list(a.shape),
                                    hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def test_oracle_reproduces_the_reference_run():
    """Bound, cost, x_mean and every parameter gradient of vae_conv.py at nf 2, z_dim 4, 3 images
    and 1 particle, run on the reference's own code."""
    g, mk, q, p = golden()
    q = [torch.tensor(a, requires_grad=True) for a in q]
    p = [torch.tensor(a, requires_grad=True) for a in p]
    x = torch.tensor(g["x"], dtype=torch.float64)
    lw, x_mean = VC.vae_conv(x, torch.tensor(g["eps"], dtype=torch.float64), q, p, mk.NF)
    bound, cost = VC.bound_and_cost(lw)
    _close(bound.detach().numpy(), g["bound"], "bound", 1e-5, 1e-6)
    _close(cost.detach().numpy(), g["cost"], "cost", 1e-5, 1e-6)
    _close(x_mean.detach().numpy(), g["x_mean"], "x_mean", 1e-4, 1e-6)
    grads = [t.numpy() for t in torch.autograd.grad(cost, q + p)]
    golden_grad_checks(g, mk, grads, lambda a, w, what: _close(a, w, what, 2e-4, 2e-5))


def test_same_pads():
    assert VC.same_pads(28, 28, 1) == (1, 1)
    assert VC.same_pads(28, 14, 2) == (0, 1)
    assert VC.same_pads(14, 7, 2) == (0, 1)
    assert VC.same_pads(13, 7, 2) == (1, 1)
    assert VC.same_pads(1, 1, 2) == (1, 1)
    assert VC.same_pads(2, 1, 2) == (0, 1)


def test_worked_4x4_example():
    """1..16 row-major, all-ones weights, stride 2: SAME gives [[54, 45], [72, 54]]; torch's
    symmetric padding=1 gives [[14, 30], [57, 99]]."""
    x = torch.arange(1, 17, dtype=torch.float64).reshape(1, 4, 4, 1)
    W = torch.ones(3, 3, 1, 1, dtype=torch.float64)
    y = VC.conv2d(x, W, stride=2)[0, :, :, 0]
    np.testing.assert_array_equal(y.numpy(), [[54, 45], [72, 54]])
    sym = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1), stride=2,
                                     padding=1)[0, 0]
    np.testing.assert_array_equal(sym.numpy(), [[14, 30], [57, 99]])


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("H,Wd", [(1, 1), (2, 2), (4, 4), (5, 9), (7, 7), (13, 14), (28, 28)])
def test_conv2d_transpose_is_the_adjoint_of_conv2d(stride, H, Wd):
    """<conv2d(u), v> = <u, conv2d_transpose(v)> with the same W, in float64."""
    rng = np.random.default_rng(H * 100 + Wd * 10 + stride)
    Cin, Cout, N = 3, 5, 2
    Ho, Wo = -(-H // stride), -(-Wd // stride)
    u = torch.as_tensor(rng.standard_normal((N, H, Wd, Cin)))
    v = torch.as_tensor(rng.standard_normal((N, Ho, Wo, Cout)))
    W = torch.as_tensor(rng.standard_normal((3, 3, Cin, Cout)))
    lhs = (VC.conv2d(u, W, stride=stride) * v).sum()
    # conv2d_transpose maps [Ho, Wo, Cout] -> [H, Wd, Cin] with its W laid out [3, 3, Cin, Cout]
    Tv = VC.conv2d_transpose(v, W, (H, Wd, Cin), stride)
    assert tuple(Tv.shape) == (N, H, Wd, Cin)
    np.testing.assert_allclose(float(lhs), float((u * Tv).sum()), rtol=1e-12)


def test_both_output_sizes_of_a_stride_2_transpose():
    """ceil(Ho / 2) == Hi: 13 and 14 both come from 7, with different pads."""
    v = torch.ones(1, 7, 7, 1, dtype=torch.float64)
    W = torch.ones(3, 3, 1, 1, dtype=torch.float64)
    assert tuple(VC.conv2d_transpose(v, W, (13, 13, 1), 2).shape) == (1, 13, 13, 1)
    assert tuple(VC.conv2d_transpose(v, W, (14, 14, 1), 2).shape) == (1, 14, 14, 1)
    with pytest.raises(AssertionError):
        VC.conv2d_transpose(v, W, (15, 15, 1), 2)


def test_example_shapes():
    """vae_conv.py at small widths: the encoder flattens 7 x 7 x 2 nf, the decoder ends at 784."""
    nf, z_dim = 2, 4
    rng = np.random.default_rng(0)
    q, p = (VC.as_torch(ps) for ps in VC.init_params(rng, nf, z_dim))
    x = torch.as_tensor((rng.random((3, 784)) < 0.5).astype(np.float64))
    eps = torch.as_tensor(rng.standard_normal((1, 3, z_dim)))
    lw, x_mean = VC.vae_conv(x, eps, q, p, nf)
    assert tuple(lw.shape) == (1, 3) and tuple(x_mean.shape) == (1, 3, 784)
    assert torch.isfinite(lw).all()
    qs, ps = VC.param_shapes(nf, z_dim)
    assert [tuple(t.shape) for t in q] == qs and [tuple(t.shape) for t in p] == ps
    assert len(qs) == 2 + 4 * 3 + 6 * 2 + 6 and len(ps) == 2 + 4 * 3 + 6 * 2 + 2


def test_public_names():
    import zhusuan_b200 as zs
    assert "conv2d" in zs.fused.__all__ and "conv2d_transpose" in zs.fused.__all__
    assert callable(zs.fused.conv2d) and callable(zs.fused.conv2d_transpose)
    from zhusuan_b200._lib import lib
    for name in ("zsb_conv3x3_fwd_f32", "zsb_conv3x3_wgrad_parts", "zsb_conv3x3_wgrad_f32"):
        assert name in lib.protos
