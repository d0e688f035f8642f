"""CPU checks of the float64 GAN-layer oracle (tests/gan_oracle.py) against TensorFlow's rules
written as plain loops: SAME / VALID output sizes and asymmetric pads for even and odd k at
strides 1 and 2, the transposed convolution as the adjoint, and the fused batch norm's Bessel
correction of the moving variance (factor 1 at one pixel)."""
import itertools

import numpy as np
import pytest
import torch

import gan_oracle as GO

GEOMS = list(itertools.product([1, 2, 3, 4, 5], [1, 2], ["SAME", "VALID"], [5, 6, 8]))


def _conv_loops(x, W, s, padding):
    """y[n, i, j, o] = sum x[n, s i + kh - pt, s j + kw - pl, c] W[kh, kw, c, o], TF's pads."""
    N, H, Wd, C = x.shape
    k = W.shape[0]
    if padding == "SAME":
        Ho, Wo = -(-H // s), -(-Wd // s)
        pt = max((Ho - 1) * s + k - H, 0) // 2
        pl = max((Wo - 1) * s + k - Wd, 0) // 2
    else:
        Ho, Wo = -(-(H - k + 1) // s), -(-(Wd - k + 1) // s)
        pt = pl = 0
    y = np.zeros((N, Ho, Wo, W.shape[3]))
    for i in range(Ho):
        for j in range(Wo):
            for kh in range(k):
                for kw in range(k):
                    yy, xx = s * i + kh - pt, s * j + kw - pl
                    if 0 <= yy < H and 0 <= xx < Wd:
                        y[:, i, j] += x[:, yy, xx] @ W[kh, kw]
    return y


@pytest.mark.parametrize("k,s,padding,H", GEOMS)
def test_conv_matches_the_loop_definition(k, s, padding, H):
    if padding == "VALID" and H < k:
        pytest.skip("no VALID output")
    rng = np.random.RandomState(k * 100 + s * 10 + H)
    x = rng.standard_normal((2, H, H + 1, 3))
    W = rng.standard_normal((k, k, 3, 4))
    got = GO.conv2d(torch.tensor(x), torch.tensor(W), s, padding).numpy()
    np.testing.assert_allclose(got, _conv_loops(x, W, s, padding), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("k,s,padding,H", GEOMS)
def test_transpose_is_the_adjoint_with_tf_output_size(k, s, padding, H):
    rng = np.random.RandomState(k * 77 + s * 7 + H)
    x = torch.tensor(rng.standard_normal((2, H, H + 1, 3)))
    W = torch.tensor(rng.standard_normal((k, k, 4, 3)))          # [k, k, Cout, Cin]
    y = GO.conv2d_transpose(x, W, s, padding)
    Hb = H * s + (0 if padding == "SAME" else max(k - s, 0))
    assert tuple(y.shape) == (2, Hb, (H + 1) * s + (0 if padding == "SAME" else max(k - s, 0)), 4)
    # <conv(u), x> = <u, conv_transpose(x)> with conv from the big grid back to x's grid
    u = torch.tensor(rng.standard_normal(tuple(y.shape)))
    cu = GO.conv2d(u, W, s, padding)
    assert tuple(cu.shape) == tuple(x.shape)
    np.testing.assert_allclose(float((cu * x).sum()), float((u * y).sum()), rtol=1e-10)


def test_fused_batch_norm_moving_variance_is_bessel_corrected():
    rng = np.random.RandomState(0)
    a = torch.tensor(rng.standard_normal((2, 3, 5, 4)))
    mm, mv = torch.zeros(4, dtype=torch.float64), torch.ones(4, dtype=torch.float64)
    y, m, v = GO.batch_norm_4d(a, None, torch.zeros(4, dtype=torch.float64), mm, mv, True,
                               momentum=0.9)
    R = 30
    var = a.reshape(-1, 4).var(0, unbiased=False)
    np.testing.assert_allclose(v.numpy(), (0.9 + 0.1 * var * R / (R - 1)).numpy(), rtol=1e-12)
    np.testing.assert_allclose(y.reshape(-1, 4).var(0, unbiased=False).numpy(),
                               (var / (var + 1e-3)).numpy(), rtol=1e-12)
    # one pixel: population variance 0, factor 1, the output is beta
    y1, m1, v1 = GO.batch_norm_4d(a[:1, :1, :1], None, torch.full((4,), 0.5, dtype=torch.float64),
                                  mm, mv, True, momentum=0.9)
    np.testing.assert_allclose(v1.numpy(), np.full(4, 0.9), rtol=1e-15)
    np.testing.assert_allclose(y1.reshape(-1).numpy(), np.full(4, 0.5), rtol=1e-15)
