"""CPU checks of zs.fused.RBFKernel and gp_conditional: the public names, the kernel's initialiser
and formula, the shape errors raised before any launch, the generic path against the float64
oracle of tests/svgp_oracle.py, and the oracle's re-associated moments against the reference
order."""
import numpy as np
import pytest
import torch

import svgp_oracle as O
import zhusuan_b200 as zs


def _data(M=7, d=3, B=11, K=4, seed=0):
    rng = np.random.default_rng(seed)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    return T(rng.uniform(-1, 1, (M, d))), T(rng.standard_normal((K, M))), \
        T(rng.standard_normal((B, d))), T(rng.uniform(-0.5, 1.0, d))


def test_public_names():
    assert "RBFKernel" in zs.fused.__all__ and "gp_conditional" in zs.fused.__all__
    assert issubclass(zs.fused.GPConditionalNormal, zs.distributions.Normal)


def test_rbf_kernel_initialiser_and_formula():
    k = zs.fused.RBFKernel(5, device="cpu")
    assert k.k_raw_scale.shape == (5,) and k.k_raw_scale.is_leaf and k.k_raw_scale.requires_grad
    assert torch.equal(k.k_raw_scale, torch.zeros(5))
    torch.testing.assert_close(k.k_scale, torch.full((5,), float(np.log(2.0))))
    with torch.no_grad():
        k.k_raw_scale.add_(1.0)
    torch.testing.assert_close(k.k_scale, torch.full((5,), float(np.log1p(np.e))))
    z, _, x, raw = _data(d=5)
    k = zs.fused.RBFKernel(5, dtype=torch.float64, device="cpu")
    with torch.no_grad():
        k.k_raw_scale.copy_(raw)
    torch.testing.assert_close(k(x, z), O.rbf(x, z, O.softplus(raw)))
    assert torch.equal(k.Kdiag(x), torch.ones(x.shape[0], dtype=torch.float64))
    assert k.Kdiag(x.expand(2, -1, -1)).shape == (2, x.shape[0])
    with pytest.raises(ValueError):
        k(x[0], z)
    with pytest.raises(ValueError):
        k(x, z[None])


@pytest.mark.parametrize("full_cov", [False, True])
def test_generic_path_against_oracle(full_cov):
    z, fz, x, raw = _data()
    k = zs.fused.RBFKernel(3, dtype=torch.float64, device="cpu")
    with torch.no_grad():
        k.k_raw_scale.copy_(raw)
    dist = zs.fused.gp_conditional(z, fz, x, full_cov, k)
    assert not isinstance(dist, zs.fused.GPConditionalNormal)
    mean, second = O.gp_conditional(z, fz, x, O.softplus(raw), full_cov)
    torch.testing.assert_close(dist.mean, mean)
    if full_cov:
        torch.testing.assert_close(dist.cov_tril, second.expand(4, 11, 11))
    else:
        torch.testing.assert_close(dist.std, second)


def test_reassociated_moments_match_reference_order():
    z, fz, x, raw = _data(M=20, d=4, B=30, K=5, seed=1)
    s = O.softplus(raw)
    L = torch.linalg.cholesky(O.rbf(z, z, s) + 0.1 * torch.eye(20, dtype=torch.float64))
    Li = torch.linalg.solve_triangular(L, torch.eye(20, dtype=torch.float64), upper=False)
    m1, s1 = O.gp_conditional(z, fz, x, s, Kzz_chol=L)
    m2, s2 = O.moments_from_factors(x, z, s, Li, fz @ Li.t())
    torch.testing.assert_close(m1, m2, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(s1, s2, rtol=1e-10, atol=1e-10)


def test_shape_errors():
    k = zs.fused.RBFKernel(3, device="cpu")
    z, x, fz = torch.zeros(5, 3), torch.zeros(7, 3), torch.zeros(2, 5)
    for args in [(z[0], fz, x), (z, fz, x[0]), (z, fz[:, :4], x), (z, fz, x[:, :2])]:
        with pytest.raises(ValueError):
            zs.fused.gp_conditional(args[0], args[1], args[2], False, k)
    with pytest.raises(ValueError):
        zs.fused.gp_conditional(z, fz, x, False, k, Kzz_chol=torch.eye(4))
    with pytest.raises(ValueError):
        zs.fused.gp_conditional(z, fz, x, False, zs.fused.RBFKernel(4, device="cpu"))
