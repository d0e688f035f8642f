"""The dense_impl=5 leapfrog pass on thread-block clusters.

Where the unit grid tiles by the cluster (an even number of 128-dimension blocks and of
128-chain blocks), the pass runs as 2 x 2 clusters that fetch each shared operand tile from L2
once and multicast it; other shapes run without clusters.  The SASS test pins that only the
cluster instantiations of the pass issue multicast TMA loads.  The GPU tests run both sides of
that rule, with ragged last chain blocks (a multicast half-tile may lie wholly past the last
chain), against the float64 oracle and against the one-launch-per-pass path (dense_impl=2)."""
import re

import numpy as np
import pytest
import torch

from oracle import hmc as OH
from oracle import models as OM
from zhusuan_b200 import _lib

from test_sass_mainloop import _cuobjdump, _tc_kernels


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def test_only_clustered_res_pass_multicasts():
    import subprocess
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout
    kernels = _tc_kernels(sass)
    clustered, plain = 0, 0
    for name, instrs in kernels.items():
        mc = sum("UTMALDG" in i and "MULTICAST" in i for i in instrs)
        # ResW<MODE, NEXT, DC, CX, CY>: the last two template arguments are the cluster shape
        m = re.search(r"ResWILi-?\d+ELi-?\d+ELi-?\d+ELi(\d+)ELi(\d+)E", name)
        if m and int(m.group(1)) * int(m.group(2)) > 1:
            clustered += 1
            assert mc > 0, name
        else:
            plain += 1
            assert mc == 0, name
    assert clustered == 6, "expected 3 pass modes x 2 dimension specialisations on clusters"
    assert plain > 0


@pytest.mark.gpu
@pytest.mark.parametrize("D,C,L", [(320, 3 * 128 + 5, 2), (256, 3 * 128 + 5, 2),
                                   (256, 300, 3), (512, 200, 3), (384, 256, 1)])
def test_resident_cluster_and_plain_shapes_vs_oracle(zs, D, C, L):
    """dense_impl=5, one iteration vs the oracle, with a mean vector: clustered shapes with a
    ragged last chain block, and shapes that run without clusters (odd dimension blocks, odd
    chain blocks)."""
    rng = np.random.RandomState(D + C + L)
    P, const = OM.make_dense_gaussian_problem(D, seed=4)
    mu = (0.3 * rng.standard_normal(D)).astype(np.float32)
    q0 = rng.standard_normal((C, D)).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    om = OM.DenseGaussian(P.astype(np.float32), mu, const)
    oq, oi = OH.HMC(step_size=0.12, n_leapfrogs=L).step([q0], om.logp, om.grad, [npz], u)
    x = T(q0)
    h = zs.HMC(step_size=0.12, n_leapfrogs=L, dense_impl=5)
    lj = zs.fused.GaussianLogJoint(P, mean=mu, log_det_cov=-2 * const - D * np.log(2 * np.pi))
    op, info = h.sample(lj, {}, {"x": x})
    assert h._res
    op(noise={"p": {"x": T(npz)}, "u": T(u)})
    op.synchronize()
    np.testing.assert_allclose(N(info.orig_hamiltonian), oi.orig_hamiltonian, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(N(info.hamiltonian), oi.hamiltonian, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(N(info.acceptance_rate), oi.acceptance_rate, rtol=2e-4, atol=1e-4)
    near = np.abs(u - oi.acceptance_rate) < 1e-3
    np.testing.assert_allclose(N(x)[~near], oq[0][~near], rtol=2e-5, atol=2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("D,C,L", [(1024, 2 * 128 + 5, 3), (1024, 5 * 128 + 5, 3),
                                   (320, 5 * 128 + 5, 2), (256, 3 * 128 + 5, 4)])
def test_resident_cluster_and_plain_shapes_match_per_pass_kernel(zs, D, C, L):
    """dense_impl=5 against dense_impl=2 (one launch per pass, no clusters): same operands and
    products, so the chains agree to fp32 rounding on both sides of the cluster rule (the
    second and last shapes run on clusters)."""
    P, _ = OM.make_dense_gaussian_problem(D, seed=2)
    res = []
    for im in (2, 5):
        torch.manual_seed(5)
        x = torch.randn(C, D, device="cuda")
        h = zs.HMC(step_size=0.1, n_leapfrogs=L, seed=7, dense_impl=im)
        op, info = h.sample(zs.fused.GaussianLogJoint(P), {}, {"x": x})
        for _ in range(2):
            op()
        op.synchronize()
        res.append((N(x), N(info.hamiltonian), N(info.acceptance_rate)))
    np.testing.assert_allclose(res[1][1], res[0][1], rtol=1e-5)
    np.testing.assert_allclose(res[1][2], res[0][2], rtol=0, atol=2e-3)
    same = np.abs(res[1][2] - res[0][2]) < 1e-6
    np.testing.assert_allclose(res[1][0][same], res[0][0][same], rtol=1e-4, atol=1e-4)
