"""The dense_impl=5 leapfrog pass on its five-stage operand ring and 2 x 1 clusters.

The GPU test runs shapes with fewer k-blocks per unit than the ring has stages (D = 64, 192), with
ragged last dimension and chain blocks, and on both sides of the cluster rule (an even number of
dimension blocks runs on clusters of two), against the one-launch-per-pass path
(dense_impl=2).  The SASS test pins that the shipped library's tensor-core kernels read no cycle
counter: the stall accounting that does (ZSB_PASS_PROFILE, scripts/pass_stalls.py) stays out of
the default build."""
import subprocess

import numpy as np
import pytest
import torch

from oracle import models as OM
from zhusuan_b200 import _lib

from test_sass_mainloop import _cuobjdump, _tc_kernels


def test_shipped_tc_kernels_read_no_clock():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout
    kernels = _tc_kernels(sass)
    assert kernels
    clocked = {name: n for name, n in
               ((k, sum("SR_CLOCKLO" in i or "SR_CLOCKHI" in i for i in v))
                for k, v in kernels.items()) if n}
    assert not clocked, "cycle-counter reads in the shipped tensor-core kernels: %r" % clocked


@pytest.mark.gpu
@pytest.mark.parametrize("D,C,L", [(64, 5, 2),              # 2 k-blocks per unit, one chain block
                                   (192, 77, 2),            # clusters, ragged blocks both ways
                                   (512, 3 * 128 + 5, 3),   # clusters, ragged last chain block
                                   (1024, 3 * 128 + 2, 2),  # clusters, 2 chains in the last block
                                   (320, 4 * 128 + 1, 3)])  # odd dimension blocks: no clusters
def test_resident_ring_and_clusters_match_per_pass_kernel(D, C, L):
    import zhusuan_b200 as zs
    P, _ = OM.make_dense_gaussian_problem(D, seed=3)
    res = []
    for im in (2, 5):
        torch.manual_seed(11)
        x = torch.randn(C, D, device="cuda")
        h = zs.HMC(step_size=0.1, n_leapfrogs=L, seed=5, dense_impl=im)
        op, info = h.sample(zs.fused.GaussianLogJoint(P), {}, {"x": x})
        for _ in range(2):
            op()
        op.synchronize()
        res.append([t.detach().cpu().numpy() for t in (x, info.hamiltonian,
                                                       info.acceptance_rate)])
    assert np.isfinite(res[1][0]).all()
    np.testing.assert_allclose(res[1][1], res[0][1], rtol=1e-5)
    np.testing.assert_allclose(res[1][2], res[0][2], rtol=0, atol=2e-3)
    same = np.abs(res[1][2] - res[0][2]) < 1e-6
    np.testing.assert_allclose(res[1][0][same], res[0][0][same], rtol=1e-4, atol=1e-4)
