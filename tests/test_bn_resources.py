"""Every batch-norm kernel (the BnEpi epilogues of the tensor-core product, the moment merge, the
affine pass and the backward passes of gemm_logjoint_tc.cu) keeps everything in registers: in the
built library each instance exists once and has no stack frame and no local memory.  CPU only
(reads the library's resource usage with cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib

# mangled-name fragment of each instance
BN_KERNELS = {
    "EPI 9": r"BnEpiELi9ELi0ELi0E",
    "EPI 9, 0/1 sample": r"BnEpiELi9ELi0ELi2E",
    "EPI 10": r"BnEpiELi10ELi0ELi0E",
    "EPI 11": r"BnEpiELi11ELi0ELi0E",
    "EPI 11, 0/1 sample": r"BnEpiELi11ELi0ELi2E",
    "stats": r"bn_stats_kernelILb0E",
    "stats, Bessel": r"bn_stats_kernelILb1E",
    "apply": r"bn_apply_kernelILb0E",
    "apply, gamma": r"bn_apply_kernelILb1E",
    "grad sums": r"bn_grad_sums_kernelE",
    "grad combine": r"bn_grad_combine_kernelE",
    "grad apply, max pass": r"bn_grad_apply_kernelILNS_9BnGradOutE0E",
    "grad apply, planes": r"bn_grad_apply_kernelILNS_9BnGradOutE1E",
    "grad apply, fp32": r"bn_grad_apply_kernelILNS_9BnGradOutE2E",
}


def test_no_bn_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    for kind, pat in BN_KERNELS.items():
        mine = [f for f in found if re.search(pat, f[0])]
        assert len(mine) == 1, (kind, [f[0] for f in mine])
        name, reg, stack, local = mine[0]
        assert int(stack) == 0 and int(local) == 0, (kind, name, reg, stack, local)
