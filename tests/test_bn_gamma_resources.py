"""The kernels of the batch-norm layer with a learned scale (zs.fused.bn_linear) keep everything in
registers: in the built library every instance exists and has no stack frame and no local memory.
CPU only (reads the library's resource usage with cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_bn_gamma_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    pat = r"(bn_\w*gamma_kernel\w*|tc_pipeline_kernel\w*BnEpiELi11\w*|" \
          r"tc_pipeline_kernel\w*BnEpiELi9ELi0ELi2\w*)"
    found = re.findall(r"Function (\S*?" + pat + r"):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ "
                       r"LOCAL:(\d+)", out)
    # bn_apply_gamma, bn_grad_combine_gamma, bn_grad_apply_gamma (x2); EPI 11 (x2), EPI 9 binary
    assert len(found) == 7, [f[0] for f in found]
    for name, _, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
