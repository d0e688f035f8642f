"""The Gaussian-sampling epilogue of the dense-layer kernel (zs.fused.LinearNormal: EPI 15) and the
layer's backward pass keep everything in registers: in the built library every instance exists and
has no stack frame and no local memory.  CPU only (reads the library's resource usage with
cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def _res_usage():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    return subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout


def test_no_normal_epilogue_spills():
    found = re.findall(r"Function (\S*?tc_pipeline_kernel\w*NormalEpiELi(\d+)ELi0ELi(\d)\w*):\s*\n"
                       r"\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", _res_usage())
    # EPI 15 on the three-product and the binary (two-product) mainloop
    assert sorted((int(e), int(z)) for _, e, z, _, _, _ in found) == [(15, 0), (15, 2)], \
        [f[0] for f in found]
    for name, _, _, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)


def test_no_normal_grad_spills():
    found = re.findall(r"Function (\S*?normal_grad_kernel\w*):\s*\n"
                       r"\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", _res_usage())
    assert len(found) == 1, found
    name, reg, stack, local = found[0]
    assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
