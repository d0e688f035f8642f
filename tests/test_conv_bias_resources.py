"""The passes of the biased tensor-core convolutions (zs.fused.conv2d_tc, conv2d_transpose_tc):
the col2im with bias, residual and ReLU and the ReLU gradient of csrc/conv_bias.cu, and the
residual epilogue of the dense-layer kernel (EPI 16), exist in the built library with no stack
frame and no local memory, so none of them spills.  CPU only (reads the library's resource usage
with cuobjdump)."""
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


def test_no_conv_bias_kernel_spills():
    found = re.findall(r"Function (\S*conv_bias\S*?(col2im_bias_kernel|relu_grad_kernel)\S*):"
                       r"\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", _res_usage())
    assert sorted(k for _, k, _, _, _ in found) == ["col2im_bias_kernel", "relu_grad_kernel"], \
        [f[0] for f in found]
    for name, _, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)


def test_no_residual_epilogue_spills():
    found = re.findall(r"Function (\S*?tc_pipeline_kernel\w*RowsEpiELi16ELi(\d)ELi(\d)\w*):\s*\n"
                       r"\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", _res_usage())
    # EPI 16 on the three-product forward mainloop only
    assert [(int(mn), int(z)) for _, mn, z, _, _, _ in found] == [(0, 0)], [f[0] for f in found]
    for name, _, _, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
