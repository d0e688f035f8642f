"""The convolution kernels of csrc/conv.cu keep their accumulators in registers: in the built
library every instance exists and has no stack frame and no local memory, so none of them spills.
CPU only (reads the library's resource usage with cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_conv_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*conv3x3_\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ "
                       r"LOCAL:(\d+)", out)
    kinds = {re.search(r"conv3x3_(fwd|wgrad_merge|wgrad)_kernel", name).group(1)
             for name, *_ in found}
    assert kinds == {"fwd", "wgrad", "wgrad_merge"}, kinds
    assert len(found) == 5, [name for name, *_ in found]
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
