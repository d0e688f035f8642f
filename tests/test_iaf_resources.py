"""The inverse-autoregressive-flow kernels of csrc/iaf.cu keep their tiles in shared memory and
their accumulators in registers: in the built library every instance has no stack frame and no
local memory, so none of them spills.  CPU only (reads the library's resource usage with
cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_iaf_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*iaf_\w+_kernel\w*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ "
                       r"LOCAL:(\d+)", out)
    kinds = {re.search(r"iaf_(fwd|bwd|merge)_kernel", name).group(1) for name, *_ in found}
    assert kinds == {"fwd", "bwd", "merge"}, kinds
    assert len(found) == 7, [f[0] for f in found]
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
