"""The categorical epilogues of the dense-layer kernel (zs.fused.LinearOnehotCategorical: EPI 12 -
14) keep everything in registers: in the built library every instance exists and has no stack frame
and no local memory.  CPU only (reads the library's resource usage with cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_categorical_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*?tc_pipeline_kernel\w*CatEpiELi(\d+)ELi0ELi(\d)\w*):\s*\n"
                       r"\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    # EPI 12, 13 and 14, each on the three-product and the binary (two-product) mainloop
    assert sorted((int(e), int(z)) for _, e, z, _, _, _ in found) == \
        [(e, z) for e in (12, 13, 14) for z in (0, 2)], [f[0] for f in found]
    for name, _, _, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
