"""The topic-model kernels of csrc/lntm.cu keep their state in registers and shared memory: in the
built library every instance (the E-step log-joint for each padded topic count, with and without
padding, phi_t and the three M-step kernels) has no stack frame and no local memory, so none of
them spills.  CPU only (reads the library's resource usage with cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_lntm_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*lntm_\w+_kernel\w*):\s*\n\s*REG:(\d+) STACK:(\d+) "
                       r"SHARED:\d+ LOCAL:(\d+)", out)
    names = [name for name, *_ in found]
    logjoint = [n for n in names if "lntm_logjoint_kernel" in n]
    # G = Kp / 16 in 1..8, padded and unpadded
    assert len(logjoint) == 16, logjoint
    for kind in ("phi_t", "mstep_fwd", "mstep_word", "mstep_topic"):
        assert sum("lntm_%s_kernel" % kind in n for n in names) == 1, (kind, names)
    assert len(found) == 20, names
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
