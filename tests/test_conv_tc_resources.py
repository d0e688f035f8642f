"""The passes of csrc/conv_tc.cu around the tensor-core products (gather-split, col2im-sum with
its epilogues, the sigmoid gradient) exist in the built library with no stack frame and no local
memory, so none of them spills.  CPU only (reads the library's resource usage with cuobjdump)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib

CONV_TC = {"conv_absmax_kernel", "conv_plane_scale_kernel", "gather_split_kernel",
           "col2im_flat_kernel", "col2im_bn_train_kernel", "sigmoid_grad_kernel",
           "col_sum_merge_kernel"}


def test_no_conv_tc_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    mine = [(n, r, st, lo) for n, r, st, lo in found if "conv_tc" in n]
    kinds = {k for n, *_ in mine for k in CONV_TC if k in n}
    assert kinds == CONV_TC, kinds
    # three col2im_flat instances (epilogues 0, 1, 3)
    assert len(mine) == len(CONV_TC) + 2, [n for n, *_ in mine]
    for name, reg, stack, local in mine:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
