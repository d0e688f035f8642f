"""The passes of csrc/conv_tc.cu around the tensor-core products (gather-split, col2im-sum with
its epilogues, the activation gradient) and the residual epilogue of the dense-layer kernel
(EPI 16) exist in the built library with no stack frame and no local memory, so none of them
spills; and the col2im and activation-gradient entries reject a bad epilogue or activation code
before any launch.  CPU only (cuobjdump reads the library's resource usage; the rejections return
before touching a device)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib

CONV_TC = {"conv_absmax_kernel", "conv_plane_scale_kernel", "gather_split_kernel",
           "col2im_flat_kernel", "col2im_bn_train_kernel", "act_grad_kernel",
           "col_sum_merge_kernel"}


def _res_usage():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    return subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout


def test_no_merged_conv_tc_kernel_spills():
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)",
                       _res_usage())
    mine = [(n, r, st, lo) for n, r, st, lo in found if "conv_tc" in n]
    kinds = {k for n, *_ in mine for k in CONV_TC if k in n}
    assert kinds == CONV_TC, kinds
    # three col2im_flat instances (epilogues 0, 1, 3)
    assert len(mine) == len(CONV_TC) + 2, [n for n, *_ in mine]
    for name, reg, stack, local in mine:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)


def test_no_residual_epilogue_spills():
    found = re.findall(r"Function (\S*?tc_pipeline_kernel\w*RowsEpiELi16ELi(\d)ELi(\d)\w*):\s*\n"
                       r"\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", _res_usage())
    # EPI 16 on the three-product forward mainloop only
    assert [(int(mn), int(z)) for _, mn, z, _, _, _ in found] == [(0, 0)], [f[0] for f in found]
    for name, _, _, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)


def test_c_abi_rejects_bad_epilogue_and_activation():
    lib = _lib.lib
    dll = lib.load()
    fake = 0x10000                      # never dereferenced: every call below is rejected first

    def col2im(epi, act):
        return dll.zsb_conv_col2im_f32(epi, fake, 2, 8, 8, 4, 4, 4, 3, 2, 1, 1, fake, fake, fake,
                                       fake, fake, fake, 1e-3, act, fake, fake, fake, fake, fake,
                                       None)
    for epi, act in ((-1, 0), (4, 0), (0, 1), (0, 2), (2, 1), (2, 2), (3, 2), (1, 3), (1, -1),
                     (3, -1)):
        assert col2im(epi, act) != 0, (epi, act)
        assert "zsb_conv_col2im_f32" in lib.last_error(), (epi, act)

    def act_grad(act, y=fake, R=10, C=4):
        return dll.zsb_conv_act_grad_f32(fake, y, R, C, act, fake, fake, fake, fake, None)
    for bad in (dict(act=3), dict(act=-1), dict(act=1, y=None), dict(act=2, y=None),
                dict(act=0, C=1 << 20), dict(act=0, R=1 << 20, C=1 << 11), dict(act=0, R=0)):
        assert act_grad(**bad) != 0, bad
        assert "zsb_conv_act_grad_f32" in lib.last_error(), bad
