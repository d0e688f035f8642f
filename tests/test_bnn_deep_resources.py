"""The deep BNN kernels of csrc/bnn_deep.cu: in the built library no instance has a stack frame
or local memory (no spill), and the C ABI rejects malformed arguments before any launch.  CPU
only (cuobjdump reads the library; the rejections return before touching a device)."""
import ctypes
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_bnn_deep_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*bnn_deep_\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ "
                       r"LOCAL:(\d+)", out)
    kinds = {re.search(r"bnn_deep_(logjoint|step|mean_k)_kernel", name).group(1)
             for name, *_ in found}
    assert kinds == {"logjoint", "step", "mean_k"}, kinds
    assert len(found) == 8, [name for name, *_ in found]      # 2 log-joint, 5 step, 1 mean_k
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)


def _arr(ctype, vals):
    a = (ctype * len(vals))(*vals)
    return a


def test_c_abi_rejects_bad_arguments():
    lib = _lib.lib
    dll = lib.load()
    fake = 0x10000                      # never dereferenced: every call below is rejected first
    keep = []

    def lj(L=3, widths=(4, 5, 3, 1), w=True, x=fake, ls_n=1, K=2, B=10):
        wa = _arr(ctypes.c_void_p, [fake if w else None] * L)
        la = _arr(ctypes.c_void_p, [fake] * L)
        wd = _arr(ctypes.c_int, list(widths)) if widths is not None else None
        keep.extend([wa, la, wd])
        return dll.zsb_bnn_deep_logjoint_f32(L, wd, ctypes.addressof(wa), x, fake, B,
                                             ctypes.addressof(la), _arr(ctypes.c_int, [ls_n] * L),
                                             fake, 100.0, fake, None, None, None, None, K, None)
    for bad in (dict(L=2, widths=(4, 5, 1)), dict(L=9, widths=(2,) * 9 + (1,)),
                dict(widths=(4, 5, 3, 2)), dict(widths=(129, 5, 3, 1)), dict(widths=(4, 129, 3, 1)),
                dict(widths=(4, 0, 3, 1)), dict(widths=(128, 128, 128, 1)), dict(widths=None),
                dict(w=False), dict(x=None), dict(ls_n=0), dict(ls_n=10 ** 6), dict(K=0),
                dict(B=0)):
        assert lj(**bad) != 0, bad
        assert "zsb_bnn_deep_logjoint_f32" in lib.last_error(), bad

    def step(method=0, L=3, v=True, part=fake, mk=True, work_n=10 ** 6, resample=0, chains=2,
             ae=False):
        wa = _arr(ctypes.c_void_p, [fake] * L)
        va = _arr(ctypes.c_void_p, [fake] * L)
        la = _arr(ctypes.c_void_p, [fake] * L)
        keep.extend([wa, va, la])
        return dll.zsb_sgmcmc_bnn_deep_step_f32(
            method, L, _arr(ctypes.c_int, [4, 5, 3, 1]), ctypes.addressof(wa),
            ctypes.addressof(va) if v else None, None,
            ctypes.addressof(va) if ae else None, fake, fake, 10,
            ctypes.addressof(la), _arr(ctypes.c_int, [1] * L), -0.9, 100.0, 1e-4, 0.1, 0.0, 0.9,
            1e-3, 0.0, 1.0, 1, resample, None, None, 1, 0, 0, part,
            ctypes.addressof(va) if mk else None, fake, work_n, chains, None)
    for bad in (dict(method=5), dict(method=-1), dict(v=False), dict(part=None), dict(mk=False),
                dict(work_n=10), dict(method=2), dict(method=3), dict(method=4, ae=False),
                dict(method=4, ae=True, resample=1),
                dict(chains=0), dict(L=2)):
        assert step(**bad) != 0, bad
        assert "zsb_sgmcmc_bnn_deep_step_f32" in lib.last_error(), bad
    assert step(method=4, ae=True, resample=1) != 0
    assert "re-draws v before the step" in lib.last_error()
