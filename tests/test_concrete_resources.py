"""The ExpConcrete / Concrete kernels of csrc/concrete.cu keep each row in registers: in the built
library no instance has a stack frame or local memory, so none of them spills.  Also checks the C
ABI of the entries and the scratch size the backward asks for.  CPU only (reads the library's
resource usage with cuobjdump; the work-size query runs on the host)."""
import os
import re
import subprocess

import pytest

from test_sass_mainloop import _cuobjdump
from zhusuan_b200 import _lib


def test_no_concrete_kernel_spills():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    out = subprocess.run([exe, "-res-usage", _lib.LIB_PATH], check=True, capture_output=True,
                         text=True).stdout
    found = re.findall(r"Function (\S*concrete_\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ "
                       r"LOCAL:(\d+)", out)
    kinds = {re.search(r"concrete_(sample|bwd|logprob|merge)_kernel", name).group(1)
             for name, *_ in found}
    assert kinds == {"sample", "bwd", "logprob", "merge"}, kinds
    # 14 row shapes (G = 1..16 with one block per lane, G = 32 with 1..9) for the sample and the
    # log-density, twice that for the two backward modes, and the merge
    assert len(found) == 14 + 14 + 28 + 1, [name for name, *_ in found]
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, (name, reg, stack, local)


def test_concrete_abi():
    src = open(_lib.HEADER_PATH).read()
    parts = int(re.search(r"#define ZSB_CONCRETE_PARTS (\d+)", src).group(1))
    protos = _lib.parse_header()
    for name in ("zsb_sample_concrete_f32", "zsb_sample_concrete_bwd_f32",
                 "zsb_logprob_concrete_f32", "zsb_logprob_concrete_bwd_f32"):
        assert name in protos, name
    assert [a[1] for a in protos["zsb_logprob_concrete_bwd_f32"]] == [
        "given", "given_rows", "logits", "logits_rows", "temperature", "n_categories",
        "log_space", "gout", "dgiven", "dlogits", "dtemp", "work", "rows", "stream"]
    work = _lib.lib.load().zsb_concrete_bwd_work
    # many logits rows: one chunk, only the temperature partials
    assert work(2000, 1024, 10 * 2000) == parts
    # broadcast logits (20 rows under 1e5 samples; 1 row under 1e6): the sample axis is split
    # and each chunk keeps a logits-gradient partial
    w = work(20, 10, 100000 * 20)
    assert w > parts and (w - parts) % (20 * 10) == 0 and (w - parts) // 200 > 100
    w = work(1, 7, 10 ** 6)
    assert w > parts and (w - parts) % 7 == 0 and (w - parts) // 7 >= 512
    assert work(3, 10, 10) < 0 and work(3, 1025, 30) < 0
