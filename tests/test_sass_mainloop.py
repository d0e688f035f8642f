"""SASS check of the tensor-core mainloop (no GPU needed).

tc_pipeline_kernel issues the wgmma of one k-block back to back and waits with
`wgmma.wait_group 1` (one k-block left in flight) inside the k-loop.  If ptxas
cannot prove a register of an in-flight wgmma is left alone, it inserts a
`WARPGROUP.DEPBAR` after every HGMMA instead (ptxas warning C7517), and each
wgmma waits for itself before the next one issues.  This test reads the SASS of
the built library and fails if a WARPGROUP.DEPBAR sits between two HGMMAs of
one k-block, i.e. between two HGMMAs with no mbarrier wait between them (every
k-block starts with the wait on its stage's full barrier)."""
import os
import re
import shutil
import subprocess

import pytest

from zhusuan_b200 import _lib


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe:
        return exe
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.exists(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


def _tc_kernels(sass):
    """-> {mangled name: [opcode text of each instruction]} of every tc_pipeline_kernel."""
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if "tc_pipeline_kernel" in m.group(1) else None
            if name:
                kernels[name] = []
            continue
        if name is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m:
            kernels[name].append(m.group(1))
    return kernels


def _serialised_kblocks(instrs):
    """Number of WARPGROUP.DEPBARs that sit between two HGMMAs of one k-block."""
    bad, seen_hgmma, pending_depbar = 0, False, 0
    for ins in instrs:
        if "SYNCS.PHASECHK" in ins:              # mbarrier wait: a new k-block may start
            seen_hgmma, pending_depbar = False, 0
        elif "WARPGROUP.DEPBAR" in ins:
            if seen_hgmma:
                pending_depbar += 1
        elif "HGMMA" in ins:
            bad += pending_depbar
            seen_hgmma, pending_depbar = True, 0
    return bad


@pytest.fixture(scope="module")
def tc_kernels():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH)")
    assert os.path.exists(_lib.LIB_PATH), "library not built: " + _lib.LIB_PATH
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout
    kernels = _tc_kernels(sass)
    assert kernels, "no tc_pipeline_kernel in " + _lib.LIB_PATH
    return kernels


def test_every_tc_pipeline_kernel_issues_hgmma(tc_kernels):
    for name, instrs in tc_kernels.items():
        assert any("HGMMA" in i for i in instrs), name


def test_no_wgmma_wait_inside_a_kblock(tc_kernels):
    bad = {name: n for name, n in ((k, _serialised_kblocks(v)) for k, v in tc_kernels.items())
           if n}
    assert not bad, ("WARPGROUP.DEPBAR between HGMMAs of one k-block (count per kernel): %r"
                     % bad)


def test_detector_on_serialised_and_pipelined_sequences():
    serialised = ["SYNCS.PHASECHK.TRANS64.TRYWAIT P0, [UR4], R0", "WARPGROUP.ARRIVE",
                  "HGMMA.64x128x16.F32 R24, gdesc[UR12], R24, gsb0",
                  "WARPGROUP.DEPBAR.LE gsb0, 0x0", "WARPGROUP.ARRIVE",
                  "HGMMA.64x128x16.F32 R24, gdesc[UR12], R24, gsb0",
                  "WARPGROUP.DEPBAR.LE gsb0, 0x0"]
    assert _serialised_kblocks(serialised) == 1
    pipelined = ["SYNCS.PHASECHK.TRANS64.TRYWAIT P0, [UR4], R0", "WARPGROUP.ARRIVE",
                 "HGMMA.64x128x16.F32 R24, gdesc[UR12], R24",
                 "HGMMA.64x128x16.F32 R24, gdesc[UR12], R24, gsb0",
                 "WARPGROUP.DEPBAR.LE gsb0, 0x1",
                 "SYNCS.PHASECHK.TRANS64.TRYWAIT P0, [UR4], R0", "WARPGROUP.ARRIVE",
                 "HGMMA.64x128x16.F32 R88, gdesc[UR12], R88, gsb0",
                 "WARPGROUP.DEPBAR.LE gsb0, 0x0"]
    assert _serialised_kblocks(pipelined) == 0
