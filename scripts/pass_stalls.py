#!/usr/bin/env python
"""Where the dense leapfrog pass waits: in-kernel stall accounting of tc_pipeline_kernel.

Builds the library with -DZSB_PASS_PROFILE into a temporary directory (or loads --lib), runs the
benchmark workload of bench.py (dense Gaussian, D = 1024, 65 536 chains, L = 50, step-size and
mass adaptation on, dense_impl 5) through its burn-in, then times --steps iterations while every
CTA of the dense pass kernels adds the clock64() cycles its roles spend waiting
(tc_common.cuh, PassProfSlot).  Prints one JSON line: each wait as a share of the MMA
warpgroup's cycles (min / median / max over CTAs), cycles per unit, the card, its power limit and
the SM clock nvidia-smi sampled during the timed steps.

The counters cost a few instructions per k-block, so the profiled pass is a little slower than
the shipped one: compare breakdowns with each other, and times with bench.py.

    python scripts/pass_stalls.py [--lib PATH] [--steps 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# tc_common.cuh: PassProfSlot, PASS_PROF_CTAS
SLOTS = ["mma_total", "mma_full", "mma_tempty", "mma_store", "prod_empty", "epi_tfull",
         "epi_unit", "units"]
PROF_CTAS = 1024


def build_profile_lib(out_dir):
    csrc = os.path.join(ROOT, "zhusuan_b200", "csrc")
    lib = os.path.join(out_dir, "libzsb200.so")
    subprocess.check_call(["make", "-C", csrc, "-j%d" % (os.cpu_count() or 8),
                           "BUILD=" + os.path.join(out_dir, "build"), "OUT=" + lib,
                           "EXTRA_NVCCFLAGS=-DZSB_PASS_PROFILE"], stdout=subprocess.DEVNULL)
    return lib


def stats(x):
    return {"min": float(np.min(x)), "median": float(np.median(x)), "max": float(np.max(x))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None,
                    help="a library built with -DZSB_PASS_PROFILE (default: build one)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--burnin", type=int, default=20)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--chains", type=int, default=65536)
    ap.add_argument("--leapfrogs", type=int, default=50)
    args = ap.parse_args()

    from zhusuan_b200 import _lib
    _lib.LIB_PATH = args.lib or build_profile_lib(tempfile.mkdtemp(prefix="zsb_prof_"))
    dll = _lib.lib.load()
    if not hasattr(dll, "zsb_pass_profile_read"):
        sys.exit("%s was not built with -DZSB_PASS_PROFILE" % _lib.LIB_PATH)
    buf = (ctypes.c_ulonglong * (PROF_CTAS * len(SLOTS)))()

    def read():
        rc = dll.zsb_pass_profile_read(buf, PROF_CTAS)
        if rc != 0:
            raise RuntimeError("zsb_pass_profile_read failed (%d)" % rc)
        return np.frombuffer(buf, dtype=np.uint64).reshape(PROF_CTAS, len(SLOTS)).astype(
            np.float64)

    import torch
    import zhusuan_b200 as zs
    from bench import ClockSampler, make_dense_gaussian_problem

    assert torch.cuda.is_available(), "pass_stalls.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    D, C, L = args.dim, args.chains, args.leapfrogs
    P, _ = make_dense_gaussian_problem(D, seed=2)
    lj = zs.fused.GaussianLogJoint(P, device=dev, impl=5)
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    q = torch.randn(C, D, device=dev, generator=g)
    hmc = zs.HMC(step_size=0.05, n_leapfrogs=L, adapt_step_size=True, adapt_mass=True,
                 mass_collect_iters=10, seed=1234, dense_impl=5)
    op, _ = hmc.sample(lj, {}, {"x": q})
    for _ in range(args.burnin):
        op(adapt_step_size=True, adapt_mass=True)
    sampler = ClockSampler(0)
    sampler.start()
    sampler.wait_first()
    op(adapt_step_size=True, adapt_mass=True)
    torch.cuda.synchronize()
    read()                                         # drop the burn-in's counts

    sampler.mark_begin("timed")
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(args.steps):
        op(adapt_step_size=True, adapt_mass=True)
    e1.record()
    torch.cuda.synchronize()
    sampler.mark_end("timed")
    ms_per_step = e0.elapsed_time(e1) / args.steps
    prof = read()
    clocks = sampler.stop().get("timed")

    live = prof[:, SLOTS.index("units")] > 0
    p = {s: prof[live, i] for i, s in enumerate(SLOTS)}
    total = p["mma_total"]
    passes = args.steps * (L + 1)
    share = {s: stats(p[s] / total) for s in ("mma_full", "mma_tempty", "mma_store",
                                              "prod_empty", "epi_tfull", "epi_unit")}
    per_unit = {"mma_total": stats(total / p["units"]),
                "epi_unit": stats(p["epi_unit"] / p["units"])}
    try:
        power_limit = float(subprocess.run(
            ["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
            capture_output=True, text=True, check=True).stdout.strip())
    except (OSError, subprocess.CalledProcessError, ValueError):
        power_limit = None
    out = {
        "what": "tc_pipeline_kernel<ResW> stall cycles per CTA, dense_impl 5, D=%d, %d chains, "
                "L=%d, adaptive, %d timed iterations (%d passes)" % (D, C, L, args.steps, passes),
        "lib": os.path.basename(os.path.dirname(os.path.abspath(_lib.LIB_PATH))),
        "ctas": int(live.sum()),
        "share_of_mma_cycles": share,
        "cycles_per_unit": per_unit,
        "units_per_cta_per_pass": stats(p["units"] / passes),
        "mma_cycles_per_pass": stats(total / passes),
        "ms_per_step": ms_per_step,
        "card": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit,
        "clocks": clocks,
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
