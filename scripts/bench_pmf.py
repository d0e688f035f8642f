#!/usr/bin/env python
"""Bayesian PMF by HMC (examples/probabilistic_matrix_factorization/pmf_hmc.py): one Gibbs epoch is
a U-sweep and a V-sweep, each ONE HMC iteration over all 50-row chunks of the factor on the fused
chunked log-joint (zs.fused.PMFLogJoint, csrc/pmf.cu).  Seeded synthetic corpora with Zipf-like
user and movie degrees at the MovieLens-1M shape (6 040 x 3 706 padded to chunks of 50, 1.0e6
draws) and the MovieLens-10M shape (69 878 x 10 677, 1.0e7 draws); repeated (user, movie) pairs are
dropped, so about 6.6e5 and 7.2e6 ratings remain (`nnz` in the output); D = 30, K = 8 particles,
L = 10, step size 1e-3 (the example's settings).  Prints one JSON line: kernel times (CUDA events
over many launches), HMC sweep and epoch times, rates, roofline counts computed from shapes, the
generic autograd path on the same model at the ML-1M shape, and the card it ran on."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zhusuan_b200 as zs  # noqa: E402
from pmf_oracle import make_corpus  # noqa: E402

K, D, CHUNK, L, STEP = 8, 30, 50, 10, 1e-3
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12          # H100 SXM data sheet (700 W card)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                             "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def events(fn, n):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def counts(nnz, n_rows, n_cols):
    """FLOPs and bytes of one gradient call from shapes.  HBM: latent read + gradient write, the
    fixed factor once, CSR once.  L2 gather: one fixed-factor row per (particle, rating)."""
    flops = 4.0 * D * K * nnz                     # dot + axpy
    hbm = 4.0 * K * D * (2 * n_rows + n_cols) + 8.0 * nnz + 8.0 * n_rows
    gather = 4.0 * D * K * nnz
    return flops, hbm, gather


def corpus(name, n_users, n_movies, nnz, seed):
    n_pad = -(-n_users // CHUNK) * CHUNK
    m_pad = -(-n_movies // CHUNK) * CHUNK
    rows, cols, r = make_corpus(n_users, n_movies, nnz, seed)
    return dict(name=name, rows=rows, cols=cols, r=r, N=n_pad, M=m_pad)


def run(c, generic=False):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(1)
    U = 0.1 * torch.randn(K, c["N"], D, device=dev, generator=g)
    V = 0.1 * torch.randn(K, c["M"], D, device=dev, generator=g)
    u, v = U.view(K, -1, CHUNK, D), V.view(K, -1, CHUNK, D)
    lj_u = zs.fused.PMFLogJoint(c["rows"], c["cols"], c["r"], fixed=v, n_rows=c["N"],
                                chunk_size=CHUNK, std=1., fixed_std=1., rating_std=0.05, name="u")
    lj_v = zs.fused.PMFLogJoint(c["cols"], c["rows"], c["r"], fixed=u, n_rows=c["M"],
                                chunk_size=CHUNK, std=1., fixed_std=1., rating_std=0.05, name="v")
    nnz = lj_u.nnz
    out = {"nnz": nnz, "users_padded": c["N"], "movies_padded": c["M"]}
    for side, lj, x in (("u", lj_u, u), ("v", lj_v, v)):
        for _ in range(3):
            lj.grad([x]); lj.logp([x])
        torch.cuda.synchronize()
        n = 200
        out["%s_grad_kernel_ms" % side] = events(lambda: lj.grad([x]), n)
        out["%s_logp_kernel_ms" % side] = events(lambda: lj.logp([x]), n)
        fl, hbm, ga = counts(nnz, lj.n_rows, lj.n_cols)
        ms = out["%s_grad_kernel_ms" % side]
        out["%s_grad_particle_ratings_per_s" % side] = K * nnz / (ms * 1e-3)
        out["%s_grad_fp32_tflops" % side] = fl / (ms * 1e-3) / 1e12
        out["%s_grad_hbm_GBps" % side] = hbm / (ms * 1e-3) / 1e9
        out["%s_grad_l2_gather_GBps" % side] = ga / (ms * 1e-3) / 1e9
        out["%s_grad_bytes" % side] = {"hbm": hbm, "l2_gathered_factor": ga, "flops": fl}
        t_hbm, t_fl = hbm / HBM_BPS * 1e3, fl / FP32_FLOPS * 1e3
        out["%s_grad_bound" % side] = (
            "HBM floor %.4f ms, FP32 floor %.4f ms (data sheet); both far below the kernel time: "
            "the kernel is bound by the per-rating gather of %.0f MB of factor rows through "
            "L2/L1 and its latency, which has no data-sheet peak" % (t_hbm, t_fl, ga / 1e6))
    op_u, info_u = zs.HMC(step_size=STEP, n_leapfrogs=L, seed=11).sample(lj_u, {}, {"u": u})
    op_v, info_v = zs.HMC(step_size=STEP, n_leapfrogs=L, seed=12).sample(lj_v, {}, {"v": v})
    for _ in range(2):
        op_u(); op_v()
    torch.cuda.synchronize()
    n = 10
    out["u_sweep_ms"] = events(op_u, n)
    out["v_sweep_ms"] = events(op_v, n)
    out["gibbs_epoch_ms"] = events(lambda: (op_u(), op_v()), n)
    chains = K * (c["N"] // CHUNK + c["M"] // CHUNK)
    out["leapfrog_steps_x_chains_per_s"] = L * chains / (out["gibbs_epoch_ms"] * 1e-3)
    out["sequential_hmc_calls_replaced_per_epoch"] = c["N"] // CHUNK + c["M"] // CHUNK
    out["u_acceptance_mean"] = float(info_u.acceptance_rate.mean())
    out["v_acceptance_mean"] = float(info_v.acceptance_rate.mean())
    if generic:
        # the same model on the generic path: torch gathers + autograd (index_add backward)
        U2 = U.clone()
        u2 = U2.view(K, -1, CHUNK, D)
        op_g, info_g = zs.HMC(step_size=STEP, n_leapfrogs=L, seed=11).sample(
            lambda obs: lj_u(obs), {}, {"u": u2})
        op_g()
        torch.cuda.synchronize()
        out["generic_autograd_u_sweep_ms"] = events(op_g, 3)
        x = u2.detach().clone().requires_grad_(True)

        def gen_grad():
            x.grad = None
            lj_u({"u": x}).sum().backward()
        gen_grad()
        torch.cuda.synchronize()
        out["generic_autograd_grad_ms"] = events(gen_grad, 10)
        out["fused_speedup_u_sweep"] = out["generic_autograd_u_sweep_ms"] / out["u_sweep_ms"]
        out["fused_speedup_grad"] = out["generic_autograd_grad_ms"] / out["u_grad_kernel_ms"]
        out["generic_u_acceptance_mean"] = float(info_g.acceptance_rate.mean())
        out["generic_peak_mem_GB"] = torch.cuda.max_memory_allocated() / 1e9
    return out


def main():
    assert torch.cuda.is_available(), "bench_pmf.py needs a CUDA device"
    name, pl = card()
    res = {"workload": "Bayesian PMF HMC Gibbs epoch (U-sweep + V-sweep, one HMC iteration each), "
                       "D=%d, K=%d, chunk=%d, L=%d, step=%g" % (D, K, CHUNK, L, STEP),
           "gpu": name, "power_limit_and_max_sm_clock": pl}
    res["ml1m"] = run(corpus("ml1m", 6040, 3706, 1000209, seed=1), generic=True)
    res["ml10m"] = run(corpus("ml10m", 69878, 10677, 10000054, seed=2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
