#!/usr/bin/env python
"""The logistic-normal topic model trained by Monte-Carlo EM and scored by AIS
(examples/topic_models/lntm_mcem.py) at the NIPS shape, fused against generic, alternating in one
process.  The corpus is synthetic: Zipf(1.1) word frequencies over V = 12 400 words, about 1300
tokens per document, 1500 documents (1200 for training, 300 for test), about 750 000 non-zeros;
K = 100 topics.  Those figures are arguments.

Arms (tests/lntm_mcem_models.py): ``fused`` runs the E-step on the sparse log-joint kernel as HMC's
provider, the M-step on ``LNTMLogJoint.cond_log_px`` and AIS on the tempered provider; ``generic``
differentiates the dense torch restatement, which forms the [rows, V] matrix doc_word.

Cases, one JSON line per case and arm:
  estep_hmc   one E-step HMC iteration, 1 chain x 100 documents, 20 leapfrog steps
  mstep       the M-step's log p(x | eta, beta) and its beta gradient, one batch
  train_batch one training batch: 5 E-step iterations, the M-step and Adam
  epoch       one epoch over the 1200 training documents (12 batches)
  ais         AIS with 25 chains x 300 test documents for --ais-temperatures temperatures after
              --ais-adapt adaptation iterations; also the time per temperature

Each line has the median, fastest and slowest window, CUDA kernel launches per call (counted by
torch.profiler in a separate call), FLOPs and bytes per call from the shapes (flops_sparse counts
4 K per (chain, word occurrence) and log-joint evaluation, flops_dense 6 K V per chain-document and
evaluation; bytes_* the eta, phi_t and doc_word traffic of one pass), and the card's name and power
limit.  Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zhusuan_b200 as zs  # noqa: E402
import lntm_mcem_models as LM  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                                "-i", str(torch.cuda.current_device())], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def corpus(n_docs, V, tokens, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    p = 1.0 / np.arange(1, V + 1) ** 1.1
    p /= p.sum()
    lengths = rng.poisson(tokens, n_docs)
    return np.stack([rng.multinomial(n, p) for n in lengths]).astype(np.float32)


def timed(fn, reps, windows):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3 / reps)
    return out


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == "CUDA")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1500)
    ap.add_argument("--train", type=int, default=1200)
    ap.add_argument("--vocab", type=int, default=12400)
    ap.add_argument("--tokens", type=int, default=1300)
    ap.add_argument("--topics", type=int, default=100)
    ap.add_argument("--ais-chains", type=int, default=25)
    ap.add_argument("--ais-temperatures", type=int, default=20)
    ap.add_argument("--ais-adapt", type=int, default=2)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--cases", default="estep_hmc,mstep,train_batch,epoch,ais")
    a = ap.parse_args()
    dev = torch.device("cuda")
    torch.backends.cuda.matmul.allow_tf32 = False        # the reference computes in float32
    name, power = card()
    X = corpus(a.docs, a.vocab, a.tokens, seed=7)
    x_train, x_test = X[:a.train], X[a.train:]
    B, K, V = 100, a.topics, a.vocab
    beta0 = 0.1 * torch.randn(K, V, device=dev, generator=torch.Generator(dev).manual_seed(3))
    models = {arm: LM.MCEM(zs, x_train, beta0, n_chains=1, batch_size=B, fused=arm == "fused")
              for arm in ("fused", "generic")}
    for m in models.values():
        m.run_epoch()                                     # warm the chains and the step size
    nnz_train = int(models["fused"].lj.nnz)
    nnz_batch = nnz_train * B / a.train
    nnz_test = int((x_test != 0).sum())
    Kp = 16 * -(-K // 16)

    def shape_cost(C, docs, nnz, evals):
        return dict(flops_sparse=4.0 * K * nnz * C * evals,
                    flops_dense=6.0 * K * V * C * docs * evals,
                    bytes_sparse=(nnz * Kp * 4.0 + 2 * C * docs * K * 4.0) * evals,
                    bytes_dense=(3 * C * docs * V * 4.0 + 2 * C * docs * K * 4.0) * evals)

    ais_state = {}

    def ais_call(arm):
        m = models[arm]
        _, bound = m.ais(x_test, n_chains=a.ais_chains, n_temperatures=a.ais_temperatures,
                         n_adapt=a.ais_adapt)
        ais_state[arm] = bound

    def prep_batch(m):
        ids = m.order[:B]
        m.lj.set_docs(ids)
        m.eta.copy_(m.Eta[:, ids])

    def mstep(m):
        b = m.beta
        lp = m.log_px()
        torch.autograd.grad(-lp, [b])

    evals_hmc = 21                                        # 20 leapfrog gradients + the MH value
    cases = {
        "estep_hmc": (lambda arm: models[arm].sample_op(), shape_cost(1, B, nnz_batch, evals_hmc),
                      prep_batch, 20),
        "mstep": (lambda arm: mstep(models[arm]), shape_cost(1, B, nnz_batch, 2), prep_batch, 20),
        "train_batch": (lambda arm: models[arm].batch(0),
                        shape_cost(1, B, nnz_batch, 5 * evals_hmc + 2), None, 3),
        "epoch": (lambda arm: models[arm].run_epoch(),
                  shape_cost(1, a.train, nnz_train, 5 * evals_hmc + 2), None, 1),
        "ais": (ais_call, shape_cost(a.ais_chains, x_test.shape[0], nnz_test,
                                     (a.ais_temperatures + a.ais_adapt) * evals_hmc),
                None, 1),
    }
    for case in a.cases.split(","):
        fn, cost, prep, reps = cases[case]
        windows = {"fused": [], "generic": []}
        for _ in range(a.windows):                        # alternate the arms
            for arm in ("fused", "generic"):
                if prep is not None:
                    prep(models[arm])
                windows[arm] += timed(lambda: fn(arm), reps, 1)
        for arm in ("fused", "generic"):
            if prep is not None:
                prep(models[arm])
            n_launch = launches(lambda: fn(arm))
            w = windows[arm]
            res = {"case": case, "arm": arm, "ms_median": statistics.median(w),
                   "ms_min": min(w), "ms_max": max(w), "windows": len(w), "calls_per_window": reps,
                   "launches_per_call": n_launch, "K": K, "V": V, "train_docs": a.train,
                   "test_docs": int(x_test.shape[0]), "nnz_train": nnz_train,
                   "nnz_test": nnz_test, "gpu": name, "power_limit": power}
            res.update(cost)
            if case == "ais":
                res.update(chains=a.ais_chains, temperatures=a.ais_temperatures,
                           adapt=a.ais_adapt, bound=ais_state[arm],
                           ms_per_temperature=res["ms_median"] / (a.ais_temperatures
                                                                  + a.ais_adapt))
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
