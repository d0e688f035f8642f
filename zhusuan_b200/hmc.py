"""Parallel-chain HMC on H100 kernels -- drop-in for ``zs.HMC`` (zhusuan/hmc.py).

Same constructor and ``sample(meta_bn, observed, latent) -> (sample_op,
HMCInfo)`` contract as hmc.py:252-255, 382-410.  Differences forced by the
absence of a TF graph/session:

* ``latent`` values are float32 CUDA ``torch.Tensor`` "variables" updated in
  place (``tf.Variable`` + ``assign``, hmc.py:497);
* ``sample_op`` is a callable: ``sample_op()`` == ``sess.run(sample_op)``.
  Per-step booleans that the reference feeds through placeholders
  (hmc.py:228-231) are passed as ``sample_op(adapt_step_size=..,
  adapt_mass=..)``; the constructor values only say whether the feature is
  configured (``is not None``) and give the default;
* ``HMCInfo`` fields are device tensors refreshed by every ``sample_op()``.

Three execution paths, all ending in the same MH / adaptation kernels:
  generic        any ``log_joint`` (callable or MetaBayesianNet); gradients by
                 torch autograd over the registry's analytic-backward kernels
                 (replaces ``tf.gradients``, hmc.py:430-432); leapfrog / MH /
                 adaptation by libzsb200.
  diag-normal    a single Normal node with group_ndims covering the data axes
                 (examples/toy_examples/gaussian.py): ONE kernel per iteration.
  dense-gaussian ``zs.fused.GaussianLogJoint``: one fused GEMM+leapfrog kernel
                 per gradient evaluation (BASELINE config 2).
"""
import ctypes
import os

import torch

from . import dist as zdist
from . import random as zrandom
from ._lib import lib, ptr, stream
from .framework.bn import StochasticTensor
from .utils import merge_dicts

__all__ = ["HMCInfo", "HMC"]

_F32 = torch.float32
# state block indices (include/zsb200.h ZSB_HMC_STATE_*)
ST_T, ST_STEP, ST_TSTEP, ST_LEB, ST_HBAR, ST_MU, ST_EWT, ST_EPS, ST_ACC, \
    ST_FLAGS, ST_SLAST, ST_SCOND = range(12)
STREAM_MOMENTUM = 1


class HMCInfo(object):
    """hmc.py:162-201 -- same eight fields; each is a device tensor view that
    the sampling op overwrites on every call (fetch after calling it)."""

    def __init__(self, samples, acceptance_rate, updated_step_size,
                 init_momentum, orig_hamiltonian, hamiltonian, orig_log_prob,
                 log_prob):
        self.samples = samples
        self.acceptance_rate = acceptance_rate
        self.updated_step_size = updated_step_size
        self.init_momentum = init_momentum
        self.orig_hamiltonian = orig_hamiltonian
        self.hamiltonian = hamiltonian
        self.orig_log_prob = orig_log_prob
        self.log_prob = log_prob


def _flag(x):
    """Resolve a per-step boolean: bool, 0-d tensor, callable or .value."""
    if x is None:
        return False
    if callable(x):
        x = x()
    if hasattr(x, "value"):
        x = x.value
    if isinstance(x, torch.Tensor):
        x = bool(x.item())
    return bool(x)


class _SampleOp(object):
    def __init__(self, hmc):
        self._hmc = hmc

    def __call__(self, adapt_step_size=None, adapt_mass=None, noise=None,
                 use_graph=None, observed=None):
        """One HMC iteration.  ``use_graph`` (default: the sampler's
        ``use_cuda_graph``) replays the iteration from a captured CUDA graph
        on the fused paths -- worthwhile when the iteration is launch-bound.
        ``observed`` replaces observed values for this and later calls (what
        ``sess.run(sample_op, feed_dict=...)`` does for placeholder-fed
        observations, evaluation.py:150-156)."""
        if observed:
            self._hmc._observed.update(observed)
        return self._hmc._iterate(adapt_step_size, adapt_mass, noise,
                                  use_graph)

    run = __call__

    def synchronize(self):
        """Drain the stream and surface the check_numerics error, if any."""
        self._hmc._check_flags(final=True)


class HMC(object):
    """hmc.py:204-522."""

    def __init__(self, step_size=1., n_leapfrogs=10, adapt_step_size=None,
                 target_acceptance_rate=0.8, gamma=0.05, t0=100, kappa=0.75,
                 adapt_mass=None, mass_collect_iters=10, mass_decay=0.99,
                 seed=None, process_group=None, chain_offset=None,
                 dense_impl=None, use_cuda_graph=False):
        self._init_step_size_value = float(step_size)
        self.n_leapfrogs = int(n_leapfrogs)
        self.target_acceptance_rate = float(target_acceptance_rate)
        self.adapt_step_size = adapt_step_size
        self._has_step = adapt_step_size is not None
        self.gamma, self.t0, self.kappa = float(gamma), float(t0), float(kappa)
        if adapt_mass is not None:
            if adapt_step_size is None:                       # hmc.py:271-272
                raise ValueError('If adapt mass is set, we should also adapt '
                                 'step size')
            self.adapt_mass = adapt_mass
        else:
            mass_collect_iters = 0                            # hmc.py:276
            self.adapt_mass = None
        self._has_mass = adapt_mass is not None
        self.mass_collect_iters = int(mass_collect_iters)
        self.mass_decay = float(mass_decay)
        self._seed = seed
        self._group = process_group
        self._chain_offset = chain_offset
        self._dense_impl = dense_impl
        self._use_graph = bool(use_cuda_graph)
        self._graphs = {}
        self._graph_launches = {}
        self._dev_mode = False   # True while capturing / replaying a graph
        self._t = 0              # host mirror of hmc.py:264 (deterministic)
        self._ewmv_t = 0         # host mirror of hmc.py:118
        self._built = False
        self.n_search_iters = 0

    # ------------------------------------------------------------------ build
    def sample(self, meta_bn, observed, latent):
        """hmc.py:382-522."""
        if self._built:
            raise RuntimeError(
                "HMC.sample() may be invoked once per HMC instance "
                "(hmc.py:218-222); declare one HMC per sample() call.")
        if callable(meta_bn):                                 # hmc.py:412-416
            self._log_joint = meta_bn
        else:
            self._log_joint = lambda obs: meta_bn.observe(**obs).log_joint()
        self._latent_k = list(latent.keys())
        self._q = []
        for k in self._latent_k:                              # hmc.py:419-423
            v = latent[k]
            if not isinstance(v, torch.Tensor):
                raise TypeError(
                    "latent['{}'] is not a Variable (a float32 CUDA "
                    "torch.Tensor updated in place).".format(k))
            if v.dtype != _F32 or not v.is_contiguous():
                raise TypeError("latent['{}'] must be a contiguous float32 "
                                "tensor.".format(k))
            self._q.append(v)
        self._observed = dict(observed)
        dev = self._q[0].device

        fused = getattr(meta_bn, "_zsb_fused", None)
        if fused is None and not callable(meta_bn):
            fused = _detect_diag_normal(meta_bn, self._observed, latent)
        # kind "provider": the log-joint object computes its own values / gradients with a
        # fused kernel (e.g. zs.fused.LNTMLogJoint); everything else runs on the generic path
        self._provider = None
        if fused is not None and fused["kind"] == "provider":
            self._provider = fused["obj"]
            fused = None
        self._fused = fused

        if fused is not None and fused["kind"] == "dense_gaussian":
            chain_shape = tuple(self._q[0].shape[:-1])
            if tuple(self._q[0].shape[-1:]) != (fused["D"],):
                raise ValueError("latent last axis must equal the Gaussian's "
                                 "dimension {}".format(fused["D"]))
        else:
            with torch.no_grad():
                lp = self._get_log_posterior(self._q)
            chain_shape = tuple(lp.shape)                     # hmc.py:436
        if len(chain_shape) == 0:                             # hmc.py:438-442
            raise ValueError(
                "HMC requires that the static shape of the value returned "
                "by log joint function should be at least partially defined. "
                "(shape: {})".format(chain_shape))
        self._chain_shape = chain_shape
        ncd = len(chain_shape)
        self._n_chain_dims = ncd
        chains = 1
        for s in chain_shape:
            chains *= int(s)
        self._chains = chains
        self._row_len = []
        for q in self._q:
            if tuple(q.shape[:ncd]) != chain_shape:
                raise ValueError("latent shape {} does not start with the "
                                 "chain shape {}".format(tuple(q.shape),
                                                         chain_shape))
            r = 1
            for s in q.shape[ncd:]:
                r *= int(s)
            self._row_len.append(r)

        world, rank = zdist.world(self._group)
        self._world = world
        self._row0 = (rank * chains if self._chain_offset is None
                      else int(self._chain_offset))
        self._n_global = float(chains * world)

        z = lambda *s: torch.zeros(*s, dtype=_F32, device=dev)
        st = z(16)
        st[ST_STEP] = self._init_step_size_value
        st[ST_MU] = 10 * self._init_step_size_value           # hmc.py:79
        self._state = st
        self._p0 = [torch.empty_like(q) for q in self._q]
        self._mass = [torch.ones(r, dtype=_F32, device=dev)
                      for r in self._row_len]
        if self._has_mass:
            self._ew_mean = [z(r) for r in self._row_len]
            self._ew_var = [z(r) for r in self._row_len]
            nparts = lib.load().zsb_hmc_mass_parts()
            self._mass_part = [z(nparts * 2 * r) for r in self._row_len]
        # one packed message [sum acc, n, S1.., S2..] -> ONE all-reduce per iteration (dist.py)
        self._pk = zdist.PackedStats(sum(self._row_len) if self._has_mass else 0, dev,
                                     self._group)
        self._stats = self._pk.acc
        self._mass_stats = self._pk.mass
        self._q_versions = None
        self._acc_part = z(lib.load().zsb_hmc_acc_parts())
        c = (chains,)
        self._k0, self._k1 = z(c), z(c)
        self._lp0, self._lp1 = z(c), z(c)
        self._h0, self._h1 = z(c), z(c)
        self._acc, self._lpsel = z(c), z(c)
        self._accept = torch.zeros(c, dtype=torch.int32, device=dev)
        self._npart = ctypes.c_int(0)
        self._flag_host = torch.zeros(1, dtype=torch.int32).pin_memory() \
            if dev.type == "cuda" else torch.zeros(1, dtype=torch.int32)
        self._flag_event = None
        if fused is not None and fused["kind"] == "dense_gaussian":
            self._setup_dense(dev)
        self._built = True

        info = HMCInfo(
            samples=dict(zip(self._latent_k, self._q)),
            acceptance_rate=self._acc.view(chain_shape),
            updated_step_size=self._state[ST_STEP],
            init_momentum=dict(zip(self._latent_k, self._p0)),
            orig_hamiltonian=self._h0.view(chain_shape),
            hamiltonian=self._h1.view(chain_shape),
            orig_log_prob=self._lp0.view(chain_shape),
            log_prob=self._lpsel.view(chain_shape))
        self._info = info
        return _SampleOp(self), info

    # ---------------------------------------------------------------- helpers
    def _get_log_posterior(self, var_list):                   # hmc.py:426-428
        if self._provider is not None:
            return self._provider.logp(var_list)
        joint_obs = merge_dicts(dict(zip(self._latent_k, var_list)),
                                self._observed)
        return self._log_joint(joint_obs)

    def _get_gradient(self, var_list):                        # hmc.py:430-432
        if self._provider is not None:
            return self._provider.grad(var_list)
        xs = [v.detach().requires_grad_(True) for v in var_list]
        with torch.enable_grad():
            lp = self._get_log_posterior(xs)
            gs = torch.autograd.grad(lp.sum(), xs, allow_unused=True)
        return [g.contiguous() if g is not None else torch.zeros_like(x)
                for g, x in zip(gs, xs)]

    def _eps_ptr(self):
        return self._state.data_ptr() + 4 * ST_EPS

    def _check_flags(self, final=False):
        """check_numerics (hmc.py:51-53) without a host sync per iteration: the flag word is
        copied to pinned memory asynchronously after every iteration and only LOOKED at here
        once its copy has completed (``final`` = wait for it: ``sample_op.synchronize()``)."""
        if self._flag_event is not None and (final or self._flag_event.query()):
            self._flag_event.synchronize()
            self._flag_event = None
            if int(self._flag_host[0]) & 1:
                # not sticky: clear the device flag so a repaired sampler can continue
                self._state[ST_FLAGS:ST_FLAGS + 1].zero_()
                self._flag_host.zero_()
                raise FloatingPointError(
                    'HMC: old_log_prob has numeric errors! Try better '
                    'initialization.')                        # hmc.py:51-53
        elif final and self._state.is_cuda:
            torch.cuda.current_stream().synchronize()

    def _mass_stats_into_packed(self, s):
        """S1/S2 of the current latent state vs the current EWMV mean -> packed buffer."""
        off = 0
        for k, q in enumerate(self._q):
            r = self._row_len[k]
            lib.call("zsb_hmc_mass_stats_f32", ptr(q), ptr(self._ew_mean[k]), self._chains, r,
                     ptr(self._mass_part[k]), self._mass_stats.data_ptr() + 4 * off, s)
            off += 2 * r

    def _prefetch_ok(self):
        """The packed mass statistics were produced by the previous iteration AND nobody wrote
        the latent tensors since (torch's version counter; our kernels write through raw
        pointers and do not bump it)."""
        return (self._pk.mass_valid and self._q_versions is not None and
                self._q_versions == [q._version for q in self._q])

    def _queue_flag_check(self):
        if self._state.is_cuda:
            self._flag_host.copy_(
                self._state[ST_FLAGS:ST_FLAGS + 1].view(torch.int32),
                non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            self._flag_event = ev

    def _seed_now(self):
        return self._seed if self._seed is not None else zrandom.get_seed()

    # -------------------------------------------------------------- iteration
    def _iterate(self, adapt_step_size, adapt_mass, noise, use_graph=None):
        if not self._built:
            raise RuntimeError("call HMC.sample() first")
        self._check_flags()
        adapt_step = _flag(self.adapt_step_size if adapt_step_size is None
                           else adapt_step_size)
        adapt_m = _flag(self.adapt_mass if adapt_mass is None else adapt_mass)
        self._t += 1                                          # hmc.py:418
        t = self._t
        init = self._has_step and (t == 1 or t == self.mass_collect_iters)
        want_graph = self._use_graph if use_graph is None else bool(use_graph)
        if (want_graph and noise is None and not init and self._fused
                and self._state.is_cuda
                and (not (adapt_m and self._has_mass) or self._prefetch_ok())):
            # (an adaptive-mass iteration without a valid statistics prefetch runs eagerly once)
            return self._iterate_graph(adapt_step, adapt_m)
        return self._iterate_eager(adapt_step, adapt_m, noise, t, init)

    def _needs_acc_exchange(self, adapt_step):
        """Does this iteration's tuner update read the GLOBAL mean acceptance?"""
        return bool(self._has_step and adapt_step)

    def _iterate_graph(self, adapt_step, adapt_m):
        """Replay (or first capture) the iteration as a CUDA graph.  All
        per-iteration scalars (t / Philox iteration, EWMV count, ones-vs-
        precision mass gating) are read from the device state block, so one
        graph per (adapt_step, adapt_mass) pair serves every non-search
        iteration.  Numerically identical to the eager path."""
        key = (adapt_step, adapt_m, self._seed_now())
        g = self._graphs.get(key)
        if g is None:
            # keep the device copy of t in step with the host mirror, then
            # capture one iteration without executing it
            self._state[ST_T] = float(self._t - 1)
            self._state[ST_EWT] = float(self._ewmv_t)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            self._dev_mode = True
            l0 = lib.launches
            try:
                with torch.cuda.graph(g):
                    self._iterate_eager(adapt_step, adapt_m, None, self._t,
                                        False)
            finally:
                self._dev_mode = False
            self._graphs[key] = g
            self._graph_launches[key] = lib.launches - l0
            lib.launches = l0              # capturing launched nothing
        if adapt_m and self._has_mass:
            self._ewmv_t += 1
        g.replay()
        lib.launches += self._graph_launches[key]   # kernels the replay launches
        if self._world > 1 and ((adapt_m and self._has_mass) or
                                self._needs_acc_exchange(adapt_step)):
            self._pk.n_collectives += 1        # the all-reduce captured in the graph
        self._pk.mass_valid = bool(adapt_m and self._has_mass)
        self._q_versions = [q._version for q in self._q]
        self._queue_flag_check()
        return None

    def _iterate_eager(self, adapt_step, adapt_m, noise, t, init):
        s = stream()
        dev = self._dev_mode
        it = 0xFFFFFFFF if dev else (t & 0xFFFFFFFF)
        seed = self._seed_now()
        noise_p = noise_u = None
        if noise is not None:
            noise_p = [noise["p"][k].contiguous() for k in self._latent_k]
            noise_u = noise["u"].contiguous().view(-1)

        # ---- begin: step size for this iteration (hmc.py:463-472); in device
        # mode the kernel also advances t (hmc.py:418)
        lib.call("zsb_hmc_begin_f32", ptr(self._state),
                 -1 if dev else int(init), s)

        # ---- mass (hmc.py:452-456, 283-305)
        if self._has_mass:
            if adapt_m:
                if not dev and not self._prefetch_ok():
                    # no valid prefetch (first iteration / latent written by the caller /
                    # adaptation was off): statistics + their own collective, now
                    self._mass_stats_into_packed(s)
                    self._pk.reduce_mass()
                if not dev:
                    self._ewmv_t += 1
            use_ones = 1 if t < self.mass_collect_iters else 0  # hmc.py:299-302
            if dev:
                use_ones = -(self.mass_collect_iters + 1)
            off = 0
            for k in range(len(self._q)):
                r = self._row_len[k]
                lib.call("zsb_hmc_mass_update_f32", ptr(self._ew_mean[k]),
                         ptr(self._ew_var[k]), ptr(self._mass[k]),
                         self._mass_stats.data_ptr() + 4 * off,
                         self._n_global, r, self.mass_decay,
                         float(self._ewmv_t), int(adapt_m), use_ones,
                         ptr(self._state), s)
                off += 2 * r
            if dev and adapt_m:
                lib.call("zsb_hmc_ewmv_bump_f32", ptr(self._state), s)

        kind = self._fused["kind"] if self._fused else "generic"
        if kind == "diag_normal":
            self._iterate_diag(noise_p, noise_u, seed, it, init, s)
        elif kind == "dense_gaussian":
            self._iterate_dense(noise_p, noise_u, seed, it, init, s)
        else:
            self._iterate_generic(noise_p, noise_u, seed, it, init, s)

        # ---- step-size adaptation (hmc.py:501-505, 374-380)
        lib.call("zsb_hmc_acc_sum_f32", ptr(self._acc_part),
                 self._npart.value, self._chains, ptr(self._stats), s)
        # the statistics the NEXT iteration's mass update needs are those of the state after
        # this iteration's select: compute them now and send them with the acceptance sum
        prefetch = bool(self._has_mass and adapt_m)
        if prefetch:
            self._mass_stats_into_packed(s)
        # The global mean acceptance only feeds the dual-averaging update (hmc.py:89-112 inside
        # tf.cond(adapt_step_size)); an iteration that adapts neither step size nor mass has no
        # exchange step at all, its ranks run unsynchronised (state[ACC_MEAN] is then rank-local).
        exchange = prefetch or self._needs_acc_exchange(adapt_step)
        if dev:
            if self._world > 1 and exchange:   # captured into the graph
                zdist.all_reduce_sum(self._pk.buf if prefetch else self._pk.acc, self._group)
        else:
            if exchange:
                self._pk.reduce_all(prefetch)  # the ONE collective of the iteration
            else:
                self._pk.mass_valid = False
            self._q_versions = [q._version for q in self._q]
        lib.call("zsb_hmc_tune_f32", ptr(self._state), ptr(self._stats),
                 int(self._has_step), int(adapt_step), 1.0 if init else 0.0,
                 self.gamma, self.t0, self.kappa, self.target_acceptance_rate,
                 -1.0 if dev else float(t), s)
        if not dev:
            self._queue_flag_check()
        return None

    def _search(self, probe, s):
        """_init_step_size (hmc.py:307-345): host loop, one scalar read-back
        per pass (fires only at t==1 and t==mass_collect_iters)."""
        while True:
            self.n_search_iters += 1
            probe()
            lib.call("zsb_hmc_acc_sum_f32", ptr(self._acc_part),
                     self._npart.value, self._chains, ptr(self._stats), s)
            self._pk.reduce_acc()
            lib.call("zsb_hmc_search_update_f32", ptr(self._state),
                     ptr(self._stats), self.target_acceptance_rate, s)
            if float(self._state[ST_SCOND].item()) == 0.0:
                break

    # ---- generic path -------------------------------------------------------
    def _momentum(self, noise_p, seed, it, s):
        for k, q in enumerate(self._q):
            lib.call("zsb_hmc_momentum_f32", ptr(self._p0[k]),
                     ptr(noise_p[k]) if noise_p else None, ptr(self._mass[k]),
                     self._row_len[k], self._chains, self._row_len[k], seed,
                     it, STREAM_MOMENTUM + 16 * k, self._row0, ptr(self._k0),
                     int(k > 0), ptr(self._state), s)

    def _lf_q(self, q, p, scale, s):
        for k in range(len(q)):
            lib.call("zsb_hmc_leapfrog_q_f32", ptr(q[k]), ptr(p[k]),
                     ptr(self._mass[k]), self._row_len[k], self._row_len[k],
                     self._eps_ptr(), scale, q[k].numel(), s)

    def _lf_p(self, p, g, scale, s):
        for k in range(len(p)):
            lib.call("zsb_hmc_leapfrog_p_f32", ptr(p[k]), ptr(g[k]),
                     self._eps_ptr(), scale, p[k].numel(), s)

    def _mh_generic(self, q_new, p_new, noise_u, seed, it, s, full):
        with torch.no_grad():                                 # hmc.py:47-50
            lp0 = self._get_log_posterior(self._q).reshape(-1).contiguous()
            lp1 = self._get_log_posterior(q_new).reshape(-1).contiguous()
        for k in range(len(p_new)):
            lib.call("zsb_hmc_kinetic_f32", ptr(p_new[k]), ptr(self._mass[k]),
                     self._row_len[k], self._chains, self._row_len[k],
                     ptr(self._k1), int(k > 0), s)
        if full:
            self._lp0.copy_(lp0)
        lib.call("zsb_hmc_mh_f32", ptr(lp0), ptr(lp1), ptr(self._k0),
                 ptr(self._k1), ptr(noise_u) if noise_u is not None else None,
                 seed, it, self._row0, self._chains,
                 ptr(self._h0) if full else None,
                 ptr(self._h1) if full else None, ptr(self._acc),
                 ptr(self._accept) if full else None,
                 ptr(self._lpsel) if full else None, ptr(self._acc_part),
                 ctypes.byref(self._npart), ptr(self._state), s)

    def _iterate_generic(self, noise_p, noise_u, seed, it, init, s):
        self._momentum(noise_p, seed, it, s)
        if init:
            def probe():                                      # hmc.py:314-326
                q = [x.clone() for x in self._q]
                p = [x.clone() for x in self._p0]
                self._lf_p(p, self._get_gradient(q), 0.5, s)
                self._lf_q(q, p, 1.0, s)
                self._lf_p(p, self._get_gradient(q), 0.5, s)
                self._mh_generic(q, p, noise_u, seed, it, s, full=False)
            self._search(probe, s)
        cq = [x.clone() for x in self._q]
        cp = [x.clone() for x in self._p0]
        L = self.n_leapfrogs
        for i in range(L + 1):                                # hmc.py:352-364
            if i > 0:
                self._lf_q(cq, cp, 1.0, s)
            g = self._get_gradient(cq)
            self._lf_p(cp, g, 1.0 if 0 < i < L else 0.5, s)
        self._mh_generic(cq, cp, noise_u, seed, it, s, full=True)
        for k, q in enumerate(self._q):                       # hmc.py:488-497
            lib.call("zsb_hmc_select_f32", ptr(q), ptr(cq[k]),
                     ptr(self._accept), self._chains, self._row_len[k], s)

    # ---- fused diagonal normal ---------------------------------------------
    def _iterate_diag(self, noise_p, noise_u, seed, it, init, s):
        f = self._fused
        q = self._q[0]

        def launch(search):
            lib.call("zsb_hmc_diag_normal_step_f32", ptr(q),
                     ptr(noise_p[0]) if noise_p else None,
                     ptr(noise_u) if noise_u is not None else None,
                     ptr(f["mean"]), f["mean"].numel(), ptr(f["logstd"]),
                     f["logstd"].numel(), ptr(self._mass[0]),
                     self._row_len[0], ptr(self._state), self.n_leapfrogs,
                     self._chains, self._row_len[0], seed, it, self._row0,
                     int(search), None if search else ptr(self._p0[0]),
                     ptr(self._h0), ptr(self._h1), ptr(self._lp0),
                     ptr(self._lpsel), ptr(self._acc), ptr(self._accept),
                     ptr(self._acc_part), ctypes.byref(self._npart), s)
        if init:
            self._search(lambda: launch(True), s)
        launch(False)

    # ---- fused dense gaussian -----------------------------------------------
    def _setup_dense(self, dev):
        f = self._fused
        D = f["D"]
        impl = self._dense_impl
        if impl is None:
            impl = f.get("impl")
        if impl is None:               # default: fastest legal tensor-core path
            impl = (5 if self.n_leapfrogs >= 1 else 2) if D % 64 == 0 else \
                (1 if D % 32 == 0 else 0)
        if int(impl) in (2, 3, 5) and D % 64 != 0:
            raise ValueError("dense_impl=2/3/5 (fp16 split) needs D % 64 == 0")
        # impl 5: whole-trajectory entry point (hmc_dense_res.cu).  The state of q inside a
        # trajectory is its fp16 hi/lo plane pair; the step-size probes are trajectories with
        # L = 1; n_leapfrogs = 0 (a single half-kick pass) runs on the per-pass kernel (impl 2).
        self._res = int(impl) == 5 and self.n_leapfrogs >= 1
        if int(impl) == 5:
            impl = 2
        # impl 4: impl 2's buffers and probe passes, the L+1 passes of the main trajectory
        # through one entry point (hmc_dense_traj.cu)
        self._traj = int(impl) == 4
        if self._traj:
            if D != 1024 or self.n_leapfrogs < 1:
                raise ValueError("dense_impl=4 needs D == 1024 and n_leapfrogs >= 1")
            impl = 2
        self._impl = int(impl)
        if self._impl >= 1:            # pipeline-shape tuning knob (same results)
            lib.call("zsb_hmc_dense_tc_config", int(os.environ.get("ZSB_TC_BK", "32")))
        nt = lib.load().zsb_hmc_dense_ntiles(D, min(self._impl, 1))
        z = lambda *s: torch.zeros(*s, dtype=_F32, device=dev)
        self._pw = torch.empty_like(self._q[0])
        self._lo = {}
        self._pass_k = 0
        self._lp0_part, self._lp1_part = z(nt * self._chains), \
            z(nt * self._chains)
        self._k_part = z(nt * self._chains)
        self._ntiles = nt
        if self._res:                  # two plane buffers + flags; no fp32 work copies of q
            shape = (2,) + tuple(self._q[0].shape)
            self._planes = [torch.empty(shape, dtype=torch.float16, device=dev)
                            for _ in range(2)]
            self._res_flags = torch.zeros(
                lib.load().zsb_hmc_dense_resident_flags(self._chains),
                dtype=torch.int32, device=dev)
            self._scales = z(4)
            self._scales[3] = f["sP"]
            return
        self._qa, self._qb = torch.empty_like(self._q[0]), \
            torch.empty_like(self._q[0])
        if self._impl == 1:            # TF32 residuals of the A operands
            for t in (self._q[0], self._qa, self._qb):
                self._lo[t.data_ptr()] = torch.empty_like(t)
        if self._impl == 2:            # fp16 hi/lo planes of q * sq
            for t in (self._q[0], self._qa, self._qb):
                self._lo[t.data_ptr()] = torch.empty(
                    (2,) + tuple(t.shape), dtype=torch.float16, device=dev)
            self._scales = z(4)
            self._scales[3] = f["sP"]
        if self._impl == 3:            # planes are built inside the kernel
            self._scales = z(8)
            self._scales[3] = f["sP"]

    def _dense_pass(self, q_cur, q_next, p_in, p_out, scale, lp_part, k_part,
                    s):
        f = self._fused
        if self._impl == 3:
            lib.call("zsb_hmc_dense_leapfrog_h16i_f32", ptr(q_cur), ptr(q_next),
                     ptr(p_in), ptr(p_out), ptr(f["P_h16"]), ptr(f["P_l16"]),
                     ptr(self._scales), self._pass_k, ptr(f.get("b")),
                     ptr(f.get("mu")), ptr(self._mass[0]), ptr(self._state),
                     scale, ptr(lp_part), ptr(k_part), self._chains, f["D"], s)
            self._pass_k += 1
            return
        if self._impl == 2:
            lib.call("zsb_hmc_dense_leapfrog_h16_f32", ptr(q_cur),
                     ptr(self._lo[q_cur.data_ptr()]), ptr(q_next),
                     ptr(self._lo[q_next.data_ptr()])
                     if q_next is not None else None, ptr(p_in), ptr(p_out),
                     ptr(f["P_h16"]), ptr(f["P_l16"]), ptr(self._scales),
                     ptr(f.get("b")), ptr(f.get("mu")), ptr(self._mass[0]),
                     ptr(self._state), scale, ptr(lp_part), ptr(k_part),
                     self._chains, f["D"], s)
            return
        tc = self._impl == 1
        lo_cur = self._lo[q_cur.data_ptr()] if tc else None
        lo_next = self._lo[q_next.data_ptr()] if tc and q_next is not None \
            else None
        lib.call("zsb_hmc_dense_leapfrog_f32", ptr(q_cur), ptr(lo_cur),
                 ptr(q_next), ptr(lo_next), ptr(p_in), ptr(p_out),
                 ptr(f["P_hi"] if tc else f["P"]),
                 ptr(f["P_lo"]) if tc else None,
                 ptr(f.get("b")), ptr(f.get("mu")), ptr(self._mass[0]),
                 ptr(self._state), scale, ptr(lp_part), ptr(k_part),
                 self._chains, f["D"], self._impl, s)

    def _dense_finish_mh(self, noise_u, seed, it, s, full):
        f = self._fused
        lib.call("zsb_hmc_dense_finish_f32", ptr(self._lp0_part), None,
                 self._ntiles, self._chains, f["const"], ptr(self._lp0), None,
                 s)
        lib.call("zsb_hmc_dense_finish_f32", ptr(self._lp1_part),
                 ptr(self._k_part), self._ntiles, self._chains, f["const"],
                 ptr(self._lp1), ptr(self._k1), s)
        lib.call("zsb_hmc_mh_f32", ptr(self._lp0), ptr(self._lp1),
                 ptr(self._k0), ptr(self._k1),
                 ptr(noise_u) if noise_u is not None else None, seed, it,
                 self._row0, self._chains,
                 ptr(self._h0) if full else None,
                 ptr(self._h1) if full else None, ptr(self._acc),
                 ptr(self._accept) if full else None,
                 ptr(self._lpsel) if full else None, ptr(self._acc_part),
                 ctypes.byref(self._npart), ptr(self._state), s)

    def _resident_trajectory(self, L, s):
        """L+1 leapfrog passes on the fp16 plane state; returns the proposal's planes."""
        f = self._fused
        lib.call("zsb_hmc_dense_resident_h16_f32", ptr(self._planes[0]),
                 ptr(self._planes[1]), ptr(self._p0[0]), ptr(self._pw),
                 ptr(f["P_h16"]), ptr(f["P_l16"]), ptr(self._scales), ptr(f.get("b")),
                 ptr(f.get("mu")), ptr(self._mass[0]), ptr(self._state),
                 ptr(self._lp0_part), ptr(self._lp1_part), ptr(self._k_part),
                 ptr(self._res_flags), self._chains, f["D"], L, s)
        return self._planes[L & 1]

    def _iterate_dense_resident(self, noise_u, seed, it, init, s):
        q0 = self._q[0]

        def prepare():
            # planes of q * sq (sq from max|q|) into buffer 0
            lib.call("zsb_hmc_dense_h16_prepare_f32", ptr(q0), ptr(self._planes[0]),
                     ptr(self._scales), q0.numel(), s)
        prepare()
        if init:
            def probe():               # hmc.py:314-326: one leapfrog step = a trajectory, L = 1
                self._resident_trajectory(1, s)
                self._dense_finish_mh(noise_u, seed, it, s, full=False)
            self._search(probe, s)
        prof = None if self._dev_mode else getattr(self, "_profile_events", None)
        if prof is not None:           # bench.py: device time of the trajectory launch
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            e0.record()
        prop = self._resident_trajectory(self.n_leapfrogs, s)
        if prof is not None:
            e1.record()
            prof.append((e0, e1))
        self._dense_finish_mh(noise_u, seed, it, s, full=True)
        lib.call("zsb_hmc_dense_select_planes_f32", ptr(q0), ptr(prop), ptr(self._scales),
                 ptr(self._accept), self._chains, self._row_len[0], s)

    def _iterate_dense(self, noise_p, noise_u, seed, it, init, s):
        q0 = self._q[0]
        self._momentum(noise_p, seed, it, s)
        if self._res:
            return self._iterate_dense_resident(noise_u, seed, it, init, s)
        if self._impl == 1:
            lib.call("zsb_hmc_dense_split_lo_f32", ptr(q0),
                     ptr(self._lo[q0.data_ptr()]), q0.numel(), s)
        elif self._impl == 2:
            lib.call("zsb_hmc_dense_h16_prepare_f32", ptr(q0),
                     ptr(self._lo[q0.data_ptr()]), ptr(self._scales),
                     q0.numel(), s)
        def prepare3():                # impl 3: seed the max|q| slot, restart the pass count
            if self._impl == 3:
                lib.call("zsb_hmc_dense_h16i_prepare_f32", ptr(q0),
                         ptr(self._scales), q0.numel(), s)
                self._pass_k = 0
        if init:
            def probe():
                prepare3()
                self._dense_pass(q0, self._qa, self._p0[0], self._pw, 0.5,
                                 self._lp0_part, None, s)
                self._dense_pass(self._qa, None, self._pw, self._pw, 0.5,
                                 self._lp1_part, self._k_part, s)
                self._dense_finish_mh(noise_u, seed, it, s, full=False)
            self._search(probe, s)
        L = self.n_leapfrogs
        cur, nxt = q0, self._qa
        p_in = self._p0[0]
        prepare3()
        if self._traj:
            f = self._fused
            prof = None if self._dev_mode else getattr(self, "_profile_events", None)
            if prof is not None:
                e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                e0.record()
            lib.call("zsb_hmc_dense_trajectory_h16_f32", ptr(q0),
                     ptr(self._lo[q0.data_ptr()]), ptr(self._qa),
                     ptr(self._lo[self._qa.data_ptr()]), ptr(self._qb),
                     ptr(self._lo[self._qb.data_ptr()]), ptr(self._p0[0]),
                     ptr(self._pw), ptr(f["P_h16"]), ptr(f["P_l16"]),
                     ptr(self._scales), ptr(f.get("b")), ptr(f.get("mu")),
                     ptr(self._mass[0]), ptr(self._state), ptr(self._lp0_part),
                     ptr(self._lp1_part), ptr(self._k_part), self._chains, f["D"],
                     L, s)
            if prof is not None:
                e1.record()
                prof.append((e0, e1))
            cur = self._qa if (L - 1) % 2 == 0 else self._qb
            self._dense_finish_mh(noise_u, seed, it, s, full=True)
            lib.call("zsb_hmc_select_f32", ptr(q0), ptr(cur), ptr(self._accept),
                     self._chains, self._row_len[0], s)
            return
        prof = getattr(self, "_profile_events", None)
        if self._dev_mode:
            prof = None
        if prof is not None:           # bench.py: device time of the L+1 passes
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            e0.record()
        for i in range(L + 1):
            last = i == L
            self._dense_pass(
                cur, None if last else nxt, p_in, self._pw,
                1.0 if 0 < i < L else 0.5,
                self._lp0_part if i == 0 else
                (self._lp1_part if last else None),
                self._k_part if last else None, s)
            p_in = self._pw
            if not last:
                cur, nxt = nxt, (self._qb if nxt is self._qa else self._qa)
        if prof is not None:
            e1.record()
            prof.append((e0, e1))
        if L == 0:
            self._lp1_part.copy_(self._lp0_part)
        self._dense_finish_mh(noise_u, seed, it, s, full=True)
        lib.call("zsb_hmc_select_f32", ptr(q0), ptr(cur), ptr(self._accept),
                 self._chains, self._row_len[0], s)

    # ----------------------------------------------------------- checkpointing
    def state_dict(self):
        """All sampler state (the reference keeps it in tf.Variables and has
        no checkpoint API, SURVEY section 5)."""
        st = self._state.clone()
        st[ST_FLAGS] = 0                       # the check_numerics flag is not sampler state
        d = {"t": self._t, "ewmv_t": self._ewmv_t, "state": st}
        if self._has_mass:
            d["ewmv_mean"] = [m.clone() for m in self._ew_mean]
            d["ewmv_var"] = [v.clone() for v in self._ew_var]
        return d

    def load_state_dict(self, d):
        self._t, self._ewmv_t = int(d["t"]), int(d["ewmv_t"])
        self._state.copy_(d["state"])
        self._state[ST_FLAGS] = 0
        self._pk.mass_valid = False            # statistics are recomputed from the latents
        self._state[ST_T] = float(self._t)
        self._state[ST_EWT] = float(self._ewmv_t)
        if self._has_mass:
            for m, s in zip(self._ew_mean, d["ewmv_mean"]):
                m.copy_(s)
            for v, s in zip(self._ew_var, d["ewmv_var"]):
                v.copy_(s)


def _suffix_ok(param_shape, data_shape):
    shape = list(param_shape)
    while shape and shape[0] == 1:
        shape.pop(0)
    n = len(shape)
    return n == 0 or list(data_shape[len(data_shape) - n:]) == shape


def _detect_diag_normal(meta_bn, observed, latent):
    """Recognise ``bn.normal(name, mean, std|logstd, group_ndims=#data axes)``
    as the only stochastic node (examples/toy_examples/gaussian.py:15-20) and
    return the fused-kernel descriptor, else None (-> generic path)."""
    from .distributions import Normal
    if len(latent) != 1 or meta_bn.log_joint is not None:
        return None
    name, q = next(iter(latent.items()))
    if not isinstance(q, torch.Tensor) or not q.is_cuda:
        return None
    try:
        bn = meta_bn.observe(**merge_dicts(latent, observed))
    except Exception:
        return None
    stoch = [n for n in bn.nodes.values() if isinstance(n, StochasticTensor)]
    if len(stoch) != 1 or stoch[0].name != name:
        return None
    d = stoch[0].dist
    if type(d) is not Normal or d.use_path_derivative:
        return None
    g = d.group_ndims
    if g < 1 or g >= q.dim() + 1:
        return None
    data_shape = tuple(q.shape[q.dim() - g:])
    if q.dim() - g < 1:
        return None
    row_len = 1
    for s in data_shape:
        row_len *= int(s)
    if row_len > 1024:
        return None
    if not (_suffix_ok(d.mean.shape, data_shape)
            and _suffix_ok(d.logstd.shape, data_shape)):
        return None
    return {"kind": "diag_normal",
            "mean": d.mean.detach().to(_F32).contiguous().reshape(-1),
            "logstd": d.logstd.detach().to(_F32).contiguous().reshape(-1)}
