"""SG-MCMC samplers on H100 kernels -- drop-in for zhusuan/sgmcmc.py
(``SGLD``, ``PSGLD``, ``SGHMC``, ``SGNHT``; same constructors and
``sample(meta_bn, observed, latent) -> (sample_op, SGMCMCInfo)`` contract,
sgmcmc.py:119-161).  As in hmc.py, ``latent`` values are float32 CUDA tensors
updated in place and ``sample_op`` is a callable; minibatches that the
reference feeds through placeholders are passed as
``sample_op(observed={...})`` overrides.  Gradients of the user log-joint
come from torch autograd over the registry kernels (replaces tf.gradients,
sgmcmc.py:96-98); the update itself is one fused kernel per latent.
"""
from collections import namedtuple

import torch

from . import dist as zdist
from . import random as zrandom
from ._lib import lib, ptr, stream
from .utils import merge_dicts

__all__ = ["SGMCMC", "SGLD", "PSGLD", "SGHMC", "SGNHT"]

_F32 = torch.float32


class _SampleOp(object):
    def __init__(self, s):
        self._s = s

    def __call__(self, observed=None, noise=None, learning_rate=None):
        return self._s._iterate(observed, noise, learning_rate)

    run = __call__


class SGMCMC(object):
    """sgmcmc.py:24-167."""

    def __init__(self, seed=None, process_group=None, chain_offset=None):
        self.t = 0                                   # sgmcmc.py:73 (int32)
        self._seed = seed
        self._group = process_group
        self._chain_offset = chain_offset

    def _make_grad_func(self, meta_bn, observed, latent):
        if callable(meta_bn):                        # sgmcmc.py:76-80
            self._log_joint = meta_bn
        else:
            self._log_joint = lambda obs: meta_bn.observe(**obs).log_joint()
        self._observed = dict(observed)
        self._latent_k = list(latent.keys())
        self._var_list = []
        for k in self._latent_k:                     # sgmcmc.py:84-88
            v = latent[k]
            if not isinstance(v, torch.Tensor):
                raise TypeError(
                    "latent['{}'] is not a Variable (a float32 CUDA "
                    "torch.Tensor updated in place).".format(k))
            if v.dtype != _F32 or not v.is_contiguous():
                raise TypeError("latent['{}'] must be a contiguous float32 "
                                "tensor.".format(k))
            self._var_list.append(v)

        def grad_func(var_list):                     # sgmcmc.py:91-100
            xs = [v.detach().requires_grad_(True) for v in var_list]
            with torch.enable_grad():
                lp = self._log_joint(merge_dicts(
                    dict(zip(self._latent_k, xs)), self._observed))
                gs = torch.autograd.grad(lp.sum(), xs, allow_unused=True)
            if self._chains is None:
                self._set_chains(lp)
            return [g.contiguous() if g is not None else torch.zeros_like(x)
                    for g, x in zip(gs, xs)]
        return grad_func

    def _set_chains(self, lp):
        ncd = lp.dim()
        chains = 1
        for s in lp.shape:
            chains *= int(s)
        self._chains = max(chains, 1)
        # every latent must carry the chain axes of the log-joint in front (as HMC.sample checks,
        # hmc.py:436-449): the kernels walk chains * row_len elements per latent
        for k, q in zip(self._latent_k, self._var_list):
            if tuple(q.shape[:ncd]) != tuple(lp.shape):
                raise ValueError(
                    "latent['{}'] has shape {} but the log joint has chain shape {}: every "
                    "latent must start with the chain axes".format(
                        k, tuple(q.shape), tuple(lp.shape)))
        self._row_len = [max(1, q.numel() // self._chains)
                         for q in self._var_list]
        w, r = zdist.world(self._group)
        self._row0 = (r * self._chains if self._chain_offset is None
                      else int(self._chain_offset))

    def sample(self, meta_bn, observed, latent):
        """sgmcmc.py:119-161."""
        self._chains = None
        self._grad_func = self._make_grad_func(meta_bn, observed, latent)
        with torch.no_grad():
            lp = self._log_joint(merge_dicts(
                dict(zip(self._latent_k, self._var_list)), self._observed))
        self._set_chains(lp)
        dev = self._var_list[0].device
        self._part = torch.zeros(lib.load().zsb_sgmcmc_parts(), dtype=_F32,
                                 device=dev)
        infos = self._define_variables(self._var_list)
        names = list(infos.keys())
        SGMCMCInfo = namedtuple("SGMCMCInfo", names)      # sgmcmc.py:109-115
        self._info = SGMCMCInfo(**infos)
        return _SampleOp(self), self._info

    def _seed_now(self):
        return self._seed if self._seed is not None else zrandom.get_seed()

    def _iterate(self, observed, noise, learning_rate):
        if observed is not None:
            self._observed.update(observed)
            f = getattr(self._log_joint, "_zsb_fused", None)
            if f is not None and "obj" in f and hasattr(f["obj"], "set_batch"):
                f["obj"].set_batch(observed)
        if learning_rate is not None:
            self.lr = float(learning_rate)
        self._update(self._var_list, self._grad_func, noise or {})
        self.t += 1                                        # sgmcmc.py:107-108
        return None

    # ----------------------------------------------------------- checkpointing
    _STATE_LISTS = ("vs", "alphas", "_alpha1", "_mean_k")

    def state_dict(self):
        """All sampler state besides the latents themselves: the iteration counter ``t``
        (sgmcmc.py:73) and the auxiliary variables of the update rule -- PSGLD's second-moment
        accumulator, SGHMC / SGNHT momenta, SGNHT thermostats (sgmcmc.py:225-226, 320-324,
        450-458).  The reference keeps them in tf.Variables and has no checkpoint API."""
        d = {"t": int(self.t), "lr": float(self.lr)}
        for name in self._STATE_LISTS:
            if hasattr(self, name):
                d[name] = [x.clone() for x in getattr(self, name)]
        return d

    def load_state_dict(self, d):
        self.t = int(d["t"])
        self.lr = float(d.get("lr", self.lr))
        for name in self._STATE_LISTS:
            if name in d:
                for dst, src in zip(getattr(self, name), d[name]):
                    dst.copy_(src)

    def _noise(self, noise, key, k):
        n = noise.get(key)
        return None if n is None else ptr(n[self._latent_k[k]].contiguous())


class SGLD(SGMCMC):
    """sgmcmc.py:170-200."""

    def __init__(self, learning_rate, **kw):
        self.lr = float(learning_rate)
        super(SGLD, self).__init__(**kw)

    def _define_variables(self, qs):
        return {"q": dict(zip(self._latent_k, qs))}

    def _update(self, qs, grad_func, noise):
        gs = grad_func(qs)
        s = stream()
        for k, (q, g) in enumerate(zip(qs, gs)):
            lib.call("zsb_sgmcmc_sgld_f32", ptr(q), ptr(g),
                     self._noise(noise, "noise", k), self.lr, self._chains,
                     self._row_len[k], self._seed_now() + k,
                     self.t & 0xFFFFFFFF, self._row0, s)


class PSGLD(SGLD):
    """sgmcmc.py:203-257 (RMSprop preconditioner)."""
    RMSHParams = namedtuple('RMSHParams', 'decay epsilon')

    def __init__(self, learning_rate, preconditioner='rms',
                 preconditioner_hparams=None, **kw):
        if preconditioner != 'rms':
            raise KeyError(preconditioner)
        if preconditioner_hparams is None:
            preconditioner_hparams = PSGLD.RMSHParams(decay=0.9, epsilon=1e-3)
        self.preconditioner_hparams = preconditioner_hparams
        super(PSGLD, self).__init__(learning_rate, **kw)

    def _define_variables(self, qs):
        self.vs = [torch.zeros_like(q) for q in qs]       # sgmcmc.py:225-226
        return {"q": dict(zip(self._latent_k, qs))}

    def _update(self, qs, grad_func, noise):
        gs = grad_func(qs)
        s = stream()
        hp = self.preconditioner_hparams
        for k, (q, g) in enumerate(zip(qs, gs)):
            lib.call("zsb_sgmcmc_psgld_f32", ptr(q), ptr(self.vs[k]), ptr(g),
                     self._noise(noise, "noise", k), self.lr, float(hp.decay),
                     float(hp.epsilon), self._chains, self._row_len[k],
                     self._seed_now() + k, self.t & 0xFFFFFFFF, self._row0, s)


class SGHMC(SGMCMC):
    """sgmcmc.py:260-371."""

    def __init__(self, learning_rate, friction=0.25, variance_estimate=0.,
                 n_iter_resample_v=20, second_order=True, use_fused=True,
                 **kw):
        self._use_fused = bool(use_fused)
        self.lr = float(learning_rate)
        self.alpha = float(friction)
        self.beta = float(variance_estimate)
        self.n_iter_resample_v = int(n_iter_resample_v or 0)
        self.second_order = bool(second_order)
        super(SGHMC, self).__init__(**kw)

    def _resample(self, k, v, noise, key, it):
        lib.call("zsb_sgmcmc_resample_v_f32", ptr(v),
                 self._noise(noise, key, k), self.lr, self._chains,
                 self._row_len[k], self._seed_now() + k, it, self._row0,
                 stream())

    def _define_variables(self, qs, noise=None):
        self.vs = [torch.empty_like(q) for q in qs]       # sgmcmc.py:320-324
        for k, v in enumerate(self.vs):
            self._resample(k, v, {}, "v0", 0xFFFFFFFF)
        self._mean_k = [torch.zeros(1, dtype=_F32, device=q.device)
                        for q in qs]
        return {"q": dict(zip(self._latent_k, qs)),
                "mean_k": dict(zip(self._latent_k,
                                   [m[0] for m in self._mean_k]))}

    def init_momentum(self, noise_v0):
        """Parity hook: v0 = N(0, sqrt(lr)) from injected standard normals."""
        for k, v in enumerate(self.vs):
            self._resample(k, v, {"v0": noise_v0}, "v0", 0)

    def _maybe_resample(self, noise):
        if self.n_iter_resample_v != 0 and \
                self.t % self.n_iter_resample_v == 0:      # sgmcmc.py:330-336
            for k, v in enumerate(self.vs):
                self._resample(k, v, noise, "resample", self.t & 0xFFFFFFFF)

    def _fused_bnn(self):
        f = getattr(self._log_joint, "_zsb_fused", None)
        if f is None or f.get("kind") != "bnn_regression":
            return None
        obj = f["obj"]
        if list(self._latent_k) != list(obj.names):
            return None
        w0, w1 = self._var_list
        if w0.dim() != 3 or w1.dim() != 3 or w1.shape[1] != 1 or \
                w1.shape[2] != w0.shape[1] + 1 or w0.shape[2] > 16 or \
                w0.shape[1] > 64 or obj.x.shape[0] > 512:
            return None
        return obj

    def _update_fused_bnn(self, obj, noise):
        """Whole step in one kernel (csrc/sgmcmc_bnn.cu)."""
        w0, w1 = self._var_list
        x, y = obj.x.contiguous(), obj.y.contiguous()
        resample = int(self.n_iter_resample_v != 0 and
                       self.t % self.n_iter_resample_v == 0)
        if not hasattr(self, "_bnn_part"):
            self._bnn_part = torch.zeros(2 * lib.load().zsb_sgmcmc_parts(),
                                         dtype=_F32, device=w0.device)
            self._bnn_mean_k = torch.zeros(2, dtype=_F32, device=w0.device)
            self._info.mean_k[self._latent_k[0]] = self._bnn_mean_k[0]
            self._info.mean_k[self._latent_k[1]] = self._bnn_mean_k[1]
        lib.call("zsb_sgmcmc_sghmc_bnn_f32", ptr(w0), ptr(w1), ptr(self.vs[0]),
                 ptr(self.vs[1]), ptr(x), ptr(y), int(x.shape[0]),
                 int(x.shape[1]), int(w0.shape[1]), ptr(obj.logstds[0]),
                 obj.logstds[0].numel(), ptr(obj.logstds[1]),
                 obj.logstds[1].numel(), obj.y_logstd, obj.n_train, self.lr,
                 self.alpha, self.beta, int(self.second_order), resample,
                 self._noise(noise, "noise", 0), self._noise(noise, "noise", 1),
                 self._noise(noise, "resample", 0),
                 self._noise(noise, "resample", 1), self._seed_now(),
                 self.t & 0xFFFFFFFF, self._row0, ptr(self._bnn_part),
                 ptr(self._bnn_mean_k), self._chains, stream())

    def _update(self, qs, grad_func, noise):
        obj = self._fused_bnn() if self._use_fused else None
        if obj is not None:
            return self._update_fused_bnn(obj, noise)
        s = stream()
        self._maybe_resample(noise)
        if self.second_order:                              # sgmcmc.py:351
            for q, v in zip(qs, self.vs):
                lib.call("zsb_sgmcmc_half_q_f32", ptr(q), ptr(v), q.numel(), s)
        gs = grad_func(qs)
        for k, (q, g) in enumerate(zip(qs, gs)):
            lib.call("zsb_sgmcmc_sghmc_f32", ptr(q), ptr(self.vs[k]), ptr(g),
                     self._noise(noise, "noise", k), self.lr, self.alpha,
                     self.beta, int(self.second_order), self._chains,
                     self._row_len[k], self._seed_now() + k,
                     self.t & 0xFFFFFFFF, self._row0, ptr(self._part),
                     ptr(self._mean_k[k]), s)


class SGNHT(SGMCMC):
    """sgmcmc.py:374-523."""

    def __init__(self, learning_rate, variance_extra=0., tune_rate=1.,
                 n_iter_resample_v=None, second_order=True,
                 use_vector_alpha=True, **kw):
        self.lr = float(learning_rate)
        self.a = float(variance_extra)
        self.tune_rate = float(tune_rate)
        self.n_iter_resample_v = int(n_iter_resample_v or 0)
        self.second_order = bool(second_order)
        self.use_vector_alpha = bool(use_vector_alpha)
        super(SGNHT, self).__init__(**kw)

    _resample = SGHMC._resample
    init_momentum = SGHMC.init_momentum
    _maybe_resample = SGHMC._maybe_resample

    def _define_variables(self, qs):
        self.vs = [torch.empty_like(q) for q in qs]        # sgmcmc.py:450-452
        for k, v in enumerate(self.vs):
            self._resample(k, v, {}, "v0", 0xFFFFFFFF)
        dev = qs[0].device
        if self.use_vector_alpha:                          # sgmcmc.py:454-458
            self.alphas = [torch.full_like(q, self.a) for q in qs]
            self._mean_k = [torch.zeros_like(q) for q in qs]
            mk = self._mean_k
            al = self.alphas
        else:
            self.alphas = [torch.full((1,), self.a, dtype=_F32, device=dev)
                           for q in qs]
            self._alpha1 = [torch.zeros(1, dtype=_F32, device=dev)
                            for q in qs]
            self._mean_k = [torch.zeros(1, dtype=_F32, device=dev)
                            for q in qs]
            mk = [m[0] for m in self._mean_k]
            al = [a[0] for a in self.alphas]
        return {"q": dict(zip(self._latent_k, qs)),
                "mean_k": dict(zip(self._latent_k, mk)),
                "alpha": dict(zip(self._latent_k, al))}

    def _update(self, qs, grad_func, noise):
        s = stream()
        it = self.t & 0xFFFFFFFF
        self._maybe_resample(noise)
        if not self.use_vector_alpha and self.second_order:
            for k, v in enumerate(self.vs):                # sgmcmc.py:494-496
                lib.call("zsb_sgmcmc_mean_sq_f32", ptr(v), v.numel(),
                         ptr(self._part), ptr(self._mean_k[k]), s)
                zdist.all_reduce_weighted_mean_(self._mean_k[k], v.numel(), self._group)
                lib.call("zsb_sgmcmc_sgnht_alpha_f32", ptr(self._alpha1[k]),
                         ptr(self.alphas[k]), ptr(self._mean_k[k]),
                         0.5 * self.tune_rate, self.lr, s)
        if self.second_order:                              # sgmcmc.py:493
            for q, v in zip(qs, self.vs):
                lib.call("zsb_sgmcmc_half_q_f32", ptr(q), ptr(v), q.numel(), s)
        gs = grad_func(qs)
        for k, (q, g) in enumerate(zip(qs, gs)):
            nz = self._noise(noise, "noise", k)
            if self.use_vector_alpha:
                lib.call("zsb_sgmcmc_sgnht_vec_f32", ptr(q), ptr(self.vs[k]),
                         ptr(self.alphas[k]), ptr(g), nz, self.lr, self.a,
                         self.tune_rate, int(self.second_order), self._chains,
                         self._row_len[k], self._seed_now() + k, it,
                         self._row0, ptr(self._mean_k[k]), s)
            else:
                a_eff = self._alpha1[k] if self.second_order \
                    else self.alphas[k]
                lib.call("zsb_sgmcmc_sgnht_scalar_f32", ptr(q),
                         ptr(self.vs[k]), ptr(a_eff), ptr(g), nz, self.lr,
                         self.a, int(self.second_order), self._chains,
                         self._row_len[k], self._seed_now() + k, it,
                         self._row0, ptr(self._part), ptr(self._mean_k[k]), s)
                # chains sharded over ranks: the thermostat is driven by the mean kinetic energy
                # of ALL chains (one 8-byte all-reduce per latent and step; no-op on one rank)
                zdist.all_reduce_weighted_mean_(self._mean_k[k], q.numel(), self._group)
                coef = 0.5 * self.tune_rate if self.second_order \
                    else self.tune_rate                    # sgmcmc.py:490, 506
                lib.call("zsb_sgmcmc_sgnht_alpha_f32", ptr(self.alphas[k]),
                         ptr(a_eff), ptr(self._mean_k[k]), coef, self.lr, s)
