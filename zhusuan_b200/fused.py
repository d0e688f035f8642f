"""Log-joint descriptors that ``HMC.sample`` recognises and runs on fused
kernels.  Each is also a plain ``log_joint(observed_dict)`` callable built
from torch ops, so it works on the generic path and as its own cross-check.
"""
import math

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .distributions.base import Distribution
from .distributions.multivariate import MultivariateNormalCholesky
from .distributions.univariate import Normal

__all__ = ["GaussianLogJoint", "BNNRegressionLogJoint", "LNTMLogJoint", "PMFLogJoint", "linear",
           "class_linear", "noisy_bn_linear", "bn_linear", "linear_bernoulli_log_prob",
           "LinearBernoulli", "LinearOnehotCategorical", "LinearNormal", "RBFKernel",
           "gp_conditional", "conv2d", "conv2d_transpose", "bn_conv2d", "bn_conv2d_transpose",
           "sigmoid_conv2d_transpose", "conv2d_tc", "conv2d_transpose_tc"]


class GaussianLogJoint(object):
    """log p(x) = -1/2 (x-mu)^T P (x-mu) - 1/2 log|2 pi Sigma|, P = Sigma^-1
    shared by all chains (BASELINE config 2; the reference can only express
    this as a callable ``log_joint`` because MultivariateNormalCholesky
    broadcasts L to every chain, multivariate.py:183-185).

    precision: [D, D] symmetric (numpy float64 preferred: the b = P mu vector
    and the hi/lo split are derived in float64 on the host, once).
    """

    def __init__(self, precision, mean=None, log_det_cov=None, name="x",
                 device="cuda", impl=None):
        P64 = np.asarray(precision.detach().cpu().numpy()
                         if isinstance(precision, torch.Tensor)
                         else precision, dtype=np.float64)
        D = P64.shape[0]
        if P64.shape != (D, D):
            raise ValueError("precision must be square")
        if D % 16 != 0:
            raise ValueError("the fused dense-Gaussian path needs D % 16 == 0")
        P64 = 0.5 * (P64 + P64.T)
        self.name = name
        self.D = D
        if log_det_cov is None:
            sign, ld = np.linalg.slogdet(P64)
            log_det_cov = -ld
        self.const = float(-0.5 * (D * math.log(2 * math.pi) + log_det_cov))
        P32 = P64.astype(np.float32)
        self.P = torch.as_tensor(P32, device=device).contiguous()
        d = {"kind": "dense_gaussian", "D": D, "P": self.P,
             "const": self.const, "impl": impl}
        self.mu = None
        if mean is not None:
            mu64 = np.asarray(mean, np.float64).reshape(D)
            self.mu = torch.as_tensor(mu64.astype(np.float32), device=device)
            d["mu"] = self.mu
            d["b"] = torch.as_tensor(
                (P32.astype(np.float64) @ mu64).astype(np.float32),
                device=device)
        # 3xTF32 split for the tensor-core path: hi = fp32 with the low 13
        # mantissa bits cleared (exactly representable in TF32), lo = P - hi.
        hi = (P32.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
        lo = (P32 - hi).astype(np.float32)
        d["P_hi"] = torch.as_tensor(hi, device=device).contiguous()
        d["P_lo"] = torch.as_tensor(lo, device=device).contiguous()
        # fp16 split for impl 2: P*sP = h + l with sP a power of two that puts
        # max|P| in [2^11, 2^12); products then fit fp32 accumulation exactly.
        pmax = float(np.abs(P32).max())
        sP = float(2.0 ** (12 - np.frexp(pmax)[1])) if pmax > 0 else 1.0
        x = P32.astype(np.float64) * sP
        h16 = x.astype(np.float16)
        l16 = (x - h16.astype(np.float64)).astype(np.float16)
        d["sP"] = sP
        # bounds the fp16-split trajectory uses to keep the planes of q inside fp16's range
        # (hmc_dense_epilogue.cuh): |g| <= max|b| + ||P||_inf max|q|
        d["P_inf"] = float(np.abs(P32.astype(np.float64)).sum(1).max())
        d["b_max"] = float(d["b"].abs().max()) if "b" in d else 0.0
        d["P_h16"] = torch.as_tensor(h16, device=device).contiguous()
        d["P_l16"] = torch.as_tensor(l16, device=device).contiguous()
        self._zsb_fused = d

    def __call__(self, observed):
        x = observed[self.name]
        if self.mu is not None:
            x = x - self.mu
        return -0.5 * ((x @ self.P) * x).sum(-1) + self.const


class BNNRegressionLogJoint(object):
    """The log-joint of examples/bayesian_neural_nets/bnn_sgmcmc.py:19-35, 74-77
    (and bnn_vi.py:18-35, 83-86) for layer sizes [n_in, H, 1] and per-particle
    weights:

        w0 [K, H, n_in+1] ~ N(0, exp(logstds[0])),
        w1 [K, 1, H+1]    ~ N(0, exp(logstds[1])),
        y ~ N(net(x; w), exp(y_logstd)),
        log_joint = sum log p(w) + mean_batch(log p(y|x,w)) * n_train.

    As a callable it is the generic-path log-joint (registry Normal kernels +
    torch einsum under the tape).  Three kinds of consumer recognise it and run
    fused kernels instead:

    * ``zs.SGHMC`` / ``SGLD`` / ``PSGLD`` / ``SGNHT`` run the whole step in one
      launch (zsb_sgmcmc_bnn_step_f32), for minibatches of up to 512 rows and
      a float ``y_logstd``.
    * ``zs.variational.elbo`` / ``iw_objective`` / ``klpq`` and
      ``zs.is_loglikelihood`` take the log-joint term from
      ``fused_log_joint`` (zsb_bnn_logjoint_f32: value and gradient in one
      launch, differentiable w.r.t. w0, w1 and a tensor ``y_logstd``).
    * ``zs.HMC`` takes ``logp`` and ``grad`` from the same kernel, one launch
      each, over any number of rows (full-batch HMC).  It decides in
      ``sample()``; rows fed later through ``sample_op(observed=...)`` that do
      not fit the kernel are evaluated on the generic path for that call.

    ``predictive(observed)`` gives y_mean and the per-point log-likelihood of
    every particle in one launch (test-set RMSE and log-likelihood of
    variational, SG-MCMC or HMC samples).

    Feed minibatches with ``sample_op(observed={'x': xb, 'y': yb})`` or in the
    objective's ``observed``; ``x`` is [B, n_in] and ``y`` holds B values.

    ``y_logstd`` is a float or a 0-d float32 CUDA tensor.  A tensor is read in
    place by the kernels (no host sync) and receives a gradient, so it can be
    learned as bnn_vi.py does; SG-MCMC then takes its generic path.

    ``logstds[k]`` broadcasts against w_k with NumPy rules.  Shapes that
    broadcast to one particle's weights -- for logstds[0] e.g. [H, n_in+1],
    [H, 1] (one scale per hidden unit), [n_in+1] or [] -- run on the fused
    kernels; shapes with chain axes, e.g. [chains, H, n_in+1] or
    [chains, 1, H+1], run on the generic path.  ``fused_inputs`` is the
    eligibility check of the objectives, HMC and ``predictive``: 3-D latents
    [K, H, n_in+1] / [K, 1, H+1] in float32 with n_in + 1 <= 16 and H <= 64,
    ``x`` [B, n_in] and B values of ``y``, all on one CUDA device, float32
    prior logstds that broadcast to one particle and do not require a
    gradient.  Under ``torch.no_grad()`` ``fused_log_joint`` launches the
    value-only kernel; its gradient is first order (no double backward).  Anything else: the objectives and
    HMC fall back to ``__call__`` under autograd, ``predictive`` raises.

    Deeper nets: ``names`` and ``logstds`` give one entry per weight layer, L >= 2 of them, at
    layer sizes [n_0, n_1, ..., n_{L-1}, 1] (layer i: w_i [K, n_{i+1}, n_i + 1], ReLU after every
    layer but the last).  L = 2 runs on the kernels above.  L >= 3 runs on csrc/bnn_deep.cu with
    the same consumers and rules -- the SG-MCMC step in one launch, ``fused_log_joint``,
    ``predictive`` and the HMC provider -- within its limits: L <= 8, n_0 <= 128, hidden widths
    <= 128, at most 32768 weights per particle, any number of rows B (minibatches included) and
    particles K.  ``fused_inputs`` then returns the L latents, ``x`` and ``y``.  Shapes past the
    limits run the generic path.
    """

    MAX_IN1, MAX_H = 16, 64      # limits of the fused kernels (n_in + 1, H)

    def __init__(self, x, y, logstds, n_train, y_logstd=-0.95,
                 names=("w0", "w1")):
        from .distributions import Normal
        self._Normal = Normal
        self.x, self.y = x, y
        self.logstds = [l.contiguous() for l in logstds]
        if len(self.logstds) != len(tuple(names)) or len(self.logstds) < 2:
            raise ValueError("BNNRegressionLogJoint needs one logstd per weight layer and at "
                             "least two layers (got %d names, %d logstds)"
                             % (len(tuple(names)), len(self.logstds)))
        self.n_train = float(n_train)
        if isinstance(y_logstd, torch.Tensor):
            if y_logstd.dim() != 0 or y_logstd.dtype != torch.float32 or \
                    not y_logstd.is_cuda:
                raise ValueError("y_logstd must be a float or a 0-d float32 CUDA tensor, "
                                 "got %s %s on %s" % (y_logstd.dtype, tuple(y_logstd.shape),
                                                      y_logstd.device))
            self.y_logstd = y_logstd
        else:
            self.y_logstd = float(y_logstd)
        self.names = tuple(names)
        self._prior_cache = {}
        self._ys_dev = None
        self._zsb_fused = {"kind": "bnn_regression", "obj": self}

    def fused_prior_logstd(self, k, shape):
        """logstds[k] as the fused kernel reads it: flat over one chain's
        weights of ``shape`` ([H, n_in+1] or [1, H+1]), index modulo its size.
        A logstd whose shape, leading 1s dropped, is a suffix of ``shape``
        already reads right and is returned as is; one that only broadcasts
        to ``shape`` (e.g. [H, 1]) is expanded once and cached until it is
        modified in place.  None if it does not broadcast to ``shape``
        (it carries chain axes)."""
        ls = self.logstds[k]
        s = list(ls.shape)
        while s and s[0] == 1:
            s.pop(0)
        shape = tuple(int(d) for d in shape)
        if len(s) > len(shape) or any(a != 1 and a != b for a, b in
                                      zip(s[::-1], shape[::-1])):
            return None
        if not s or tuple(s) == shape[len(shape) - len(s):]:
            return ls
        key = (k, shape, ls.data_ptr(), tuple(ls.shape), ls._version)
        e = self._prior_cache.get(k)
        if e is None or e[0] != key:
            e = (key, ls.reshape(s).expand(shape).contiguous())
            self._prior_cache[k] = e
        return e[1]

    def set_batch(self, observed):
        if "x" in observed:
            self.x = observed["x"]
        if "y" in observed:
            self.y = observed["y"]

    def _y_logstd_dev(self, device):
        """y_logstd as the one-element device array the kernel reads: the tensor itself, or a
        copy of the float, made once per value and device."""
        if isinstance(self.y_logstd, torch.Tensor):
            return self.y_logstd
        e = self._ys_dev
        if e is None or e[0] != (self.y_logstd, device):
            e = ((self.y_logstd, device),
                 torch.tensor(self.y_logstd, dtype=torch.float32, device=device))
            self._ys_dev = e
        return e[1]

    def fused_inputs(self, observed):
        """``(w0, w1, x, y)`` when the fused log-joint kernel can evaluate ``observed``, else
        None (the caller runs ``__call__`` under autograd).  ``x`` / ``y`` come from
        ``observed``, else from the object; latents that are ``StochasticTensor`` samples of a
        variational net are unwrapped."""
        if len(self.names) > 2:
            return self._deep_fused_inputs(observed)
        try:
            w0, w1 = (_unwrap(observed[n]) for n in self.names)
        except KeyError:
            return None
        x, y = _unwrap(observed.get("x", self.x)), _unwrap(observed.get("y", self.y))
        ts = (w0, w1, x, y)
        if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in ts) or \
                w0.dtype != torch.float32 or w1.dtype != torch.float32:
            return None
        if w0.dim() != 3 or w1.dim() != 3:
            return None
        K, H, in1 = (int(d) for d in w0.shape)
        if tuple(w1.shape) != (K, 1, H + 1) or not (2 <= in1 <= self.MAX_IN1) or \
                not (1 <= H <= self.MAX_H) or K < 1:
            return None
        if x.dim() != 2 or int(x.shape[1]) + 1 != in1 or x.shape[0] < 1 or \
                y.numel() != x.shape[0]:
            return None
        dev = w0.device
        if w1.device != dev or x.device != dev or y.device != dev:
            return None
        # the kernel reads the prior and y_logstd scales as float32 on w0's device
        if any(ls.requires_grad or ls.dtype != torch.float32 or ls.device != dev
               for ls in self.logstds):
            return None
        if isinstance(self.y_logstd, torch.Tensor) and self.y_logstd.device != dev:
            return None
        if self.fused_prior_logstd(0, w0.shape[1:]) is None or \
                self.fused_prior_logstd(1, w1.shape[1:]) is None:
            return None
        return w0, w1, x, y

    def _deep_fused_inputs(self, observed):
        """fused_inputs for L >= 3 layers: ``(w_0, ..., w_{L-1}, x, y)`` or None.  The rules of
        the two-layer check, per layer, with the deep kernels' limits: L <= DEEP_MAX_L, n_0 and
        every hidden width <= DEEP_MAX_WIDTH, at most DEEP_MAX_WEIGHTS weights per particle."""
        try:
            ws = [_unwrap(observed[n]) for n in self.names]
        except KeyError:
            return None
        x, y = _unwrap(observed.get("x", self.x)), _unwrap(observed.get("y", self.y))
        if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in ws + [x, y]) or \
                any(w.dtype != torch.float32 or w.dim() != 3 for w in ws):
            return None
        if not self.deep_shape_ok([tuple(int(d) for d in w.shape) for w in ws]):
            return None
        if x.dim() != 2 or int(x.shape[1]) + 1 != ws[0].shape[2] or x.shape[0] < 1 or \
                y.numel() != x.shape[0]:
            return None
        dev = ws[0].device
        if any(t.device != dev for t in ws + [x, y]):
            return None
        if any(ls.requires_grad or ls.dtype != torch.float32 or ls.device != dev
               for ls in self.logstds):
            return None
        if isinstance(self.y_logstd, torch.Tensor) and self.y_logstd.device != dev:
            return None
        if any(self.fused_prior_logstd(i, w.shape[1:]) is None for i, w in enumerate(ws)):
            return None
        return tuple(ws) + (x, y)

    DEEP_MAX_L, DEEP_MAX_WIDTH, DEEP_MAX_WEIGHTS = 8, 128, 32768   # limits of csrc/bnn_deep.cu

    @classmethod
    def deep_shape_ok(cls, shapes):
        """Whether latents of these shapes ([K, n_{i+1}, n_i + 1] per layer, L >= 3) chain into
        one net within the deep kernels' limits."""
        L = len(shapes)
        if not 3 <= L <= cls.DEEP_MAX_L:
            return False
        K = shapes[0][0]
        if K < 1 or any(len(s) != 3 or s[0] != K for s in shapes) or shapes[-1][1] != 1:
            return False
        widths = [s[2] - 1 for s in shapes]
        if any(shapes[i][1] != widths[i + 1] for i in range(L - 1)):
            return False
        if any(not 1 <= n <= cls.DEEP_MAX_WIDTH for n in widths):
            return False
        return sum(s[1] * s[2] for s in shapes) <= cls.DEEP_MAX_WEIGHTS

    def _deep_prior(self, ws):
        """(logstd tensors, host arrays of their pointers and sizes) as the deep kernels read
        them; the tensors must outlive the call."""
        import ctypes
        from ._lib import ptr
        lss = [self.fused_prior_logstd(i, w.shape[1:]).detach() for i, w in enumerate(ws)]
        L = len(ws)
        return (lss, (ctypes.c_void_p * L)(*[ptr(l) for l in lss]),
                (ctypes.c_int * L)(*[l.numel() for l in lss]))

    def _launch_deep(self, ws, x, y, ys, lp=False, gs=(), gys=False, ym=False, ll=False):
        """One zsb_bnn_deep_logjoint_f32 launch; returns ``(lp, [g_i], gys, y_mean, log_lik)``
        with None where not requested (``gs``: per layer whether its gradient is wanted)."""
        import ctypes
        from ._lib import lib, ptr, stream
        L = len(ws)
        ws = [w.detach().contiguous() for w in ws]
        K, B, dev = int(ws[0].shape[0]), int(x.shape[0]), ws[0].device
        x = x.detach().to(torch.float32).contiguous()
        y = y.detach().to(torch.float32).contiguous().view(-1)
        gs = list(gs) + [False] * (L - len(gs))
        widths = (ctypes.c_int * (L + 1))(*([int(w.shape[2]) - 1 for w in ws] + [1]))
        lss, ls_p, ls_n = self._deep_prior(ws)
        e = lambda want, *s: torch.empty(s, dtype=torch.float32, device=dev) if want else None  # noqa: E731
        g = [e(want, *w.shape) for want, w in zip(gs, ws)]
        out = (e(lp, K), e(gys, K), e(ym, K, B), e(ll, K, B))
        w_p = (ctypes.c_void_p * L)(*[ptr(w) for w in ws])
        g_p = (ctypes.c_void_p * L)(*[ptr(t) for t in g])
        lib.call("zsb_bnn_deep_logjoint_f32", L, widths, ctypes.addressof(w_p), ptr(x), ptr(y), B,
                 ctypes.addressof(ls_p), ls_n, ptr(ys.detach()), self.n_train, ptr(out[0]),
                 ctypes.addressof(g_p), ptr(out[1]), ptr(out[2]), ptr(out[3]), K, stream())
        return out[0], g, out[1], out[2], out[3]

    def _launch(self, w0, w1, x, y, ys, lp=False, g0=False, g1=False, gys=False,
                ym=False, ll=False):
        """One zsb_bnn_logjoint_f32 launch; returns the requested outputs (None elsewhere)."""
        from ._lib import lib, ptr, stream
        K, H, in1 = (int(d) for d in w0.shape)
        B = int(x.shape[0])
        dev = w0.device
        w0, w1 = w0.detach().contiguous(), w1.detach().contiguous()
        x = x.detach().to(torch.float32).contiguous()
        y = y.detach().to(torch.float32).contiguous().view(-1)
        ys = ys.detach()
        ls0 = self.fused_prior_logstd(0, w0.shape[1:]).detach()
        ls1 = self.fused_prior_logstd(1, w1.shape[1:]).detach()
        e = lambda want, *s: torch.empty(s, dtype=torch.float32, device=dev) if want else None  # noqa: E731
        out = (e(lp, K), e(g0, K, H, in1), e(g1, K, 1, H + 1), e(gys, K), e(ym, K, B),
               e(ll, K, B))
        lib.call("zsb_bnn_logjoint_f32", ptr(w0), ptr(w1), ptr(x), ptr(y), B, in1 - 1, H,
                 ptr(ls0), ls0.numel(), ptr(ls1), ls1.numel(), ptr(ys), self.n_train,
                 *[ptr(o) for o in out], K, stream())
        return out

    def fused_log_joint(self, observed):
        """The log-joint [K] of ``observed`` on the fused kernel, differentiable w.r.t. w0, w1
        and a tensor ``y_logstd``: the forward launch also computes the gradients of the inputs
        that need one, and backward scales them by the upstream [K] gradient.  ValueError when
        ``fused_inputs(observed)`` is None."""
        got = self.fused_inputs(observed)
        if got is None:
            raise ValueError("BNNRegressionLogJoint.fused_log_joint: these inputs need the "
                             "generic path (see fused_inputs)")
        ys = self._y_logstd_dev(got[0].device)
        if len(got) > 4:
            ws, x, y = got[:-2], got[-2], got[-1]
            if not torch.is_grad_enabled():
                return self._launch_deep(ws, x, y, ys, lp=True)[0]
            return _BNNDeepLogJoint.apply(ys, self, x, y, *[w.contiguous() for w in ws])
        w0, w1, x, y = got
        if not torch.is_grad_enabled():        # nothing is recorded: the value-only launch
            return self._launch(w0, w1, x, y, ys, lp=True)[0]
        return _BNNLogJoint.apply(w0.contiguous(), w1.contiguous(), ys, self, x, y)

    def predictive(self, observed):
        """``(y_mean [K, B], log_lik [K, B])`` of every particle ``observed[names]`` at the rows
        ``observed['x']`` (else the object's x), with log_lik = log N(y_b; y_mean, exp(y_logstd))
        unscaled -- the prediction fetches of bnn_vi.py:98-103 -- from one launch, no gradient.
        E.g. RMSE = ((y_mean.mean(0) - y) ** 2).mean().sqrt() and test log-likelihood =
        (log_lik.logsumexp(0) - log K).mean()."""
        got = self.fused_inputs(observed)
        if got is None:
            raise ValueError("BNNRegressionLogJoint.predictive: shapes outside the fused "
                             "kernel's limits (see fused_inputs)")
        if len(got) > 4:
            _, _, _, ym, ll = self._launch_deep(got[:-2], got[-2], got[-1],
                                                self._y_logstd_dev(got[0].device), ym=True,
                                                ll=True)
            return ym, ll
        w0, w1, x, y = got
        _, _, _, _, ym, ll = self._launch(w0, w1, x, y, self._y_logstd_dev(w0.device),
                                          ym=True, ll=True)
        return ym, ll

    def hmc_provider(self, latent_names, observed, latents):
        """The provider ``zs.HMC`` uses instead of autograd (logp / grad, one launch each) when
        the latents are the object's weight layers and ``fused_inputs`` accepts them; else
        None."""
        if list(latent_names) != list(self.names):
            return None
        obs = dict(observed)
        obs.update(zip(self.names, latents))
        if self.fused_inputs(obs) is None:
            return None
        return _BNNProvider(self, observed)

    def __call__(self, observed):
        x = observed.get("x", self.x)
        y = observed.get("y", self.y)
        ws = [observed[n] for n in self.names]
        C = ws[0].shape[0]
        h = x.unsqueeze(0).expand(C, -1, -1)
        lp = 0.0
        for i, (w, ls) in enumerate(zip(ws, self.logstds)):
            ones = torch.ones(h.shape[:-1] + (1,), device=h.device)
            h = torch.cat([h, ones], -1)
            h = torch.einsum("imk,ijk->ijm", w, h) / math.sqrt(h.shape[2])
            if i < len(ws) - 1:
                h = torch.relu(h)
            lp = lp + self._Normal(torch.zeros_like(ls), logstd=ls,
                                   group_ndims=2).log_prob(w)
        y_mean = h.squeeze(2)
        if isinstance(self.y_logstd, torch.Tensor):
            y_ls = self.y_logstd.to(y_mean.dtype).expand_as(y_mean)
        else:
            y_ls = torch.full_like(y_mean, self.y_logstd)
        lpy = self._Normal(y_mean, logstd=y_ls).log_prob(y.unsqueeze(0))
        return lp + lpy.mean(1) * self.n_train


def _unwrap(v):
    """The tensor of a ``StochasticTensor`` (a variational net's sample), else ``v``."""
    return v if isinstance(v, torch.Tensor) else getattr(v, "tensor", v)


class _BNNLogJoint(torch.autograd.Function):
    """lp [K] of BNNRegressionLogJoint over (w0, w1, y_logstd) on zsb_bnn_logjoint_f32.  The
    forward launch writes the gradients of the inputs that need one; backward only scales
    them by the upstream gradient (any [K] weights, e.g. iw_objective's normalised ones)."""

    @staticmethod
    def forward(ctx, w0, w1, ys, obj, x, y):
        need = ctx.needs_input_grad
        lp, g0, g1, gys, _, _ = obj._launch(w0, w1, x, y, ys, lp=True, g0=need[0], g1=need[1],
                                            gys=need[2])
        ctx.save_for_backward(g0, g1, gys)
        return lp

    @staticmethod
    @once_differentiable
    def backward(ctx, glp):
        g0, g1, gys = ctx.saved_tensors
        glp = glp.to(torch.float32)
        d0 = g0 * glp.view(-1, 1, 1) if g0 is not None else None
        d1 = g1 * glp.view(-1, 1, 1) if g1 is not None else None
        dys = (gys * glp).sum() if gys is not None else None
        return d0, d1, dys, None, None, None


class _BNNDeepLogJoint(torch.autograd.Function):
    """lp [K] of an L >= 3 layer BNNRegressionLogJoint over (y_logstd, w_0, ..., w_{L-1}) on
    zsb_bnn_deep_logjoint_f32; as _BNNLogJoint, the forward launch writes the gradients the
    inputs need and backward scales them."""

    @staticmethod
    def forward(ctx, ys, obj, x, y, *ws):
        need = ctx.needs_input_grad
        lp, gs, gys, _, _ = obj._launch_deep(ws, x, y, ys, lp=True, gs=need[4:], gys=need[0])
        ctx.save_for_backward(gys, *gs)
        return lp

    @staticmethod
    @once_differentiable
    def backward(ctx, glp):
        gys, *gs = ctx.saved_tensors
        glp = glp.to(torch.float32)
        dws = [g * glp.view(-1, 1, 1) if g is not None else None for g in gs]
        dys = (gys * glp).sum() if gys is not None else None
        return (dys, None, None, None) + tuple(dws)


class _BNNProvider(object):
    """HMC's provider interface over BNNRegressionLogJoint: values and gradients of the latents
    (w0, w1) at the observed rows, one zsb_bnn_logjoint_f32 launch each.  HMC picks the provider
    once, in sample(); should later ``sample_op(observed=...)`` rows not fit the kernel, that call
    runs the generic path (``__call__``, under autograd for the gradient) instead."""

    def __init__(self, obj, observed):
        self.obj, self.observed = obj, observed

    def _obs(self, var_list):
        obs = dict(self.observed)
        obs.update(zip(self.obj.names, var_list))
        return obs

    def logp(self, var_list):
        obs = self._obs(var_list)
        got = self.obj.fused_inputs(obs)
        if got is None:
            return self.obj(obs)
        if len(got) > 4:
            return self.obj._launch_deep(got[:-2], got[-2], got[-1],
                                         self.obj._y_logstd_dev(got[0].device), lp=True)[0]
        w0, w1, x, y = got
        return self.obj._launch(w0, w1, x, y, self.obj._y_logstd_dev(w0.device), lp=True)[0]

    def grad(self, var_list):
        got = self.obj.fused_inputs(self._obs(var_list))
        if got is None:
            xs = [v.detach().requires_grad_(True) for v in var_list]
            with torch.enable_grad():
                gs = torch.autograd.grad(self.obj(self._obs(xs)).sum(), xs, allow_unused=True)
            return [g.contiguous() if g is not None else torch.zeros_like(x)
                    for g, x in zip(gs, xs)]
        if len(got) > 4:
            ws = got[:-2]
            return self.obj._launch_deep(ws, got[-2], got[-1],
                                         self.obj._y_logstd_dev(ws[0].device),
                                         gs=[True] * len(ws))[1]
        w0, w1, x, y = got
        out = self.obj._launch(w0, w1, x, y, self.obj._y_logstd_dev(w0.device), g0=True,
                               g1=True)
        return [out[1], out[2]]


class LNTMLogJoint(object):
    """Logistic-Normal Topic Model, examples/topic_models/lntm_mcem.py:33-48: the E-step objective
    with ``model.log_joint = e_obj`` (:97-99), the M-step likelihood (:106-114) and AIS's tempered
    log-joint (evaluation.py:91-94):

        eta [chains, docs, K] ~ Normal(eta_mean, exp(eta_logstd)), group_ndims=1
        log p = cond_log_prob('eta') + UnnormalizedMultinomial(log(softmax(eta) @ softmax(beta)),
                                                                normalize_logits=False).log_prob(x)

    ``zs.HMC.sample`` recognises it (``_zsb_fused`` kind "provider") and takes log-joint values
    and gradients from ONE fused, sparsity-aware kernel (zsb_lntm_logjoint_f32): the corpus is held
    in CSR, only the words a document contains are formed, and the [chains*docs, V] matrix
    ``doc_word`` of the reference never exists (335 TB at BASELINE config 5).  As a plain callable
    it is the dense torch restatement of the reference graph (small shapes / cross-check).

    x: dense [n_docs, V] counts (any float/int tensor), the whole corpus; beta: [K, V] (fixed
    during the E-step; call ``set_beta`` after every M-step); 1 <= K <= 128 on the kernels.  A CPU
    ``beta`` or K > 128 leaves only the dense restatement: HMC then differentiates ``__call__``.

    ``set_docs(doc_ids)`` selects a batch of corpus rows (a device int64 tensor of distinct rows,
    or None for all of them) with no host sync: eta is then ``[chains, len(doc_ids), K]`` for the
    E-step, the dense callable and ``cond_log_px``.  One training batch of the example::

        lj.set_docs(ids)                               # ids = perm[t * 100:(t + 1) * 100]
        eta.copy_(Eta[:, ids])
        for _ in range(num_e_steps):
            sample_op()                                # zs.HMC(...).sample(lj, {}, {"eta": eta})
        Eta[:, ids] = eta
        log_px = lj.cond_log_px(eta, beta).mean(0).sum()
        log_p_beta = Normal(torch.zeros_like(beta), logstd=log_delta).log_prob(beta).sum()
        (-(log_p_beta + log_px)).backward()            # then the Adam step on beta
    """

    def __init__(self, x, beta, eta_mean, eta_logstd, name="eta"):
        from ._lib import lib  # noqa: F401  (fail early without the library)
        self.name = name
        dev = beta.device
        x = torch.as_tensor(x, device=dev)
        self.x = x.to(torch.float32)
        self.n_docs, self.n_vocab = int(x.shape[0]), int(x.shape[1])
        nz = (self.x != 0)
        per_doc = nz.sum(1)
        self.doc_ptr = torch.zeros(self.n_docs + 1, dtype=torch.int64, device=dev)
        self.doc_ptr[1:] = torch.cumsum(per_doc, 0)
        idx = nz.nonzero(as_tuple=False)                  # row-major: sorted by document
        self.word_idx = idx[:, 1].to(torch.int32).contiguous()
        self.word_cnt = self.x[idx[:, 0], idx[:, 1]].contiguous()
        self.nnz = int(idx.shape[0])
        # the same entries grouped by word, documents ascending (the M-step's fixed summation order)
        order = torch.sort(idx[:, 1], stable=True)[1]
        self.csc_entry = order.to(torch.int32).contiguous()
        self.entry_doc = idx[order, 0].to(torch.int32).contiguous()
        self.csc_ptr = torch.zeros(self.n_vocab + 1, dtype=torch.int64, device=dev)
        self.csc_ptr[1:] = torch.cumsum(torch.bincount(idx[:, 1], minlength=self.n_vocab), 0)
        self.eta_mean = eta_mean.detach().to(torch.float32).contiguous()
        self.eta_logstd = eta_logstd.detach().to(torch.float32).contiguous()
        self.n_topics = int(beta.shape[0])
        if self.n_topics < 1:
            raise ValueError("LNTMLogJoint: n_topics must be at least 1")
        self.n_topics_padded = 16 * -(-self.n_topics // 16)
        self.fused = dev.type == "cuda" and self.n_topics <= 128
        self.set_docs(None)
        self.set_beta(beta)
        if self.fused:
            self._zsb_fused = {"kind": "provider", "obj": self}

    def set_beta(self, beta):
        """Take ``beta`` for the E-step: phi_t [V, Kp] = softmax(beta)^T with zero pad columns,
        in a new buffer (a pending ``cond_log_px`` backward keeps the one it read)."""
        from ._lib import lib, ptr, stream
        self.beta = beta.detach().to(torch.float32).contiguous()
        if not self.fused:
            return
        self.phi_t = torch.empty((self.n_vocab, self.n_topics_padded), dtype=torch.float32,
                                 device=self.beta.device)
        lib.call("zsb_lntm_phi_t_f32", ptr(self.beta), self.n_topics, self.n_vocab,
                 ptr(self.phi_t), stream())

    def set_docs(self, doc_ids):
        """Work on corpus rows ``doc_ids`` (int64 tensor on the corpus' device, distinct rows) or,
        for None, on every row.  No CSR rebuild and no host sync."""
        if doc_ids is None:
            self.doc_ids, self._doc_slot, self.n_batch = None, None, self.n_docs
            return
        if not isinstance(doc_ids, torch.Tensor) or doc_ids.dim() != 1 or \
                doc_ids.dtype != torch.int64 or doc_ids.device != self.doc_ptr.device:
            raise ValueError("doc_ids must be a 1-D int64 tensor on %s" % self.doc_ptr.device)
        self.doc_ids = doc_ids.contiguous()
        self.n_batch = int(doc_ids.shape[0])
        # batch row of each corpus document, -1 outside the batch (the M-step skips those)
        self._doc_slot = torch.full((self.n_docs,), -1, dtype=torch.int32,
                                    device=doc_ids.device).scatter_(
            0, self.doc_ids, torch.arange(self.n_batch, dtype=torch.int32,
                                          device=doc_ids.device))

    def _check_eta(self, eta):
        if eta.dim() != 3 or int(eta.shape[1]) != self.n_batch or \
                int(eta.shape[2]) != self.n_topics:
            raise ValueError("eta must be [chains, %d, %d]" % (self.n_batch, self.n_topics))
        return eta.detach().to(torch.float32).contiguous()

    def _launch(self, eta, want_lp, want_grad, temperature=None):
        from ._lib import lib, ptr, stream
        if not self.fused:
            raise ValueError("LNTMLogJoint: the fused kernels need 1 <= n_topics <= 128 and a "
                             "CUDA beta (got %d topics on %s); call the object for the dense "
                             "log-joint" % (self.n_topics, self.beta.device))
        eta = self._check_eta(eta)
        chains = int(eta.shape[0])
        lp = torch.empty((chains, self.n_batch), dtype=torch.float32, device=eta.device) \
            if want_lp else None
        g = torch.empty_like(eta) if want_grad else None
        lib.call("zsb_lntm_logjoint_f32", ptr(eta), ptr(self.eta_mean), ptr(self.eta_logstd),
                 ptr(self.phi_t), ptr(self.doc_ptr), ptr(self.word_idx), ptr(self.word_cnt),
                 ptr(self.doc_ids), ptr(temperature), ptr(lp), ptr(g), chains, self.n_batch,
                 self.n_topics, stream())
        return lp, g

    # provider interface used by HMC's generic path instead of autograd
    def logp(self, var_list):
        return self._launch(var_list[0], True, False)[0]

    def grad(self, var_list):
        return [self._launch(var_list[0], False, True)[1]]

    def tempered(self, temperature):
        """The provider of ``prior + t * likelihood`` for a 0-d float32 device tensor ``t`` read
        by the kernel at every call: AIS's log-joint ``log_prior * (1 - t) + log_joint * t``
        (evaluation.py:91-94) when the proposal's log-joint is this object's eta prior."""
        return _LNTMTempered(self, temperature)

    def _batch_x(self):
        return self.x if self.doc_ids is None else self.x.index_select(0, self.doc_ids)

    def _dense_log_px(self, eta, beta):
        theta = torch.softmax(eta, -1)
        phi = torch.softmax(beta, -1)
        doc_word = theta.reshape(-1, self.n_topics) @ phi
        doc_word = doc_word.reshape(tuple(eta.shape[:-1]) + (self.n_vocab,))
        return (self._batch_x().to(doc_word.dtype) * torch.log(doc_word)).sum(-1)

    def cond_log_px(self, eta, beta):
        """log p(x_d | eta_c, beta) [chains, B] of the selected documents (the reference's
        ``cond_log_prob('x')``, lntm_mcem.py:106-110), differentiable w.r.t. ``beta`` only: eta
        is a constant, as ``var_list=[beta]`` makes it.  Refreshes phi_t from ``beta``.  On the
        kernels (zsb_lntm_mstep_f32, and zsb_lntm_mstep_grad_f32 for the gradient) nothing
        [chains * B, V]-sized is formed; a float64 or CPU ``beta``, or K > 128, takes the dense
        restatement."""
        eta = eta.detach()
        if not (self.fused and beta.dtype == torch.float32 and beta.is_cuda):
            return self._dense_log_px(eta.to(beta.dtype), beta)
        self.set_beta(beta)
        return _LNTMLogPx.apply(beta, self._check_eta(eta), self)

    def __call__(self, observed):
        """Dense restatement of the reference graph in torch (lntm_mcem.py:33-48)."""
        eta = observed[self.name]
        prec = torch.exp(-2 * self.eta_logstd)
        prior = (-0.5 * math.log(2 * math.pi) - self.eta_logstd
                 - 0.5 * prec * (eta - self.eta_mean) ** 2).sum(-1)
        return prior + self._dense_log_px(eta, self.beta)


class _LNTMTempered(object):
    """HMC's provider interface (and the callable AIS evaluates at t = 0) over
    ``LNTMLogJoint.tempered``: zsb_lntm_logjoint_f32 with a device temperature."""

    def __init__(self, obj, temperature):
        self.obj, self.temperature = obj, temperature
        self._zsb_fused = {"kind": "provider", "obj": self}

    def logp(self, var_list):
        return self.obj._launch(var_list[0], True, False, self.temperature)[0]

    def grad(self, var_list):
        return [self.obj._launch(var_list[0], False, True, self.temperature)[1]]

    def __call__(self, observed):
        return self.logp([observed[self.obj.name]])


class _LNTMLogPx(torch.autograd.Function):
    """lp [chains, B] of LNTMLogJoint.cond_log_px on zsb_lntm_mstep_f32; backward is
    zsb_lntm_mstep_grad_f32 on the theta / ratio the forward wrote."""

    @staticmethod
    def forward(ctx, beta, eta, obj):
        from ._lib import lib, ptr, stream
        chains, dev = int(eta.shape[0]), eta.device
        lp = torch.empty((chains, obj.n_batch), dtype=torch.float32, device=dev)
        ratio = torch.empty((chains, obj.nnz), dtype=torch.float32, device=dev)
        theta = torch.empty((chains, obj.n_batch, obj.n_topics_padded), dtype=torch.float32,
                            device=dev)
        lib.call("zsb_lntm_mstep_f32", ptr(eta), ptr(obj.phi_t), ptr(obj.doc_ptr),
                 ptr(obj.word_idx), ptr(obj.word_cnt), ptr(obj.doc_ids), ptr(lp), ptr(ratio),
                 ptr(theta), chains, obj.n_batch, obj.nnz, obj.n_topics, stream())
        ctx.obj, ctx.phi_t, ctx.doc_slot = obj, obj.phi_t, obj._doc_slot
        ctx.save_for_backward(ratio, theta)
        return lp

    @staticmethod
    @once_differentiable
    def backward(ctx, glp):
        from ._lib import lib, ptr, stream
        obj = ctx.obj
        ratio, theta = ctx.saved_tensors
        glp = glp.to(torch.float32).contiguous()
        G = torch.empty((obj.n_vocab, obj.n_topics_padded), dtype=torch.float32,
                        device=glp.device)
        dbeta = torch.empty((obj.n_topics, obj.n_vocab), dtype=torch.float32, device=glp.device)
        lib.call("zsb_lntm_mstep_grad_f32", ptr(glp), ptr(ratio), ptr(theta), ptr(ctx.phi_t),
                 ptr(obj.csc_ptr), ptr(obj.csc_entry), ptr(obj.entry_doc), ptr(ctx.doc_slot),
                 ptr(G), ptr(dbeta), int(glp.shape[0]), int(glp.shape[1]), obj.nnz,
                 obj.n_topics, obj.n_vocab, stream())
        return dbeta, None, None


def _as_numpy(a, dtype):
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().numpy()
    return np.asarray(a).astype(dtype, copy=False)


class PMFLogJoint(object):
    """One HMC sweep over every chunk of one factor of Bayesian probabilistic matrix factorisation,
    examples/probabilistic_matrix_factorization/pmf_hmc.py:19-31 with its log_joint override
    (136-144):

        u [K, n, D] ~ N(0, std), v [K, m, D] ~ N(0, fixed_std),
        r_ij ~ N(sigmoid(u_i . v_j), rating_std)    for every observed rating (i, j).

    The example runs one HMC per chunk of ``chunk_size`` users with the movie factor fixed, then
    one per chunk of movies.  Given the other factor the chunks are independent, so one HMC
    iteration whose latent is ``[K, n_chunks, chunk_size, D]`` (chain shape ``[K, n_chunks]``)
    performs the example's whole sequential sweep; each chain's log-joint is the example's own
    for its chunk: the prior of its rows, the prior of the fixed factor over the columns the chunk's
    ratings touch (its neighbour set), and the chunk's rating terms.  ``zs.HMC.sample`` recognises
    the object (``_zsb_fused`` kind "provider") and takes values and gradients from one
    deterministic kernel (zsb_pmf_logjoint_f32) that never forms the [K, nnz, D] gathered
    factors.  Called as ``lj(observed)`` it is the torch restatement of the example's graph
    (gather, sigmoid, Normal log-probs summed per chunk), differentiable, for small shapes.

    rows, cols, ratings: COO ratings (already normalised); ``rows`` index the sampled factor,
    ``cols`` the fixed one.  fixed: the other factor, float32 ``[K, n_cols, D]`` or
    ``[K, n_col_chunks, col_chunk, D]``, read in place on every call -- pass the other sampler's
    latent and no copy is ever needed (``set_fixed`` rebinds it).  n_rows: rows of the sampled
    factor, a multiple of chunk_size (pad as the example does).  1 <= D <= 128.

    A Gibbs epoch of the example, and its RMSE recipe (lines 114-120) in torch::

        U = torch.randn(K, N_pad, D, device="cuda") * 0.1
        V = torch.randn(K, M_pad, D, device="cuda") * 0.1
        u = U.view(K, N_pad // 50, 50, D)
        v = V.view(K, M_pad // 50, 50, D)
        lj_u = zs.fused.PMFLogJoint(user, movie, r_norm, fixed=v, n_rows=N_pad, chunk_size=50,
                                    std=1., fixed_std=1., rating_std=0.05, name="u")
        lj_v = zs.fused.PMFLogJoint(movie, user, r_norm, fixed=u, n_rows=M_pad, chunk_size=50,
                                    std=1., fixed_std=1., rating_std=0.05, name="v")
        op_u, _ = zs.HMC(step_size=1e-3, n_leapfrogs=10).sample(lj_u, {}, {"u": u})
        op_v, _ = zs.HMC(step_size=1e-3, n_leapfrogs=10).sample(lj_v, {}, {"v": v})
        for epoch in range(n_epochs):
            op_u(); op_v()
            pred = torch.sigmoid((U[:, su] * V[:, sv]).sum(-1)).mean(0)
            rmse = torch.sqrt(((pred - (true_rating - 1.) / 4.) ** 2).mean()) * 4
    """

    def __init__(self, rows, cols, ratings, fixed, n_rows, chunk_size=50, std=1.0,
                 fixed_std=1.0, rating_std=1.0, name="u"):
        rows, cols = _as_numpy(rows, np.int64), _as_numpy(cols, np.int64)
        r = _as_numpy(ratings, np.float32)
        if rows.ndim != 1 or cols.ndim != 1 or r.ndim != 1:
            raise ValueError("rows, cols and ratings must be 1-D")
        if not (rows.shape[0] == cols.shape[0] == r.shape[0]):
            raise ValueError("rows, cols and ratings have different lengths (%d, %d, %d)"
                             % (rows.shape[0], cols.shape[0], r.shape[0]))
        n_rows, chunk_size = int(n_rows), int(chunk_size)
        if n_rows <= 0 or chunk_size <= 0 or n_rows % chunk_size != 0:
            raise ValueError("n_rows (%d) must be a positive multiple of chunk_size (%d)"
                             % (n_rows, chunk_size))
        for nm, s in (("std", std), ("fixed_std", fixed_std), ("rating_std", rating_std)):
            if not (float(s) > 0 and math.isfinite(float(s))):
                raise ValueError("%s must be positive and finite" % nm)
        if not np.all(np.isfinite(r)):
            raise ValueError("ratings must be finite")
        self.name = name
        self.n_rows, self.chunk_size = n_rows, chunk_size
        self.n_chunks = n_rows // chunk_size
        self.std, self.fixed_std, self.rating_std = float(std), float(fixed_std), float(rating_std)
        self.set_fixed(fixed)
        if rows.size and (rows.min() < 0 or rows.max() >= n_rows):
            raise ValueError("rows index outside [0, %d)" % n_rows)
        if cols.size and (cols.min() < 0 or cols.max() >= self.n_cols):
            raise ValueError("cols index outside [0, %d)" % self.n_cols)
        if rows.size >= (1 << 31):
            raise ValueError("at most 2^31 - 1 ratings")
        # CSR by latent row; the stable sort keeps each row's ratings in input order
        order = np.argsort(rows, kind="stable")
        self.nnz = int(rows.size)
        row_ptr = np.zeros(n_rows + 1, np.int64)
        row_ptr[1:] = np.cumsum(np.bincount(rows, minlength=n_rows))
        # per chunk: the distinct columns its ratings touch (select_from_corpus, pmf_hmc.py:34-60)
        key = np.unique((rows // chunk_size) * self.n_cols + cols)
        nbr_ptr = np.zeros(self.n_chunks + 1, np.int64)
        nbr_ptr[1:] = np.cumsum(np.bincount(key // self.n_cols, minlength=self.n_chunks))
        dev = self.fixed.device
        pad1 = lambda a: a if a.size else np.zeros(1, a.dtype)      # noqa: E731 (no NULL pointers)
        self.row_ptr = torch.as_tensor(row_ptr, device=dev)
        self.row_idx = torch.as_tensor(rows[order], device=dev)
        self.col_idx = torch.as_tensor(pad1(cols[order].astype(np.int32)), device=dev)
        self.rating = torch.as_tensor(pad1(r[order]), device=dev)
        self.nbr_ptr = torch.as_tensor(nbr_ptr, device=dev)
        self.nbr_idx = torch.as_tensor(pad1((key % self.n_cols).astype(np.int32)), device=dev)
        self.nbr_chunk = torch.as_tensor(key // self.n_cols, device=dev)
        self._zsb_fused = {"kind": "provider", "obj": self}

    def set_fixed(self, fixed):
        """Rebind the fixed factor ([K, n_cols, D] or [K, n_col_chunks, col_chunk, D])."""
        if not isinstance(fixed, torch.Tensor) or fixed.dtype != torch.float32 or \
                fixed.dim() not in (3, 4) or not fixed.is_contiguous():
            raise ValueError("fixed must be a contiguous float32 tensor [K, n_cols, D] or "
                             "[K, n_col_chunks, col_chunk, D]")
        K, D = int(fixed.shape[0]), int(fixed.shape[-1])
        n_cols = int(np.prod(fixed.shape[1:-1]))
        if K < 1 or n_cols < 1 or not 1 <= D <= 128:
            raise ValueError("fixed has shape %s: need K >= 1, n_cols >= 1 and 1 <= D <= 128"
                             % (tuple(fixed.shape),))
        if getattr(self, "n_cols", n_cols) != n_cols:
            raise ValueError("fixed has %d columns, the ratings were built for %d"
                             % (n_cols, self.n_cols))
        self.fixed, self.K, self.D, self.n_cols = fixed, K, D, n_cols

    def _latent(self, var_list):
        lat = var_list[0].detach()
        want = (self.K, self.n_chunks, self.chunk_size, self.D)
        if tuple(lat.shape) != want or lat.dtype != torch.float32:
            raise ValueError("latent must be float32 %s, got %s %s"
                             % (list(want), lat.dtype, list(lat.shape)))
        return lat.contiguous()

    def _launch(self, lat, want_lp, want_grad):
        from ._lib import lib, ptr, stream
        dev = lat.device
        lp = torch.empty((self.K, self.n_chunks), dtype=torch.float32, device=dev) \
            if want_lp else None
        work = torch.empty((self.K, self.n_rows), dtype=torch.float32, device=dev) \
            if want_lp else None
        g = torch.empty_like(lat) if want_grad else None
        lib.call("zsb_pmf_logjoint_f32", ptr(lat), ptr(self.fixed), ptr(self.row_ptr),
                 ptr(self.col_idx), ptr(self.rating), ptr(self.nbr_ptr), ptr(self.nbr_idx),
                 math.log(self.std), math.log(self.fixed_std), math.log(self.rating_std),
                 ptr(lp), ptr(g), ptr(work), self.K, self.n_rows, self.n_cols, self.D,
                 self.chunk_size, stream())
        return lp, g

    # provider interface used by HMC's generic path instead of autograd
    def logp(self, var_list):
        return self._launch(self._latent(var_list), True, False)[0]

    def grad(self, var_list):
        return [self._launch(self._latent(var_list), False, True)[1]]

    def __call__(self, observed):
        """Torch restatement of pmf_hmc.py:19-31, 136-144 per chunk: [K, n_chunks]."""
        lat = observed[self.name]
        K, D = int(lat.shape[0]), self.D
        u = lat.reshape(K, self.n_rows, D)
        v = self.fixed.reshape(self.K, self.n_cols, D).to(lat.dtype)
        nnz = self.nnz
        col = self.col_idx[:nnz].long()
        c = -0.5 * math.log(2 * math.pi)

        def normal(x, std):                               # Normal._log_prob, univariate.py
            logstd = math.log(std)
            return c - logstd - 0.5 * math.exp(-2 * logstd) * x * x
        s = torch.sigmoid((u[:, self.row_idx] * v[:, col]).sum(-1))                # [K, nnz]
        lp_r = normal(self.rating[:nnz].to(lat.dtype) - s, self.rating_std)
        out = normal(u, self.std).sum(-1).reshape(K, self.n_chunks, self.chunk_size).sum(-1)
        out = out.index_add(1, self.row_idx // self.chunk_size, lp_r)
        lp_v = normal(v[:, self.nbr_idx[:self.nbr_chunk.numel()].long()], self.fixed_std).sum(-1)
        return out.index_add(1, self.nbr_chunk, lp_v)


# ---------------------------------------------------------------------------
# K8: dense layers of a VAE / BNN log-joint on the tensor cores (gemm_logjoint_tc.cu)
# ---------------------------------------------------------------------------
def _tc_split(t2d):
    """fp32 [rows, K] -> (fp16 planes [2, rows, Kp], scale float[4]) for the
    tensor-core dense kernels (zsb_split16_pad_f32)."""
    from ._lib import lib, ptr, stream
    t2d = t2d.detach().to(torch.float32).contiguous()
    rows, K = int(t2d.shape[0]), int(t2d.shape[1])
    Kp = lib.load().zsb_linear_tc_kpad(K)
    planes = torch.empty((2, rows, Kp), dtype=torch.float16, device=t2d.device)
    scale = torch.zeros(4, dtype=torch.float32, device=t2d.device)
    lib.call("zsb_split16_pad_f32", ptr(t2d), rows, K, ptr(planes), ptr(scale),
             stream())
    return planes, scale


class _Planes(object):
    """fp16 hi/lo operand planes ``planes`` [2, rows, Kp] of one [rows, K] matrix times a
    power-of-two scale, read by all three products of a layer; ``scale`` = device float[4].
    ``binary``: a 0/1 sample of LinearBernoulli.sample -- ``planes`` [1, rows, Kp] is the hi plane
    only (the lo plane is identically zero), read by the two-product kernels; valid while the
    sample's ``_version`` is ``version``."""
    __slots__ = ("planes", "scale", "rows", "K", "binary", "version")

    def __init__(self, planes, scale, rows, K, binary=False, version=None):
        self.planes, self.scale, self.rows, self.K = planes, scale, rows, K
        self.binary, self.version = binary, version


def _tc_split_dual(t2d, mask=None, amax=None, col_sum=None):
    """One pass over fp32 ``t2d`` [R, K] (times the ReLU mask ``mask > 0``) -> its _Planes;
    ``amax`` = scale slot whose max-|.| word a producing GEMM already filled (no max pass then);
    ``col_sum`` [K] += column sums."""
    from ._lib import lib, ptr, stream
    t2d = t2d.detach().to(torch.float32).contiguous()
    R, K = int(t2d.shape[0]), int(t2d.shape[1])
    dev = t2d.device
    if K % 2:                      # odd widths: mask and column sums in torch, then the plain split
        if mask is not None:
            t2d = t2d * (mask > 0)
        if col_sum is not None:
            col_sum += t2d.sum(0)
        return _Planes(*_tc_split(t2d), R, K)
    Kp = lib.load().zsb_linear_tc_kpad(K)
    planes = torch.empty((2, R, Kp), dtype=torch.float16, device=dev)
    scale = amax if amax is not None else torch.zeros(4, dtype=torch.float32, device=dev)
    m = None if mask is None else mask.detach().to(torch.float32).contiguous()
    lib.call("zsb_split16_dual_f32", ptr(t2d), ptr(m), R, K, ptr(planes), ptr(col_sum),
             ptr(scale), int(amax is not None), stream())
    return _Planes(planes, scale, R, K)


def _planes_of(h2, src):
    """Operand planes of activation ``h2`` (= ``src`` flattened to 2-D), cached on ``src``: the
    producing GEMM left the max |.| in ``src._zsb_amax`` (no max pass), and every consumer of the
    same activation (e.g. the two heads of the encoder) shares one split."""
    R, K = int(h2.shape[0]), int(h2.shape[1])
    pl = getattr(src, "_zsb_pl", None)
    if (pl is not None and pl.rows == R and pl.K == K
            and (not pl.binary or (pl.version is not None and pl.version == _version(src)))):
        return pl
    amax = getattr(src, "_zsb_amax", None)
    pl = _tc_split_dual(h2, amax=None if K % 2 else amax)
    try:
        src._zsb_pl = pl
        if amax is not None:
            del src._zsb_amax
    except (AttributeError, RuntimeError):
        pass
    return pl


def _tc_grad_input(gpl, W, R, wp=None, ws=None):
    """dh [R, K] = g [R, J] @ W [J, K] on the tensor cores (+ the scale slot holding max|dh|).
    ``wp, ws``: the forward planes of W when the caller still has them (else W is split again) --
    the product reads them as an MN-major operand (zsb_linear_tc_dgrad_f32), so W^T is never
    formed."""
    from ._lib import lib, ptr, stream
    amax = torch.zeros(4, dtype=torch.float32, device=W.device)
    if wp is None:
        wp, ws = _tc_split(W)
    J, K = int(W.shape[0]), int(W.shape[1])
    dh = torch.empty((R, K), dtype=torch.float32, device=W.device)
    lib.call("zsb_linear_tc_dgrad_f32", ptr(wp), ptr(ws), ptr(gpl.planes), ptr(gpl.scale),
             R, J, K, ptr(dh), ptr(amax), stream())
    return dh, amax


def _tc_grad_weight(gpl, hpl, R):
    """dW [J, K] = g^T [J, R] @ h [R, K]: contraction over the rows, split-K over the CTA pairs.
    Both operands are the row-major planes of g and h (MN-major wgmma operands,
    zsb_linear_tc_wgrad_f32)."""
    from ._lib import lib, ptr, stream
    J, K = gpl.K, hpl.K
    dev = gpl.planes.device
    slices = lib.load().zsb_linear_tc_slices(J, K, R)
    part = torch.empty(slices * J * K, dtype=torch.float32, device=dev) if slices > 1 else None
    out = torch.empty((J, K), dtype=torch.float32, device=dev)
    lib.call("zsb_linear_tc_wgrad_bin_f32" if hpl.binary else "zsb_linear_tc_wgrad_f32",
             ptr(hpl.planes), ptr(hpl.scale), K, ptr(gpl.planes), ptr(gpl.scale), J, R, ptr(out),
             ptr(part), stream())
    return out


def _tc_linear(epi, wp, ws, hp, hs, bias, x, gout, R, J, K, relu=False, amax=None,
               binary=False):
    """One product on the wgmma kernel; ``binary``: ``hp`` is the one plane of a 0/1 sample."""
    from ._lib import lib, ptr, stream
    dev = hp.device
    part = None
    if epi == 1:
        out = torch.empty(R, dtype=torch.float32, device=dev)
        part = torch.empty(lib.load().zsb_linear_tc_nparts(J) * R,
                           dtype=torch.float32, device=dev)
    else:
        out = torch.empty((R, J), dtype=torch.float32, device=dev)
    lib.call("zsb_linear_tc_bin_f32" if binary else "zsb_linear_tc_amax_f32", epi, ptr(wp),
             ptr(ws), ptr(hp), ptr(hs),
             ptr(bias), ptr(x), int(x.shape[0]) if x is not None else 0,
             ptr(gout), ptr(out), ptr(part), R, J, K, int(bool(relu)), ptr(amax), stream())
    return out


def _tag(t, amax):
    try:
        t._zsb_amax = amax
    except (AttributeError, RuntimeError):
        pass
    return t


def _grad_weight_release(ctx, gpl, R, need):
    """dW from the planes ``gpl`` of d/d(pre-activation) and the layer's saved input planes
    ``ctx.hpl``; the layer then drops its saved planes."""
    dW = _tc_grad_weight(gpl, ctx.hpl, R) if need else None
    ctx.hpl = None
    ctx.wpl = None
    return dW


def _grad_products(ctx, gpl, W, R, wpl, dh_shape, need_dh, need_dW):
    """The backward products of a dense layer from the planes ``gpl`` of d/d(pre-activation): dh
    (shaped ``dh_shape`` and tagged with its max |.|, from the forward planes ``wpl`` of W) and
    dW (_grad_weight_release)."""
    dh = None
    if need_dh:
        dh2, amax = _tc_grad_input(gpl, W, R, *wpl)
        dh = _tag(dh2.reshape(dh_shape), amax)
    return dh, _grad_weight_release(ctx, gpl, R, need_dW)


class _Linear(torch.autograd.Function):
    """y = relu?(h W^T + b): forward and both backward products on the wgmma kernel at fp32
    accuracy (epi 0; the weight gradient reads the same row-major planes as MN-major operands, split-K).
    Memory passes around the GEMMs are fused: every GEMM leaves max|out| for its consumer's
    scale, ONE pass (zsb_split16_dual_f32) turns an activation / gradient into its operand planes,
    applies the ReLU mask and accumulates the bias gradient."""

    @staticmethod
    def forward(ctx, h, W, b, relu):
        lead = h.shape[:-1]
        h2 = h if h.dim() == 2 else h.reshape(-1, h.shape[-1])
        R, K, J = int(h2.shape[0]), int(h2.shape[1]), int(W.shape[0])
        hpl = _planes_of(h2, h)
        wp, ws = _tc_split(W)
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        amax = torch.zeros(4, dtype=torch.float32, device=h2.device)
        y = _tc_linear(0, wp, ws, hpl.planes, hpl.scale, bias, None, None, R, J, K, relu,
                       amax=amax, binary=hpl.binary)
        ctx.save_for_backward(W, y if relu else None)
        ctx.hpl = hpl
        ctx.wpl = (wp, ws)
        ctx.meta = (lead, relu, b is not None, R, K, J)
        return _tag(y.reshape(tuple(lead) + (J,)), amax)

    @staticmethod
    def backward(ctx, gy):
        W, y = ctx.saved_tensors
        lead, relu, has_b, R, K, J = ctx.meta
        need = ctx.needs_input_grad
        g = gy.reshape(-1, J)
        db = torch.zeros(J, dtype=torch.float32, device=g.device) \
            if (has_b and need[2]) else None
        gpl = _tc_split_dual(g, mask=y if relu else None, amax=getattr(gy, "_zsb_amax", None),
                             col_sum=db)
        dh, dW = _grad_products(ctx, gpl, W, R, ctx.wpl or (None, None), tuple(lead) + (K,),
                                need[0], need[1])
        return dh, dW, db, None


def linear(h, W, b=None, relu=False):
    """``relu?(h @ W.T + b)`` (``tf.layers.dense``) on the wgmma kernel.  ``h`` may be a
    ``StochasticTensor``, as a model's node fed straight to a dense layer is (vae_nf.py:23-24)."""
    return _Linear.apply(_unwrap(h), W, b, bool(relu))


class _LinearBernoulliLogProb(torch.autograd.Function):
    """sum_j Bernoulli(logits = h W^T + b).log_prob(x)[..., j] without ever
    writing the logits: forward = GEMM with the Bernoulli row-sum epilogue
    (epi 1); backward = the same GEMM with the d/dlogits epilogue (epi 2),
    then the input / weight gradient products on the same kernel."""

    @staticmethod
    def forward(ctx, h, W, b, x):
        lead = h.shape[:-1]
        h2 = h if h.dim() == 2 else h.reshape(-1, h.shape[-1])
        R, K, J = int(h2.shape[0]), int(h2.shape[1]), int(W.shape[0])
        x2 = x.reshape(-1, J).to(torch.float32).contiguous()
        if R % int(x2.shape[0]) != 0:
            raise ValueError("rows of the observation (%d) must divide the rows "
                             "of the activations (%d)" % (x2.shape[0], R))
        wp, ws = _tc_split(W)
        hpl = _planes_of(h2, h)
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        lp = _tc_linear(1, wp, ws, hpl.planes, hpl.scale, bias, x2, None, R, J, K,
                        binary=hpl.binary)
        ctx.save_for_backward(W, bias, x2, wp, ws)
        ctx.hpl = hpl
        ctx.meta = (lead, R, J, K, b is not None)
        return lp.reshape(tuple(lead))

    @staticmethod
    def backward(ctx, glp):
        W, bias, x2, wp, ws = ctx.saved_tensors
        lead, R, J, K, has_b = ctx.meta
        hpl = ctx.hpl
        need = ctx.needs_input_grad
        g = glp.reshape(-1).to(torch.float32).contiguous()
        db = torch.zeros(J, dtype=torch.float32, device=g.device) \
            if (has_b and need[2]) else None
        amax = torch.zeros(4, dtype=torch.float32, device=g.device)
        dl = _tc_linear(2, wp, ws, hpl.planes, hpl.scale, bias, x2, g, R, J, K, amax=amax,
                        binary=hpl.binary)
        dlpl = _tc_split_dual(dl, amax=amax, col_sum=db)
        dh, dW = _grad_products(ctx, dlpl, W, R, (wp, ws), tuple(lead) + (K,), need[0], need[1])
        return dh, dW, db, None


def _class_indices(y, lead, C):
    """``y`` as the int32 class indices [n_y] the class kernel reads (row r of the flattened
    ``lead`` takes index r % n_y): int indices whose shape is a suffix of ``lead``, or a one-hot
    ``[..., C]`` whose leading shape is (turned into indices on the device, no host sync; an
    unchanged LinearOnehotCategorical sample brings its own).  A shape that fits both is read as
    indices."""
    lead = tuple(int(d) for d in lead)
    ys = tuple(int(d) for d in y.shape)

    def suffix(s):
        return len(s) <= len(lead) and s == lead[len(lead) - len(s):]
    if not y.is_floating_point() and suffix(ys):
        idx = y
    elif ys and ys[-1] == C and suffix(ys[:-1]):
        own = getattr(y, "_zsb_cls", None)     # the class indices of a LinearOnehotCategorical draw
        if own is not None and own[1] is not None and own[1] == _version(y):
            return own[0]
        idx = y.detach().argmax(-1)
    else:
        raise ValueError("y %s is neither class indices whose shape is a suffix of %s nor a "
                         "one-hot [..., %d] over such a shape" % (ys, lead, C))
    return idx.detach().reshape(-1).to(torch.int32).contiguous()


def _tc_split_class(g2, R, cls, C, mask=None, amax=None, col_sum=None, dtab=None):
    """The backward pass of the class-conditioned layer (zsb_split16_class_f32): _Planes [2, R, Jp]
    of the upstream gradient ``g2`` (times the ReLU mask ``mask > 0``) -- of its class fold
    ``sum_c g2[c R + r]`` when ``cls`` is None -- with ``col_sum`` [J] and ``dtab`` [C, J]
    accumulating the bias and class-table gradients."""
    from ._lib import lib, ptr, stream
    g2 = g2.detach().to(torch.float32).contiguous()
    J = int(g2.shape[1])
    dev = g2.device
    planes = torch.empty((2, R, lib.load().zsb_linear_tc_kpad(J)), dtype=torch.float16,
                         device=dev)
    scale = amax if amax is not None else torch.zeros(4, dtype=torch.float32, device=dev)
    m = None if mask is None else mask.detach().to(torch.float32).contiguous()
    lib.call("zsb_split16_class_f32", ptr(g2), ptr(m), R, J, ptr(cls),
             0 if cls is None else int(cls.numel()), C, ptr(planes), ptr(col_sum), ptr(dtab),
             ptr(scale), int(amax is not None), stream())
    return _Planes(planes, scale, R, J)


class _ClassLinear(torch.autograd.Function):
    """relu?(h W^T + b + W_class[:, y]) on the class epilogue of the wgmma kernel, per row (``cls``)
    or for every class (``cls`` None, class-major).  Backward: one pass over the upstream gradient
    gives the class-table and bias gradients and the operand planes of the input- and
    weight-gradient products -- over the rows of h also in the enumerated form, whose gradient is
    first folded over the classes."""

    @staticmethod
    def forward(ctx, h, W, W_class, b, cls, relu):
        from ._lib import lib, ptr, stream
        lead = h.shape[:-1]
        h2 = h if h.dim() == 2 else h.reshape(-1, h.shape[-1])
        R, K, J, C = int(h2.shape[0]), int(h2.shape[1]), int(W.shape[0]), int(W_class.shape[1])
        hpl = _planes_of(h2, h)
        wp, ws = _tc_split(W)
        tab = W_class.detach().to(torch.float32).t().contiguous()          # [C, J]
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        amax = torch.zeros(4, dtype=torch.float32, device=h2.device)
        y = torch.empty(((C if cls is None else 1) * R, J), dtype=torch.float32, device=h2.device)
        lib.call("zsb_linear_tc_class_f32", ptr(wp), ptr(ws), ptr(hpl.planes), ptr(hpl.scale),
                 int(hpl.binary), ptr(bias), ptr(tab), C, ptr(cls),
                 0 if cls is None else int(cls.numel()), ptr(y), R, J, K, int(bool(relu)),
                 ptr(amax), stream())
        ctx.save_for_backward(W, y if relu else None)
        ctx.cls = cls
        ctx.hpl = hpl
        ctx.wpl = (wp, ws)
        ctx.meta = (lead, relu, b is not None, R, K, J, C)
        shape = tuple(lead) + (J,) if cls is not None else (C,) + tuple(lead) + (J,)
        return _tag(y.reshape(shape), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        W, y = ctx.saved_tensors
        lead, relu, has_b, R, K, J, C = ctx.meta
        need = ctx.needs_input_grad
        dev = gy.device
        db = torch.zeros(J, dtype=torch.float32, device=dev) if (has_b and need[3]) else None
        dtab = torch.zeros((C, J), dtype=torch.float32, device=dev) if need[2] else None
        gpl = _tc_split_class(gy.reshape(-1, J), R, ctx.cls, C, mask=y if relu else None,
                              amax=getattr(gy, "_zsb_amax", None), col_sum=db, dtab=dtab)
        dh, dW = _grad_products(ctx, gpl, W, R, ctx.wpl, tuple(lead) + (K,), need[0], need[1])
        return dh, dW, None if dtab is None else dtab.t(), db, None, None


def class_linear(h, W, W_class, y=None, b=None, relu=False):
    """``relu?(h @ W.T + onehot(y) @ W_class.T + b)`` -- ``tf.layers.dense`` of ``[h, onehot(y)]``
    (vae_ssl.py:38), or the sum of two dense layers of ``h`` and ``onehot(y)`` (vae_ssl.py:24-28)
    with their biases added into one ``b`` -- on the wgmma kernel, where the one-hot block of the
    product is the gather ``W_class[:, y]`` in the epilogue (exact, no C-wide product).

    ``W`` [J, K] and ``W_class`` [J, C] are ``tf.layers.dense`` kernels transposed, as in
    ``linear``.  ``y``: int class indices whose shape is a suffix of ``h.shape[:-1]`` (broadcast
    over the leading axes), or a one-hot ``[..., C]`` over such a shape; the result is
    ``h.shape[:-1] + (J,)``.  A class index outside ``[0, C)`` gives a NaN row.

    ``y=None`` enumerates every class from one product over the rows of h: the result is
    ``[C, *h.shape[:-1], J]``, class-major, bit for bit the per-row layer on h tiled C times.
    This differs from the reference's unlabeled bound (vae_ssl.py:108-124), which tiles each row
    of x C times (row ``n C + c``): here class c of row n sits at ``[c, n]``, so per-datum bounds
    built on it come out ``[C, N]`` where the reference reshapes to ``[N, C]``.

    Differentiable w.r.t. h, W, W_class and b.  The output carries the max |.| that the next
    ``linear`` / ``LinearBernoulli`` uses for its operand split."""
    C = int(W_class.shape[1])
    if int(W_class.shape[0]) != int(W.shape[0]):
        raise ValueError("W %s and W_class %s have different output widths"
                         % (tuple(W.shape), tuple(W_class.shape)))
    cls = None if y is None else _class_indices(y, h.shape[:-1], C)
    return _ClassLinear.apply(h, W, W_class, b, cls, bool(relu))


def _bn_check(name, J, dev, gamma, beta, moving_mean, moving_variance):
    """ValueError naming the first of gamma (None: no learned scale), beta, moving_mean and
    moving_variance that is not a float32 [J] tensor on dev; the moving statistics, which are
    updated in place, must also be contiguous."""
    for nm, t, contig in (("gamma", gamma, False), ("beta", beta, False),
                          ("moving_mean", moving_mean, True),
                          ("moving_variance", moving_variance, True)):
        if t is None and nm == "gamma":
            continue
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != (J,) or \
                t.dtype != torch.float32 or t.device != dev or (contig and not t.is_contiguous()):
            raise ValueError("%s: %s must be a %sfloat32 [%d] tensor on %s"
                             % (name, nm, "contiguous " if contig else "", J, dev))


def _bn_buffers(R, J, dev, training, keep_pre):
    """stats [2, J], the output y [R, J], the pre-activation a [R, J] (training, or keep_pre: an
    evaluation whose gamma needs a gradient; else None), the moment partials of 128-row tiles
    (training; else None) and the amax slot of a batch-normalised layer's forward."""
    f32 = dict(dtype=torch.float32, device=dev)
    a = torch.empty((R, J), **f32) if training or keep_pre else None
    part = torch.empty(-(-R // 128) * 2 * J, **f32) if training else None
    return torch.empty((2, J), **f32), torch.empty((R, J), **f32), a, part, torch.zeros(4, **f32)


def _bn_save(ctx, training, relu, gm, y, a, stats, *extra):
    """Keeps what _bn_backward reads, then ``extra`` (ctx.saved_tensors[4:])."""
    ctx.save_for_backward(gm, y if relu else None, a, stats, *extra)
    ctx.bn = (training, relu)


def _bn_forward(ctx, hpl, wpl, J, gamma, beta, stats_bufs, training, relu, rate, eps, bessel,
                keep_pre, *extra):
    """y [R, J] = relu?(BN(h W^T) * gamma + beta) (gamma None: no scale) and its amax slot, from
    the operand planes hpl of h and wpl of W (zsb_linear_tc_bn_f32; bessel: TF's fused-batch-norm
    update of the moving variance); saves the layer for _bn_backward."""
    from ._lib import lib, ptr, stream
    moving_mean, moving_variance = stats_bufs
    R, K = hpl.rows, hpl.K
    gm = None if gamma is None else gamma.detach().to(torch.float32).contiguous()
    b = beta.detach().to(torch.float32).contiguous()
    stats, y, a, part, amax = _bn_buffers(R, J, b.device, training, keep_pre)
    lib.call("zsb_linear_tc_bn_f32", int(training), int(bessel), ptr(wpl[0]), ptr(wpl[1]),
             ptr(hpl.planes), ptr(hpl.scale), int(hpl.binary), ptr(gm), ptr(b), ptr(moving_mean),
             ptr(moving_variance), rate, eps, ptr(stats), ptr(a), ptr(part), ptr(y), R, J, K,
             int(relu), ptr(amax), stream())
    _bn_save(ctx, training, relu, gm, y, a, stats, *extra)
    return y, amax


def _bn_backward(ctx, gy, need_gamma, need_beta, planes=True):
    """d gamma, d beta (each None unless needed) and G = d/d(pre-activation) of a layer saved by
    _bn_save: G's operand planes (zsb_bn_grad_f32), or with planes=False G [R, J] in fp32 and the
    scale slot holding its max |.| (zsb_bn_grad_f32out)."""
    from ._lib import lib, ptr, stream
    gm, y, a, stats = ctx.saved_tensors[:4]
    training, relu = ctx.bn
    J = int(stats.shape[1])
    R = gy.numel() // J
    f32 = dict(dtype=torch.float32, device=gy.device)
    g = gy.reshape(R, J).to(torch.float32).contiguous()
    dgamma = torch.empty(J, **f32) if need_gamma else None
    dbeta = torch.empty(J, **f32) if need_beta else None
    part = torch.empty((-(-R // 128) + 1) * 2 * J, **f32)
    scale = torch.zeros(4, **f32)
    args = (int(training), ptr(g), ptr(y), ptr(a), ptr(stats), ptr(gm), int(relu), R, J,
            ptr(part), ptr(dbeta), ptr(dgamma))
    if planes:
        pl = torch.empty((2, R, lib.load().zsb_linear_tc_kpad(J)), dtype=torch.float16,
                         device=gy.device)
        lib.call("zsb_bn_grad_f32", *args, ptr(pl), ptr(scale), stream())
        return dgamma, dbeta, _Planes(pl, scale, R, J)
    da = torch.empty((R, J), **f32)
    lib.call("zsb_bn_grad_f32out", *args, ptr(da), ptr(scale), stream())
    return dgamma, dbeta, (da, scale)


class _NoisyBNLinear(torch.autograd.Function):
    """relu?(BN((h * noise) W^T)) on the batch-norm epilogues of the wgmma kernel.  Forward: one
    split pass turns h * noise into operand planes (zsb_split16_noisy_f32), then _bn_forward with
    no gamma.  Backward: _bn_backward gives d beta and the planes of the pre-activation gradient,
    the unchanged input- and weight-gradient products read them, and one pass turns d(h * noise)
    into d noise and d h (zsb_noisy_grad_f32)."""

    @staticmethod
    def forward(ctx, h, noise, W, beta, stats_bufs, training, relu, rate, eps):
        from ._lib import lib, ptr, stream
        K, J = int(noise.shape[-1]), int(W.shape[0])
        lead = noise.shape[:-1]
        n2 = noise.detach().to(torch.float32).reshape(-1, K).contiguous()
        h2 = h.detach().to(torch.float32).reshape(-1, K).contiguous()
        R, n_h = int(n2.shape[0]), int(h2.shape[0])
        dev = n2.device
        Kp = lib.load().zsb_linear_tc_kpad(K)
        planes = torch.empty((2, R, Kp), dtype=torch.float16, device=dev)
        scale = torch.zeros(4, dtype=torch.float32, device=dev)
        lib.call("zsb_split16_noisy_f32", ptr(h2), n_h, ptr(n2), R, K, ptr(planes), ptr(scale),
                 stream())
        ctx.hpl = _Planes(planes, scale, R, K)
        ctx.wpl = _tc_split(W)
        y, amax = _bn_forward(ctx, ctx.hpl, ctx.wpl, J, None, beta, stats_bufs, training, relu,
                              rate, eps, False, False, W, h2, n2)
        ctx.meta = (tuple(h.shape), lead, R, n_h, K)
        return _tag(y.reshape(tuple(lead) + (J,)), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        from ._lib import lib, ptr, stream
        W, h2, n2 = ctx.saved_tensors[4:]
        h_shape, lead, R, n_h, K = ctx.meta
        need = ctx.needs_input_grad
        dev = gy.device
        _, dbeta, gpl = _bn_backward(ctx, gy, False, need[3])
        dh = dnoise = None
        if need[0] or need[1]:
            dx, _ = _tc_grad_input(gpl, W, R, *ctx.wpl)
            dnoise = torch.empty((R, K), dtype=torch.float32, device=dev) if need[1] else None
            dh = torch.empty((n_h, K), dtype=torch.float32, device=dev) if need[0] else None
            lib.call("zsb_noisy_grad_f32", ptr(dx), ptr(h2), n_h, ptr(n2), R, K, ptr(dnoise),
                     ptr(dh), stream())
            dh = None if dh is None else dh.reshape(h_shape)
            dnoise = None if dnoise is None else dnoise.reshape(tuple(lead) + (K,))
        dW = _grad_weight_release(ctx, gpl, R, need[2])
        return dh, dnoise, dW, dbeta, None, None, None, None, None


def noisy_bn_linear(h, noise, W, beta, moving_mean, moving_variance, training, relu=True,
                    decay=0.999, epsilon=1e-3):
    """``relu?(BN((h * noise) @ W.T))``, shape ``noise.shape[:-1] + (J,)``: one layer of
    examples/bayesian_neural_nets/variational_dropout.py:26-37, ``layers.fully_connected(h * eps,
    n_out, normalizer_fn=layers.batch_norm)`` with the defaults of tf.contrib.layers:

    * no bias (``fully_connected`` drops it when a normalizer is given);
    * batch norm with ``center=True`` (``beta`` [J]), ``scale=False`` (no gamma) and ``epsilon``;
      ``training``: the moments over all ``noise.shape[:-1]`` rows with the population variance, and
      ``moving_mean`` / ``moving_variance`` (float32 [J]) updated in place as ``m -= (m - batch) *
      (1 - decay)`` (``updates_collections=None``, no zero-debiasing); otherwise the moving
      statistics normalise and stay unchanged;
    * then ``relu``.  ``fully_connected``'s default activation is ReLU, so the example applies it
      to every layer, the 10-unit logits layer included (its explicit ``tf.nn.relu`` for the hidden
      layers is redundant): keep ``relu=True`` on the last layer to reproduce it.

    ``noise`` is ``[*lead, K]`` and ``h``'s shape is a suffix of it, so ``x`` [n, K] broadcasts
    over the particle axis without being tiled; ``h`` may also have ``noise``'s full shape.
    ``W`` is [J, K] (the kernel transposed, as in ``linear``).  The product of ``h * noise`` is
    never formed in fp32: its operand planes are made in one pass over ``h`` and ``noise``.

    Differentiable w.r.t. ``h``, ``noise``, ``W`` and ``beta``; the moving statistics receive no
    gradient.  The batch moments and every gradient's column sums are reduced in a fixed order, so
    two identical calls give identical bits.  The output carries the max |.| that a following
    ``linear`` uses for its operand split."""
    noise_s, h_s = tuple(noise.shape), tuple(h.shape)
    if noise.dim() < 1 or not noise.is_floating_point():
        raise ValueError("noise must be a floating tensor [*lead, K], got %s %s"
                         % (noise.dtype, noise_s))
    if len(h_s) < 1 or len(h_s) > len(noise_s) or noise_s[len(noise_s) - len(h_s):] != h_s:
        raise ValueError("the shape of h %s must be a suffix of the shape of noise %s"
                         % (h_s, noise_s))
    K = noise_s[-1]
    if W.dim() != 2 or int(W.shape[1]) != K:
        raise ValueError("W %s must be [J, %d]" % (tuple(W.shape), K))
    J = int(W.shape[0])
    _bn_check("noisy_bn_linear", J, W.device, None, beta, moving_mean, moving_variance)
    if any(int(d) == 0 for d in noise_s) or J == 0:
        raise ValueError("empty shapes are not supported: noise %s, W %s"
                         % (noise_s, tuple(W.shape)))
    return _NoisyBNLinear.apply(h, noise, W, beta, (moving_mean, moving_variance), bool(training),
                                bool(relu), float(1.0 - decay), float(epsilon))


class _BNLinear(torch.autograd.Function):
    """relu?(BN(h W^T) * gamma + beta): _bn_forward from the cached operand planes of h -- a 0/1
    sample's one plane included.  Backward: _bn_backward gives d beta, d gamma and the planes of
    the pre-activation gradient, which the unchanged input- and weight-gradient products read."""

    @staticmethod
    def forward(ctx, h, W, gamma, beta, stats_bufs, training, relu, rate, eps, keep_pre):
        lead = h.shape[:-1]
        K, J = int(h.shape[-1]), int(W.shape[0])
        h2 = h.reshape(-1, K)
        R = int(h2.shape[0])
        ctx.hpl = _planes_of(h2, h)
        ctx.wpl = _tc_split(W)
        y, amax = _bn_forward(ctx, ctx.hpl, ctx.wpl, J, gamma, beta, stats_bufs, training, relu,
                              rate, eps, False, keep_pre, W)
        ctx.meta = (lead, R, K)
        return _tag(y.reshape(tuple(lead) + (J,)), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        W, = ctx.saved_tensors[4:]
        lead, R, K = ctx.meta
        need = ctx.needs_input_grad
        dgamma, dbeta, gpl = _bn_backward(ctx, gy, need[2], need[3])
        dh, dW = _grad_products(ctx, gpl, W, R, ctx.wpl, tuple(lead) + (K,), need[0], need[1])
        return dh, dW, dgamma, dbeta, None, None, None, None, None, None


def bn_linear(h, W, gamma, beta, moving_mean, moving_variance, training, relu=True, momentum=0.99,
              epsilon=1e-3):
    """``relu?(BN(h @ W.T))``, shape ``h.shape[:-1] + (J,)``: ``tf.layers.dense(h, J,
    use_bias=False)`` followed by ``tf.layers.batch_normalization(..., training=training)`` and
    ``tf.nn.relu``, as in examples/variational_autoencoders/bernoulli_latent_vae.py:25-30 and 39-44,
    with the defaults of ``tf.layers.batch_normalization`` on its non-fused path (TF 1.x fuses only
    4-D inputs):

    * ``center=True`` and ``scale=True``: ``y = xhat * gamma + beta`` with ``xhat = (a - mean) *
      rsqrt(var + epsilon)``, ``a = h @ W.T``;
    * ``training``: the moments over all ``h.shape[:-1]`` rows with the population variance, and
      ``moving_mean`` / ``moving_variance`` (contiguous float32 [J]) updated in place as ``m -= (m -
      batch) * (1 - momentum)``, with no zero-debiasing; otherwise the moving statistics normalise
      and stay unchanged.

    ``h`` [*lead, K] may be an activation of another fused layer, a ``StochasticTensor``, or a
    ``LinearBernoulli`` sample, whose one 0/1 operand plane is multiplied as it is (never split
    again).  ``W`` is [J, K] (the kernel transposed, as in ``linear``); ``gamma`` and ``beta`` are
    [J].  Differentiable w.r.t. ``h``, ``W``, ``gamma`` and ``beta``; the moving statistics receive
    no gradient.  In evaluation with a ``gamma`` that requires a gradient, the forward also keeps
    the pre-activation, from which the gradient of gamma is computed.  The batch moments and every
    gradient's column sums are reduced in a fixed order, so two identical calls give identical
    bits.  The output carries the max |.| that a following fused layer uses for its operand
    split."""
    h = _unwrap(h)
    if not isinstance(h, torch.Tensor) or h.dim() < 1:
        raise ValueError("h must be a tensor [*lead, K], got %r" % (type(h),))
    if h.dtype != torch.float32 and (h.is_floating_point() or h.is_complex()):
        raise ValueError("h must be float32 or a 0/1 integer sample, got %s" % h.dtype)
    K = int(h.shape[-1])
    if not isinstance(W, torch.Tensor) or W.dim() != 2 or int(W.shape[1]) != K or \
            W.dtype != torch.float32:
        raise ValueError("W %s must be a float32 [J, %d] tensor"
                         % (tuple(getattr(W, "shape", ())), K))
    dev = W.device
    if dev.type != "cuda":
        raise ValueError("bn_linear runs on a CUDA device; W is on %s" % dev)
    J = int(W.shape[0])
    if h.device != dev:
        raise ValueError("h is on %s and W on %s" % (h.device, dev))
    if gamma is None:
        raise ValueError("bn_linear: gamma must be a float32 [%d] tensor on %s" % (J, dev))
    _bn_check("bn_linear", J, dev, gamma, beta, moving_mean, moving_variance)
    if h.numel() == 0 or J == 0:
        raise ValueError("empty shapes are not supported: h %s, W %s"
                         % (tuple(h.shape), tuple(W.shape)))
    keep_pre = (not training) and torch.is_grad_enabled() and gamma.requires_grad
    return _BNLinear.apply(h, W, gamma, beta, (moving_mean, moving_variance), bool(training),
                           bool(relu), float(1.0 - momentum), float(epsilon), bool(keep_pre))


def linear_bernoulli_log_prob(h, W, b, x):
    """log p(x | logits = h @ W.T + b) summed over the last axis, fused.
    ``x`` ([n_x, J], 0/1) is broadcast over the leading rows of ``h``
    (row r of h uses x[r % n_x]: the [particles, batch] layout of
    iwae.py:23-32 flattened)."""
    return _LinearBernoulliLogProb.apply(h, W, b, x)


_BIN_SCALES = {}


def _bin_scale(device):
    """The scale slot of a sample's binary plane: 2048, the power of two the split of a 0/1
    matrix picks (zsb_linear_tc_bern_sample_f32).  One read-only tensor per device."""
    t = _BIN_SCALES.get(device)
    if t is None:
        t = torch.tensor([2048.0, 0.0, 0.0, 0.0], dtype=torch.float32, device=device)
        _BIN_SCALES[device] = t
    return t


class _LinearBernoulliGiven(torch.autograd.Function):
    """log Bernoulli(logits = h W^T + b).log_prob(x[s]) summed over the features, [S, *lead], for
    S given rows per logit row (x2 = [S * rows, J]), differentiable w.r.t. h, W and b.  Forward:
    the epi-1 launch with S given rows, or -- for the layer's own sample -- the log q its sampling
    launch already wrote (``lq``).  Backward: d/dlogits summed over the S draws, so the input and
    weight gradients stay products over the rows of h (nothing is expanded S-fold)."""

    @staticmethod
    def forward(ctx, h, W, b, x2, S, lq, wp, ws, hpl):
        from ._lib import lib, ptr, stream
        lead = h.shape[:-1]
        R, K, J = hpl.rows, hpl.K, int(W.shape[0])
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        if lq is None:
            lq = torch.empty(S * R, dtype=torch.float32, device=x2.device)
            part = torch.empty(lib.load().zsb_linear_tc_nparts(J) * S * R, dtype=torch.float32,
                               device=x2.device)
            lib.call("zsb_linear_tc_bern_given_f32", 1, ptr(wp), ptr(ws), ptr(hpl.planes),
                     ptr(hpl.scale), int(hpl.binary), ptr(bias), ptr(x2), S, None, ptr(lq),
                     ptr(part), R, J, K, None, stream())
        else:
            lq = lq.clone()
        ctx.save_for_backward(W, bias, x2, wp, ws)
        ctx.hpl = hpl
        ctx.meta = (lead, S, R, J, K, b is not None)
        return lq.reshape((S,) + tuple(lead))

    @staticmethod
    @once_differentiable
    def backward(ctx, glq):
        from ._lib import lib, ptr, stream
        W, bias, x2, wp, ws = ctx.saved_tensors
        lead, S, R, J, K, has_b = ctx.meta
        hpl = ctx.hpl
        need = ctx.needs_input_grad
        g = glq.reshape(-1).to(torch.float32).contiguous()
        db = torch.zeros(J, dtype=torch.float32, device=g.device) if (has_b and need[2]) else None
        amax = torch.zeros(4, dtype=torch.float32, device=g.device)
        dl = torch.empty((R, J), dtype=torch.float32, device=g.device)
        lib.call("zsb_linear_tc_bern_given_f32", 2, ptr(wp), ptr(ws), ptr(hpl.planes),
                 ptr(hpl.scale), int(hpl.binary), ptr(bias), ptr(x2), S, ptr(g), ptr(dl), None,
                 R, J, K, ptr(amax), stream())
        dlpl = _tc_split_dual(dl, amax=amax, col_sum=db)
        dh, dW = _grad_products(ctx, dlpl, W, R, (wp, ws), tuple(lead) + (K,), need[0], need[1])
        return dh, dW, db, None, None, None, None, None, None


def _version(t):
    """The in-place version counter of ``t``; None for an inference tensor, which has none (it is
    then never trusted as an unchanged cache key)."""
    try:
        return t._version
    except RuntimeError:
        return None


def _versions(*ts):
    return tuple(None if t is None else _version(t) for t in ts)


class LinearBernoulli(object):
    """Drop-in for ``Bernoulli(logits=dense(h), group_ndims=1)`` as a
    distribution plugin (duck-typed contract of bn.py:96-115): ``log_prob`` runs
    the fused GEMM + Bernoulli epilogue; the logits never reach memory.

    ``sample(n_samples)`` is one launch (zsb_linear_tc_bern_sample_f32) that draws the sample --
    element for element what ``Bernoulli(linear(h, W, b)).sample(n_samples)`` draws from the same
    ``zs.random`` state -- together with its log-probability and its operand plane for the next
    layer.  ``log_prob`` of that very sample returns the stored log-probability (no second GEMM),
    differentiable w.r.t. h, W and b.  A sample fed to ``linear`` or to another ``LinearBernoulli``
    (the sigmoid belief nets of examples/sigmoid_belief_nets, where every activation is a 0/1
    sample) is multiplied on the two-product mainloop: same result bit for bit, a third fewer
    tensor-core products and operand bytes.  ``given`` with leading sample axes beyond the rows of
    ``h`` ([S, *h.shape[:-1], J]) is scored against the shared logits without expanding them."""

    def __init__(self, h, W, b=None, dtype=torch.int32, group_ndims=1):
        if group_ndims != 1:
            raise ValueError("LinearBernoulli sums over the feature axis: "
                             "group_ndims must be 1")
        self._h, self._W, self._b = h, W, b
        self.dtype = dtype
        self.param_dtype = torch.float32
        self.is_continuous = False
        self.is_reparameterized = False
        self.group_ndims = 1

    @property
    def logits(self):
        return linear(self._h, self._W, self._b)

    def get_batch_shape(self):
        return torch.Size(tuple(self._h.shape[:-1]) + (int(self._W.shape[0]),))

    def get_value_shape(self):
        return torch.Size([])

    batch_shape = property(lambda self: self.get_batch_shape())
    value_shape = property(lambda self: self.get_value_shape())

    def sample(self, n_samples=None, u=None):
        """``n_samples`` as in ``Bernoulli.sample``; ``u``: injected uniforms that broadcast to the
        sample's shape (``Bernoulli._sample(n, u=...)``), else the Philox stream of
        ``zs.random``."""
        from . import random as zrandom
        from ._lib import lib, ptr, stream
        if isinstance(n_samples, torch.Tensor):
            n_samples = int(n_samples.item())
        S = 1 if n_samples is None else int(n_samples)
        h, W, b = self._h, self._W, self._b
        lead = tuple(h.shape[:-1])
        J, K = int(W.shape[0]), int(h.shape[-1])
        h2 = h.reshape(-1, K)
        R = int(h2.shape[0])
        dev = W.device
        hpl = _planes_of(h2, h)
        wp, ws = _tc_split(W)
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        seed, it = zrandom.get_seed(), zrandom.next_counter()
        full = (S,) + lead + (J,)
        h_int = self.dtype == torch.int32
        hs = torch.empty(full, dtype=torch.int32 if h_int else torch.float32, device=dev)
        planes = torch.empty((1, S * R, lib.load().zsb_linear_tc_kpad(J)), dtype=torch.float16,
                             device=dev)
        lq = torch.empty(S * R, dtype=torch.float32, device=dev)
        part = torch.empty(lib.load().zsb_linear_tc_nparts(J) * S * R, dtype=torch.float32,
                           device=dev)
        uu = None if u is None else u.to(torch.float32).expand(full).contiguous()
        lib.call("zsb_linear_tc_bern_sample_f32", ptr(wp), ptr(ws), ptr(hpl.planes),
                 ptr(hpl.scale), int(hpl.binary), ptr(bias), ptr(uu), int(seed), int(it), S,
                 ptr(hs), int(h_int), ptr(planes), ptr(lq), ptr(part), R, J, K, stream())
        if self.dtype not in (torch.int32, torch.float32):
            hs = hs.to(self.dtype)
        if n_samples is None:
            hs = hs.squeeze(0)
        vs = _versions(hs, h, W, b)
        if all(v is not None for t, v in zip((hs, h, W, b), vs) if t is not None):
            # (inference tensors of torch.inference_mode() have no version: nothing is cached)
            hs._zsb_pl = _Planes(planes, _bin_scale(dev), S * R, J, binary=True, version=vs[0])
            self._own = (hs, lq, S, wp, ws, hpl, vs)
        else:
            self._own = None
        return hs

    def log_prob(self, given):
        J = int(self._W.shape[0])
        lead = tuple(self._h.shape[:-1])
        own = getattr(self, "_own", None)
        if own is not None and given is own[0] and \
                own[6] == _versions(given, self._h, self._W, self._b):
            hs, lq, S, wp, ws, hpl, _ = own
            x2 = hs.reshape(-1, J).to(torch.float32).contiguous()
            return _LinearBernoulliGiven.apply(self._h, self._W, self._b, x2, S, lq, wp, ws, hpl)\
                .reshape(tuple(given.shape[:-1]))
        nd = len(lead) + 1
        if given.dim() > nd and tuple(given.shape[-nd:]) == lead + (J,):
            # leading sample axes beyond the rows of h: [S, *lead, J] against the [*lead, J] logits
            S = 1
            for d in given.shape[:-nd]:
                S *= int(d)
            h2 = self._h.reshape(-1, int(self._h.shape[-1]))
            hpl = _planes_of(h2, self._h)
            wp, ws = _tc_split(self._W)
            x2 = given.reshape(-1, J).to(torch.float32).contiguous()
            return _LinearBernoulliGiven.apply(self._h, self._W, self._b, x2, S, None, wp, ws,
                                               hpl).reshape(tuple(given.shape[:-1]))
        g = given.reshape(-1, J)
        n_x = int(g.shape[0])
        rows = 1
        for d in lead:
            rows *= int(d)
        if tuple(given.shape) != lead + (J,):
            # suffix-broadcast observation (e.g. x [N, J] against h [K, N, H])
            if rows % n_x != 0 or tuple(given.shape[:-1]) != lead[len(lead) - (given.dim() - 1):]:
                raise ValueError("given %s is not a suffix-broadcast of the "
                                 "batch shape %s" % (tuple(given.shape), lead + (J,)))
        return linear_bernoulli_log_prob(self._h, self._W, self._b, g)

    def prob(self, given):
        return torch.exp(self.log_prob(given))


CAT_MAX_C = 128


class _LinearCategoricalGiven(torch.autograd.Function):
    """OnehotCategorical(logits = h W^T + b).log_prob(given) for S draws per logit row, [S R]: draw
    d = s R + r against given row d % n_g (g2 = [n_g, C] float).  Forward: the given epilogue, or --
    for the layer's own sample -- the log q its sampling launch already wrote (``lq``).  Backward:
    d/dlogits summed over the S draws in one launch, then the input and weight gradients as products
    over the rows of h."""

    @staticmethod
    def forward(ctx, h, W, b, g2, S, lq, wp, ws, hpl):
        R, K, C = hpl.rows, hpl.K, int(W.shape[0])
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        if lq is None:
            lq = torch.empty(S * R, dtype=torch.float32, device=g2.device)
            _cat_given(1, wp, ws, hpl, bias, g2, S, None, lq, R, C, K, None)
        else:
            lq = lq.clone()
        ctx.save_for_backward(W, bias, g2, wp, ws)
        ctx.hpl = hpl
        ctx.meta = (tuple(h.shape[:-1]), S, R, C, K, b is not None)
        return lq

    @staticmethod
    @once_differentiable
    def backward(ctx, glq):
        W, bias, g2, wp, ws = ctx.saved_tensors
        lead, S, R, C, K, has_b = ctx.meta
        need = ctx.needs_input_grad
        g = glq.reshape(-1).to(torch.float32).contiguous()
        db = torch.zeros(C, dtype=torch.float32, device=g.device) if (has_b and need[2]) else None
        amax = torch.zeros(4, dtype=torch.float32, device=g.device)
        dl = torch.empty((R, C), dtype=torch.float32, device=g.device)
        _cat_given(2, wp, ws, ctx.hpl, bias, g2, S, g, dl, R, C, K, amax)
        dlpl = _tc_split_dual(dl, amax=amax, col_sum=db)
        dh, dW = _grad_products(ctx, dlpl, W, R, (wp, ws), lead + (K,), need[0], need[1])
        return dh, dW, db, None, None, None, None, None, None


def _cat_given(epi, wp, ws, hpl, bias, g2, S, gout, out, R, C, K, amax):
    from ._lib import lib, ptr, stream
    lib.call("zsb_linear_tc_cat_given_f32", epi, ptr(wp), ptr(ws), ptr(hpl.planes),
             ptr(hpl.scale), int(hpl.binary), ptr(bias), ptr(g2), int(g2.shape[0]), S, ptr(gout),
             ptr(out), R, C, K, ptr(amax), stream())


class _CachedHPlanes(object):
    """The operand planes of a layer's input ``self._h``, kept with h's version in ``self._hpl``."""

    def _h_planes(self):
        """The operand planes of h.  The planes cached on h do not track its version, so the layer
        keeps the planes it last read with h's version: while that version holds it reuses them;
        once h has been rewritten in place it splits h afresh and caches the new planes on h as
        well, so the next reader (this layer or another) does not find the old ones.  An inference
        tensor has no version and is read through the cache on h, as ``linear`` reads it."""
        h2 = self._h.reshape(-1, int(self._h.shape[-1]))
        v = _version(self._h)
        if v is not None and self._hpl is not None and self._hpl[1] == v:
            return self._hpl[0]
        if v is not None and self._hpl is not None:
            pl = _tc_split_dual(h2)
            try:
                self._h._zsb_pl = pl
            except (AttributeError, RuntimeError):
                pass
        else:
            pl = _planes_of(h2, self._h)
        self._hpl = (pl, v)
        return pl


class LinearOnehotCategorical(_CachedHPlanes):
    """Drop-in for ``OnehotCategorical(logits=dense(h))`` as a distribution plugin of
    ``bn.stochastic`` (the ``y`` of vae_ssl_adaptive_is.py:61-68), with the logits never leaving the
    dense layer's epilogue.  ``W`` [C, H] and ``b`` [C] are the ``tf.layers.dense`` kernel
    transposed and its bias, as in ``linear``.

    ``sample(n_samples)`` is one launch (zsb_linear_tc_cat_sample_f32) that draws the one-hot sample
    -- element for element what ``OnehotCategorical(linear(h, W, b)).sample(n_samples)`` draws from
    the same ``zs.random`` state -- together with its log-probability and its class indices.
    ``log_prob`` of that very sample returns the stored log-probability (no second product);
    ``log_prob`` of any other ``given`` ([S, *h.shape[:-1], C] with leading sample axes, or a
    suffix-broadcast [..., C] such as labels [N, C] against h [K, N, H]; one-hot or not) runs the
    given epilogue.  Both are differentiable w.r.t. h, W and b.  The sample carries its class
    indices, so ``class_linear(x, W, W_class, y)`` reads them instead of taking an argmax.

    Outside the fused domain -- more than 128 classes, parameters that are not float32, tensors not
    on one CUDA device -- the layer is ``OnehotCategorical(linear(h, W, b))`` (``F.linear`` for
    tensors off the GPU), which draws the same samples by construction."""

    def __init__(self, h, W, b=None, dtype=torch.int32, group_ndims=0):
        h = _unwrap(h)
        self._h, self._W, self._b = h, W, b
        self.dtype = dtype
        self.param_dtype = torch.float32
        self.is_continuous = False
        self.is_reparameterized = False
        self.group_ndims = group_ndims
        self._n_categories = int(W.shape[0])
        ts = [t for t in (h, W, b) if t is not None]
        self._hpl = None
        self._fused = (1 <= self._n_categories <= CAT_MAX_C and h.numel() > 0
                       and all(t.is_cuda and t.dtype == torch.float32 and t.device == W.device
                               for t in ts))

    n_categories = property(lambda self: self._n_categories)

    @property
    def logits(self):
        if self._W.is_cuda:
            return linear(self._h, self._W, self._b)
        return torch.nn.functional.linear(self._h, self._W, self._b)

    def _registry(self):
        from .distributions.multivariate import OnehotCategorical
        return OnehotCategorical(self.logits, dtype=self.dtype, group_ndims=self.group_ndims)

    def get_batch_shape(self):
        return torch.Size(tuple(self._h.shape[:-1]))

    def get_value_shape(self):
        return torch.Size([self._n_categories])

    batch_shape = property(lambda self: self.get_batch_shape())
    value_shape = property(lambda self: self.get_value_shape())

    def sample(self, n_samples=None, u=None):
        """``n_samples`` as in ``OnehotCategorical.sample``; ``u``: injected uniforms, one per draw,
        that broadcast to ``[n_samples, *batch_shape]`` (those of ``ops.sample_categorical``), else
        the Philox stream of ``zs.random``."""
        from . import random as zrandom
        from ._lib import lib, ptr, stream
        if isinstance(n_samples, torch.Tensor):
            n_samples = int(n_samples.item())
        S = 1 if n_samples is None else int(n_samples)
        if not self._fused:
            if u is None:
                out = self._registry().sample(n_samples)
            else:
                from . import ops
                draws = ops.sample_categorical(self.logits, S, u=u.to(torch.float32),
                                               seed=zrandom.get_seed(), it=zrandom.next_counter())
                out = torch.nn.functional.one_hot(draws.long(), self._n_categories).to(self.dtype)
                if n_samples is None:
                    out = out.squeeze(0)
            self._own = None
            return out
        h, W, b = self._h, self._W, self._b
        lead = tuple(h.shape[:-1])
        C, K = self._n_categories, int(h.shape[-1])
        R = h.numel() // K
        dev = W.device
        hpl = self._h_planes()
        wp, ws = _tc_split(W)
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        seed, it = zrandom.get_seed(), zrandom.next_counter()
        h_int = self.dtype != torch.float32
        ys = torch.empty((S,) + lead + (C,), dtype=torch.int32 if h_int else torch.float32,
                         device=dev)
        cls = torch.empty(S * R, dtype=torch.int32, device=dev)
        lq = torch.empty(S * R, dtype=torch.float32, device=dev)
        uu = None if u is None else u.to(torch.float32).expand((S,) + lead).contiguous()
        lib.call("zsb_linear_tc_cat_sample_f32", ptr(wp), ptr(ws), ptr(hpl.planes),
                 ptr(hpl.scale), int(hpl.binary), ptr(bias), ptr(uu), int(seed), int(it), S,
                 ptr(cls), ptr(ys), int(h_int), ptr(lq), R, C, K, stream())
        if self.dtype not in (torch.int32, torch.float32):
            ys = ys.to(self.dtype)
        if n_samples is None:
            ys = ys.squeeze(0)
        vs = _versions(ys, h, W, b)
        if all(v is not None for t, v in zip((ys, h, W, b), vs) if t is not None):
            # (inference tensors of torch.inference_mode() have no version: nothing is cached)
            ys._zsb_cls = (cls, vs[0])
            self._own = (ys, lq, S, wp, ws, hpl, vs)
        else:
            self._own = None
        return ys

    def log_prob(self, given):
        if not self._fused:
            return self._registry().log_prob(given)
        from . import ops
        C = self._n_categories
        lead = tuple(self._h.shape[:-1])
        own = getattr(self, "_own", None)
        if own is not None and given is own[0] and \
                own[6] == _versions(given, self._h, self._W, self._b):
            ys, lq, S, wp, ws, hpl, _ = own
            g2 = ys.reshape(-1, C).to(torch.float32).contiguous()
            lp = _LinearCategoricalGiven.apply(self._h, self._W, self._b, g2, S, lq, wp, ws, hpl)
            return ops.group_sum(lp.reshape(tuple(given.shape[:-1])), self.group_ndims)
        gs = tuple(given.shape)
        nd = len(lead)
        if not gs or gs[-1] != C:
            raise ValueError("given %s is not a one-hot over the %d classes" % (gs, C))
        gb = gs[:-1]
        if len(gb) >= nd and gb[len(gb) - nd:] == lead:
            S = 1                   # [S..., *lead, C]: leading sample axes against the shared logits
            for d in gb[:len(gb) - nd]:
                S *= int(d)
            out_shape = gb
        elif gb == lead[nd - len(gb):]:
            S, out_shape = 1, lead  # suffix broadcast: given row r % n_g for logit row r
        else:
            return self._registry().log_prob(given)
        if given.numel() == 0:
            return self._registry().log_prob(given)
        hpl = self._h_planes()
        wp, ws = _tc_split(self._W)
        g2 = given.reshape(-1, C).to(torch.float32).contiguous()
        lp = _LinearCategoricalGiven.apply(self._h, self._W, self._b, g2, S, None, wp, ws, hpl)
        return ops.group_sum(lp.reshape(out_shape), self.group_ndims)

    def prob(self, given):
        return torch.exp(self.log_prob(given))


NORMAL_MAX_D = 256


def _pack_heads(a, b, D):
    """The heads ``a``, ``b`` ([D, ...]) stacked along axis 0 in blocks of 64 rows, [a 0..63 |
    b 0..63 | a 64..127 | ...], each zero padded to Dp = kpad(D) rows: the weight (or bias) layout
    of zsb_linear_tc_normal_sample_f32.  Differentiable."""
    Dp = (D + 63) // 64 * 64
    pad = (0, 0) * (a.dim() - 1) + (0, Dp - D)
    blocks = [torch.nn.functional.pad(t, pad).reshape((Dp // 64, 64) + tuple(t.shape[1:]))
              for t in (a, b)]
    return torch.stack(blocks, 1).reshape((2 * Dp,) + tuple(a.shape[1:]))


def _unpack_heads(y, D):
    """(a, b) of a packed [..., 2 Dp] output, each [..., D]."""
    Dp = int(y.shape[-1]) // 2
    y4 = y.reshape(tuple(y.shape[:-1]) + (Dp // 64, 2, 64))
    lead = tuple(y.shape[:-1])
    return (y4[..., 0, :].reshape(lead + (Dp,))[..., :D],
            y4[..., 1, :].reshape(lead + (Dp,))[..., :D])


class _LinearNormalSample(torch.autograd.Function):
    """(z, log q(z)) of S draws per row of h from N(mu, exp(ls)), [mu | ls] = h Wp^T + bp with the
    packed heads Wp [2 Dp, K], bp [2 Dp]: one launch of the Gaussian-sampling epilogue (EPI 15).
    Backward receives the gradients of z and log q together and runs one pass over the draws
    (zsb_linear_normal_grad_f32, eps recomputed from Philox or read when injected) that gives the
    gradient of the packed pre-activation, then the layer's input- and weight-gradient products.
    ``reparam`` False: z is a constant (Normal._sample stop-gradients mean and std) and log q keeps
    its partials w.r.t. mu and ls."""

    @staticmethod
    def forward(ctx, h, Wp, bp, eps, S, D, reparam, hpl, seed, it, keep):
        from ._lib import lib, ptr, stream
        lead = tuple(h.shape[:-1])
        R, K, J = hpl.rows, hpl.K, int(Wp.shape[0])
        dev = Wp.device
        wp, ws = _tc_split(Wp)
        bias = bp.detach().to(torch.float32).contiguous() if bp is not None else None
        z = torch.empty((S,) + lead + (D,), dtype=torch.float32, device=dev)
        lq = torch.empty((S,) + lead, dtype=torch.float32, device=dev)
        part = torch.empty(J // 64 * S * R, dtype=torch.float32, device=dev)
        ls = torch.empty((R, D), dtype=torch.float32, device=dev) if keep else None
        amax = torch.zeros(4, dtype=torch.float32, device=dev)
        e = None if eps is None else eps.detach().to(torch.float32).expand(z.shape).contiguous()
        lib.call("zsb_linear_tc_normal_sample_f32", ptr(wp), ptr(ws), ptr(hpl.planes),
                 ptr(hpl.scale), int(hpl.binary), ptr(bias), ptr(e), int(seed), int(it), S,
                 ptr(z), ptr(lq), ptr(part), None, ptr(ls), R, D, K, ptr(amax), stream())
        if keep:
            # the device epoch the launch added to `it`, copied on the stream right after it: the
            # backward pass recomputes these draws even if the epoch moves before it runs
            from . import random as zrandom
            ep = zrandom._epoch["tensor"]
            ctx.epoch = None if (ep is None or e is not None) else ep.clone()
            ctx.save_for_backward(Wp, ls, e)
            ctx.hpl = hpl
            ctx.wpl = (wp, ws)
        ctx.meta = (lead, S, R, D, K, bp is not None, reparam, int(seed), int(it))
        ctx.set_materialize_grads(False)     # an unused z or log q sends None, not zeros
        if not reparam:
            ctx.mark_non_differentiable(z)
        return _tag(z, amax), lq

    @staticmethod
    @once_differentiable
    def backward(ctx, gz, glq):
        from ._lib import lib, ptr, stream
        Wp, ls, e = ctx.saved_tensors
        lead, S, R, D, K, has_b, reparam, seed, it = ctx.meta
        need = ctx.needs_input_grad
        dev = Wp.device
        J = int(Wp.shape[0])
        g_z = gz.to(torch.float32).contiguous() if (gz is not None and reparam) else None
        g_lq = glq.to(torch.float32).contiguous() if glq is not None else None
        dpre = torch.empty((R, J), dtype=torch.float32, device=dev)
        amax = torch.zeros(4, dtype=torch.float32, device=dev)
        lib.call("zsb_linear_normal_grad_f32", ptr(ls), ptr(g_z), ptr(g_lq), ptr(e), seed, it,
                 ptr(ctx.epoch), int(reparam), S, R, D, ptr(dpre), ptr(amax), stream())
        db = torch.zeros(J, dtype=torch.float32, device=dev) if (has_b and need[2]) else None
        dpl = _tc_split_dual(dpre, amax=amax, col_sum=db)
        dh, dW = _grad_products(ctx, dpl, Wp, R, ctx.wpl, lead + (K,), need[0], need[1])
        return dh, dW, db, None, None, None, None, None, None, None, None


class LinearNormal(_CachedHPlanes):
    """Drop-in for ``Normal(dense(h), logstd=dense(h), ...)`` as a distribution plugin of
    ``bn.stochastic`` (the z heads of vae_ssl_adaptive_is.py:53-68, and the Gaussian latent head of
    the VAE examples), with the two heads never leaving the dense layer's epilogue.  ``W_mean``,
    ``W_logstd`` [D, H] and ``b_mean``, ``b_logstd`` [D] (either bias may be None) are the
    ``tf.layers.dense`` kernels transposed and their biases, as in ``linear``.

    ``sample(n_samples)`` is one launch (zsb_linear_tc_normal_sample_f32) that draws z -- element
    for element what ``Normal(layer.mean, logstd=layer.logstd).sample(n_samples)`` draws from the
    same ``zs.random`` state, or from the same injected ``eps`` -- together with ``log q(z)`` summed
    over the features; no [n_samples, *batch, D] tensor besides z is written.  ``log_prob`` of that
    very sample with ``group_ndims >= 1`` returns the stored sum (no second pass); any other
    ``given``, and ``group_ndims = 0``, is scored by ``Normal`` on ``mean`` / ``logstd``.  Both are
    differentiable w.r.t. h and the four parameters: z by the reparameterisation when
    ``is_reparameterized``, else z is a constant and log q keeps its partials (univariate.py:161-172).
    The sample carries its max |.|, so the next ``linear`` of it skips its max pass.

    ``mean`` / ``logstd`` are one ``linear`` over the packed heads, sliced: they read the operand
    planes the sampling launch reads.  Outside the fused domain -- more than 256 features,
    parameters that are not float32, tensors not on one CUDA device -- the layer is
    ``Normal(linear(h, W_mean, b_mean), logstd=linear(h, W_logstd, b_logstd))`` (``F.linear`` for
    tensors off the GPU)."""

    def __init__(self, h, W_mean, b_mean, W_logstd, b_logstd, group_ndims=0,
                 is_reparameterized=True):
        h = _unwrap(h)
        self._h = h
        self._params = (W_mean, b_mean, W_logstd, b_logstd)
        self._D = int(W_mean.shape[0])
        if tuple(W_logstd.shape) != tuple(W_mean.shape):
            raise ValueError("W_mean %s and W_logstd %s differ in shape"
                             % (tuple(W_mean.shape), tuple(W_logstd.shape)))
        self.dtype = torch.float32
        self.param_dtype = torch.float32
        self.is_continuous = True
        self.is_reparameterized = bool(is_reparameterized)
        self.group_ndims = group_ndims
        self._hpl = None
        self._heads = None
        self._own = None
        ts = [t for t in (h,) + self._params if t is not None]
        self._fused = (1 <= self._D <= NORMAL_MAX_D and h.numel() > 0
                       and all(t.is_cuda and t.dtype == torch.float32
                               and t.device == W_mean.device for t in ts))

    def _packed(self):
        W_mean, b_mean, W_logstd, b_logstd = self._params
        Wp = _pack_heads(W_mean, W_logstd, self._D)
        if b_mean is None and b_logstd is None:
            return Wp, None
        zero = torch.zeros(self._D, dtype=torch.float32, device=W_mean.device)
        return Wp, _pack_heads(zero if b_mean is None else b_mean,
                               zero if b_logstd is None else b_logstd, self._D)

    def _mean_logstd(self):
        ts = (self._h,) + self._params
        vs = _versions(*ts)
        key = (vs, torch.is_grad_enabled())
        if not all(v is not None for t, v in zip(ts, vs) if t is not None):
            key = None                       # an inference tensor: nothing is cached
        if key is not None and self._heads is not None and self._heads[0] == key:
            return self._heads[1]
        W_mean, b_mean, W_logstd, b_logstd = self._params
        if self._fused:
            self._h_planes()                 # h's cached planes follow its in-place changes
            Wp, bp = self._packed()
            heads = _unpack_heads(linear(self._h, Wp, bp), self._D)
        elif W_mean.is_cuda:
            heads = (linear(self._h, W_mean, b_mean), linear(self._h, W_logstd, b_logstd))
        else:
            F = torch.nn.functional
            heads = (F.linear(self._h, W_mean, b_mean), F.linear(self._h, W_logstd, b_logstd))
        self._heads = (key, heads)
        return heads

    mean = property(lambda self: self._mean_logstd()[0])
    logstd = property(lambda self: self._mean_logstd()[1])

    def _registry(self):
        mean, logstd = self._mean_logstd()
        return Normal(mean, logstd=logstd, group_ndims=self.group_ndims,
                      is_reparameterized=self.is_reparameterized)

    def get_batch_shape(self):
        return torch.Size(tuple(self._h.shape[:-1]) + (self._D,))

    def get_value_shape(self):
        return torch.Size([])

    batch_shape = property(lambda self: self.get_batch_shape())
    value_shape = property(lambda self: self.get_value_shape())

    def sample(self, n_samples=None, eps=None):
        """``n_samples`` as in ``Normal.sample``; ``eps``: injected standard normals that broadcast
        to ``[n_samples, *batch_shape]`` (``Normal._sample(n, eps=...)``), else the Philox stream of
        ``zs.random``."""
        from . import random as zrandom
        if isinstance(n_samples, torch.Tensor):
            n_samples = int(n_samples.item())
        S = 1 if n_samples is None else int(n_samples)
        self._own = None
        if not self._fused:
            out = self._registry()._sample(S, eps=eps)
            return out.squeeze(0) if n_samples is None else out
        hpl = self._h_planes()
        Wp, bp = self._packed()
        keep = torch.is_grad_enabled() and any(
            t is not None and t.requires_grad for t in (self._h, Wp, bp))
        seed, it = zrandom.get_seed(), zrandom.next_counter()
        z, lq = _LinearNormalSample.apply(self._h, Wp, bp, eps, S, self._D,
                                          self.is_reparameterized, hpl, seed, it, keep)
        if n_samples is None:
            amax = getattr(z, "_zsb_amax", None)
            z, lq = z.squeeze(0), lq.squeeze(0)
            if amax is not None:
                _tag(z, amax)
        vs = _versions(z, self._h, *self._params)
        if all(v is not None for t, v in zip((z, self._h) + self._params, vs) if t is not None):
            # (inference tensors of torch.inference_mode() have no version: nothing is cached)
            self._own = (z, lq, vs)
        return z

    def log_prob(self, given):
        from . import ops
        own = self._own
        if (own is not None and self.group_ndims >= 1 and given is own[0]
                and own[2] == _versions(given, self._h, *self._params)):
            return ops.group_sum(own[1], self.group_ndims - 1)
        return self._registry().log_prob(given)

    def prob(self, given):
        return torch.exp(self.log_prob(given))


# ---- Sparse GP conditional (examples/gaussian_process/utils.py) on csrc/gp.cu ---------------------

GP_MAX_M = 256
GP_MAX_D = 64


class RBFKernel(object):
    """utils.py:10-49.  Owns ``k_raw_scale`` [n_covariates], a zeros leaf with ``requires_grad``
    (the reference's ``k_log_scale_<name>`` variable and initialiser); ``k_scale`` is its softplus,
    recomputed on each access so it follows optimiser steps.  ``device`` defaults to the current
    CUDA device.  ``gp_conditional`` runs this kernel on the fused path; ``__call__`` is the
    reference's broadcast formula in torch, the generic path and the cross-check."""

    def __init__(self, n_covariates, name='rbf_kernel', dtype=torch.float32, device=None):
        device = torch.device("cuda") if device is None else torch.device(device)
        self.name = name
        self.k_raw_scale = torch.zeros(int(n_covariates), dtype=dtype, device=device,
                                       requires_grad=True)

    @property
    def k_scale(self):
        return torch.nn.functional.softplus(self.k_raw_scale)

    def __call__(self, x, y):
        """K(x, y) [..., n_x, n_y] for x [..., n_x, n_covariates], y [..., n_y, n_covariates]."""
        if x.dim() < 2:
            raise ValueError("RBFKernel: rank(x) should be static and >=2")
        if x.dim() != y.dim():
            raise ValueError("RBFKernel: x and y should have the same rank")
        diff = x.unsqueeze(-2) - y.unsqueeze(-3)
        return torch.exp(-(diff * diff / self.k_scale).sum(-1) / 2)

    def Kdiag(self, x):
        """diag_part(self(x, x)): ones of x.shape[:-1] (rank 2 or 3, as in the reference)."""
        shape = (x.shape[0],) if x.dim() == 2 else (x.shape[0], x.shape[1])
        return torch.ones(shape, dtype=x.dtype, device=x.device)


class _GPCondMoments(torch.autograd.Function):
    """(mean [K, B], std [B]) of utils.py:69-87 with full_cov=False on zsb_gp_cond_fwd_f32, as
    functions of (z, s, Li, V); x is data.  When a gradient is needed the forward pass also keeps
    A = Kxz Li^T ([B, M] floats); the backward pass (zsb_gp_cond_bwd_f32) recomputes Kxz from x
    and z, and sums over B in a fixed order."""

    @staticmethod
    def forward(ctx, x, z, s, Li, V, need_grad):
        from ._lib import lib, ptr, stream
        B, d = int(x.shape[0]), int(x.shape[1])
        M, K = int(z.shape[0]), int(V.shape[0])
        xx, zz, ss, LL, VV = (t.detach().contiguous() for t in (x, z, s, Li, V))
        mean = torch.empty((K, B), dtype=torch.float32, device=x.device)
        std = torch.empty((B,), dtype=torch.float32, device=x.device)
        A = torch.empty((B, M), dtype=torch.float32, device=x.device) if need_grad else None
        if B > 0:
            lib.call("zsb_gp_cond_fwd_f32", ptr(xx), ptr(zz), ptr(ss), ptr(LL), ptr(VV),
                     ptr(mean), ptr(std), ptr(A), B, M, d, K, stream())
        if need_grad:
            ctx.save_for_backward(xx, zz, ss, LL, VV, A, std)
        ctx.set_materialize_grads(False)
        return mean, std

    @staticmethod
    @once_differentiable
    def backward(ctx, g_mean, g_std):
        from ._lib import lib, ptr, stream
        xx, zz, ss, LL, VV, A, std = ctx.saved_tensors
        B, d = int(xx.shape[0]), int(xx.shape[1])
        M, K = int(zz.shape[0]), int(VV.shape[0])
        if B == 0 or (g_mean is None and g_std is None):
            return None, torch.zeros_like(zz), torch.zeros_like(ss), torch.zeros_like(LL), \
                torch.zeros_like(VV), None
        dz, ds = torch.empty_like(zz), torch.empty_like(ss)          # the merge writes every entry
        dLi, dV = torch.empty_like(LL), torch.empty_like(VV)
        gm = None if g_mean is None else g_mean.to(torch.float32).contiguous()
        gs = None if g_std is None else g_std.to(torch.float32).contiguous()
        part = torch.empty((lib.load().zsb_gp_cond_parts(B, M, d, K), K * M + M * M + M * d + d),
                           dtype=torch.float32, device=xx.device)
        lib.call("zsb_gp_cond_bwd_f32", ptr(xx), ptr(zz), ptr(ss), ptr(LL), ptr(VV), ptr(A),
                 ptr(std), ptr(gm), ptr(gs), ptr(part), ptr(dz), ptr(ds), ptr(dLi), ptr(dV),
                 B, M, d, K, stream())
        return None, dz, ds, dLi, dV, None


def _gp_factors(z, fz, kernel, Kzz_chol):
    """Li = chol(Kzz)^-1 and V = fz Li^T in torch (utils.py:63-69), so autograd carries the
    gradients of Li and V back to Kzz_chol, fz, z and the kernel's scales.  Without ``Kzz_chol``
    the factor comes from ``cholesky_ex``: no host sync, and a Kzz that is not positive definite
    gives NaN moments rather than an error."""
    if Kzz_chol is None:
        Kzz_chol = torch.linalg.cholesky_ex(kernel(z, z))[0]
    eye = torch.eye(int(z.shape[0]), dtype=z.dtype, device=z.device)
    Li = torch.linalg.solve_triangular(Kzz_chol, eye, upper=False)
    return Li, torch.matmul(fz, Li.transpose(-1, -2))


class GPConditionalNormal(Normal):
    """The registry ``Normal(mean, std, group_ndims=1)`` of a fused ``gp_conditional``, whose
    moments are computed on first use (sampling, ``log_prob``, ``.mean`` / ``.std``) and then
    kept.  Building it launches nothing, so a conditional that is never read costs nothing.

    The moments use the values of z, fz, Kzz_chol and the kernel's scales at first use: an
    in-place optimiser step between building the conditional and reading it changes them.  When
    they were first computed without a gradient (under ``no_grad`` or ``inference_mode``) and
    are read again with grad mode on and an input that requires a gradient, they are computed
    again, so the later read carries the gradient."""

    def __init__(self, z, fz, x, kernel, Kzz_chol):
        self._args = (z, fz, x, kernel, Kzz_chol)
        self._moments = None
        self._moments_grad = False
        self._check_numerics = False
        Distribution.__init__(self, dtype=torch.float32, param_dtype=torch.float32,
                              is_continuous=True, is_reparameterized=True, group_ndims=1)

    def _compute(self):
        z, fz, x, kernel, Kzz_chol = self._args
        wants_grad = torch.is_grad_enabled() and any(
            t is not None and t.requires_grad for t in (z, fz, Kzz_chol, kernel.k_raw_scale))
        if self._moments is None or (wants_grad and not self._moments_grad):
            s = kernel.k_scale
            Li, V = _gp_factors(z, fz, kernel, Kzz_chol)
            need_grad = torch.is_grad_enabled() and any(t.requires_grad for t in (z, s, Li, V))
            mean, std = _GPCondMoments.apply(x, z, s, Li, V, need_grad)
            self._moments = (mean, std, torch.log(std))
            self._moments_grad = need_grad
        return self._moments

    _mean = property(lambda self: self._compute()[0])
    _std = property(lambda self: self._compute()[1])
    _logstd = property(lambda self: self._compute()[2])

    def _get_batch_shape(self):
        return torch.Size([int(self._args[1].shape[0]), int(self._args[2].shape[0])])


def _gp_fused_ok(z, fz, x, full_cov, kernel, Kzz_chol):
    """The one eligibility check of the fused path; anything else runs the reference's torch
    arithmetic."""
    if full_cov or not isinstance(kernel, RBFKernel):
        return False
    ts = [z, fz, x, kernel.k_raw_scale] + ([] if Kzz_chol is None else [Kzz_chol])
    if any(t.dtype != torch.float32 or not t.is_cuda or t.device != z.device for t in ts):
        return False
    if x.requires_grad or fz.dim() != 2:
        return False
    M, d = int(z.shape[0]), int(z.shape[1])
    return 1 <= M <= GP_MAX_M and 1 <= d <= GP_MAX_D


def gp_conditional(z, fz, x, full_cov, kernel, Kzz_chol=None):
    """GP conditional f(x) | f(z) = fz (utils.py:52-90): z [n_z, n_covariates], fz
    [n_particles, n_z] (a tensor or a ``StochasticTensor``, whose value is taken now), x
    [n_x, n_covariates].  Returns ``Normal(mean, std, group_ndims=1)`` [n_particles, n_x] for
    ``full_cov=False`` and ``MultivariateNormalCholesky`` for ``full_cov=True``.

    With an ``RBFKernel``, ``full_cov=False``, float32 CUDA inputs on one device, an ``x`` that
    needs no gradient, a rank-2 ``fz``, 1 <= n_z <= 256 and 1 <= n_covariates <= 64, the moments
    run on csrc/gp.cu and are computed lazily, on first use of the returned ``Normal``.  With
    A = Kxz Li^T and V = fz Li^T (Li = Kzz_chol^-1) they are mean = V A^T and
    var = 1 - rowsum(A^2): the reference's products re-associated, equal up to rounding.  var is
    not clamped, as in the reference.  Without ``Kzz_chol`` the Cholesky factor comes from
    ``torch.linalg.cholesky_ex``, so a Kzz that is not positive definite gives NaN, not an error.
    Everything else runs the reference's arithmetic in torch."""
    fz = _unwrap(fz)
    x = _unwrap(x)
    if z.dim() != 2:
        raise ValueError("RBFKernel: rank(x) should be static and >=2" if z.dim() < 2 else
                         "gp_conditional: z should have shape [n_z, n_covariates], got %s"
                         % (tuple(z.shape),))
    if x.dim() != z.dim():
        raise ValueError("RBFKernel: x and y should have the same rank")
    n_z, n_cov = int(z.shape[0]), int(z.shape[1])
    if int(x.shape[-1]) != n_cov:
        raise ValueError("gp_conditional: x has %d covariates, z has %d"
                         % (int(x.shape[-1]), n_cov))
    if fz.dim() < 1 or int(fz.shape[-1]) != n_z:
        raise ValueError("gp_conditional: fz should have shape [n_particles, %d], got %s"
                         % (n_z, tuple(fz.shape)))
    if isinstance(kernel, RBFKernel) and int(kernel.k_raw_scale.shape[0]) != n_cov:
        raise ValueError("gp_conditional: the kernel has %d covariates, z has %d"
                         % (int(kernel.k_raw_scale.shape[0]), n_cov))
    if Kzz_chol is not None and tuple(Kzz_chol.shape) != (n_z, n_z):
        raise ValueError("gp_conditional: Kzz_chol should have shape [%d, %d], got %s"
                         % (n_z, n_z, tuple(Kzz_chol.shape)))
    if _gp_fused_ok(z, fz, x, full_cov, kernel, Kzz_chol):
        return GPConditionalNormal(z, fz, x, kernel, Kzz_chol)
    return _gp_conditional_generic(z, fz, x, full_cov, kernel, Kzz_chol)


def _gp_conditional_generic(z, fz, x, full_cov, kernel, Kzz_chol=None):
    """utils.py:60-90 in torch ops, the Kzz_inv form included."""
    if Kzz_chol is None:
        Kzz_chol = torch.linalg.cholesky_ex(kernel(z, z))[0]
    eye = torch.eye(int(z.shape[0]), dtype=z.dtype, device=z.device)
    Kzz_chol_inv = torch.linalg.solve_triangular(Kzz_chol, eye, upper=False)
    Kzz_inv = torch.matmul(Kzz_chol_inv.t(), Kzz_chol_inv)
    Kxz = kernel(x, z)
    Kxziz = torch.matmul(Kxz, Kzz_inv)
    mean = torch.matmul(fz, Kxziz.transpose(-1, -2))
    if full_cov:
        cov = kernel(x, x) - torch.matmul(Kxziz, Kxz.t())
        tril = torch.linalg.cholesky_ex(cov)[0]
        tril = tril.unsqueeze(0).expand((int(fz.shape[0]),) + tuple(tril.shape))
        return MultivariateNormalCholesky(mean, tril)
    var = kernel.Kdiag(x) - (torch.matmul(Kxz, Kzz_chol_inv.transpose(-1, -2)) ** 2).sum(-1)
    return Normal(mean=mean, std=torch.sqrt(var), group_ndims=1)


# ---- 3x3 SAME convolutions (examples/variational_autoencoders/vae_conv.py) on csrc/conv.cu -------

CONV_MAX_C = 64


def _same_pads(big, small, stride):
    """TensorFlow "SAME" padding of a 3x3 window: (before, after) for an input of ``big`` rows
    giving ``small = ceil(big / stride)`` rows."""
    total = max((small - 1) * stride + 3 - big, 0)
    return total // 2, total - total // 2


def _conv_launch(x, gate, W, b, res, R, Hc, Wc, Cin, Cout, stride, transpose, relu, out_shape):
    from ._lib import lib, ptr, stream
    y = torch.empty(out_shape, dtype=torch.float32, device=x.device)
    lib.call("zsb_conv3x3_fwd_f32", ptr(x), ptr(gate), ptr(W), ptr(b), ptr(res), ptr(y), R, Hc,
             Wc, Cin, Cout, int(stride), int(transpose), int(bool(relu)), stream())
    return y


class _Conv3x3(torch.autograd.Function):
    """relu?(conv(x) + b + residual) on zsb_conv3x3_fwd_f32, as a function of (x, W, b, residual).
    ``geom`` = (transpose, stride, R, Hc, Wc, Hs, Ws, Cin, Cout): the convolution's big grid
    Hc x Wc and small grid Hs x Ws, as in include/zsb200.h.  Backward: the input gradient is the
    other mode on the output gradient, masked by y > 0 as it is loaded; dW and db come from
    zsb_conv3x3_wgrad_f32.  The masked gradient is written only when the residual needs it."""

    @staticmethod
    def forward(ctx, x, W, b, res, geom, relu):
        transpose, stride, R, Hc, Wc, Hs, Ws, Cin, Cout = geom
        out = (R, Hc, Wc, Cout) if transpose else (R, Hs, Ws, Cout)
        xx, WW = x.detach().contiguous(), W.detach().contiguous()
        bb = None if b is None else b.detach().contiguous()
        rr = None if res is None else res.detach().contiguous()
        y = _conv_launch(xx, None, WW, bb, rr, R, Hc, Wc, Cin, Cout, stride, transpose, relu, out)
        ctx.save_for_backward(xx, WW, y if relu else None)
        ctx.meta = (geom, relu, b is not None, res is not None)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        from ._lib import lib, ptr, stream
        xx, WW, y = ctx.saved_tensors
        geom, relu, has_b, has_r = ctx.meta
        transpose, stride, R, Hc, Wc, Hs, Ws, Cin, Cout = geom
        need = ctx.needs_input_grad
        g = gy.to(torch.float32).contiguous()
        gate = y if relu else None
        dres = None
        if has_r and need[3]:
            dres = torch.where(y > 0, g, torch.zeros((), dtype=g.dtype, device=g.device)) \
                if relu else g
            if relu:
                g, gate = dres, None
        dx = dW = db = None
        if need[0]:
            # the adjoint: conv2d's input gradient is the transpose on g, and the reverse
            dx = _conv_launch(g, gate, WW, None, None, R, Hc, Wc, Cout, Cin, stride,
                              not transpose, False, tuple(xx.shape))
        if need[1] or (has_b and need[2]):
            big, small = (g, xx) if transpose else (xx, g)
            Ca, Cb = (Cout, Cin) if transpose else (Cin, Cout)
            # the merge writes every entry; without dW only the bias sums run
            dW = torch.empty_like(WW) if need[1] else None
            db = torch.empty((Cout,), dtype=torch.float32, device=g.device) \
                if (has_b and need[2]) else None
            part = torch.empty((lib.load().zsb_conv3x3_wgrad_parts(R, Hc, Wc, stride), Ca * Cb),
                               dtype=torch.float32, device=g.device)
            lib.call("zsb_conv3x3_wgrad_f32", ptr(big), ptr(small), ptr(gate), int(transpose),
                     ptr(part), ptr(dW), ptr(db), R, Hc, Wc, Ca, Cb, stride, stream())
        return dx, dW, db, dres, None, None


def _conv_check(name, x, W, b, residual, stride, Cin, Cout, in_hw):
    if not isinstance(x, torch.Tensor) or not isinstance(W, torch.Tensor):
        raise ValueError("%s: x and W should be tensors" % name)
    ts = [x, W] + [t for t in (b, residual) if t is not None]
    for t in ts:
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda \
                or t.device != x.device:
            raise ValueError("%s: x, W, b and residual should be float32 tensors on one CUDA "
                             "device" % name)
    if x.dim() < 3:
        raise ValueError("%s: x should have shape [..., H, W, C], got %s"
                         % (name, tuple(x.shape)))
    if isinstance(stride, bool) or stride not in (1, 2):
        raise ValueError("%s: stride should be 1 or 2, got %r" % (name, stride))
    if W.dim() != 4 or tuple(W.shape[:2]) != (3, 3):
        raise ValueError("%s: W should be a 3x3 kernel [3, 3, ., .], got %s"
                         % (name, tuple(W.shape)))
    if not (1 <= Cin <= CONV_MAX_C and 1 <= Cout <= CONV_MAX_C):
        raise ValueError("%s: channels should be in [1, %d], got Cin %d, Cout %d"
                         % (name, CONV_MAX_C, Cin, Cout))
    if int(x.shape[-1]) != Cin:
        raise ValueError("%s: x has %d channels, W expects %d" % (name, int(x.shape[-1]), Cin))
    if min(in_hw) < 1:
        raise ValueError("%s: H and W should be >= 1, got %s" % (name, tuple(in_hw)))
    if b is not None and tuple(b.shape) != (Cout,):
        raise ValueError("%s: b should have shape [%d], got %s" % (name, Cout, tuple(b.shape)))


def _conv_apply(name, x, W, b, residual, geom, relu, lead, out_hw):
    transpose, stride, R, Hc, Wc, Hs, Ws, Cin, Cout = geom
    out_shape = tuple(lead) + tuple(out_hw) + (Cout,)
    if residual is not None and tuple(residual.shape) != out_shape:
        raise ValueError("%s: residual should have the output's shape %s, got %s"
                         % (name, out_shape, tuple(residual.shape)))
    if max(R * Hc * Wc * (Cout if transpose else Cin),
           R * Hs * Ws * (Cin if transpose else Cout)) >= 2 ** 31:
        raise ValueError("%s: R*H*W*C should be below 2^31" % name)
    if R == 0:
        return torch.empty(out_shape, dtype=torch.float32, device=x.device)
    x4 = x.reshape((R,) + tuple(x.shape[-3:]))
    r4 = None if residual is None else residual.reshape((R,) + tuple(out_hw) + (Cout,))
    ts = [t for t in (x, W, b, residual) if t is not None]
    if torch.is_grad_enabled() and any(t.requires_grad for t in ts):
        y = _Conv3x3.apply(x4, W, b, r4, geom, bool(relu))
    else:
        y = _conv_launch(x4.contiguous(), None, W.contiguous(),
                         None if b is None else b.contiguous(),
                         None if r4 is None else r4.contiguous(), R, Hc, Wc, Cin, Cout, stride,
                         transpose, relu, (R,) + tuple(out_hw) + (Cout,))
    return y.reshape(out_shape)


def conv2d(x, W, b=None, stride=1, relu=False, residual=None):
    """``relu?(tf.layers.conv2d(x, Cout, 3, strides=stride, padding="same") + residual)``
    (vae_conv.py:39-53, 80) on csrc/conv.cu, in FP32 FFMA.

    x [..., H, W, Cin] is NHWC, any leading shape flattened to R images; W [3, 3, Cin, Cout] is
    the ``tf.layers.conv2d`` kernel layout; b [Cout]; ``residual`` has the output's shape and is
    added before the ReLU.  The output is [..., Ho, Wo, Cout] with Ho = ceil(H / stride) and

        y[n, i, j, co] = b[co] + sum_{kh, kw, ci} x[n, s i + kh - pt, s j + kw - pl, ci] W[kh, kw, ci, co]

    where out-of-range x counts as 0 and the pads are TensorFlow's SAME rule:
    pad_total = max((Ho - 1) s + 3 - H, 0), pt = pad_total // 2 (pl likewise).  So stride 1 pads
    1 before and 1 after; stride 2 pads 0 before and 1 after an even H, and 1 and 1 an odd H --
    unlike torch's symmetric ``padding=1``.

    Differentiable w.r.t. x, W, b and residual; under ``inference_mode`` nothing is kept.  The
    gradients are deterministic: two identical calls give identical bits.  Supported: float32
    CUDA tensors on one device, stride 1 or 2, 1 <= Cin, Cout <= 64, H, W >= 1 and
    R*H*W*C < 2^31; anything else raises ValueError before any launch."""
    x = _unwrap(x)
    Cin = int(W.shape[2]) if isinstance(W, torch.Tensor) and W.dim() == 4 else 0
    Cout = int(W.shape[3]) if isinstance(W, torch.Tensor) and W.dim() == 4 else 0
    hw = tuple(int(v) for v in x.shape[-3:-1]) if isinstance(x, torch.Tensor) \
        and x.dim() >= 3 else (0, 0)
    _conv_check("conv2d", x, W, b, residual, stride, Cin, Cout, hw)
    H, Wd = hw
    lead = tuple(x.shape[:-3])
    R = 1
    for d in lead:
        R *= int(d)
    Hs, Ws = -(-H // stride), -(-Wd // stride)
    geom = (False, int(stride), R, H, Wd, Hs, Ws, Cin, Cout)
    return _conv_apply("conv2d", x, W, b, residual, geom, relu, lead, (Hs, Ws))


def conv2d_transpose(x, W, out_shape, stride=1, b=None, relu=False, residual=None):
    """``relu?(conv2d_transpose(x, out_shape, (3, 3), stride) + residual)`` of
    examples/utils/utils.py:74-113 (``tf.nn.conv2d_transpose(..., padding="SAME")`` plus
    ``bias_add``; vae_conv.py:20-36, 63-68) on csrc/conv.cu, in FP32 FFMA.

    x [..., Hi, Wi, Cin] is NHWC; W [3, 3, Cout, Cin] is that helper's ``weights`` layout;
    ``out_shape`` = (Ho, Wo, Cout) with ceil(Ho / stride) == Hi and ceil(Wo / stride) == Wi (TF
    rejects anything else too); b [Cout]; ``residual`` has the output's shape, added before the
    ReLU.  The map is the adjoint of ``conv2d`` from [Ho, Wo, Cout] to [Hi, Wi, Cin] with the
    same W and the SAME pads of (Ho -> Hi):

        y[n, h, w, co] = b[co] + sum x[n, i, j, ci] W[kh, kw, co, ci]  over h = s i + kh - pt,
                                                                      w = s j + kw - pl

    i.e. ``F.conv_transpose2d(..., padding=0)`` cropped by pt rows and pl columns at the start and
    cut to Ho x Wo.  At stride 2 the kernel enumerates output pixels by parity, and a warp
    skips the taps none of its pixels needs.  Gradients, determinism, inference mode and the supported range
    are those of ``conv2d``."""
    x = _unwrap(x)
    if not isinstance(W, torch.Tensor) or W.dim() != 4:
        raise ValueError("conv2d_transpose: W should be a 3x3 kernel [3, 3, Cout, Cin]")
    Cout, Cin = int(W.shape[2]), int(W.shape[3])
    try:
        Ho, Wo, Co = (int(v) for v in out_shape)
    except (TypeError, ValueError):
        raise ValueError("conv2d_transpose: out_shape should be (Ho, Wo, Cout), got %r"
                         % (out_shape,))
    hw = tuple(int(v) for v in x.shape[-3:-1]) if isinstance(x, torch.Tensor) \
        and x.dim() >= 3 else (0, 0)
    _conv_check("conv2d_transpose", x, W, b, residual, stride, Cin, Cout, hw)
    if Co != Cout:
        raise ValueError("conv2d_transpose: out_shape has %d channels, W has %d" % (Co, Cout))
    Hi, Wi = hw
    if Ho < 1 or Wo < 1 or -(-Ho // stride) != Hi or -(-Wo // stride) != Wi:
        raise ValueError("conv2d_transpose: out_shape %s does not give the input's %dx%d at "
                         "stride %d (ceil(Ho / stride) must equal Hi)" % ((Ho, Wo, Co), Hi, Wi,
                                                                          stride))
    lead = tuple(x.shape[:-3])
    R = 1
    for d in lead:
        R *= int(d)
    geom = (True, int(stride), R, Ho, Wo, Hi, Wi, Cin, Cout)
    return _conv_apply("conv2d_transpose", x, W, b, residual, geom, relu, lead, (Ho, Wo))


# ---------------------------------------------------------------------------
# k x k convolutions on the tensor-core products (csrc/conv_tc.cu): the GAN examples
# ---------------------------------------------------------------------------
CONV_TC_MAX_K = 7


class _ConvGeom(object):
    """A k x k convolution from the big grid Hb x Wb (its input) to the small grid Hs x Ws (its
    output) over N images, with TF's pads before (pt, pl); the transposed convolution runs the
    same geometry the other way.  Cin / Cout are the channels of the layer's input / output."""
    __slots__ = ("N", "Hb", "Wb", "Hs", "Ws", "k", "s", "pt", "pl", "Cin", "Cout")

    def __init__(self, N, Hb, Wb, Hs, Ws, k, s, pt, pl, Cin, Cout):
        self.N, self.Hb, self.Wb, self.Hs, self.Ws = N, Hb, Wb, Hs, Ws
        self.k, self.s, self.pt, self.pl, self.Cin, self.Cout = k, s, pt, pl, Cin, Cout

    def args(self, C):
        """(N, Hb, Wb, C, Hs, Ws, k, s, pt, pl) of a conv_tc.cu pass over C channels."""
        return (self.N, self.Hb, self.Wb, C, self.Hs, self.Ws, self.k, self.s, self.pt, self.pl)


def _tf_pad_before(big, small, k, s, padding):
    """TF's pad before the first row: SAME pads pad_total = max((small - 1) s + k - big, 0) rows,
    pad_total // 2 of them before (asymmetric for even k and at stride 2); VALID pads nothing."""
    return max((small - 1) * s + k - big, 0) // 2 if padding == "SAME" else 0


def _conv_tc_geom(name, x, W, stride, padding, transpose, out_hw=None, empty_batch=False):
    """Validate the arguments of a tensor-core convolution before any launch and return its
    _ConvGeom and the leading shape of x.  ``out_hw`` (transposed only): the output's (Ho, Wo), as
    ``tf.nn.conv2d_transpose``'s ``output_shape`` gives it, instead of the size ``tf.layers``
    picks; it must satisfy ceil(Ho / s) == Hi (SAME) or ceil((Ho - k + 1) / s) == Hi (VALID), as
    TF requires.  ``empty_batch``: zero images (a leading dimension of 0) are valid, N = 0."""
    if not isinstance(x, torch.Tensor) or not isinstance(W, torch.Tensor):
        raise ValueError("%s: x and W should be tensors" % name)
    if x.dtype != torch.float32 or W.dtype != torch.float32:
        raise ValueError("%s: x and W should be float32, got %s and %s" % (name, x.dtype, W.dtype))
    if not x.is_cuda or x.device != W.device:
        raise ValueError("%s: x and W should be on one CUDA device, got %s and %s"
                         % (name, x.device, W.device))
    if x.dim() < 3:
        raise ValueError("%s: x should be NHWC [..., H, W, C], got %s" % (name, tuple(x.shape)))
    if W.dim() != 4 or int(W.shape[0]) != int(W.shape[1]) or \
            not 1 <= int(W.shape[0]) <= CONV_TC_MAX_K:
        raise ValueError("%s: W should be a square k x k kernel [k, k, ., .] with 1 <= k <= %d, "
                         "got %s" % (name, CONV_TC_MAX_K, tuple(W.shape)))
    if isinstance(stride, bool) or stride not in (1, 2):
        raise ValueError("%s: stride should be 1 or 2, got %r" % (name, stride))
    if not isinstance(padding, str) or padding.upper() not in ("SAME", "VALID"):
        raise ValueError("%s: padding should be 'SAME' or 'VALID', got %r" % (name, padding))
    padding = padding.upper()
    k, s = int(W.shape[0]), int(stride)
    # tf.layers kernels: conv2d [k, k, Cin, Cout], conv2d_transpose [k, k, Cout, Cin]
    Cin, Cout = (int(W.shape[3]), int(W.shape[2])) if transpose else \
        (int(W.shape[2]), int(W.shape[3]))
    if int(x.shape[-1]) != Cin:
        raise ValueError("%s: x has %d channels, W expects %d" % (name, int(x.shape[-1]), Cin))
    empty_lead = empty_batch and min(int(d) for d in x.shape[-3:]) > 0
    if (x.numel() == 0 and not empty_lead) or W.numel() == 0:
        raise ValueError("%s: empty shapes are not supported: x %s, W %s"
                         % (name, tuple(x.shape), tuple(W.shape)))
    lead = tuple(int(d) for d in x.shape[:-3])
    N = 1
    for d in lead:
        N *= d
    H, Wd = int(x.shape[-3]), int(x.shape[-2])
    if transpose:
        Hs, Ws = H, Wd
        if out_hw is None:
            grow = 0 if padding == "SAME" else max(k - s, 0)
            Hb, Wb = Hs * s + grow, Ws * s + grow
        else:
            Hb, Wb = out_hw
            for big, small in ((Hb, Hs), (Wb, Ws)):
                n = big if padding == "SAME" else big - k + 1
                if n < 1 or -(-n // s) != small:
                    raise ValueError(
                        "%s: an output of %dx%d does not give the input's %dx%d at stride %d, %s "
                        "(ceil(%s / stride) must equal Hi)" % (
                            name, Hb, Wb, Hs, Ws, s, padding,
                            "Ho" if padding == "SAME" else "(Ho - k + 1)"))
    else:
        Hb, Wb = H, Wd
        if padding == "SAME":
            Hs, Ws = -(-Hb // s), -(-Wb // s)
        else:
            Hs, Ws = -(-(Hb - k + 1) // s), -(-(Wb - k + 1) // s)
        if Hs < 1 or Ws < 1:
            raise ValueError("%s: a %dx%d input is smaller than the %dx%d kernel (VALID)"
                             % (name, Hb, Wb, k, k))
    pt, pl = _tf_pad_before(Hb, Hs, k, s, padding), _tf_pad_before(Wb, Ws, k, s, padding)
    kk = k * k
    big, small = N * Hb * Wb, N * Hs * Ws
    C_big, C_small = (Cout, Cin) if transpose else (Cin, Cout)
    if max(big * C_big, small * C_small, small * kk * C_big,
           small * (-(-(kk * C_big) // 64) * 64), big * (-(-C_big // 64) * 64)) >= 2 ** 31:
        raise ValueError("%s: too large: every tensor and operand of the layer must have fewer "
                         "than 2^31 entries (N*H*W*k*k*C)" % name)
    return _ConvGeom(N, Hb, Wb, Hs, Ws, k, s, pt, pl, Cin, Cout), lead


def _gather_planes(x4, g, C, tag=None):
    """The fp16 operand planes of the im2col matrix [N Hs Ws, k k C] of x4 [N, Hb, Wb, C]
    (zsb_conv_gather_split_f32), at the scale of ``tag`` (a scale slot holding max |x4|) when
    given, else of one max pass."""
    from ._lib import lib, ptr, stream
    R, K = g.N * g.Hs * g.Ws, g.k * g.k * C
    planes = torch.empty((2, R, lib.load().zsb_linear_tc_kpad(K)), dtype=torch.float16,
                         device=x4.device)
    scale = tag if tag is not None else torch.zeros(4, dtype=torch.float32, device=x4.device)
    lib.call("zsb_conv_gather_split_f32", ptr(x4), *g.args(C), ptr(planes), ptr(scale),
             int(tag is not None), stream())
    return _Planes(planes, scale, R, K)


def _take_tag(x):
    """The max |.| scale slot a producing fused layer left on x (consumed: its word 2 is cleared
    by the split that reads it), or None."""
    tag = getattr(x, "_zsb_amax", None)
    if tag is not None:
        try:
            del x._zsb_amax
        except (AttributeError, RuntimeError):
            pass
    return tag


# the activation codes of zsb_conv_col2im_f32 and zsb_conv_act_grad_f32
_ACT_NONE, _ACT_RELU, _ACT_SIGMOID = 0, 1, 2


def _col2im(epi, cols, g, C, out=None, bias=None, gamma=None, beta=None, mm=None, mv=None,
            eps=0.0, act=_ACT_NONE, stats=None, pre=None, part=None, amax=None, residual=None):
    from ._lib import lib, ptr, stream
    lib.call("zsb_conv_col2im_f32", epi, ptr(cols), *g.args(C), ptr(bias), ptr(residual),
             ptr(gamma), ptr(beta), ptr(mm), ptr(mv), float(eps), act, ptr(stats),
             ptr(pre), ptr(part), ptr(out), ptr(amax), stream())


def _ones_like_gamma(gamma, Cout, dev):
    return gamma.detach().contiguous() if gamma is not None else \
        torch.ones(Cout, dtype=torch.float32, device=dev)


class _BNConv2d(torch.autograd.Function):
    """relu?(BN(conv(x, W)) * gamma + beta): _conv_planes, then _bn_forward with TF's
    fused-batch-norm update over R = N Ho Wo rows, J = Cout features and K = k k Cin.  Backward:
    _bn_backward gives d beta, d gamma and the planes of G = d/d(pre-activation), then
    _conv_grads."""

    @staticmethod
    def forward(ctx, x, W, gamma, beta, stats_bufs, g, training, relu, rate, eps, keep_pre):
        ctx.hpl, ctx.wpl = _conv_planes(x, W, g)
        y, amax = _bn_forward(ctx, ctx.hpl, ctx.wpl, g.Cout,
                              _ones_like_gamma(gamma, g.Cout, W.device), beta, stats_bufs,
                              training, relu, rate, eps, True, keep_pre)
        ctx.meta = (g, tuple(x.shape))
        return _tag(y.reshape(tuple(x.shape[:-3]) + (g.Hs, g.Ws, g.Cout)), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        g, x_shape = ctx.meta
        need = ctx.needs_input_grad
        dgamma, dbeta, gpl = _bn_backward(ctx, gy, need[2], need[3])
        dx, dW = _conv_grads(ctx, gpl, g, need[0], need[1], x_shape)
        return dx, dW, dgamma, dbeta, None, None, None, None, None, None, None


class _ShapeOnly(object):
    """Stands for a weight matrix whose operand planes the caller already has: _tc_grad_input
    reads only its shape and device."""
    __slots__ = ("shape", "device")

    def __init__(self, shape, device):
        self.shape, self.device = shape, device


def _conv_planes(x, W, g):
    """The planes of a convolution's product over R = N Ho Wo rows, J = Cout features and K = k k
    Cin: the gather-split of x (at its max |.| tag when it has one) and the planes of
    W^T [Cout, k k Cin]."""
    tag = _take_tag(x)
    x4 = x.detach().reshape(g.N, g.Hb, g.Wb, g.Cin).contiguous()
    hpl = _gather_planes(x4, g, g.Cin, tag)
    return hpl, _tc_split(W.detach().reshape(hpl.K, g.Cout).t())


def _conv_grads(ctx, gpl, g, need_x, need_W, x_shape):
    """dx and dW of a convolution from the planes gpl of G = d/d(its pre-activation)
    [N Ho Wo, Cout]: dx is the col2im-sum of G W (the MN-major input-gradient product with the
    forward planes of W^T) and dW the weight-gradient product of G and the saved gather planes."""
    R, K = g.N * g.Hs * g.Ws, g.k * g.k * g.Cin
    dev = gpl.planes.device
    dx = dW = None
    if need_x:
        wp, ws = ctx.wpl
        dcols, _ = _tc_grad_input(gpl, _ShapeOnly((g.Cout, K), dev), R, wp, ws)
        dx = torch.empty((g.N, g.Hb, g.Wb, g.Cin), dtype=torch.float32, device=dev)
        amax = torch.zeros(4, dtype=torch.float32, device=dev)
        _col2im(0, dcols, g, g.Cin, out=dx, amax=amax)
        del dcols
        dx = _tag(dx.reshape(x_shape), amax)
    if need_W:
        dW = _tc_grad_weight(gpl, ctx.hpl, R).t().reshape(g.k, g.k, g.Cin, g.Cout)
    ctx.hpl = ctx.wpl = None
    return dx, dW


def _conv_t_product(x, W, g):
    """cols [N Hs Ws, k k Cout] = x W'^T with W' = W.reshape(k k Cout, Cin) on the epi-0 product,
    from the planes of x (scaled by its max |.| tag when it has one); returns cols, the planes of
    x and of W'.  The planes are not cached on x: only the layer's backward keeps them."""
    kk = g.k * g.k
    x2 = x.detach().reshape(-1, g.Cin)
    tag = _take_tag(x)
    hpl = _tc_split_dual(x2, amax=None if g.Cin % 2 else tag)
    wp, ws = _tc_split(W.detach().reshape(kk * g.Cout, g.Cin))
    cols = _tc_linear(0, wp, ws, hpl.planes, hpl.scale, None, None, None, hpl.rows,
                      kk * g.Cout, g.Cin)
    return cols, hpl, (wp, ws)


def _conv_t_grads(ctx, gp, gscale, g, need_x, need_W, x_shape):
    """dx and dW of a transposed convolution from gp = d/d(its output) [N Hb Wb, Cout] in fp32
    with its max |.| in gscale: the gather-split of gp on the small grid, then the input-gradient
    product with the forward planes of W' and the weight-gradient product with the planes of x."""
    R = g.N * g.Hs * g.Ws
    gpl = _gather_planes(gp.reshape(g.N, g.Hb, g.Wb, g.Cout), g, g.Cout, gscale)
    dx = dW = None
    if need_x:
        wp, ws = ctx.wpl
        dx2, amax = _tc_grad_input(gpl, _ShapeOnly((gpl.K, g.Cin), gp.device), R, wp, ws)
        dx = _tag(dx2.reshape(x_shape), amax)
    if need_W:
        dW = _tc_grad_weight(gpl, ctx.hpl, R).reshape(g.k, g.k, g.Cout, g.Cin)
    ctx.hpl = ctx.wpl = None
    return dx, dW


class _BNConv2dT(torch.autograd.Function):
    """relu?(BN(conv_transpose(x, W)) * gamma + beta): the epi-0 product x W'^T gives the columns
    [N Hi Wi, k k Cout]; their col2im-sum onto the output grid runs the batch-norm epilogue
    (training: pre-activation and moment partials, then zsb_bn_finish_fused_f32; evaluation:
    the affine step in place).  Backward: _bn_backward gives d beta, d gamma and da in fp32, then
    _conv_t_grads."""

    @staticmethod
    def forward(ctx, x, W, gamma, beta, stats_bufs, g, training, relu, rate, eps, keep_pre):
        from ._lib import lib, ptr, stream
        moving_mean, moving_variance = stats_bufs
        dev = W.device
        J, Rb = g.Cout, g.N * g.Hb * g.Wb
        cols, hpl, wpl = _conv_t_product(x, W, g)
        gm = _ones_like_gamma(gamma, J, dev)
        b = beta.detach().contiguous()
        stats, y, a, part, amax = _bn_buffers(Rb, J, dev, training, keep_pre)
        if training:
            _col2im(2, cols, g, J, pre=a, part=part)
            del cols
            lib.call("zsb_bn_finish_fused_f32", ptr(a), ptr(part), Rb, J, ptr(gm), ptr(b),
                     ptr(moving_mean), ptr(moving_variance), rate, eps, ptr(stats), ptr(y),
                     int(relu), ptr(amax), stream())
        else:
            _col2im(3, cols, g, J, out=y, gamma=gm, beta=b, mm=moving_mean, mv=moving_variance,
                    eps=eps, act=_ACT_RELU if relu else _ACT_NONE, stats=stats, pre=a, amax=amax)
            del cols
        _bn_save(ctx, training, relu, gm, y, a, stats)
        ctx.hpl, ctx.wpl = hpl, wpl
        ctx.meta = (g, tuple(x.shape))
        return _tag(y.reshape(tuple(x.shape[:-3]) + (g.Hb, g.Wb, J)), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        g, x_shape = ctx.meta
        need = ctx.needs_input_grad
        dgamma, dbeta, (da, scale) = _bn_backward(ctx, gy, need[2], need[3], planes=False)
        dx, dW = _conv_t_grads(ctx, da, scale, g, need[0], need[1], x_shape)
        return dx, dW, dgamma, dbeta, None, None, None, None, None, None, None


def _bn_conv_apply(fn, name, x, W, gamma, beta, moving_mean, moving_variance, training, stride,
                   padding, relu, momentum, epsilon, transpose):
    x = _unwrap(x)
    g, _ = _conv_tc_geom(name, x, W, stride, padding, transpose)
    _bn_check(name, g.Cout, W.device, gamma, beta, moving_mean, moving_variance)
    keep_pre = (not training) and torch.is_grad_enabled() and gamma is not None and \
        gamma.requires_grad
    return fn.apply(x, W, gamma, beta, (moving_mean, moving_variance), g, bool(training),
                    bool(relu), float(1.0 - momentum), float(epsilon), bool(keep_pre))


def bn_conv2d(x, W, gamma, beta, moving_mean, moving_variance, training, stride=1,
              padding="SAME", relu=True, momentum=0.99, epsilon=1e-3):
    """``relu?(BN(tf.layers.conv2d(x, Cout, k, stride, padding, use_bias=False)))``, the conv ->
    batch norm -> ReLU layer of examples/generative_adversarial_nets (dcgan.py, wasserstein_gan.py)
    on the tensor-core products at fp32 accuracy.

    x [..., H, W, Cin] is NHWC, any leading shape flattened to images; W [k, k, Cin, Cout] is the
    ``tf.layers.conv2d`` kernel, 1 <= k <= 7; gamma (or None) and beta [Cout].  The output is
    [..., Ho, Wo, Cout] with Ho = ceil(H / s) (SAME) or ceil((H - k + 1) / s) (VALID), and

        a[n, i, j, co] = sum_{kh, kw, ci} x[n, s i + kh - pt, s j + kw - pl, ci] W[kh, kw, ci, co]

    where out-of-range x counts as 0.  SAME pads by TF's rule, pad_total = max((Ho - 1) s + k - H,
    0) and pt = pad_total // 2 (pl likewise): asymmetric for even k and at stride 2.  VALID pads
    nothing.

    Batch norm is ``tf.layers.batch_normalization(training=training)`` with its defaults
    (``center=True``, ``scale=True``: ``y = xhat * gamma + beta``, ``xhat = (a - mean) *
    rsqrt(var + epsilon)``) on TF 1.x's FUSED path, which ``tf.layers`` takes for 4-D inputs
    (``BatchNormalization._fused_batch_norm`` with ``_bessels_correction_test_only = True``, its
    default).  This differs from ``bn_linear``, which keeps the non-fused rule of 2-D inputs:

    * ``training``: ``mean`` and the population variance ``var`` over all N*H*W pixels normalise
      the output, but the moving variance moves towards the Bessel-corrected ``var * R / (R - 1)``
      (``R = N*H*W``); the moving mean towards ``mean``.  Both in place, as ``m -= (m - batch) *
      (1 - momentum)``, with no zero-debiasing.  At ``R = 1`` the moving variance moves towards
      ``var = 0``: the factor is 1 there, as in the CPU kernel of TF's ``fused_batch_norm``.
    * otherwise the moving statistics normalise and stay unchanged.

    ``gamma=None`` is ``scale=False`` (wasserstein_gan.py) and gives the bits of ``gamma = ones``.
    ``moving_mean`` / ``moving_variance`` are contiguous float32 [Cout] and get no gradient.

    Differentiable w.r.t. x, W, gamma and beta; under ``inference_mode`` nothing is kept.  The
    batch moments and every gradient are reduced in a fixed order with no float atomics, so two
    identical calls give identical bits.  The output carries the max |.| that a following fused
    layer uses for its operand split.  Supported: float32 CUDA tensors on one device, stride 1 or
    2, padding "SAME" or "VALID", no empty shapes, fewer than 2^31 entries in every tensor and
    operand; anything else raises ValueError before any launch."""
    return _bn_conv_apply(_BNConv2d, "bn_conv2d", x, W, gamma, beta, moving_mean, moving_variance,
                          training, stride, padding, relu, momentum, epsilon, False)


def bn_conv2d_transpose(x, W, gamma, beta, moving_mean, moving_variance, training, stride=1,
                        padding="SAME", relu=True, momentum=0.99, epsilon=1e-3):
    """``relu?(BN(tf.layers.conv2d_transpose(x, Cout, k, stride, padding, use_bias=False)))``, the
    generators' deconv -> batch norm -> ReLU layer of examples/generative_adversarial_nets, on the
    tensor-core products at fp32 accuracy.

    x [..., Hi, Wi, Cin] is NHWC; W [k, k, Cout, Cin] is the ``tf.layers.conv2d_transpose``
    kernel, 1 <= k <= 7.  The output is [..., Ho, Wo, Cout] as ``tf.layers`` sizes it: Ho = Hi s
    (SAME) or Hi s + max(k - s, 0) (VALID).  The map is the adjoint of ``bn_conv2d``'s
    convolution from [Ho, Wo, Cout] to [Hi, Wi, Cin] with the same W and pads:

        a[n, h, w, co] = sum x[n, i, j, ci] W[kh, kw, co, ci]  over h = s i + kh - pt, w = s j + kw - pl

    computed as the product x W'^T (W' = W.reshape(k k Cout, Cin)) followed by a gather of its
    columns onto the output grid, so no structural zero is multiplied.  Batch norm, ``gamma=None``
    and the moving statistics are those of ``bn_conv2d`` (TF's fused rule for 4-D inputs, not
    ``bn_linear``'s).  Gradients, determinism, inference mode, the amax tag and the supported
    range are those of ``bn_conv2d``."""
    return _bn_conv_apply(_BNConv2dT, "bn_conv2d_transpose", x, W, gamma, beta, moving_mean,
                          moving_variance, training, stride, padding, relu, momentum, epsilon,
                          True)


def sigmoid_conv2d_transpose(x, W, b=None, stride=1, padding="SAME"):
    """``tf.layers.conv2d_transpose(x, Cout, k, stride, padding, activation=tf.sigmoid)`` with its
    bias b [Cout] (None: no bias), the generators' output layers of
    examples/generative_adversarial_nets.  Geometry and W as in ``bn_conv2d_transpose``.
    Differentiable w.r.t. x, W and b; the bias gradient is a column sum merged in a fixed order.
    Determinism, inference mode, the amax tag and the supported range are those of
    ``bn_conv2d``, and both channel counts must be below 2^20."""
    x = _unwrap(x)
    g, lead = _conv_tc_geom("sigmoid_conv2d_transpose", x, W, stride, padding, True)
    return _conv_tc_apply(_Conv2dTransposeTC, "sigmoid_conv2d_transpose", x, W, b, None, g, lead,
                          _ACT_SIGMOID, (g.Hb, g.Wb))


# Biased layers act(conv(x) + b + residual) on the same products: the convolutions of vae_conv.py
# at any k <= 7, channel count and padding, and the GAN generators' sigmoid output layers
CONV_TC_MAX_C = 2 ** 20


def _act_grad(gy, y, R, J, act, need_db):
    """gp = d/d(pre-activation) [R, J] of act(a) with output y (gy itself without an activation,
    copied), db [J] (None unless ``need_db``) and the scale slot holding max |gp|
    (zsb_conv_act_grad_f32)."""
    from ._lib import lib, ptr, stream
    dev = gy.device
    g = gy.reshape(R, J).to(torch.float32).contiguous()
    gp = torch.empty((R, J), dtype=torch.float32, device=dev)
    part = torch.empty(-(-R // 128) * J, dtype=torch.float32, device=dev)
    db = torch.empty(J, dtype=torch.float32, device=dev) if need_db else None
    scale = torch.zeros(4, dtype=torch.float32, device=dev)
    lib.call("zsb_conv_act_grad_f32", ptr(g), ptr(y if act else None), R, J, act, ptr(gp),
             ptr(part), ptr(db), ptr(scale), stream())
    return gp, db, scale


class _Conv2dTC(torch.autograd.Function):
    """act(conv(x, W) + b + residual), act none or ReLU: _conv_planes, then the product over
    R = N Ho Wo rows, J = Cout features and K = k k Cin with the bias + ReLU epilogue (epi 0), or
    with the residual added before the ReLU (epi 16).  Backward: gp = d/d(pre-activation) and db
    from _act_grad (gp is the residual's gradient too), the plain split of gp at the max |gp| that
    pass left, then _conv_grads."""

    @staticmethod
    def forward(ctx, x, W, b, res, g, act):
        hpl, (wp, ws) = _conv_planes(x, W, g)
        R, K, J = hpl.rows, hpl.K, g.Cout
        bias = None if b is None else b.detach().contiguous()
        r2 = None if res is None else res.detach().reshape(R, J).contiguous()
        amax = torch.zeros(4, dtype=torch.float32, device=W.device)
        y = _tc_linear(0 if r2 is None else 16, wp, ws, hpl.planes, hpl.scale, bias, r2, None, R,
                       J, K, act == _ACT_RELU, amax=amax)
        ctx.save_for_backward(y if act else None)
        ctx.hpl, ctx.wpl = hpl, (wp, ws)
        ctx.meta = (g, tuple(x.shape), act)
        return _tag(y.reshape(tuple(x.shape[:-3]) + (g.Hs, g.Ws, J)), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        y, = ctx.saved_tensors
        g, x_shape, act = ctx.meta
        need = ctx.needs_input_grad
        gp, db, scale = _act_grad(gy, y, g.N * g.Hs * g.Ws, g.Cout, act, need[2])
        dx = dW = None
        if need[0] or need[1]:
            dx, dW = _conv_grads(ctx, _tc_split_dual(gp, amax=scale), g, need[0], need[1],
                                 x_shape)
        ctx.hpl = ctx.wpl = None
        dres = gp.reshape(gy.shape) if need[3] else None
        return dx, dW, db, dres, None, None


class _Conv2dTransposeTC(torch.autograd.Function):
    """act(conv_transpose(x, W) + b + residual): the epi-0 product x W'^T gives the columns
    [N Hi Wi, k k Cout]; their col2im-sum onto the output grid adds the bias and the residual and
    applies the activation (epi 1).  Backward: gp and db from _act_grad (gp is the residual's
    gradient too), then _conv_t_grads at the max |gp| that pass left."""

    @staticmethod
    def forward(ctx, x, W, b, res, g, act):
        J, Rb = g.Cout, g.N * g.Hb * g.Wb
        dev = W.device
        cols, hpl, wpl = _conv_t_product(x, W, g)
        bias = None if b is None else b.detach().contiguous()
        r2 = None if res is None else res.detach().reshape(Rb, J).contiguous()
        y = torch.empty((Rb, J), dtype=torch.float32, device=dev)
        amax = torch.zeros(4, dtype=torch.float32, device=dev)
        _col2im(1, cols, g, J, out=y, bias=bias, residual=r2, act=act, amax=amax)
        del cols
        ctx.save_for_backward(y if act else None)
        ctx.hpl, ctx.wpl = hpl, wpl
        ctx.meta = (g, tuple(x.shape), act)
        return _tag(y.reshape(tuple(x.shape[:-3]) + (g.Hb, g.Wb, J)), amax)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        y, = ctx.saved_tensors
        g, x_shape, act = ctx.meta
        need = ctx.needs_input_grad
        gp, db, scale = _act_grad(gy, y, g.N * g.Hb * g.Wb, g.Cout, act, need[2])
        dx = dW = None
        if need[0] or need[1]:
            dx, dW = _conv_t_grads(ctx, gp, scale, g, need[0], need[1], x_shape)
        ctx.hpl = ctx.wpl = None
        dres = gp.reshape(gy.shape) if need[3] else None
        return dx, dW, db, dres, None, None


def _conv_tc_apply(fn, name, x, W, b, residual, g, lead, act, out_hw):
    """Check b and residual against the layer's geometry and the channel and weight-operand
    limits, all before any launch; then zero images give an empty result without a launch."""
    out_shape = tuple(lead) + tuple(out_hw) + (g.Cout,)
    for what, t, shape in (("b", b, (g.Cout,)), ("residual", residual, out_shape)):
        if t is not None and (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or
                              t.device != W.device or tuple(t.shape) != shape):
            raise ValueError("%s: %s should be a float32 tensor of shape %s on %s, got %s"
                             % (name, what, shape, W.device,
                                (t.dtype, tuple(t.shape), t.device)
                                if isinstance(t, torch.Tensor) else type(t).__name__))
    if max(g.Cin, g.Cout) >= CONV_TC_MAX_C:
        raise ValueError("%s: channels should be below 2^20, got Cin %d, Cout %d"
                         % (name, g.Cin, g.Cout))
    kk = g.k * g.k
    # the weight operand: W^T [Cout, k k Cin] (conv2d_tc) or W' [k k Cout, Cin] (transposed), in
    # rows padded to 64 entries
    w_rows, w_cols = (kk * g.Cout, g.Cin) if fn is _Conv2dTransposeTC else (g.Cout, kk * g.Cin)
    if w_rows * (-(-w_cols // 64) * 64) >= 2 ** 31:
        raise ValueError("%s: too large: the weight operand must have fewer than 2^31 entries"
                         % name)
    if g.N == 0:
        return torch.empty(out_shape, dtype=torch.float32, device=x.device)
    return fn.apply(x, W, b, residual, g, act)


def conv2d_tc(x, W, b=None, stride=1, relu=False, residual=None, padding="SAME"):
    """``relu?(tf.layers.conv2d(x, Cout, k, stride, padding) + residual)`` with its bias b, the
    convolutions of vae_conv.py's encoder and resnet blocks (vae_conv.py:39-53, 80), on the
    tensor-core products at fp32 accuracy: ``conv2d`` beyond the 3 x 3, 64-channel, SAME range of
    its FFMA kernels.

    x [..., H, W, Cin] is NHWC, any leading shape flattened to images; W [k, k, Cin, Cout] is the
    ``tf.layers.conv2d`` kernel, 1 <= k <= 7; b [Cout] or None; ``residual`` (or None) has the
    output's shape and is added before the ReLU.  The output is [..., Ho, Wo, Cout], sized and
    padded as in ``bn_conv2d``:

        y[n, i, j, co] = b[co] + residual[n, i, j, co]
                         + sum_{kh, kw, ci} x[n, s i + kh - pt, s j + kw - pl, ci] W[kh, kw, ci, co]

    Differentiable w.r.t. x, W, b and residual; under ``inference_mode`` nothing is kept.  Every
    reduction runs in a fixed order with no float atomics, so two identical calls give identical
    bits.  The output carries the max |.| that a following fused layer uses for its operand split,
    and a tagged x is split at its tag.  Supported: float32 CUDA tensors on one device, stride 1
    or 2, padding "SAME" or "VALID", 1 <= Cin, Cout < 2^20, fewer than 2^31 entries in every
    tensor and operand; zero images give an empty result without a launch; anything else raises
    ValueError before any launch."""
    x = _unwrap(x)
    g, lead = _conv_tc_geom("conv2d_tc", x, W, stride, padding, False, empty_batch=True)
    return _conv_tc_apply(_Conv2dTC, "conv2d_tc", x, W, b, residual, g, lead,
                          _ACT_RELU if relu else _ACT_NONE, (g.Hs, g.Ws))


def conv2d_transpose_tc(x, W, out_shape, stride=1, b=None, relu=False, residual=None,
                        padding="SAME"):
    """``relu?(conv2d_transpose(x, out_shape, (k, k), stride) + residual)`` of
    examples/utils/utils.py:74-113 (``tf.nn.conv2d_transpose`` plus ``bias_add``; vae_conv.py:20-36,
    63-68) on the tensor-core products at fp32 accuracy: ``conv2d_transpose`` beyond the 3 x 3,
    64-channel, SAME range of its FFMA kernels.

    x [..., Hi, Wi, Cin] is NHWC; W [k, k, Cout, Cin] is that helper's ``weights`` layout, 1 <= k
    <= 7; ``out_shape`` = (Ho, Wo, Cout) with ceil(Ho / stride) == Hi for SAME and
    ceil((Ho - k + 1) / stride) == Hi for VALID (Wo likewise), as TF requires; b [Cout] or None;
    ``residual`` (or None) has the output's shape and is added before the ReLU.  The map is the
    adjoint of ``conv2d_tc``'s convolution from [Ho, Wo, Cout] to [Hi, Wi, Cin] with the same W
    and pads, computed as in ``bn_conv2d_transpose``.  Gradients, determinism, inference mode, the
    max |.| tag and the supported range are those of ``conv2d_tc``."""
    x = _unwrap(x)
    try:
        Ho, Wo, Co = (int(v) for v in out_shape)
    except (TypeError, ValueError):
        raise ValueError("conv2d_transpose_tc: out_shape should be (Ho, Wo, Cout), got %r"
                         % (out_shape,))
    g, lead = _conv_tc_geom("conv2d_transpose_tc", x, W, stride, padding, True, out_hw=(Ho, Wo),
                            empty_batch=True)
    if Co != g.Cout:
        raise ValueError("conv2d_transpose_tc: out_shape has %d channels, W has %d"
                         % (Co, g.Cout))
    return _conv_tc_apply(_Conv2dTransposeTC, "conv2d_transpose_tc", x, W, b, residual, g, lead,
                          _ACT_RELU if relu else _ACT_NONE, (Ho, Wo))
