"""Log-joint descriptors that ``HMC.sample`` recognises and runs on fused
kernels.  Each is also a plain ``log_joint(observed_dict)`` callable built
from torch ops, so it works on the generic path and as its own cross-check.
"""
import math
import os

import numpy as np
import torch

__all__ = ["GaussianLogJoint", "BNNRegressionLogJoint", "LNTMLogJoint", "linear",
           "linear_bernoulli_log_prob", "LinearBernoulli"]


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
    for layer sizes [n_in, H, 1] and per-chain weights:

        w0 [chains, H, n_in+1] ~ N(0, exp(logstds[0])),
        w1 [chains, 1, H+1]    ~ N(0, exp(logstds[1])),
        y ~ N(net(x; w), exp(y_logstd)),
        log_joint = sum log p(w) + mean_batch(log p(y|x,w)) * n_train.

    As a callable it is the generic-path log-joint (registry Normal kernels +
    torch einsum under the tape); ``zs.SGHMC.sample`` recognises it and runs
    the whole step in one fused kernel (zsb_sgmcmc_sghmc_bnn_f32).  Feed
    minibatches with ``sample_op(observed={'x': xb, 'y': yb})``.
    """

    def __init__(self, x, y, logstds, n_train, y_logstd=-0.95,
                 names=("w0", "w1")):
        from .distributions import Normal
        self._Normal = Normal
        self.x, self.y = x, y
        self.logstds = [l.contiguous() for l in logstds]
        self.n_train = float(n_train)
        self.y_logstd = float(y_logstd)
        self.names = tuple(names)
        self._zsb_fused = {"kind": "bnn_regression", "obj": self}

    def set_batch(self, observed):
        if "x" in observed:
            self.x = observed["x"]
        if "y" in observed:
            self.y = observed["y"]

    def __call__(self, observed):
        x = observed.get("x", self.x)
        y = observed.get("y", self.y)
        w0, w1 = observed[self.names[0]], observed[self.names[1]]
        C = w0.shape[0]
        h = x.unsqueeze(0).expand(C, -1, -1)
        lp = 0.0
        for w, ls in zip((w0, w1), self.logstds):
            ones = torch.ones(h.shape[:-1] + (1,), device=h.device)
            h = torch.cat([h, ones], -1)
            h = torch.einsum("imk,ijk->ijm", w, h) / math.sqrt(h.shape[2])
            if w is w0:
                h = torch.relu(h)
            lp = lp + self._Normal(torch.zeros_like(ls), logstd=ls,
                                   group_ndims=2).log_prob(w)
        y_mean = h.squeeze(2)
        lpy = self._Normal(y_mean, logstd=torch.full_like(y_mean,
                                                         self.y_logstd)
                           ).log_prob(y.unsqueeze(0))
        return lp + lpy.mean(1) * self.n_train



class LNTMLogJoint(object):
    """E-step objective of the Logistic-Normal Topic Model, examples/topic_models/
    lntm_mcem.py:33-48 with ``model.log_joint = e_obj`` (:97-99):

        eta [chains, docs, K] ~ Normal(eta_mean, exp(eta_logstd)), group_ndims=1
        log p = cond_log_prob('eta') + UnnormalizedMultinomial(log(softmax(eta) @ softmax(beta)),
                                                                normalize_logits=False).log_prob(x)

    ``zs.HMC.sample`` recognises it (``_zsb_fused`` kind "provider") and takes log-joint values
    and gradients from ONE fused, sparsity-aware kernel (zsb_lntm_logjoint_f32): the corpus is held
    in CSR, only the words a document contains are formed, and the [chains*docs, V] matrix
    ``doc_word`` of the reference never exists (335 TB at BASELINE config 5).  As a plain callable
    it is the dense torch restatement of the reference graph (small shapes / cross-check).

    x: dense [docs, V] counts (any float/int tensor); beta: [K, V] (fixed during the E-step; call
    ``set_beta`` after every M-step); K in {16, 32, 64, 128}.
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
        self.eta_mean = eta_mean.detach().to(torch.float32).contiguous()
        self.eta_logstd = eta_logstd.detach().to(torch.float32).contiguous()
        self.n_topics = int(beta.shape[0])
        if self.n_topics not in (16, 32, 64, 128):
            raise ValueError("LNTMLogJoint: n_topics must be 16, 32, 64 or 128")
        self.phi_t = torch.empty((self.n_vocab, self.n_topics), dtype=torch.float32, device=dev)
        self.set_beta(beta)
        self._zsb_fused = {"kind": "provider", "obj": self}

    def set_beta(self, beta):
        from ._lib import lib, ptr, stream
        self.beta = beta.detach().to(torch.float32).contiguous()
        lib.call("zsb_lntm_phi_t_f32", ptr(self.beta), self.n_topics, self.n_vocab,
                 ptr(self.phi_t), stream())

    def _launch(self, eta, want_lp, want_grad):
        from ._lib import lib, ptr, stream
        eta = eta.detach()
        if eta.dim() != 3 or int(eta.shape[1]) != self.n_docs or \
                int(eta.shape[2]) != self.n_topics:
            raise ValueError("eta must be [chains, %d, %d]" % (self.n_docs, self.n_topics))
        eta = eta.to(torch.float32).contiguous()
        chains = int(eta.shape[0])
        lp = torch.empty((chains, self.n_docs), dtype=torch.float32, device=eta.device) \
            if want_lp else None
        g = torch.empty_like(eta) if want_grad else None
        lib.call("zsb_lntm_logjoint_f32", ptr(eta), ptr(self.eta_mean), ptr(self.eta_logstd),
                 ptr(self.phi_t), ptr(self.doc_ptr), ptr(self.word_idx), ptr(self.word_cnt),
                 ptr(lp), ptr(g), chains, self.n_docs, self.n_topics, stream())
        return lp, g

    # provider interface used by HMC's generic path instead of autograd
    def logp(self, var_list):
        return self._launch(var_list[0], True, False)[0]

    def grad(self, var_list):
        return [self._launch(var_list[0], False, True)[1]]

    def __call__(self, observed):
        """Dense restatement of the reference graph in torch (lntm_mcem.py:33-48)."""
        eta = observed[self.name]
        theta = torch.softmax(eta, -1)
        phi = torch.softmax(self.beta, -1)
        doc_word = theta.reshape(-1, self.n_topics) @ phi
        doc_word = doc_word.reshape(tuple(eta.shape[:-1]) + (self.n_vocab,))
        prec = torch.exp(-2 * self.eta_logstd)
        prior = (-0.5 * math.log(2 * math.pi) - self.eta_logstd
                 - 0.5 * prec * (eta - self.eta_mean) ** 2).sum(-1)
        return prior + (self.x * torch.log(doc_word)).sum(-1)


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


def _tc_split_t(t2d):
    """fp32 [R, C] -> (fp16 planes [2, C, Rp] of the transpose, scale)."""
    from ._lib import lib, ptr, stream
    t2d = t2d.detach().to(torch.float32).contiguous()
    R, C = int(t2d.shape[0]), int(t2d.shape[1])
    Rp = lib.load().zsb_linear_tc_kpad(R)
    planes = torch.empty((2, C, Rp), dtype=torch.float16, device=t2d.device)
    scale = torch.zeros(4, dtype=torch.float32, device=t2d.device)
    lib.call("zsb_split16_pad_t_f32", ptr(t2d), R, C, ptr(planes), ptr(scale),
             stream())
    return planes, scale


class _Planes(object):
    """fp16 hi/lo operand planes of one [rows, K] matrix times a power-of-two scale: row-major
    ``planes`` [2, rows, Kp] (all three products of a layer) and, only with ZSB_WGRAD_T=1, transposed ``planes_t``
    [2, K, Rp] (weight-gradient product, contraction over the rows); ``scale`` = device float[4]."""
    __slots__ = ("planes", "planes_t", "scale", "rows", "K")

    def __init__(self, planes, planes_t, scale, rows, K):
        self.planes, self.planes_t, self.scale, self.rows, self.K = planes, planes_t, scale, rows, K


def _tc_split_dual(t2d, mask=None, want=(True, True), amax=None, col_sum=None):
    """One pass over fp32 ``t2d`` [R, K] (times the ReLU mask ``mask > 0``) -> _Planes with the
    layouts asked for in ``want`` = (row-major, transposed); ``amax`` = scale slot whose max-|.|
    word a producing GEMM already filled (no max pass then); ``col_sum`` [K] += column sums."""
    from ._lib import lib, ptr, stream
    t2d = t2d.detach().to(torch.float32).contiguous()
    R, K = int(t2d.shape[0]), int(t2d.shape[1])
    dev = t2d.device
    if K % 2:                      # odd widths: the two single-layout kernels (same max|.| in
        if mask is not None:       # both -> the same power-of-two scale)
            t2d = t2d * (mask > 0)
        if col_sum is not None:
            col_sum += t2d.sum(0)
        pl, sc = _tc_split(t2d) if want[0] else (None, None)
        plt, sct = _tc_split_t(t2d) if want[1] else (None, None)
        return _Planes(pl, plt, sc if sc is not None else sct, R, K)
    Kp = lib.load().zsb_linear_tc_kpad(K)
    Rp = lib.load().zsb_linear_tc_kpad(R)
    planes = torch.empty((2, R, Kp), dtype=torch.float16, device=dev) if want[0] else None
    planes_t = torch.empty((2, K, Rp), dtype=torch.float16, device=dev) if want[1] else None
    scale = amax if amax is not None else torch.zeros(4, dtype=torch.float32, device=dev)
    m = None if mask is None else mask.detach().to(torch.float32).contiguous()
    lib.call("zsb_split16_dual_f32", ptr(t2d), ptr(m), R, K, ptr(planes), ptr(planes_t),
             ptr(col_sum), ptr(scale), int(amax is not None), stream())
    return _Planes(planes, planes_t, scale, R, K)


def _planes_of(h2, src, need_t):
    """Operand planes of activation ``h2`` (= ``src`` flattened to 2-D), cached on ``src``: the
    producing GEMM left the max |.| in ``src._zsb_amax`` (no max pass), and every consumer of the
    same activation (e.g. the two heads of the encoder) shares one split."""
    R, K = int(h2.shape[0]), int(h2.shape[1])
    pl = getattr(src, "_zsb_pl", None)
    if (pl is not None and pl.rows == R and pl.K == K and pl.planes is not None
            and (not need_t or pl.planes_t is not None)):
        return pl
    amax = getattr(src, "_zsb_amax", None)
    pl = _tc_split_dual(h2, want=(True, need_t), amax=None if K % 2 else amax)
    try:
        src._zsb_pl = pl
        if amax is not None:
            del src._zsb_amax
    except (AttributeError, RuntimeError):
        pass
    return pl


def _tc_grad_input(gpl, W, R, wp=None, ws=None):
    """dh [R, K] = g [R, J] @ W [J, K] on the tensor cores (+ the scale slot holding max|dh|).
    ``wp, ws``: the forward planes of W when the caller still has them -- the product reads them
    as an MN-major operand (zsb_linear_tc_dgrad_f32), so W^T is never formed; ZSB_DGRAD_MN=0 (or
    ZSB_WGRAD_T=1): split of W^T, K-major operands."""
    amax = torch.zeros(4, dtype=torch.float32, device=W.device)
    if _WGRAD_T or not _DGRAD_MN:
        wtp, wts = _tc_split(W.detach().t())
        dh = _tc_linear(0, wtp, wts, gpl.planes, gpl.scale, None, None, None, R,
                        int(W.shape[1]), int(W.shape[0]), amax=amax)
        return dh, amax
    from ._lib import lib, ptr, stream
    if wp is None:
        wp, ws = _tc_split(W)
    J, K = int(W.shape[0]), int(W.shape[1])
    dh = torch.empty((R, K), dtype=torch.float32, device=W.device)
    lib.call("zsb_linear_tc_dgrad_f32", ptr(wp), ptr(ws), ptr(gpl.planes), ptr(gpl.scale),
             R, J, K, ptr(dh), ptr(amax), stream())
    return dh, amax


# ZSB_WGRAD_T=1: the weight gradient reads TRANSPOSED operand planes (the round-2 scheme, kept as a
# cross-check); default: MN-major operands straight from the row-major planes.
_WGRAD_T = os.environ.get("ZSB_WGRAD_T", "0") == "1"
# The input gradient reads the forward weight planes as an MN-major operand
# (zsb_linear_tc_dgrad_f32) instead of splitting W^T; ZSB_DGRAD_MN=0 restores the W^T split.
_DGRAD_MN = os.environ.get("ZSB_DGRAD_MN", "1") == "1"
# ZSB_BERN_FUSED=1: the Bernoulli layer's backward emits d/dlogits directly as operand planes from
# the GEMM epilogue (zsb_linear_tc_bern_grad_planes_f32, epi 3).  Correct (tests) but MEASURED SLOWER
# than fp32 dlogits + one split pass (1.47 vs 0.75 + 0.5 ms at config 3: the longer epilogue is no
# longer hidden behind the next unit's MMAs), so it is opt-in.
_BERN_UNFUSED = os.environ.get("ZSB_BERN_FUSED", "0") != "1"


def _tc_grad_weight(gpl, hpl, R):
    """dW [J, K] = g^T [J, R] @ h [R, K]: contraction over the rows, split-K over the CTA pairs.
    Both operands are the row-major planes of g and h (MN-major wgmma operands,
    zsb_linear_tc_wgrad_f32); with ZSB_WGRAD_T=1 the transposed plane layout instead."""
    if _WGRAD_T:
        return _tc_linear(0, hpl.planes_t, hpl.scale, gpl.planes_t, gpl.scale, None, None, None,
                          gpl.K, hpl.K, R, split_k=True)
    from ._lib import lib, ptr, stream
    J, K = gpl.K, hpl.K
    dev = gpl.planes.device
    slices = lib.load().zsb_linear_tc_slices(J, K, R)
    part = torch.empty(slices * J * K, dtype=torch.float32, device=dev) if slices > 1 else None
    out = torch.empty((J, K), dtype=torch.float32, device=dev)
    lib.call("zsb_linear_tc_wgrad_f32", ptr(hpl.planes), ptr(hpl.scale), K, ptr(gpl.planes),
             ptr(gpl.scale), J, R, ptr(out), ptr(part), stream())
    return out


def _tc_linear(epi, wp, ws, hp, hs, bias, x, gout, R, J, K, relu=False,
               split_k=False, amax=None):
    from ._lib import lib, ptr, stream
    dev = hp.device
    part = None
    if epi == 0 and split_k:
        slices = lib.load().zsb_linear_tc_slices(R, J, K)
        if slices > 1:
            part = torch.empty(slices * R * J, dtype=torch.float32, device=dev)
    if epi == 1:
        out = torch.empty(R, dtype=torch.float32, device=dev)
        part = torch.empty(lib.load().zsb_linear_tc_nparts(J) * R,
                           dtype=torch.float32, device=dev)
    else:
        out = torch.empty((R, J), dtype=torch.float32, device=dev)
    lib.call("zsb_linear_tc_amax_f32", epi, ptr(wp), ptr(ws), ptr(hp), ptr(hs),
             ptr(bias), ptr(x), int(x.shape[0]) if x is not None else 0,
             ptr(gout), ptr(out), ptr(part), R, J, K, int(bool(relu)), ptr(amax), stream())
    return out


def _tag(t, amax):
    try:
        t._zsb_amax = amax
    except (AttributeError, RuntimeError):
        pass
    return t


class _Linear(torch.autograd.Function):
    """y = relu?(h W^T + b): forward and both backward products on the wgmma kernel at fp32
    accuracy (epi 0; the weight gradient reads the same row-major planes as MN-major operands, split-K).
    Memory passes around the GEMMs are fused (round 2): every GEMM leaves max|out| for its
    consumer's scale, ONE pass (zsb_split16_dual_f32) turns an activation / gradient into both
    operand layouts, applies the ReLU mask and accumulates the bias gradient."""

    @staticmethod
    def forward(ctx, h, W, b, relu):
        lead = h.shape[:-1]
        h2 = h if h.dim() == 2 else h.reshape(-1, h.shape[-1])
        R, K, J = int(h2.shape[0]), int(h2.shape[1]), int(W.shape[0])
        need_dw = bool(ctx.needs_input_grad[1])
        hpl = _planes_of(h2, h, need_dw and _WGRAD_T)
        wp, ws = _tc_split(W)
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        amax = torch.zeros(4, dtype=torch.float32, device=h2.device)
        y = _tc_linear(0, wp, ws, hpl.planes, hpl.scale, bias, None, None, R, J, K, relu,
                       amax=amax)
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
        gpl = _tc_split_dual(g, mask=y if relu else None,
                             want=(bool(need[0]) or (bool(need[1]) and not _WGRAD_T),
                                   bool(need[1]) and _WGRAD_T),
                             amax=getattr(gy, "_zsb_amax", None), col_sum=db)
        dh = None
        if need[0]:
            dh2, amax = _tc_grad_input(gpl, W, R, *(ctx.wpl or (None, None)))
            dh = _tag(dh2.reshape(tuple(lead) + (K,)), amax)
        dW = _tc_grad_weight(gpl, ctx.hpl, R) if need[1] else None
        ctx.hpl = None
        ctx.wpl = None
        return dh, dW, db, None


def linear(h, W, b=None, relu=False):
    """``relu?(h @ W.T + b)`` (``tf.layers.dense``) on the wgmma kernel."""
    return _Linear.apply(h, W, b, bool(relu))


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
        hpl = _planes_of(h2, h, bool(ctx.needs_input_grad[1]) and _WGRAD_T)
        bias = b.detach().to(torch.float32).contiguous() if b is not None else None
        lp = _tc_linear(1, wp, ws, hpl.planes, hpl.scale, bias, x2, None, R, J, K)
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
        if _WGRAD_T or _BERN_UNFUSED:        # round-2 scheme: fp32 dl, then one split pass
            amax = torch.zeros(4, dtype=torch.float32, device=g.device)
            dl = _tc_linear(2, wp, ws, hpl.planes, hpl.scale, bias, x2, g, R, J, K, amax=amax)
            dlpl = _tc_split_dual(dl, want=(bool(need[0]) or (bool(need[1]) and not _WGRAD_T),
                                            bool(need[1]) and _WGRAD_T), amax=amax, col_sum=db)
        else:                                # dl leaves the GEMM epilogue as operand planes
            from ._lib import lib, ptr, stream
            Jp = lib.load().zsb_linear_tc_kpad(J)
            planes = torch.empty((2, R, Jp), dtype=torch.float16, device=g.device)
            scale = torch.zeros(4, dtype=torch.float32, device=g.device)
            lib.call("zsb_linear_tc_bern_grad_planes_f32", ptr(wp), ptr(ws), ptr(hpl.planes),
                     ptr(hpl.scale), ptr(bias), ptr(x2), int(x2.shape[0]), ptr(g), ptr(planes),
                     ptr(db), ptr(scale), R, J, K, stream())
            dlpl = _Planes(planes, None, scale, R, J)
        dh = None
        if need[0]:
            dh2, a2 = _tc_grad_input(dlpl, W, R, wp, ws)
            dh = _tag(dh2.reshape(tuple(lead) + (K,)), a2)
        dW = _tc_grad_weight(dlpl, hpl, R) if need[1] else None
        ctx.hpl = None
        return dh, dW, db, None


def linear_bernoulli_log_prob(h, W, b, x):
    """log p(x | logits = h @ W.T + b) summed over the last axis, fused.
    ``x`` ([n_x, J], 0/1) is broadcast over the leading rows of ``h``
    (row r of h uses x[r % n_x]: the [particles, batch] layout of
    iwae.py:23-32 flattened)."""
    return _LinearBernoulliLogProb.apply(h, W, b, x)


class LinearBernoulli(object):
    """Drop-in for ``Bernoulli(logits=dense(h), group_ndims=1)`` as a
    distribution plugin (duck-typed contract of bn.py:96-115): ``log_prob`` runs
    the fused GEMM + Bernoulli epilogue; the logits are only materialised when
    the node is *sampled* rather than observed."""

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

    def sample(self, n_samples=None):
        from .distributions import Bernoulli
        return Bernoulli(self.logits, dtype=self.dtype).sample(n_samples)

    def log_prob(self, given):
        J = int(self._W.shape[0])
        lead = tuple(self._h.shape[:-1])
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
