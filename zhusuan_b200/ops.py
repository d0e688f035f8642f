"""torch.autograd wrappers around the libzsb200 kernels.

This is the "generic path": every distribution ``log_prob`` / reduction is an
individually callable CUDA kernel with an analytic backward, so an arbitrary
user ``log_joint`` composed from the registry is differentiable without
TensorFlow's ``tf.gradients`` (zhusuan/hmc.py:430-432).  torch supplies device
memory, streams and the tape; the arithmetic is ours.
"""
import math

import torch

from ._lib import lib, ptr, stream, ZsbError

_F32 = torch.float32


def _f32c(t):
    if t.dtype != _F32:
        raise TypeError("zhusuan_b200 computes in float32; got %s" % t.dtype)
    return t.contiguous()


def _prep(t, full_shape):
    """Return (contiguous tensor, numel) usable with the kernels' modular
    broadcast: the operand's shape must be a suffix of ``full_shape`` after
    dropping its leading 1-dims, otherwise it is materialised
    (what maybe_explicit_broadcast always does, distributions/utils.py:52-78)."""
    shape = list(t.shape)
    while shape and shape[0] == 1:
        shape.pop(0)
    n = len(shape)
    if n == 0 or list(full_shape[len(full_shape) - n:]) == shape:
        return _f32c(t).reshape(-1), max(1, int(t.numel()))
    e = t.expand(full_shape).contiguous()
    return e.reshape(-1), int(e.numel())


def _group_of(shape, group_ndims):
    if group_ndims == 0:
        return 1, tuple(shape)
    if group_ndims > len(shape):
        raise ValueError("group_ndims (%d) exceeds the rank of the batch "
                         "shape %s" % (group_ndims, tuple(shape)))
    g = 1
    for s in shape[len(shape) - group_ndims:]:
        g *= int(s)
    return g, tuple(shape[:len(shape) - group_ndims])


def _sum_to(t, shape):
    return t.sum_to_size(tuple(shape)) if tuple(t.shape) != tuple(shape) else t


class _NormalLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, mean, logstd, group_ndims):
        full = torch.broadcast_shapes(given.shape, mean.shape, logstd.shape)
        group, out_shape = _group_of(full, group_ndims)
        g, gn = _prep(given, full)
        m, mn = _prep(mean, full)
        s, sn = _prep(logstd, full)
        n_out = 1
        for d in out_shape:
            n_out *= int(d)
        out = torch.empty(out_shape, dtype=_F32, device=given.device)
        lib.call("zsb_logprob_normal_f32", ptr(g), gn, ptr(m), mn, ptr(s), sn,
                 ptr(out), n_out, group, stream())
        ctx.save_for_backward(g, m, s)
        ctx.meta = (gn, mn, sn, n_out, group, full, given.shape, mean.shape,
                    logstd.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        g, m, s = ctx.saved_tensors
        gn, mn, sn, n_out, group, full, gs, ms, ss = ctx.meta
        need = ctx.needs_input_grad
        gout = _f32c(gout)
        dev = gout.device
        dg = torch.empty(full, dtype=_F32, device=dev) if need[0] else None
        dm = torch.empty(full, dtype=_F32, device=dev) if need[1] else None
        ds = torch.empty(full, dtype=_F32, device=dev) if need[2] else None
        lib.call("zsb_logprob_normal_bwd_f32", ptr(g), gn, ptr(m), mn, ptr(s),
                 sn, ptr(gout), n_out, group, ptr(dg), ptr(dm), ptr(ds),
                 stream())
        return (_sum_to(dg, gs) if need[0] else None,
                _sum_to(dm, ms) if need[1] else None,
                _sum_to(ds, ss) if need[2] else None, None)


def normal_log_prob(given, mean, logstd, group_ndims=0):
    """Normal._log_prob + group sum (univariate.py:174-181, base.py:303)."""
    return _NormalLogProb.apply(given, mean, logstd, int(group_ndims))


class _BernoulliLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, logits, group_ndims):
        full = torch.broadcast_shapes(given.shape, logits.shape)
        group, out_shape = _group_of(full, group_ndims)
        g, gn = _prep(given, full)
        l, ln = _prep(logits, full)
        n_out = 1
        for d in out_shape:
            n_out *= int(d)
        out = torch.empty(out_shape, dtype=_F32, device=logits.device)
        lib.call("zsb_logprob_bernoulli_f32", ptr(g), gn, ptr(l), ln, ptr(out),
                 n_out, group, stream())
        ctx.save_for_backward(g, l)
        ctx.meta = (gn, ln, n_out, group, full, logits.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        g, l = ctx.saved_tensors
        gn, ln, n_out, group, full, ls = ctx.meta
        if not ctx.needs_input_grad[1]:
            return None, None, None
        gout = _f32c(gout)
        dl = torch.empty(full, dtype=_F32, device=gout.device)
        lib.call("zsb_logprob_bernoulli_bwd_f32", ptr(g), gn, ptr(l), ln,
                 ptr(gout), n_out, group, ptr(dl), stream())
        return None, _sum_to(dl, ls), None


def bernoulli_log_prob(given, logits, group_ndims=0):
    """Bernoulli._log_prob (univariate.py:398-403); ``given`` is cast to the
    param dtype first (:399)."""
    return _BernoulliLogProb.apply(given.to(_F32), logits, int(group_ndims))


# ids of zsb_logprob_univariate_f32 (include/zsb200.h)
UNI_FOLDNORMAL, UNI_UNIFORM, UNI_GAMMA, UNI_BETA, UNI_POISSON, UNI_BINOMIAL, \
    UNI_INVGAMMA, UNI_LAPLACE, UNI_BINCONCRETE = range(9)


class _UnivariateLogProb(torch.autograd.Function):
    """Elementwise density ``dist`` of ``given`` under parameters (a, b) with
    the group sum; analytic gradients wrt all three (univariate_ext.cu)."""

    @staticmethod
    def forward(ctx, dist, given, a, b, group_ndims):
        shapes = [given.shape, a.shape] + ([b.shape] if b is not None else [])
        full = torch.broadcast_shapes(*shapes)
        group, out_shape = _group_of(full, group_ndims)
        g, gn = _prep(given, full)
        pa, an = _prep(a, full)
        pb, bn = _prep(b, full) if b is not None else (None, 0)
        n_out = 1
        for d in out_shape:
            n_out *= int(d)
        out = torch.empty(out_shape, dtype=_F32, device=a.device)
        lib.call("zsb_logprob_univariate_f32", dist, ptr(g), gn, ptr(pa), an,
                 ptr(pb), bn, ptr(out), n_out, group, stream())
        ctx.save_for_backward(g, pa, pb)
        ctx.meta = (dist, gn, an, bn, n_out, group, full, given.shape, a.shape,
                    b.shape if b is not None else None)
        return out

    @staticmethod
    def backward(ctx, gout):
        g, pa, pb = ctx.saved_tensors
        dist, gn, an, bn, n_out, group, full, gs, as_, bs = ctx.meta
        need = ctx.needs_input_grad
        gout = _f32c(gout)
        dev = gout.device
        dg = torch.empty(full, dtype=_F32, device=dev) if need[1] else None
        da = torch.empty(full, dtype=_F32, device=dev) if need[2] else None
        db = torch.empty(full, dtype=_F32, device=dev) \
            if (need[3] and pb is not None) else None
        lib.call("zsb_logprob_univariate_bwd_f32", dist, ptr(g), gn, ptr(pa),
                 an, ptr(pb), bn, ptr(gout), n_out, group, ptr(dg), ptr(da),
                 ptr(db), stream())
        return (None, _sum_to(dg, gs) if dg is not None else None,
                _sum_to(da, as_) if da is not None else None,
                _sum_to(db, bs) if db is not None else None, None)


def univariate_log_prob(dist, given, a, b=None, group_ndims=0):
    """log-density of one of the UNI_* families + group sum."""
    return _UnivariateLogProb.apply(int(dist), given.to(_F32), a, b,
                                    int(group_ndims))


def _rows_prep(t, batch_shape, C):
    """[..., C] operand against a broadcast batch shape -> (flat, rows)."""
    full = tuple(batch_shape) + (C,)
    flat, n = _prep(t, full)
    return flat, n // C


class _CategoricalLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, logits):
        C = int(logits.shape[-1])
        bshape = torch.broadcast_shapes(given.shape, logits.shape[:-1])
        gi = given.to(torch.int32)
        gshape = list(gi.shape)
        while gshape and gshape[0] == 1:
            gshape.pop(0)
        if len(gshape) == 0 or list(bshape[len(bshape) - len(gshape):]) == gshape:
            g = gi.contiguous().reshape(-1)
        else:
            g = gi.expand(bshape).contiguous().reshape(-1)
        gn = max(1, int(g.numel()))
        l, lrows = _rows_prep(logits, bshape, C)
        rows = 1
        for d in bshape:
            rows *= int(d)
        out = torch.empty(bshape, dtype=_F32, device=logits.device)
        lib.call("zsb_logprob_categorical_f32", ptr(g), gn, ptr(l), lrows, C,
                 ptr(out), rows, stream())
        ctx.save_for_backward(g, l)
        ctx.meta = (gn, lrows, C, rows, tuple(bshape), logits.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        g, l = ctx.saved_tensors
        gn, lrows, C, rows, bshape, ls = ctx.meta
        if not ctx.needs_input_grad[1]:
            return None, None
        gout = _f32c(gout)
        dl = torch.empty(bshape + (C,), dtype=_F32, device=gout.device)
        lib.call("zsb_logprob_categorical_bwd_f32", ptr(g), gn, ptr(l), lrows,
                 C, ptr(gout), ptr(dl), rows, stream())
        return None, _sum_to(dl, ls)


def categorical_log_prob(given, logits, group_ndims=0):
    """Categorical._log_prob (univariate.py:496-548) + group sum."""
    lp = _CategoricalLogProb.apply(given, logits)
    return group_sum(lp, group_ndims)


class _DirichletLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, alpha):
        full = torch.broadcast_shapes(given.shape, alpha.shape)
        C = int(full[-1])
        bshape = tuple(full[:-1])
        g, grows = _rows_prep(given, bshape, C)
        a, arows = _rows_prep(alpha, bshape, C)
        rows = 1
        for d in bshape:
            rows *= int(d)
        out = torch.empty(bshape, dtype=_F32, device=given.device)
        lib.call("zsb_logprob_dirichlet_f32", ptr(g), grows, ptr(a), arows, C,
                 ptr(out), rows, stream())
        ctx.save_for_backward(g, a, given, alpha)
        ctx.meta = (grows, arows, C, rows, bshape, given.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        g, a, given, alpha = ctx.saved_tensors
        grows, arows, C, rows, bshape, gs = ctx.meta
        gout = _f32c(gout)
        dgiven = dalpha = None
        if ctx.needs_input_grad[1]:
            # d/d alpha_i = psi(sum alpha) - psi(alpha_i) + log x_i  (multivariate.py:665-677
            # differentiated); parameter gradients are off the hot path: composed from torch ops
            al = alpha.to(_F32)
            full = (torch.digamma(al.sum(-1, keepdim=True)) - torch.digamma(al)
                    + torch.log(given.to(_F32)))
            dalpha = _sum_to(gout.reshape(bshape + (1,)) * full, alpha.shape)
        if ctx.needs_input_grad[0]:
            dg = torch.empty(bshape + (C,), dtype=_F32, device=gout.device)
            lib.call("zsb_logprob_dirichlet_bwd_given_f32", ptr(g), grows, ptr(a),
                     arows, C, ptr(gout), ptr(dg), rows, stream())
            dgiven = _sum_to(dg, gs)
        return dgiven, dalpha


def dirichlet_log_prob(given, alpha, group_ndims=0):
    """Dirichlet._log_prob (multivariate.py:665-677) + group sum."""
    return group_sum(_DirichletLogProb.apply(given, alpha), group_ndims)


class _UnnormMultinomialLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, logits, normalize):
        full = torch.broadcast_shapes(given.shape, logits.shape)
        C = int(full[-1])
        bshape = tuple(full[:-1])
        g, grows = _rows_prep(given, bshape, C)
        l, lrows = _rows_prep(logits, bshape, C)
        rows = 1
        for d in bshape:
            rows *= int(d)
        out = torch.empty(bshape, dtype=_F32, device=logits.device)
        lib.call("zsb_logprob_unnorm_multinomial_f32", ptr(g), grows, ptr(l),
                 lrows, C, int(normalize), ptr(out), rows, stream())
        ctx.save_for_backward(g, l)
        ctx.meta = (grows, lrows, C, rows, bshape, logits.shape, int(normalize))
        return out

    @staticmethod
    def backward(ctx, gout):
        g, l = ctx.saved_tensors
        grows, lrows, C, rows, bshape, ls, normalize = ctx.meta
        if not ctx.needs_input_grad[1]:
            return None, None, None
        gout = _f32c(gout)
        dl = torch.empty(bshape + (C,), dtype=_F32, device=gout.device)
        lib.call("zsb_logprob_unnorm_multinomial_bwd_f32", ptr(g), grows,
                 ptr(l), lrows, C, normalize, ptr(gout), ptr(dl), rows,
                 stream())
        return None, _sum_to(dl, ls), None


def unnormalized_multinomial_log_prob(given, logits, normalize_logits=True,
                                      group_ndims=0):
    """UnnormalizedMultinomial._log_prob (multivariate.py:435-443)."""
    lp = _UnnormMultinomialLogProb.apply(given.to(_F32), logits,
                                         bool(normalize_logits))
    return group_sum(lp, group_ndims)


class _MVNCholLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, mean, cov_tril):
        D = int(mean.shape[-1])
        bshape = tuple(torch.broadcast_shapes(given.shape[:-1],
                                              mean.shape[:-1],
                                              cov_tril.shape[:-2]))
        g, grows = _rows_prep(given, bshape, D)
        m, mrows = _rows_prep(mean, bshape, D)
        full_l = bshape + (D, D)
        lt, ln = _prep(cov_tril, full_l)
        lmats = ln // (D * D)
        rows = 1
        for d in bshape:
            rows *= int(d)
        out = torch.empty(bshape, dtype=_F32, device=given.device)
        x = torch.empty(bshape + (D,), dtype=_F32, device=given.device)
        lib.call("zsb_logprob_mvn_chol_f32", ptr(g), grows, ptr(m), mrows,
                 ptr(lt), lmats, D, ptr(out), ptr(x), rows, stream())
        ctx.save_for_backward(x, lt, cov_tril)
        ctx.meta = (lmats, D, rows, bshape, given.shape, mean.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        x, lt, cov_tril = ctx.saved_tensors
        lmats, D, rows, bshape, gs, ms = ctx.meta
        gout = _f32c(gout)
        dg = torch.empty(bshape + (D,), dtype=_F32, device=gout.device)
        lib.call("zsb_logprob_mvn_chol_bwd_given_f32", ptr(x), ptr(lt), lmats,
                 D, ptr(gout), ptr(dg), rows, stream())
        dtril = None
        if ctx.needs_input_grad[2]:
            # y = L^-1 (x - mu) (saved), dg = -gout * L^-T y:
            #   d log p / dL = gout * tril(L^-T y y^T) - gout * diag(1 / L_ii)
            # (multivariate.py:169-189 differentiated).  Parameter gradient: off the hot path,
            # composed from torch ops on the kernel's intermediates.
            outer = torch.tril(-dg.unsqueeze(-1) * x.unsqueeze(-2))
            inv_diag = 1.0 / torch.diagonal(cov_tril.to(_F32), dim1=-2, dim2=-1)
            full = outer - torch.diag_embed(
                gout.reshape(bshape + (1,)) * inv_diag.expand(bshape + (D,)))
            dtril = _sum_to(full, cov_tril.shape)
        return (_sum_to(dg, gs) if ctx.needs_input_grad[0] else None,
                _sum_to(-dg, ms) if ctx.needs_input_grad[1] else None, dtril)


def mvn_cholesky_log_prob(given, mean, cov_tril, group_ndims=0):
    """MultivariateNormalCholesky._log_prob (multivariate.py:169-189)."""
    return group_sum(_MVNCholLogProb.apply(given, mean, cov_tril), group_ndims)


# ---------------------------------------------------------------- reductions
OP_LME, OP_MEAN, OP_LSE, OP_SUM = 0, 1, 2, 3


class _Reduce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, op, outer, K, inner):
        x = _f32c(x)
        out = torch.empty((outer, inner), dtype=_F32, device=x.device)
        lib.call("zsb_reduce_fwd_f32", op, ptr(x), ptr(out), outer, K, inner,
                 stream())
        ctx.save_for_backward(x, out)
        ctx.meta = (op, outer, K, inner)
        return out

    @staticmethod
    def backward(ctx, gout):
        x, y = ctx.saved_tensors
        op, outer, K, inner = ctx.meta
        gout = _f32c(gout)
        dx = torch.empty_like(x)
        lib.call("zsb_reduce_bwd_f32", op, ptr(x), ptr(y), ptr(gout), ptr(dx),
                 outer, K, inner, stream())
        return dx, None, None, None, None


def reduce_axes(x, op, axis=None, keepdims=False):
    """Reduce ``x`` over ``axis`` (int, tuple or None = all) with kernel op."""
    nd = x.dim()
    if axis is None:
        axes = list(range(nd))
    elif isinstance(axis, (tuple, list)):
        axes = sorted(a % nd for a in axis)
    else:
        axes = [int(axis) % nd]
    if nd == 0:
        axes = []
    if not axes:
        return x
    kept = [a for a in range(nd) if a not in axes]
    contiguous_block = axes == list(range(axes[0], axes[-1] + 1))
    if contiguous_block:
        xv = x.contiguous()
        outer = 1
        for a in range(axes[0]):
            outer *= int(x.shape[a])
        K = 1
        for a in axes:
            K *= int(x.shape[a])
        inner = 1
        for a in range(axes[-1] + 1, nd):
            inner *= int(x.shape[a])
    else:
        xv = x.permute(kept + axes).contiguous()
        outer = 1
        for a in kept:
            outer *= int(x.shape[a])
        K = 1
        for a in axes:
            K *= int(x.shape[a])
        inner = 1
    if K == 0:
        raise ValueError("cannot reduce over an empty axis")
    out = _Reduce.apply(xv.reshape(outer, K, inner), op, outer, K, inner)
    out = out.reshape([int(x.shape[a]) for a in kept])
    if keepdims:
        shape = [1 if a in axes else int(x.shape[a]) for a in range(nd)]
        out = out.reshape(shape)
    return out


def _single_axis_view(x, axis):
    """[outer, K, inner] view of ``x`` for one axis (int)."""
    nd = x.dim()
    ax = int(axis) % nd
    outer = 1
    for a in range(ax):
        outer *= int(x.shape[a])
    inner = 1
    for a in range(ax + 1, nd):
        inner *= int(x.shape[a])
    return ax, outer, int(x.shape[ax]), inner


def vimco_signal(log_w, axis):
    """VIMCO learning signal and log_mean_exp(log_w, axis, keepdims=True)
    (monte_carlo.py:194-223) in one kernel; both are constants for autograd
    (the reference stops the gradient of the signal)."""
    x = _f32c(log_w.detach())
    ax, outer, K, inner = _single_axis_view(x, axis)
    if K < 2:
        raise ValueError(
            "VIMCO is a multi-sample gradient estimator, size along "
            "`axis` in the objective should be larger than 1.")
    sig = torch.empty_like(x)
    shape = list(x.shape)
    shape[ax] = 1
    lme = torch.empty(shape, dtype=torch.float32, device=x.device)
    lib.call("zsb_vimco_signal_f32", ptr(x), ptr(sig), ptr(lme), outer, K,
             inner, stream())
    return sig, lme


def normalized_weights(log_w, axis):
    """Self-normalised importance weights softmax_axis(log_w), detached
    (inclusive_kl.py:139-143)."""
    x = _f32c(log_w.detach())
    ax, outer, K, inner = _single_axis_view(x, axis)
    w = torch.empty_like(x)
    lib.call("zsb_normalized_weights_f32", ptr(x), ptr(w), outer, K, inner,
             stream())
    return w


def group_sum(x, group_ndims):
    """reduce_sum over the last ``group_ndims`` axes (base.py:303-304)."""
    if group_ndims == 0:
        return x
    nd = x.dim()
    if group_ndims > nd:
        raise ValueError("group_ndims (%d) exceeds the rank of the batch "
                         "shape %s" % (group_ndims, tuple(x.shape)))
    return reduce_axes(x, OP_SUM, tuple(range(nd - group_ndims, nd)))


# ------------------------------------------------------------------ sampling
class _ReparamNormal(torch.autograd.Function):
    """z = mean + exp(logstd) * eps (univariate.py:161-172); eps injected or
    drawn in-kernel.  Backward is the reparameterisation path derivative."""

    @staticmethod
    def forward(ctx, mean, logstd, eps, n_samples, seed, it):
        bshape = torch.broadcast_shapes(mean.shape, logstd.shape)
        full = (int(n_samples),) + tuple(bshape)
        m, mn = _prep(mean, full)
        s, sn = _prep(logstd, full)
        n = 1
        for d in full:
            n *= int(d)
        z = torch.empty(full, dtype=_F32, device=mean.device)
        eps_out = torch.empty(full, dtype=_F32, device=mean.device)
        e = None
        if eps is not None:
            e = _f32c(eps.expand(full)).reshape(-1)
        lib.call("zsb_reparam_normal_f32", ptr(m), mn, ptr(s), sn, ptr(e),
                 int(seed), int(it), ptr(z), ptr(eps_out), None, n, 1,
                 stream())
        ctx.save_for_backward(eps_out, s)
        ctx.meta = (sn, full, mean.shape, logstd.shape)
        return z

    @staticmethod
    def backward(ctx, gz):
        eps, s = ctx.saved_tensors
        sn, full, ms, ss = ctx.meta
        gm = gs = None
        if ctx.needs_input_grad[0]:
            gm = _sum_to(gz, ms)
        if ctx.needs_input_grad[1]:
            std = torch.exp(s).reshape(-1)
            idx_std = std if sn == eps.numel() else std.repeat(
                eps.numel() // sn)
            gs = _sum_to(gz * eps * idx_std.reshape(full), ss)
        return gm, gs, None, None, None, None


def reparam_normal(mean, logstd, n_samples, eps=None, seed=0, it=0):
    return _ReparamNormal.apply(mean, logstd, eps, n_samples, seed, it)


def sample_bernoulli(logits, n_samples, u=None, seed=0, it=0,
                     dtype=torch.int32):
    full = (int(n_samples),) + tuple(logits.shape)
    l, ln = _prep(logits.detach(), full)
    n = 1
    for d in full:
        n *= int(d)
    out = torch.empty(full, dtype=torch.int32, device=logits.device)
    uu = None if u is None else _f32c(u.expand(full)).reshape(-1)
    lib.call("zsb_sample_bernoulli_i32", ptr(l), ln, ptr(uu), int(seed),
             int(it), ptr(out), n, stream())
    return out if dtype == torch.int32 else out.to(dtype)


def sample_categorical(logits, n_samples, u=None, seed=0, it=0):
    """Categorical._sample (univariate.py:478-494) on the device sampler: int32
    [n_samples] + logits.shape[:-1]; ``u`` = injected uniforms of that shape."""
    lg = _f32c(logits.detach())
    C = int(lg.shape[-1])
    bshape = tuple(lg.shape[:-1])
    rows = 1
    for d in bshape:
        rows *= int(d)
    out = torch.empty((int(n_samples),) + bshape, dtype=torch.int32, device=lg.device)
    uu = None if u is None else _f32c(u.expand(out.shape)).reshape(-1)
    lib.call("zsb_sample_categorical_i32", ptr(lg.reshape(-1)), max(rows, 1), max(rows, 1), C,
             int(n_samples), ptr(uu), int(seed), int(it), ptr(out), stream())
    return out


def sample_dirichlet(alpha, n_samples, gammas=None, seed=0, it=0):
    """Dirichlet._sample (multivariate.py:660-663): float32 [n_samples] + alpha.shape;
    ``gammas`` = injected Gamma(alpha, 1) variates of that shape."""
    a = _f32c(alpha.detach())
    C = int(a.shape[-1])
    arows = max(1, a.numel() // C)
    out = torch.empty((int(n_samples),) + tuple(a.shape), dtype=_F32, device=a.device)
    g = None if gammas is None else _f32c(gammas.expand(out.shape)).reshape(-1)
    lib.call("zsb_sample_dirichlet_f32", ptr(a.reshape(-1)), arows, int(n_samples) * arows, C,
             ptr(g), int(seed), int(it), ptr(out), stream())
    return out


def sample_gamma(alpha, beta, shape, seed=0, it=0):
    """Gamma(alpha, beta) draws of ``shape`` (alpha / beta broadcast against it)."""
    a = _f32c(alpha.detach().to(_F32).expand(shape))
    b = None if beta is None else _f32c(beta.detach().to(_F32).expand(shape))
    out = torch.empty(tuple(shape), dtype=_F32, device=a.device)
    n = out.numel()
    if n == 0:
        return out
    row_len = int(shape[-1]) if len(shape) else 1
    rows = n // row_len
    lib.call("zsb_sample_gamma_f32", ptr(a.reshape(-1)), rows, ptr(b.reshape(-1)) if b is not None
             else None, rows, rows, row_len, int(seed), int(it), ptr(out), stream())
    return out


def base_noise(kind, shape, device, seed=0, it=0):
    """U[0,1) (``kind`` 0) or N(0,1) (1) float32 noise of ``shape`` from the in-kernel Philox."""
    out = torch.empty(tuple(shape), dtype=_F32, device=device)
    lib.call("zsb_sample_base_noise_f32", int(kind), ptr(out), out.numel(), int(seed), int(it),
             stream())
    return out


def sample_count(kind, param, n_experiments, shape, u=None, seed=0, it=0):
    """Poisson (kind 0, param = rate) / Binomial (kind 1, param = logits) draws of ``shape``
    (the parameter broadcast against it): int32, one uniform per draw."""
    p = _f32c(param.detach().to(_F32).expand(shape))
    out = torch.empty(tuple(shape), dtype=torch.int32, device=p.device)
    n = out.numel()
    if n == 0:
        return out
    uu = None if u is None else _f32c(u.expand(shape)).reshape(-1)
    lib.call("zsb_sample_count_i32", int(kind), ptr(p.reshape(-1)), n, int(n_experiments),
             ptr(uu), int(seed), int(it), ptr(out), n, stream())
    return out


# ------------------------------------------------------- ExpConcrete / Concrete
CONCRETE_MAX_CATEGORIES = 1024


def _concrete_work(logits_rows, C, rows, device):
    n = lib.load().zsb_concrete_bwd_work(int(logits_rows), int(C), int(rows))
    if n < 0:
        raise ZsbError("zsb_concrete_bwd_work: bad sizes")
    return torch.empty(n, dtype=_F32, device=device)


class _ConcreteSample(torch.autograd.Function):
    """ExpConcrete / Concrete ._sample (multivariate.py:768-782, 905-919) in one pass: y =
    log_softmax((l + g) / t) or softmax(...), u injected or drawn as base_noise(0, ...) would
    draw it.  Backward: the reparameterisation gradient from the saved sample alone."""

    @staticmethod
    def forward(ctx, logits, temperature, n_samples, log_space, u, seed, it):
        l = _f32c(logits)
        t = _f32c(temperature)
        C = int(l.shape[-1])
        lrows = max(1, l.numel() // C)
        full = (int(n_samples),) + tuple(l.shape)
        out = torch.empty(full, dtype=_F32, device=l.device)
        rows = out.numel() // C
        uu = None if u is None else _f32c(u.expand(full)).reshape(-1)
        lib.call("zsb_sample_concrete_f32", ptr(l), lrows, ptr(t), C, int(log_space), ptr(uu),
                 int(seed), int(it), ptr(out), rows, stream())
        ctx.save_for_backward(out, t)
        ctx.meta = (lrows, C, int(log_space), rows, tuple(l.shape))
        return out

    @staticmethod
    def backward(ctx, gy):
        y, t = ctx.saved_tensors
        lrows, C, log_space, rows, lshape = ctx.meta
        need = ctx.needs_input_grad
        if rows == 0:
            return (torch.zeros(lshape, dtype=_F32, device=y.device) if need[0] else None,
                    torch.zeros_like(t) if need[1] else None, None, None, None, None, None)
        dl = torch.empty(lshape, dtype=_F32, device=y.device) if need[0] else None
        dt = torch.empty((), dtype=_F32, device=y.device) if need[1] else None
        if need[0] or need[1]:
            lib.call("zsb_sample_concrete_bwd_f32", ptr(y), ptr(_f32c(gy)), lrows, ptr(t), C,
                     log_space, ptr(dl), ptr(dt), ptr(_concrete_work(lrows, C, rows, y.device)),
                     rows, stream())
        return dl, dt.reshape(t.shape) if dt is not None else None, None, None, None, None, None


def sample_concrete(logits, temperature, n_samples, log_space, u=None, seed=0, it=0):
    """[n_samples] + logits.shape relaxed one-hot draws (log-probabilities when ``log_space``);
    ``u``: injected uniforms of that shape."""
    return _ConcreteSample.apply(logits, temperature, int(n_samples), bool(log_space), u,
                                 seed, it)


class _ConcreteLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, given, logits, temperature, log_space):
        full = torch.broadcast_shapes(given.shape, logits.shape)
        C = int(full[-1])
        bshape = tuple(full[:-1])
        g, grows = _rows_prep(given, bshape, C)
        l, lrows = _rows_prep(logits, bshape, C)
        t = _f32c(temperature)
        rows = 1
        for d in bshape:
            rows *= int(d)
        out = torch.empty(bshape, dtype=_F32, device=logits.device)
        if rows > 0:
            lib.call("zsb_logprob_concrete_f32", ptr(g), grows, ptr(l), lrows, ptr(t), C,
                     int(log_space), ptr(out), rows, stream())
        ctx.save_for_backward(g, l, t)
        ctx.meta = (grows, lrows, C, int(log_space), rows, bshape, given.shape, logits.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        g, l, t = ctx.saved_tensors
        grows, lrows, C, log_space, rows, bshape, gs, ls = ctx.meta
        need = ctx.needs_input_grad
        dev = l.device
        alloc = torch.empty if rows > 0 else torch.zeros
        dg = alloc(bshape + (C,), dtype=_F32, device=dev) if need[0] else None
        dl = alloc(lrows * C, dtype=_F32, device=dev) if need[1] else None
        dt = alloc((), dtype=_F32, device=dev) if need[2] else None
        if rows > 0 and any(need[:3]):
            lib.call("zsb_logprob_concrete_bwd_f32", ptr(g), grows, ptr(l), lrows, ptr(t), C,
                     log_space, ptr(_f32c(gout)), ptr(dg), ptr(dl), ptr(dt),
                     ptr(_concrete_work(lrows, C, rows, dev)), rows, stream())
        if dl is not None:
            # a suffix-broadcast parameter comes back in its own shape; an expanded one in full
            dl = dl.reshape(ls) if dl.numel() == math.prod(ls) else \
                _sum_to(dl.reshape(bshape + (C,)), ls)
        return (_sum_to(dg, gs) if dg is not None else None, dl,
                dt.reshape(t.shape) if dt is not None else None, None)


def concrete_log_prob(given, logits, temperature, log_space):
    """ExpConcrete._log_prob (log_space) / Concrete._log_prob (multivariate.py:800-812,
    938-955), before the group sum."""
    return _ConcreteLogProb.apply(given, logits, temperature, bool(log_space))


LOG_2PI = math.log(2.0 * math.pi)
