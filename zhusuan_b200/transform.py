"""zhusuan/transform.py: planar normalizing flows on the H100 kernels of csrc/flows.cu, and inverse
autoregressive flows with a linear autoregressive network on those of csrc/iaf.cu."""
import torch
from torch.autograd.function import once_differentiable

__all__ = ["planar_normalizing_flow", "planar_flow_parameters", "inv_autoregressive_flow",
           "LinearAR"]

MAX_D = 1024


class _PlanarFlow(torch.autograd.Function):
    """The whole stack in one launch (zsb_planar_flow_fwd_f32).  When a gradient is needed the
    forward pass also keeps every flow's input z_{k-1}; the backward pass (zsb_planar_flow_bwd_f32)
    recomputes each flow's activation from it and runs one reverse sweep plus one merge."""

    @staticmethod
    def forward(ctx, samples, log_probs, b, aux_u, w, need_grad):
        from ._lib import lib, ptr, stream
        n, d = int(aux_u.shape[0]), int(aux_u.shape[1])
        z = samples.detach().to(torch.float32).reshape(-1, d).contiguous()
        lq = log_probs.detach().to(torch.float32).reshape(-1).contiguous()
        bb, uu, ww = (t.detach().to(torch.float32).contiguous() for t in (b, aux_u, w))
        R = int(z.shape[0])
        z_out, lq_out = torch.empty_like(z), torch.empty_like(lq)
        ck = torch.empty((n, R, d), dtype=torch.float32, device=z.device) if need_grad else None
        lib.call("zsb_planar_flow_fwd_f32", ptr(z), ptr(lq), ptr(bb), ptr(uu), ptr(ww), ptr(z_out),
                 ptr(lq_out), ptr(ck), R, d, n, stream())
        if need_grad:
            ctx.save_for_backward(ck, bb, uu, ww)
        ctx.shapes = (tuple(samples.shape), tuple(log_probs.shape), R, d, n)
        return z_out.reshape(samples.shape), lq_out.reshape(log_probs.shape)

    @staticmethod
    @once_differentiable
    def backward(ctx, gz, glq):
        from ._lib import lib, ptr, stream
        ck, bb, uu, ww = ctx.saved_tensors
        z_shape, lq_shape, R, d, n = ctx.shapes
        dev = ck.device
        g = gz.to(torch.float32).reshape(R, d).contiguous()
        gl = glq.to(torch.float32).reshape(R).contiguous()
        gz_in = torch.empty_like(g)
        part = torch.empty((lib.load().zsb_planar_flow_warps(R, d, n), n, 2 * d + 2),
                           dtype=torch.float32, device=dev)
        db, daux, dw = torch.empty_like(bb), torch.empty_like(uu), torch.empty_like(ww)
        lib.call("zsb_planar_flow_bwd_f32", ptr(ck), ptr(g), ptr(gl), ptr(bb), ptr(uu), ptr(ww),
                 ptr(gz_in), ptr(part), ptr(db), ptr(daux), ptr(dw), R, d, n, stream())
        return gz_in.reshape(z_shape), glq.reshape(lq_shape), db, daux, dw, None


def planar_normalizing_flow(samples, log_probs, n_iters, b, aux_u, w):
    """``n_iters`` planar flows (Rezende & Mohamed, 2015) along the last axis of ``samples``:
    transform.py:70-198 with the parameters passed in, not created by the call.

    ``samples`` is ``[..., d]`` (rank >= 2, 1 <= d <= 1024) and ``log_probs`` is
    ``samples.shape[:-1]``.  ``b`` [n_iters], ``aux_u`` and ``w`` [n_iters, d] are the reference's
    ``param_b_i`` [1], ``aux_u_i`` [d, 1] and ``para_w_i`` [d, 1] of every flow, stacked (see
    ``planar_flow_parameters``).  Flow k computes

        u = aux_u_k + w_k / (w_k.w_k) * (softplus(w_k.aux_u_k) - 1 - w_k.aux_u_k)
        a = tanh(z.w_k + b_k),  log_q -= log(1 + (u.w_k)(1 - a^2)),  z += a u

    and the call returns ``(z, log_q)`` after the last flow.  Differentiable w.r.t. ``samples``,
    ``log_probs``, ``b``, ``aux_u`` and ``w``; two identical calls give identical bits.  The whole
    stack is one kernel launch, and its gradient one sweep plus one merge.

    Two deliberate differences from the reference: softplus is computed stably (the reference's
    ``log(exp(c) + 1)`` is inf for ``c > 88`` in float32), and there is no run-time check of
    ``u.w >= -1`` (it would need a host sync; ``u.w = softplus(w.aux_u) - 1 > -1`` by
    construction).  ``n_iters = 0`` returns the inputs unchanged."""
    if not isinstance(n_iters, int):
        raise ValueError("n_iters should be type 'int'")
    if samples.dim() < 2:
        raise ValueError("samples should have rank >= 2")
    if log_probs.dim() != samples.dim() - 1:
        raise ValueError("log_probs should have rank (N-1), while N is the rank of samples")
    if tuple(log_probs.shape) != tuple(samples.shape[:-1]):
        raise ValueError("samples and log_probs don't have same shape of (N-1) dims, while N is "
                         "the rank of samples")
    d = int(samples.shape[-1])
    if d < 1 or d > MAX_D:
        raise ValueError("the last axis of samples has %d elements: planar flows here take "
                         "1 <= d <= %d" % (d, MAX_D))
    for nm, t, shape in (("b", b, (n_iters,)), ("aux_u", aux_u, (n_iters, d)),
                         ("w", w, (n_iters, d))):
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape:
            raise ValueError("%s must be a tensor of shape %s, got %s"
                             % (nm, list(shape), tuple(t.shape) if isinstance(t, torch.Tensor)
                                else type(t).__name__))
        if t.device != samples.device:
            raise ValueError("%s is on %s, samples on %s" % (nm, t.device, samples.device))
    if log_probs.device != samples.device:
        raise ValueError("log_probs is on %s, samples on %s" % (log_probs.device, samples.device))
    if n_iters == 0:
        return samples, log_probs
    need_grad = torch.is_grad_enabled() and any(
        t.requires_grad for t in (samples, log_probs, b, aux_u, w))
    return _PlanarFlow.apply(samples, log_probs, b, aux_u, w, need_grad)


def planar_flow_parameters(d, n_iters, device=None, generator=None):
    """``(b, aux_u, w)`` for ``planar_normalizing_flow``: leaf float32 tensors with
    ``requires_grad=True``, initialised as transform.py:148-160 does: ``b`` [n_iters] zeros, and
    for each flow in turn ``aux_u`` then ``w`` ([d] each) drawn from N(0, 0.005^2) with
    ``generator``.  ``device`` defaults to the current CUDA device.  Each call of the flow in a
    model needs a set of its own, as each reference call creates its own variables."""
    device = torch.device("cuda") if device is None else torch.device(device)
    draws = torch.randn((n_iters, 2, d), generator=generator, device=device) * 0.005
    b = torch.zeros(n_iters, device=device).requires_grad_(True)
    aux_u = draws[:, 0].contiguous().requires_grad_(True)
    w = draws[:, 1].contiguous().requires_grad_(True)
    return b, aux_u, w


IAF_MAX_D = 256
_UPDATES = {"normal": 0, "gru": 1}


class LinearAR(object):
    """The linear autoregressive network of transform.py:17-67 for ``n_iters`` flows of
    ``inv_autoregressive_flow`` on samples of width ``d``.

    ``m_w`` and ``s_w`` are ``[n_iters, d, d]`` float32 leaves with ``requires_grad=True``; flow
    ``k`` reads only their entries ``i < j`` (the reference's ``mask``).  They are drawn from
    N(0, 0.005^2) with ``generator`` in the reference's creation order: ``m_w`` of flow 0, ``s_w``
    of flow 0, then flow 1, and so on.  ``device`` defaults to the current CUDA device.

    The reference's ``linear_ar`` creates fresh variables inside every call; here the caller
    creates a ``LinearAR`` once and passes it in, and each flow call in a model needs an object of
    its own.  ``inv_autoregressive_flow`` runs the whole stack on fused kernels when it is given
    one of these."""

    def __init__(self, d, n_iters, device=None, generator=None):
        device = torch.device("cuda") if device is None else torch.device(device)
        self.d, self.n_iters = int(d), int(n_iters)
        draws = torch.randn((self.n_iters, 2, self.d, self.d), generator=generator,
                            device=device) * 0.005
        self.m_w = draws[:, 0].contiguous().requires_grad_(True)
        self.s_w = draws[:, 1].contiguous().requires_grad_(True)

    def parameters(self):
        return [self.m_w, self.s_w]

    def __call__(self, name, id, z, hidden=None):
        """``(m, s)`` of flow ``id`` (transform.py:30-67) in torch; ``hidden`` is ignored, as in
        the reference."""
        d = self.d
        mask = torch.ones(d, d, dtype=z.dtype, device=z.device).triu(1)
        zz = z.reshape(-1, d)
        m = zz @ (mask * self.m_w[id].to(z.dtype))
        s = torch.exp(zz @ (mask * self.s_w[id].to(z.dtype)))
        return m.reshape(z.shape), s.reshape(z.shape)


class _LinearIAF(torch.autograd.Function):
    """The whole stack in one launch (zsb_iaf_fwd_f32).  When a gradient is needed the forward
    pass also keeps every flow's input z; the backward pass (zsb_iaf_bwd_f32) recomputes each
    flow's m and t from it and runs one reverse sweep plus one merge."""

    @staticmethod
    def forward(ctx, samples, log_probs, m_w, s_w, update, need_grad):
        from ._lib import lib, ptr, stream
        n, d = int(m_w.shape[0]), int(m_w.shape[1])
        z = samples.detach().reshape(-1, d).contiguous()
        lq = log_probs.detach().reshape(-1).contiguous()
        mw, sw = m_w.detach().contiguous(), s_w.detach().contiguous()
        R = int(z.shape[0])
        z_out, lq_out = torch.empty_like(z), torch.empty_like(lq)
        ck = torch.empty((n, R, d), dtype=torch.float32, device=z.device) if need_grad else None
        if R > 0:
            lib.call("zsb_iaf_fwd_f32", ptr(z), ptr(lq), ptr(mw), ptr(sw), ptr(z_out),
                     ptr(lq_out), ptr(ck), R, d, n, update, stream())
        if need_grad:
            ctx.save_for_backward(ck, mw, sw)
        ctx.shapes = (tuple(samples.shape), tuple(log_probs.shape), R, d, n, update)
        return z_out.reshape(samples.shape), lq_out.reshape(log_probs.shape)

    @staticmethod
    @once_differentiable
    def backward(ctx, gz, glq):
        from ._lib import lib, ptr, stream
        ck, mw, sw = ctx.saved_tensors
        z_shape, lq_shape, R, d, n, update = ctx.shapes
        if R == 0:
            return (gz.new_zeros(z_shape), glq.reshape(lq_shape), torch.zeros_like(mw),
                    torch.zeros_like(sw), None, None)
        g = gz.to(torch.float32).reshape(R, d).contiguous()
        gl = glq.to(torch.float32).reshape(R).contiguous()
        gz_in = torch.empty_like(g)
        part = torch.empty((lib.load().zsb_iaf_slices(R, d, n), n, 2, d, d), dtype=torch.float32,
                           device=ck.device)
        dmw, dsw = torch.empty_like(mw), torch.empty_like(sw)
        lib.call("zsb_iaf_bwd_f32", ptr(ck), ptr(g), ptr(gl), ptr(mw), ptr(sw), ptr(gz_in),
                 ptr(part), ptr(dmw), ptr(dsw), R, d, n, update, stream())
        return gz_in.reshape(z_shape), glq.reshape(lq_shape), dmw, dsw, None, None


def inv_autoregressive_flow(samples, hidden, log_probs, autoregressive_nn, n_iters,
                            update='normal'):
    """``n_iters`` Inverse Autoregressive Flows (Kingma et al., 2016) along the last axis of
    ``samples``: transform.py:200-282.

    ``samples`` is ``[..., d]`` (rank >= 2) and ``log_probs`` is ``samples.shape[:-1]``.  For each
    flow ``k`` the call takes ``m, s = autoregressive_nn('iaf', k, z, hidden)`` and computes

        update='normal':  z = s z + m,                   log_q -= sum(log s)
        update='gru':     g = sigmoid(s), z = g z + (1 - g) m,  log_q -= sum(log g)
        z = reverse(z, last axis)          (after every flow, the last one included)

    and returns ``(z, log_q)`` after the last flow.  Differentiable w.r.t. ``samples``,
    ``log_probs`` and the network's parameters.

    When ``autoregressive_nn`` is a ``LinearAR`` for ``n_iters`` flows, ``samples`` and
    ``log_probs`` are float32 CUDA tensors on its device and ``1 <= d <= 256``, the whole stack is
    one kernel launch and its gradient one sweep plus one merge; two identical calls give identical
    bits.  There ``log s`` is ``t`` itself rather than ``log(exp(t))``, and ``log sigmoid(s)`` is
    computed stably as ``-softplus(-s)``.  Any other callable, CPU or float64 tensors, or
    ``d > 256`` run the reference's loop in torch through ``autoregressive_nn``.

    One deliberate difference from the reference: an ``update`` other than ``'normal'`` or
    ``'gru'`` raises ``ValueError``, where the reference silently only reverses ``z``.
    ``n_iters = 0`` returns the inputs unchanged."""
    if not isinstance(n_iters, int):
        raise ValueError("n_iters should be type 'int'")
    if samples.dim() < 2:
        raise ValueError("samples should have rank >= 2")
    if log_probs.dim() != samples.dim() - 1:
        raise ValueError("log_probs should have rank (N-1), while N is the rank of samples")
    if tuple(log_probs.shape) != tuple(samples.shape[:-1]):
        raise ValueError("samples and log_probs don't have same shape of (N-1) dims, while N is "
                         "the rank of samples")
    if update not in _UPDATES:
        raise ValueError("update should be 'normal' or 'gru', got %r" % (update,))
    if log_probs.device != samples.device:
        raise ValueError("log_probs is on %s, samples on %s" % (log_probs.device, samples.device))
    d = int(samples.shape[-1])
    fused = isinstance(autoregressive_nn, LinearAR)
    if fused:
        if autoregressive_nn.d != d or autoregressive_nn.n_iters != n_iters:
            raise ValueError("the LinearAR is for d = %d and %d flows, the call has d = %d and "
                             "n_iters = %d" % (autoregressive_nn.d, autoregressive_nn.n_iters, d,
                                               n_iters))
        if autoregressive_nn.m_w.device != samples.device:
            raise ValueError("the LinearAR is on %s, samples on %s"
                             % (autoregressive_nn.m_w.device, samples.device))
    if n_iters <= 0:
        return samples, log_probs
    if (fused and samples.is_cuda and samples.dtype == torch.float32
            and log_probs.dtype == torch.float32 and 1 <= d <= IAF_MAX_D):
        ar = autoregressive_nn
        need_grad = torch.is_grad_enabled() and any(
            t.requires_grad for t in (samples, log_probs, ar.m_w, ar.s_w))
        return _LinearIAF.apply(samples, log_probs, ar.m_w, ar.s_w, _UPDATES[update], need_grad)
    z, log_q = samples, log_probs
    for k in range(n_iters):                          # transform.py:262-275
        m, s = autoregressive_nn('iaf', k, z, hidden)
        if update == 'gru':
            sigma = torch.sigmoid(s)
            z = sigma * z + (1 - sigma) * m
            log_q = log_q - torch.log(sigma).sum(-1)
        else:
            z = s * z + m
            log_q = log_q - torch.log(s).sum(-1)
        z = torch.flip(z, [-1])
    return z, log_q
