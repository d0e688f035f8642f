"""GPU tests of zs.fused.LinearOnehotCategorical, the one-hot categorical dense layer of the
semi-supervised VAE trained by adaptive importance sampling
(examples/semi_supervised_vae/vae_ssl_adaptive_is.py): its draws against the registry's sampler bit
for bit, its log-probabilities and their gradients against float64, the cache of its own sample's
log q, the class indices its samples hand to class_linear, and the fallback outside the fused
domain."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

K_IN = 50


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return torch.tensor(t.detach().cpu().numpy(), dtype=torch.float64)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _weights(rng, C, K, scale=2.0):
    return (T(rng.standard_normal((C, K)) * scale / np.sqrt(K)), T(0.3 * rng.standard_normal(C)))


def _input(zs, rng, R, kind):
    """A dense float activation [R, K_IN], or a 0/1 sample [R, 200] of a fused Bernoulli layer (it
    carries its binary operand plane)."""
    x = T(rng.standard_normal((R, K_IN)))
    if kind == "dense":
        return x
    W, b = _weights(rng, 200, K_IN)
    h = zs.fused.LinearBernoulli(x, W, b, dtype=torch.float32).sample()
    assert h._zsb_pl.binary
    return h


def _registry_sample(zs, logits, S, u):
    """OnehotCategorical(logits).sample(S) -- or, with injected uniforms, the registry's sampler
    fed them -- as float32 one-hot rows [S, *batch, C]."""
    C = int(logits.shape[-1])
    if u is None:
        return zs.distributions.OnehotCategorical(logits, dtype=torch.float32).sample(S)
    draws = zs.ops.sample_categorical(logits, S, u=u)
    return F.one_hot(draws.long(), C).to(torch.float32)


@pytest.mark.parametrize("C", [1, 2, 10, 31, 32, 33, 100, 128])
@pytest.mark.parametrize("R", [1, 127, 129, 1000])
def test_sample_equals_the_registry(zs, C, R):
    """LinearOnehotCategorical.sample == OnehotCategorical(linear(h, W, b)).sample(n) bit for bit,
    from the same zs.random state or the same injected uniforms, for n in {None, 1, 3, 17}, dense
    and binary h; the stored class indices are the one-hot's classes."""
    rng = np.random.RandomState(C * 7 + R)
    for kind in ("dense", "binary"):
        h = _input(zs, rng, R, kind)
        W, b = _weights(rng, C, int(h.shape[-1]))
        logits = zs.fused.linear(h, W, b)
        for n in (None, 1, 3, 17):
            S = 1 if n is None else n
            for inject in (False, True):
                u = T(rng.random_sample((S, R))) if inject else None
                zs.random.set_random_seed(99 + C + S)
                zs.random.set_counter(40)
                got = zs.fused.LinearOnehotCategorical(h, W, b, dtype=torch.float32).sample(n, u=u)
                zs.random.set_counter(40)
                want = _registry_sample(zs, logits, S, u)
                if n is None:
                    want = want.squeeze(0)
                assert got.shape == want.shape and got.dtype == torch.float32
                assert torch.equal(got, want), (kind, n, inject)
                assert inject or zs.random.counter() == 41
                cls, _ = got._zsb_cls
                assert torch.equal(cls.long(), got.reshape(-1, C).argmax(-1))


@pytest.mark.parametrize("C", [2, 10, 33, 128])
def test_sample_edge_uniforms_and_one_class_rows(zs, C):
    """u = 0, u just below 1, and rows where one class holds all the mass (logits around +-80):
    the same classes as the registry's sampler, round-off resolved towards the last class with
    mass."""
    rng = np.random.RandomState(C)
    R, S = 300, 4
    h = T(rng.standard_normal((R, K_IN)))
    W = T(rng.standard_normal((C, K_IN)) * 0.01)
    b = np.full(C, -80.0)
    b[rng.randint(C)] = 80.0
    for bias in (T(0.3 * rng.standard_normal(C)), T(b)):
        logits = zs.fused.linear(h, W, bias)
        for uval in (0.0, 1.0 - 2.0 ** -24, None):
            u = T(rng.random_sample((S, R))) if uval is None else T(np.full((S, R), uval))
            got = zs.fused.LinearOnehotCategorical(h, W, bias, dtype=torch.float32).sample(S, u=u)
            assert torch.equal(got, _registry_sample(zs, logits, S, u)), uval


@pytest.mark.parametrize("dtype", [torch.int32, torch.float32])
def test_sample_dtypes_and_device_epoch(zs, dtype):
    """int32 and float32 one-hot samples, and the device epoch that CUDA-graph replays add to the
    Philox counter."""
    rng = np.random.RandomState(3)
    h = T(rng.standard_normal((300, K_IN)))
    W, b = _weights(rng, 10, K_IN)
    zs.random.enable_device_epoch()
    try:
        zs.random.bump_device_epoch(17)
        zs.random.set_counter(5)
        got = zs.fused.LinearOnehotCategorical(h, W, b, dtype=dtype).sample(4)
        zs.random.set_counter(5)
        want = zs.distributions.OnehotCategorical(zs.fused.linear(h, W, b), dtype=dtype).sample(4)
    finally:
        zs.random.disable_device_epoch()
    assert got.dtype == dtype and torch.equal(got, want)
    assert torch.equal(got.sum(-1), torch.ones_like(got.sum(-1)))


def _lp64(h, W, b, given):
    """float64 OnehotCategorical(h W^T + b).log_prob(given): sum_j given_j log_softmax(l)_j."""
    l = h @ W.t() + b
    return (given * torch.log_softmax(l, -1)).sum(-1)


def _check_lp_and_grads(zs, h, W, b, lp, given64, reduce_w):
    """lp against float64, and the gradients of sum(w * lp) w.r.t. h, W and b."""
    h64, W64, b64 = (N64(t).requires_grad_() for t in (h, W, b))
    want = _lp64(h64, W64, b64, given64)
    np.testing.assert_allclose(lp.detach().cpu().numpy(), want.detach().numpy(), rtol=1e-4,
                               atol=2e-4)
    w = torch.tensor(reduce_w, dtype=torch.float64)
    g = torch.autograd.grad((want * w).sum(), (h64, W64, b64))
    got = torch.autograd.grad((lp * T(reduce_w)).sum(), (h, W, b))
    for name, a, e in zip("hWb", got, g):
        e = e.numpy()
        tol = 2e-4 * max(1.0, float(np.abs(e).max()))
        np.testing.assert_allclose(a.cpu().numpy(), e, rtol=1e-3, atol=tol, err_msg=name)


@pytest.mark.parametrize("C", [1, 10, 33, 128])
@pytest.mark.parametrize("R", [1, 129, 1000])
def test_log_prob_of_own_sample(zs, C, R):
    """log_prob of the layer's own sample returns the stored log q (no second product) and matches
    float64, with its gradients."""
    rng = np.random.RandomState(C + R)
    h = T(rng.standard_normal((R, K_IN))).requires_grad_()
    W, b = (t.requires_grad_() for t in _weights(rng, C, K_IN))
    d = zs.fused.LinearOnehotCategorical(h, W, b)
    y = d.sample(3)
    launches = zs._lib.lib.launches
    lp = d.log_prob(y)
    assert zs._lib.lib.launches == launches          # no launch: the stored log q
    assert lp.shape == (3, R)
    _check_lp_and_grads(zs, h, W, b, lp, N64(y), rng.standard_normal((3, R)))


@pytest.mark.parametrize("C", [1, 10, 33, 128])
@pytest.mark.parametrize("shape", [((5,), (40,)), ((2, 3), (7, 20)), ((), (129,))])
def test_log_prob_of_given_samples(zs, C, shape):
    """[S..., *lead, C] given one-hot rows against the shared logits, with gradients."""
    sax, lead = shape
    rng = np.random.RandomState(C + len(sax))
    h = T(rng.standard_normal(lead + (K_IN,))).requires_grad_()
    W, b = (t.requires_grad_() for t in _weights(rng, C, K_IN))
    cls = rng.randint(C, size=sax + lead)
    given = T(np.eye(C)[cls])
    lp = zs.fused.LinearOnehotCategorical(h, W, b).log_prob(given)
    assert lp.shape == sax + lead
    _check_lp_and_grads(zs, h, W, b, lp, N64(given), rng.standard_normal(sax + lead))


@pytest.mark.parametrize("C", [2, 10, 128])
def test_log_prob_of_suffix_broadcast_labels(zs, C):
    """Labels [N, C] against h [K, N, H] (row r of the flattened lead reads label r % N), and
    labels against h [N, H] itself."""
    rng = np.random.RandomState(C)
    N, K = 100, 10
    W, b = (t.requires_grad_() for t in _weights(rng, C, K_IN))
    labels = T(np.eye(C)[rng.randint(C, size=N)])
    for lead in ((K, N), (N,)):
        h = T(rng.standard_normal(lead + (K_IN,))).requires_grad_()
        lp = zs.fused.LinearOnehotCategorical(h, W, b).log_prob(labels)
        assert lp.shape == lead
        _check_lp_and_grads(zs, h, W, b, lp, N64(labels).expand(lead + (C,)),
                            rng.standard_normal(lead))


def test_log_prob_of_non_one_hot_given(zs):
    """A given that is not one-hot (counts, fractions, negatives) is scored exactly as
    OnehotCategorical._log_prob scores it: sum_j given_j log_softmax(l)_j."""
    rng = np.random.RandomState(11)
    C, R = 33, 300
    h = T(rng.standard_normal((R, K_IN))).requires_grad_()
    W, b = (t.requires_grad_() for t in _weights(rng, C, K_IN))
    given = T(rng.standard_normal((2, R, C)))
    lp = zs.fused.LinearOnehotCategorical(h, W, b).log_prob(given)
    _check_lp_and_grads(zs, h, W, b, lp, N64(given), rng.standard_normal((2, R)))


def test_log_prob_group_ndims(zs):
    rng = np.random.RandomState(12)
    h = T(rng.standard_normal((6, 40, K_IN)))
    W, b = _weights(rng, 10, K_IN)
    d0 = zs.fused.LinearOnehotCategorical(h, W, b)
    d1 = zs.fused.LinearOnehotCategorical(h, W, b, group_ndims=1)
    y = d0.sample(2)
    assert torch.allclose(d1.log_prob(y), d0.log_prob(y).sum(-1), rtol=1e-6, atol=1e-5)
    assert d1.batch_shape == (6, 40) and d1.value_shape == (10,)


def test_in_place_changes_invalidate_the_cached_log_q(zs):
    """An in-place change of h, W, b or the sample makes log_prob score the sample anew, on every
    later call and after a second change; a draw after the change uses the changed parameters."""
    rng = np.random.RandomState(21)
    C, R = 10, 200
    for which in ("h", "W", "b", "y"):
        h = T(rng.standard_normal((R, K_IN)))
        W, b = _weights(rng, C, K_IN)
        d = zs.fused.LinearOnehotCategorical(h, W, b, dtype=torch.float32)
        y = d.sample(2)
        for scale in (1.7, -0.6):
            if which == "h":
                h.mul_(scale)
            elif which == "W":
                W.mul_(scale)
            elif which == "b":
                b.add_(scale)
            else:
                y.copy_(torch.roll(y, 1, -1))
            for _ in range(2):
                lp = d.log_prob(y)
                want = _lp64(N64(h), N64(W), N64(b), N64(y))
                np.testing.assert_allclose(lp.cpu().numpy(), want.numpy(), rtol=1e-4, atol=2e-4,
                                           err_msg=which)
        zs.random.set_counter(3)
        got = d.sample(2)
        zs.random.set_counter(3)
        # the logits of the changed parameters, through a copy of h that has no cached planes
        ref = zs.distributions.OnehotCategorical(zs.fused.linear(h.clone(), W, b),
                                                 dtype=torch.float32)
        assert torch.equal(got, ref.sample(2)), which


def test_inference_mode(zs):
    """Inference tensors carry no version counter: sample() runs and equals the sample drawn
    outside inference mode; nothing is cached; log_prob and class_linear still work."""
    rng = np.random.RandomState(5)
    h = T(rng.standard_normal((200, K_IN)))
    W, b = _weights(rng, 10, K_IN)
    Wx, Wy = _weights(rng, 30, K_IN)[0], _weights(rng, 30, 10)[0]
    zs.random.set_counter(9)
    want = zs.fused.LinearOnehotCategorical(h, W, b).sample(2)
    with torch.inference_mode():
        zs.random.set_counter(9)
        d = zs.fused.LinearOnehotCategorical(h, W, b)
        got = d.sample(2)
        assert getattr(got, "_zsb_cls", None) is None
        lq = d.log_prob(got)
        z = zs.fused.class_linear(h.expand(2, 200, K_IN), Wx, Wy, got)
    assert torch.equal(got, want)
    np.testing.assert_allclose(lq.cpu().numpy(),
                               _lp64(N64(h), N64(W), N64(b), N64(got)).numpy(), rtol=1e-4,
                               atol=2e-4)
    assert z.shape == (2, 200, 30)


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.name for e in prof.events() if e.device_type.name == "CUDA"]


def test_class_linear_reads_the_sample_class_indices(zs):
    """class_linear fed a sampled y gives bit for bit what it gives for a copy of its one-hot,
    without the argmax launch the copy needs."""
    rng = np.random.RandomState(8)
    h = T(rng.standard_normal((3, 100, K_IN)))
    x = T(rng.standard_normal((100, 64)))
    W, b = _weights(rng, 10, K_IN)
    Wx, Wy = _weights(rng, 40, 64)[0], _weights(rng, 40, 10)[0]
    y = zs.fused.LinearOnehotCategorical(h, W, b).sample()          # [3, 100, 10]
    xs = x.expand(3, 100, 64).contiguous()
    ycopy = y.clone().to(torch.float32)
    zs.fused.class_linear(xs, Wx, Wy, ycopy)        # the operand planes of xs, cached on it
    got, k_got = _kernel_names(lambda: zs.fused.class_linear(xs, Wx, Wy, y))
    want, k_want = _kernel_names(lambda: zs.fused.class_linear(xs, Wx, Wy, ycopy))
    assert torch.equal(got, want)
    argmax = [k for k in k_want if "rgMax" in k or "argmax" in k.lower()]
    assert argmax, k_want
    assert not [k for k in k_got if "rgMax" in k or "argmax" in k.lower()], k_got
    assert len(k_got) < len(k_want)
    y.zero_()                        # the indices no longer describe y: back to the argmax
    assert torch.equal(zs.fused.class_linear(xs, Wx, Wy, y),
                       zs.fused.class_linear(xs, Wx, Wy, torch.zeros_like(ycopy)))


def test_fallback_outside_the_fused_domain(zs):
    """C = 129 and float64 parameters run OnehotCategorical(linear(h, W, b)): the same samples and
    log-probabilities exactly; CPU tensors raise what the registry raises for them."""
    from zhusuan_b200._lib import ZsbError
    rng = np.random.RandomState(4)
    h = T(rng.standard_normal((120, K_IN)))
    for C, dt in ((129, torch.float32), (10, torch.float64)):
        W, b = (t.to(dt) for t in _weights(rng, C, K_IN))
        hh = h.to(dt)
        d = zs.fused.LinearOnehotCategorical(hh, W, b)
        assert not d._fused
        zs.random.set_counter(70)
        got = d.sample(3)
        zs.random.set_counter(70)
        ref = zs.distributions.OnehotCategorical(zs.fused.linear(hh, W, b))
        want = ref.sample(3)
        assert torch.equal(got, want)
        assert torch.equal(d.log_prob(got), ref.log_prob(got))
        u = T(rng.random_sample((3, 120)))
        want_u = F.one_hot(zs.ops.sample_categorical(zs.fused.linear(hh, W, b), 3, u=u).long(),
                           C).to(torch.int32)
        assert torch.equal(d.sample(3, u=u), want_u)
    hc, (Wc, bc) = h.cpu(), (t.cpu() for t in _weights(rng, 10, K_IN))
    d = zs.fused.LinearOnehotCategorical(hc, Wc, bc)
    ref = zs.distributions.OnehotCategorical(F.linear(hc, Wc, bc))
    for fn in (lambda o: o.sample(2), lambda o: o.log_prob(torch.eye(10)[:1].expand(120, 10))):
        with pytest.raises(ZsbError):
            fn(ref)
        with pytest.raises(ZsbError):
            fn(d)
