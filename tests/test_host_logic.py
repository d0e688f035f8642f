"""CPU tests of the host side: the C-ABI library loads and exports every
symbol include/zsb200.h declares, the plugin (BayesianNet / StochasticTensor /
MetaBayesianNet) contract, error conventions, and that the product path fails
loudly without a GPU (no CPU fallback).  No kernel is launched here."""
import os
import re
from unittest import mock

import numpy as np
import pytest
import torch

import zhusuan_b200 as zs
from zhusuan_b200 import _lib
from zhusuan_b200.framework.meta_bn import Local

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    protos = _lib.parse_header()
    assert len(protos) >= 54
    dll = _lib.lib.load()
    for name in protos:
        assert hasattr(dll, name), name
    assert dll.zsb_version() >= 100
    # every extern "C" zsb_* definition in csrc is declared in the header
    src = ""
    for f in os.listdir(os.path.join(ROOT, "zhusuan_b200", "csrc")):
        if f.endswith(".cu"):
            src += open(os.path.join(ROOT, "zhusuan_b200", "csrc", f)).read()
    defined = set(re.findall(r"^int (zsb_\w+)\(", src, flags=re.M))
    internal = {"zsb_check_launch", "zsb_dense_leapfrog_tc_launch",
                "zsb_dense_tc_ntiles", "zsb_dense_split_lo_launch",
                "zsb_dense_leapfrog_h16_launch", "zsb_dense_h16_prepare_launch",
                "zsb_dense_res_h16_launch", "zsb_dense_select_planes_launch"}
    assert defined - internal <= set(protos), defined - internal - set(protos)


@pytest.mark.parametrize("impl", [3, 4, 6, -1])
def test_dense_impl_outside_the_four_paths_is_rejected(impl):
    """dense_impl / GaussianLogJoint(impl=) take None, 0, 1, 2 or 5; anything else raises before
    any launch, so this runs on host tensors."""
    P = np.eye(64)
    x = torch.zeros(4, 64)
    with pytest.raises(ValueError, match="dense_impl must be"):
        zs.HMC(dense_impl=impl).sample(zs.fused.GaussianLogJoint(P, device="cpu"), {}, {"x": x})
    with pytest.raises(ValueError, match="dense_impl must be"):
        zs.HMC().sample(zs.fused.GaussianLogJoint(P, device="cpu", impl=impl), {}, {"x": x})


def test_header_cites_reference_lines():
    h = open(os.path.join(ROOT, "include", "zsb200.h")).read()
    for cite in ["hmc.py:21-23", "hmc.py:46-61", "hmc.py:89-112",
                 "univariate.py:174-181", "utils.py:177-196",
                 "sgmcmc.py:195-200", "multivariate.py:435-443"]:
        assert cite in h, cite


def test_no_cpu_fallback_and_error_string():
    dll = _lib.lib.load()
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert dll.zsb_device_count() == 0
    # a compute entry point with host tensors must raise, not fall back
    d = zs.distributions.Normal(torch.zeros(3), std=torch.ones(3))
    with pytest.raises(_lib.ZsbError, match="no CPU fallback"):
        d.log_prob(torch.zeros(3))
    with pytest.raises(_lib.ZsbError, match="no CPU fallback"):
        zs.log_mean_exp(torch.zeros(4, 3), 0)
    # argument validation happens before any launch and sets the message
    with pytest.raises(_lib.ZsbError, match="bad sizes"):
        _lib.lib.call("zsb_logprob_normal_f32", None, 0, None, 0, None, 0,
                      None, 0, 0, None)


def test_no_environment_switches():
    """What runs is chosen by arguments, never by the environment: no kernel source calls getenv
    and no module of the package reads os.environ."""
    csrc = os.path.join(ROOT, "zhusuan_b200", "csrc")
    for f in sorted(os.listdir(csrc)):
        if f.endswith((".cu", ".cuh")):
            assert "getenv" not in open(os.path.join(csrc, f)).read(), f
    for dirpath, _, files in os.walk(os.path.join(ROOT, "zhusuan_b200")):
        for f in files:
            if f.endswith(".py"):
                s = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"\benviron\b|\bgetenv\b", s), os.path.join(dirpath, f)


def test_product_does_not_import_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "zhusuan_b200")):
        for f in files:
            if f.endswith(".py"):
                s = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", s, re.M), f


# ------------------------------------------------------------ plugin contract
def test_stochastic_tensor_duck_typed_distribution():
    """tests/framework/test_base.py:16-40 with unittest.mock."""
    static_shape = mock.Mock()
    samples = mock.Mock(shape=static_shape)
    log_probs, probs = mock.Mock(), mock.Mock()
    distribution = mock.Mock(sample=mock.Mock(return_value=samples),
                             log_prob=mock.Mock(return_value=log_probs),
                             prob=mock.Mock(return_value=probs),
                             dtype=torch.int32)
    bn = zs.BayesianNet()
    s_tensor = bn.stochastic('test', distribution)
    assert s_tensor.name == 'test'
    assert s_tensor.dist is distribution
    with pytest.warns(FutureWarning):
        assert s_tensor.distribution is distribution
    assert s_tensor.dtype == torch.int32
    assert s_tensor.tensor is samples
    assert s_tensor.cond_log_p is log_probs
    distribution.log_prob.assert_called_once_with(samples)
    with pytest.warns(FutureWarning):
        assert s_tensor.log_prob(None) is log_probs
    with pytest.warns(FutureWarning):
        assert s_tensor.prob(None) is probs
    assert s_tensor.get_shape() is static_shape
    assert s_tensor.shape is static_shape
    assert s_tensor.bn is bn
    assert not s_tensor.is_observed()


def test_bayesian_net_names_and_queries():
    dist = mock.Mock(dtype=torch.float32,
                     sample=mock.Mock(return_value=torch.zeros(2)),
                     log_prob=mock.Mock(return_value=torch.ones(2)))
    del dist.get_batch_shape
    bn = zs.BayesianNet()
    a = bn.stochastic('a', dist)
    with pytest.raises(ValueError, match="Names should be unique"):
        bn.stochastic('a', dist)
    c = bn.deterministic('c', torch.arange(3.))
    assert bn['a'] is a and bn.get('c') is c
    assert bn.get(['a', 'c'])[0] is a
    with pytest.raises(ValueError, match="There isn't a node named 'z'"):
        bn['z']
    with pytest.raises(TypeError, match="Expected string"):
        bn[3]
    with pytest.raises(ValueError, match="is deterministic"):
        bn.cond_log_prob('c')
    with pytest.raises(TypeError, match="does not support replacement"):
        bn['a'] = a
    assert torch.equal(bn.cond_log_prob('a'), torch.ones(2))
    assert torch.equal(bn.log_joint(), torch.ones(2))
    assert set(bn.nodes) == {'a', 'c'}


def test_meta_bayesian_net_observe_and_log_joint_override():
    calls = []

    def make_dist(val):
        d = mock.Mock(dtype=torch.float32)
        d.sample = mock.Mock(return_value=torch.full((2,), val))
        d.log_prob = mock.Mock(side_effect=lambda given: given * 2)
        del d.get_batch_shape
        return d

    @zs.meta_bayesian_net(scope="model")
    def build(k):
        calls.append(k)
        bn = zs.BayesianNet()
        z = bn.stochastic('z', make_dist(1.0))
        bn.stochastic('x', make_dist(5.0))
        bn.deterministic('zz', z.tensor + k)
        return bn
    m = build(10.)
    assert isinstance(m, zs.MetaBayesianNet)
    bn = m.observe()
    assert not bn['z'].is_observed() and calls == [10.]
    assert torch.equal(bn.log_joint(), torch.full((2,), 12.0))
    obs = torch.tensor([3., 4.])
    bn2 = m.observe(x=obs)
    assert bn2['x'].is_observed() and bn2['x'].tensor is obs
    assert torch.equal(bn2.log_joint(), torch.tensor([8., 10.]))
    assert torch.equal(bn2['zz'], torch.full((2,), 11.0))
    m.log_joint = lambda b: b.cond_log_prob('x') * 100
    assert torch.equal(m.observe(x=obs).log_joint(), obs * 200)
    m.log_joint = 3
    with pytest.raises(TypeError, match="non-callable"):
        m.observe().log_joint()
    with pytest.raises(RuntimeError, match="No contexts"):
        Local.get_context()
    with pytest.raises(ValueError, match="Cannot reuse"):
        zs.meta_bayesian_net(reuse_variables=True)(lambda: None)()


def test_tensor_like_arithmetic():
    dist = mock.Mock(dtype=torch.float32,
                     sample=mock.Mock(return_value=torch.tensor([1., 2.])))
    del dist.get_batch_shape
    s = zs.BayesianNet().stochastic('s', dist)
    assert torch.equal(s + 1, torch.tensor([2., 3.]))
    assert torch.equal(2 * s, torch.tensor([2., 4.]))
    assert torch.equal(-s, torch.tensor([-1., -2.]))
    assert torch.equal(torch.exp(s), torch.exp(torch.tensor([1., 2.])))
    assert float(torch.mean(s)) == 1.5
    with pytest.raises(TypeError, match="as a Python `bool`"):
        bool(s)
    with pytest.raises(TypeError, match="not iterable"):
        iter(s)


def test_observation_shape_and_dtype_checks():
    d = zs.distributions.Normal(torch.zeros(2, 3), std=torch.ones(3))
    bn = zs.BayesianNet(observed={'a': torch.zeros(5, 4)})
    with pytest.raises(ValueError, match=r"Incompatible shapes of "
                                         r"StochasticTensor\('a'\)"):
        bn.stochastic('a', d)
    bn = zs.BayesianNet(observed={'a': torch.zeros(2, 3, dtype=torch.int32)})
    with pytest.raises(ValueError, match=r"Incompatible types of "
                                         r"StochasticTensor\('a'\)"):
        bn.stochastic('a', d)


def test_distribution_constructor_contract():
    N = zs.distributions.Normal
    with pytest.raises(ValueError, match="Either `std` or `logstd`"):
        N(0.)
    with pytest.raises(ValueError, match="Either `std` or `logstd`"):
        N(0., std=1., logstd=0.)
    with pytest.raises(ValueError, match="broadcastable"):
        N(torch.zeros(2, 3), std=torch.ones(4))
    with pytest.raises(TypeError, match="must have the same dtype as"):
        N(torch.zeros(2), std=torch.ones(2, dtype=torch.float64))
    with pytest.raises(TypeError, match="must have a dtype in"):
        zs.distributions.Bernoulli(torch.zeros(2, dtype=torch.int32))
    with pytest.raises(ValueError, match="group_event_ndims"):
        N(0., std=1., group_event_ndims=1)
    with pytest.raises(ValueError, match="non-negative"):
        N(0., std=1., group_ndims=-1)
    d = N(torch.zeros(4, 1), logstd=torch.zeros(3), group_ndims=1)
    assert tuple(d.get_batch_shape()) == (4, 3)
    assert tuple(d.batch_shape) == (4, 3) and tuple(d.value_shape) == ()
    assert d.dtype == torch.float32 and d.is_continuous \
        and d.is_reparameterized
    with pytest.raises(ValueError, match="broadcast to match"):
        d._check_input_shape(torch.zeros(5, 7))
    c = zs.distributions.Categorical(torch.zeros(2, 5))
    assert tuple(c.get_batch_shape()) == (2,) and c.n_categories == 5
    assert zs.distributions.Discrete is zs.distributions.Categorical
    with pytest.raises(ValueError, match="rank >= 1"):
        zs.distributions.Categorical(torch.tensor(0.))
    with pytest.raises(ValueError, match="at least 2"):
        zs.distributions.Dirichlet(torch.ones(3, 1))
    m = zs.distributions.MultivariateNormalCholesky(
        torch.zeros(2, 3), torch.eye(3).expand(2, 3, 3).contiguous())
    assert tuple(m.get_value_shape()) == (3,)
    with pytest.raises(ValueError, match="compatible shape with mean"):
        zs.distributions.MultivariateNormalCholesky(torch.zeros(2, 3),
                                                    torch.eye(4))
    u = zs.distributions.UnnormalizedMultinomial(torch.zeros(2, 6))
    assert tuple(u.get_value_shape()) == (6,)
    with pytest.raises(NotImplementedError, match="does not support sampling"):
        u.sample(1)


def test_sampler_and_objective_argument_contract():
    with pytest.raises(ValueError, match="If adapt mass is set"):
        zs.HMC(adapt_mass=True)
    h = zs.HMC(step_size=0.1, adapt_step_size=True, adapt_mass=True,
               mass_collect_iters=7)
    assert h.mass_collect_iters == 7
    assert zs.HMC(mass_collect_iters=7).mass_collect_iters == 0  # hmc.py:276
    with pytest.raises(TypeError, match=r"latent\['x'\] is not a"):
        zs.HMC().sample(lambda o: 0, {}, {"x": 1.0})
    with pytest.raises(TypeError, match=r"latent\['w'\] is not a"):
        zs.SGHMC(1e-3).sample(lambda o: 0, {}, {"w": np.zeros(3)})
    # a latent that does not carry the chain axes of the log-joint is rejected up front (the
    # kernels would otherwise walk chains * row_len elements of a shorter tensor)
    import torch
    with pytest.raises(ValueError, match="must start with the chain axes"):
        zs.SGLD(1e-3).sample(lambda o: torch.zeros(10) + o["w"].sum(), {},
                             {"w": torch.zeros(5)})
    s = zs.SGHMC(1e-3, n_iter_resample_v=None)
    assert s.n_iter_resample_v == 0 and s.second_order
    p = zs.PSGLD(1e-3)
    assert p.preconditioner_hparams.decay == 0.9
    assert p.preconditioner_hparams.epsilon == 1e-3
    with pytest.raises(ValueError, match="the `axis` argument must be"):
        zs.variational.iw_objective(lambda o: 0, {}, latent={})
    with pytest.raises(ValueError, match="both are specified or both are not"):
        zs.variational.elbo(lambda o: 0, {})
    with pytest.raises(ValueError, match="both are specified or both are not"):
        zs.variational.elbo(lambda o: 0, {}, latent={},
                            variational=zs.BayesianNet())
    with pytest.raises(TypeError, match="should be a BayesianNet instance"):
        zs.variational.elbo(lambda o: 0, {}, variational=3)
    assert zs.variational.iw_objective is \
        zs.variational.importance_weighted_objective


def test_variational_objective_wiring_with_mocks():
    """base.py:70-73, 117-138, 169-183: latent nodes of `variational` become
    observations of the model; entropy = -sum log q."""
    z_sample = torch.tensor([1., 2., 3.])
    qd = mock.Mock(dtype=torch.float32,
                   sample=mock.Mock(return_value=z_sample),
                   log_prob=mock.Mock(return_value=torch.tensor([.1, .2, .3])))
    del qd.get_batch_shape
    variational = zs.BayesianNet()
    variational.stochastic('z', qd)
    seen = {}

    @zs.meta_bayesian_net()
    def model():
        bn = zs.BayesianNet()
        pd = mock.Mock(dtype=torch.float32,
                       log_prob=mock.Mock(side_effect=lambda g: g * 10))
        del pd.get_batch_shape
        node = bn.stochastic('z', pd)
        seen['z'] = node
        xd = mock.Mock(dtype=torch.float32,
                       log_prob=mock.Mock(return_value=torch.zeros(3)))
        del xd.get_batch_shape
        bn.stochastic('x', xd)
        return bn
    obj = zs.variational.elbo(model(), {'x': torch.zeros(3)},
                              variational=variational)
    assert obj.variational is variational and obj.meta_bn is not None
    lj = obj._log_joint_term()
    assert seen['z'].is_observed() and seen['z'].tensor is z_sample
    assert torch.equal(lj, z_sample * 10)
    assert torch.allclose(obj._entropy_term(), -torch.tensor([.1, .2, .3]))
    assert torch.allclose(obj.tensor, z_sample * 10 - torch.tensor([.1, .2, .3]))
    assert torch.allclose(obj.sgvb(), -obj.tensor)
    # un-modelled latent -> ValueError (base.py:91-97)
    obj2 = zs.variational.elbo(model(), {}, variational=variational)
    with pytest.raises(ValueError, match="neither observed nor provided"):
        obj2.bn


def test_shard_chains_partition():
    from zhusuan_b200 import dist
    assert dist.world() == (1, 0)
    assert dist.shard_chains(65536) == (0, 65536)


def test_added_distribution_and_estimator_contracts_need_no_gpu():
    """Argument checks of the added distributions / objectives fire before any kernel call
    (messages of zhusuan/distributions/univariate.py and variational/*.py)."""
    import warnings
    import torch
    import zhusuan_b200 as zs
    D = zs.distributions
    one = torch.ones(3)
    with pytest.raises(ValueError, match="should be broadcastable to match"):
        D.Beta(torch.ones(2), one)
    with pytest.raises(ValueError, match="Either std or logstd"):
        D.FoldNormal(one, std=one, logstd=one)
    with pytest.raises(ValueError, match="n_experiments must be positive"):
        D.Binomial(one, -1)
    with pytest.raises(TypeError, match="must have the same dtype as"):
        D.Uniform(one, one.double())
    with pytest.raises(TypeError):
        D.Poisson(torch.ones(3, dtype=torch.int32))
    assert tuple(D.Laplace(torch.zeros(4, 1), one).get_batch_shape()) == (4, 3)
    assert D.Gamma(one, one).is_reparameterized is False and D.Poisson(one).dtype == torch.int32
    with pytest.raises(ValueError, match="group_ndims must be 1"):
        zs.fused.LinearBernoulli(torch.ones(2, 4), torch.ones(5, 4), group_ndims=0)
    x = torch.zeros(6)
    lj = lambda obs: -obs["x"] ** 2
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj = zs.variational.klpq(lj, observed={}, latent={"x": [x, -x]}, axis=0)
        iw = zs.variational.iw_objective(lj, observed={}, latent={"x": [x[:1], -x[:1]]}, axis=0)
    with pytest.raises(NotImplementedError, match="can only be optimized"):
        obj.tensor
    with pytest.raises(ValueError, match="larger than 1"):
        iw.vimco()
    bn = zs.BayesianNet()
    for name in ("gamma", "beta", "inverse_gamma", "poisson", "binomial", "laplace", "uniform",
                 "fold_normal", "bin_concrete", "bin_gumbel_softmax"):
        assert callable(getattr(bn, name))


def test_user_defined_distribution_subclass_gets_the_group_sum():
    """tests/distributions/test_base.py:15-140: a plugin subclass returns the UN-grouped log
    density from `_log_prob`; the base class checks shapes and sums the last `group_ndims`
    axes (here with the kernel entry point patched by a torch sum: no GPU in this test)."""
    from zhusuan_b200.distributions import Distribution
    from zhusuan_b200 import ops

    class Dist(Distribution):
        def __init__(self, group_ndims=0):
            super(Dist, self).__init__(torch.float32, torch.float32, is_continuous=True,
                                       is_reparameterized=True, group_ndims=group_ndims)

        def _get_value_shape(self):
            return torch.Size([5])

        def _get_batch_shape(self):
            return torch.Size([2, 3, 4])

        def _sample(self, n_samples):
            return torch.ones(n_samples, 2, 3, 4, 5)

        def _log_prob(self, given):
            return torch.zeros_like(given).sum(-1)

    base = Distribution(torch.float32, torch.float32, True, True, group_ndims=2)
    assert (base.dtype, base.is_continuous, base.group_ndims) == (torch.float32, True, 2)
    for call in (base._get_value_shape, base._get_batch_shape) if hasattr(
            base, "_get_value_shape") else ():
        with pytest.raises((NotImplementedError, AttributeError)):
            call()
    with pytest.raises(NotImplementedError):
        base._sample(1)
    with pytest.raises(NotImplementedError):
        base._log_prob(torch.ones(2, 3, 4, 5))
    with pytest.raises(ValueError, match="must be non-negative"):
        Distribution(torch.float32, torch.float32, True, True, False, -1)

    d = Dist(group_ndims=2)
    assert tuple(d.get_value_shape()) == (5,) and tuple(d.batch_shape) == (2, 3, 4)
    assert tuple(d.sample().shape) == (2, 3, 4, 5)
    for n in (1, 2):
        assert tuple(d.sample(n_samples=n).shape) == (n, 2, 3, 4, 5)
    assert tuple(d.sample(torch.tensor(3)).shape) == (3, 2, 3, 4, 5)
    with pytest.raises(ValueError, match="should be a scalar"):
        d.sample(torch.tensor([1, 2]))
    fake = lambda x, g: x.sum(dim=tuple(range(-g, 0))) if g else x
    with mock.patch.object(ops, "group_sum", side_effect=fake) as gs:
        lp = d.log_prob(torch.ones(2, 3, 4, 5))
        assert tuple(lp.shape) == (2,) and float(lp.abs().sum()) == 0.0
        assert tuple(d.log_prob(torch.ones(1, 2, 3, 4, 5)).shape) == (1, 2)
        assert gs.call_count == 2
        assert tuple(Dist(0).log_prob(torch.ones(2, 3, 4, 5)).shape) == (2, 3, 4)
        assert gs.call_count == 2                      # group_ndims = 0: no call
    with pytest.raises(ValueError, match=r"broadcast to match batch_shape \+ value_shape"):
        d.log_prob(torch.ones(3, 3, 4, 5))
    # built-in classes fuse the sum into their kernels
    assert zs.distributions.Normal(0., std=1.)._group_sum_in_log_prob is True


def test_deprecated_query_api_of_bayesian_net():
    """bn.py:1200-1249: outputs / local_log_prob / query still answer, with FutureWarnings."""
    def dist(v):
        d = mock.Mock(dtype=torch.float32, sample=mock.Mock(return_value=torch.full((2,), v)),
                      log_prob=mock.Mock(side_effect=lambda g: g * 3))
        del d.get_batch_shape
        return d
    bn = zs.BayesianNet()
    bn.stochastic('a', dist(1.)); bn.stochastic('b', dist(2.))
    with pytest.warns(FutureWarning, match="outputs"):
        assert torch.equal(bn.outputs('a'), torch.full((2,), 1.))
    with pytest.warns(FutureWarning):
        outs = bn.outputs(['a', 'b'])
    assert torch.equal(outs[1], torch.full((2,), 2.))
    with pytest.warns(FutureWarning, match="local_log_prob"):
        assert torch.equal(bn.local_log_prob('b'), torch.full((2,), 6.))
    with pytest.warns(FutureWarning, match="query"):
        o, lp = bn.query('a', outputs=True, local_log_prob=True)
    assert torch.equal(o, torch.full((2,), 1.)) and torch.equal(lp, torch.full((2,), 3.))
    with pytest.warns(FutureWarning):
        pairs = bn.query(['a', 'b'], outputs=True, local_log_prob=True)
    assert torch.equal(pairs[1][0], torch.full((2,), 2.)) and torch.equal(pairs[1][1],
                                                                          torch.full((2,), 6.))
    with pytest.warns(FutureWarning), pytest.raises(ValueError, match="No query options"):
        bn.query('a')


def test_top_level_names_of_the_reference_package():
    """zhusuan/__init__.py and the `__all__` lists it pulls in (hmc.py:15-18, sgmcmc.py:15-21,
    evaluation.py:17-19, utils.py:11-15, framework/{bn,meta_bn,utils}.py)."""
    for name in ["distributions", "variational", "StochasticTensor", "BayesianNet",
                 "MetaBayesianNet", "meta_bayesian_net", "reuse_variables", "reuse", "HMCInfo",
                 "HMC", "SGMCMC", "SGLD", "PSGLD", "SGHMC", "SGNHT", "is_loglikelihood", "AIS",
                 "TensorArithmeticMixin", "log_mean_exp", "merge_dicts"]:
        assert hasattr(zs, name), name
    for name in ["elbo", "klpq", "iw_objective", "importance_weighted_objective",
                 "EvidenceLowerBoundObjective", "InclusiveKLObjective",
                 "ImportanceWeightedObjective", "VariationalObjective"]:
        assert hasattr(zs.variational, name), name
    with pytest.warns(FutureWarning, match="renamed to `reuse_variables\\(\\)`"):
        deco = zs.reuse("scope")
    assert deco(lambda: 3)() == 3
    assert zs.merge_dicts({"a": 1}, {"b": 2}, {"a": 3}) == {"a": 3, "b": 2}


def test_context_frames_are_per_thread():
    """framework/utils.py Context: frames nest per class and per thread."""
    import threading
    from zhusuan_b200.framework.utils import Context

    class A(Context):
        pass

    class B(Context):
        pass
    seen = {}
    with A() as a:
        with B() as b:
            assert A.get_context() is a and B.get_context() is b

            def other():
                try:
                    A.get_context()
                    seen["other"] = "found"
                except RuntimeError as e:
                    seen["other"] = str(e)
            t = threading.Thread(target=other)
            t.start()
            t.join()
        with pytest.raises(RuntimeError, match="No contexts on the stack"):
            B.get_context()
    assert seen["other"] == "No contexts on the stack."


def test_bnn_prior_logstd_as_the_fused_kernel_reads_it():
    """BNNRegressionLogJoint.fused_prior_logstd: the fused BNN kernel reads a prior log-stddev by
    flat index modulo its size over one chain's weights.  Suffix shapes go through untouched,
    shapes that only broadcast are expanded (once, until modified in place), and shapes with
    chain axes are refused so the step takes the generic path."""
    H, in1 = 5, 4
    lj = lambda ls: zs.fused.BNNRegressionLogJoint(torch.zeros(2, in1 - 1), torch.zeros(2),
                                                   [ls, torch.zeros(1, H + 1)], 10)
    for shape in [(H, in1), (in1,), (), (1, 1), (1, H, in1)]:
        m = lj(torch.randn(shape))
        assert m.fused_prior_logstd(0, (H, in1)) is m.logstds[0], shape
    for shape in [(3, H, in1), (3, H, 1), (H, 2), (H + 1, in1)]:
        assert lj(torch.randn(shape)).fused_prior_logstd(0, (H, in1)) is None, shape
    for shape in [(H, 1), (1, H, 1)]:
        m = lj(torch.randn(shape))
        e = m.fused_prior_logstd(0, (H, in1))
        assert e.shape == (H, in1) and e.is_contiguous()
        flat = e.reshape(-1)
        for i in range(H * in1):              # the kernel's index: i % numel over [H, n_in+1]
            assert flat[i % flat.numel()] == m.logstds[0].reshape(H)[i // in1]
        assert m.fused_prior_logstd(0, (H, in1)) is e           # cached: no launch per step
        m.logstds[0].add_(1.0)
        e2 = m.fused_prior_logstd(0, (H, in1))
        assert torch.equal(e2, e + 1.0)
    m = lj(torch.randn(H, in1))
    m.logstds[1] = torch.randn(3, 1, H + 1)
    assert m.fused_prior_logstd(1, (1, H + 1)) is None
