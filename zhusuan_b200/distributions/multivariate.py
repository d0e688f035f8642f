"""MultivariateNormalCholesky / UnnormalizedMultinomial / Dirichlet on the
H100 kernels (zhusuan/distributions/multivariate.py:41-192, 339-446, 570-680)."""
import torch

from .. import ops
from ..utils import convert_to_tensor
from .base import Distribution
from .utils import (assert_same_float_dtype, assert_dtype_is_int_or_float,
                    assert_rank_at_least)

__all__ = ["MultivariateNormalCholesky", "UnnormalizedMultinomial",
           "BagofCategoricals", "Dirichlet", "Multinomial",
           "OnehotCategorical", "OnehotDiscrete"]


class MultivariateNormalCholesky(Distribution):
    """multivariate.py:41-192."""
    _group_sum_in_log_prob = True

    def __init__(self, mean, cov_tril, group_ndims=0, is_reparameterized=True,
                 use_path_derivative=False, check_numerics=False, **kwargs):
        self._check_numerics = check_numerics
        self._mean = convert_to_tensor(mean)
        assert_rank_at_least(self._mean, 1, 'MultivariateNormalCholesky.mean')
        self._n_dim = int(self._mean.shape[-1])
        self._cov_tril = convert_to_tensor(cov_tril, device=self._mean.device)
        assert_rank_at_least(self._cov_tril, 2,
                             'MultivariateNormalCholesky.cov_tril')
        expected = tuple(self._mean.shape) + (self._n_dim,)
        if tuple(self._cov_tril.shape) != expected:
            raise ValueError(
                'MultivariateNormalCholesky.cov_tril should have compatible '
                'shape with mean. Expected {} got {}'.format(
                    expected, tuple(self._cov_tril.shape)))
        dtype = assert_same_float_dtype(
            [(self._mean, 'MultivariateNormalCholesky.mean'),
             (self._cov_tril, 'MultivariateNormalCholesky.cov_tril')])
        super(MultivariateNormalCholesky, self).__init__(
            dtype=dtype, param_dtype=dtype, is_continuous=True,
            is_reparameterized=is_reparameterized,
            use_path_derivative=use_path_derivative, group_ndims=group_ndims,
            **kwargs)

    mean = property(lambda self: self._mean)
    cov_tril = property(lambda self: self._cov_tril)

    def _get_value_shape(self):
        return torch.Size([self._n_dim])

    def _get_batch_shape(self):
        return self._mean.shape[:-1]

    def _sample(self, n_samples, eps=None):
        """multivariate.py:145-167: mean + L eps (eps via the Normal kernel)."""
        mean, tril = self._mean, self._cov_tril
        if not self.is_reparameterized:
            mean, tril = mean.detach(), tril.detach()
        seed, it = self._next_rng()
        zeros = torch.zeros_like(mean)
        noise = ops.reparam_normal(zeros, zeros, n_samples, eps=eps,
                                   seed=seed, it=it)
        return torch.matmul(tril, noise.unsqueeze(-1)).squeeze(-1) + mean

    def _log_prob(self, given):
        return ops.mvn_cholesky_log_prob(
            given, self.path_param(self._mean),
            self.path_param(self._cov_tril), self._group_ndims)


class UnnormalizedMultinomial(Distribution):
    """multivariate.py:339-446 (a.k.a. BagofCategoricals)."""
    _group_sum_in_log_prob = True

    def __init__(self, logits, normalize_logits=True, dtype=torch.int32,
                 group_ndims=0, **kwargs):
        self._logits = convert_to_tensor(logits)
        param_dtype = assert_same_float_dtype(
            [(self._logits, 'UnnormalizedMultinomial.logits')])
        assert_dtype_is_int_or_float(dtype)
        assert_rank_at_least(self._logits, 1,
                             'UnnormalizedMultinomial.logits')
        self._n_categories = int(self._logits.shape[-1])
        self.normalize_logits = normalize_logits
        super(UnnormalizedMultinomial, self).__init__(
            dtype=dtype, param_dtype=param_dtype, is_continuous=False,
            is_reparameterized=False, group_ndims=group_ndims, **kwargs)

    logits = property(lambda self: self._logits)
    n_categories = property(lambda self: self._n_categories)

    def _get_value_shape(self):
        return torch.Size([self._n_categories])

    def _get_batch_shape(self):
        return self._logits.shape[:-1]

    def _sample(self, n_samples):
        raise NotImplementedError("Unnormalized multinomial distribution"
                                  " does not support sampling because"
                                  " n_experiments is not given. Please use"
                                  " class Multinomial to sample")

    def _log_prob(self, given):
        return ops.unnormalized_multinomial_log_prob(
            given, self._logits, self.normalize_logits, self._group_ndims)


BagofCategoricals = UnnormalizedMultinomial


class Multinomial(UnnormalizedMultinomial):
    """multivariate.py:195-336: counts over ``n_categories`` from
    ``n_experiments`` draws (``None``: inferred from ``given``, no sampling).
    log_prob = log n! - sum log k_i! + sum k_i * log-softmax(logits)_i: the
    last term is the zsb_logprob_unnorm_multinomial_f32 kernel, the
    combinatorial term has no gradient."""

    def __init__(self, logits, n_experiments, normalize_logits=True,
                 dtype=torch.int32, group_ndims=0, **kwargs):
        super(Multinomial, self).__init__(
            logits, normalize_logits=normalize_logits, dtype=dtype,
            group_ndims=group_ndims, **kwargs)
        if n_experiments is not None:
            if isinstance(n_experiments, torch.Tensor):
                if n_experiments.dtype not in (torch.int32, torch.int64) or \
                        n_experiments.dim() != 0:
                    raise TypeError("Multinomial.n_experiments must be a 0-D "
                                    "int32 Tensor")
                n_experiments = int(n_experiments)
            elif not isinstance(n_experiments, int):
                raise TypeError("Multinomial.n_experiments must be int32")
            if n_experiments <= 0:
                raise ValueError("Multinomial.n_experiments must be positive")
        self._n_experiments = n_experiments

    n_experiments = property(lambda self: self._n_experiments)

    def _sample(self, n_samples):
        if self._n_experiments is None:
            raise ValueError('Cannot sample when `n_experiments` is None')
        # n_experiments categorical draws per sample on the device sampler, then counted
        seed, it = self._next_rng()
        draws = ops.sample_categorical(self._logits, int(n_samples) * self._n_experiments,
                                       seed=seed, it=it).long()     # [S * n] + batch
        onehot = torch.nn.functional.one_hot(draws, self._n_categories)
        counts = onehot.reshape((int(n_samples), self._n_experiments)
                                + tuple(self._logits.shape)).sum(1)
        return counts.to(self.dtype)

    def _log_prob(self, given):
        g = given.to(torch.float32)
        n = g.sum(-1) if self._n_experiments is None else \
            torch.full((), float(self._n_experiments), device=g.device)
        log_comb = torch.lgamma(n + 1) - torch.lgamma(g + 1).sum(-1)
        lp = ops.unnormalized_multinomial_log_prob(
            given, self._logits, self.normalize_logits, 0)
        return ops.group_sum(log_comb.detach() + lp, self._group_ndims)


class OnehotCategorical(Distribution):
    """multivariate.py:452-567: one-hot valued categorical;
    log_prob = -softmax_cross_entropy(labels=given, logits) = sum_i given_i *
    log-softmax(logits)_i, i.e. the same kernel with normalised logits."""
    _group_sum_in_log_prob = True

    def __init__(self, logits, dtype=torch.int32, group_ndims=0, **kwargs):
        self._logits = convert_to_tensor(logits)
        param_dtype = assert_same_float_dtype(
            [(self._logits, 'OnehotCategorical.logits')])
        assert_dtype_is_int_or_float(dtype)
        assert_rank_at_least(self._logits, 1, 'OnehotCategorical.logits')
        self._n_categories = int(self._logits.shape[-1])
        super(OnehotCategorical, self).__init__(
            dtype=dtype, param_dtype=param_dtype, is_continuous=False,
            is_reparameterized=False, group_ndims=group_ndims, **kwargs)

    logits = property(lambda self: self._logits)
    n_categories = property(lambda self: self._n_categories)

    def _get_value_shape(self):
        return torch.Size([self._n_categories])

    def _get_batch_shape(self):
        return self._logits.shape[:-1]

    def _sample(self, n_samples):
        seed, it = self._next_rng()
        draws = ops.sample_categorical(self._logits, int(n_samples), seed=seed, it=it).long()
        onehot = torch.nn.functional.one_hot(draws, self._n_categories)
        return onehot.to(self.dtype)

    def _log_prob(self, given):
        return ops.unnormalized_multinomial_log_prob(
            given, self._logits, True, self._group_ndims)


OnehotDiscrete = OnehotCategorical


class Dirichlet(Distribution):
    """multivariate.py:570-680."""
    _group_sum_in_log_prob = True

    def __init__(self, alpha, group_ndims=0, check_numerics=False, **kwargs):
        self._alpha = convert_to_tensor(alpha)
        dtype = assert_same_float_dtype([(self._alpha, 'Dirichlet.alpha')])
        if self._alpha.dim() < 1:
            raise ValueError("`alpha` should have rank >= 1.")
        self._n_categories = int(self._alpha.shape[-1])
        if self._n_categories < 2:
            raise ValueError("`n_categories` (length of the last axis "
                             "of `alpha`) should be at least 2.")
        self._check_numerics = check_numerics
        super(Dirichlet, self).__init__(
            dtype=dtype, param_dtype=dtype, is_continuous=True,
            is_reparameterized=False, group_ndims=group_ndims, **kwargs)

    alpha = property(lambda self: self._alpha)
    n_categories = property(lambda self: self._n_categories)

    def _get_value_shape(self):
        return torch.Size([self._n_categories])

    def _get_batch_shape(self):
        return self._alpha.shape[:-1]

    def _sample(self, n_samples, gammas=None):
        # multivariate.py:660-663: Gamma(alpha, 1) normalised -> device sampler
        # (Marsaglia-Tsang on Philox; ``gammas``: injected variates for parity)
        seed, it = self._next_rng()
        return ops.sample_dirichlet(self._alpha, n_samples, gammas=gammas, seed=seed, it=it)

    def _log_prob(self, given):
        return ops.dirichlet_log_prob(given, self._alpha, self._group_ndims)
