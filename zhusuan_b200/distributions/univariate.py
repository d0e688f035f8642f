"""Normal / Bernoulli / Categorical on the H100 kernels
(zhusuan/distributions/univariate.py:43-184, 334-406, 409-551)."""
import torch

from .. import ops
from ..utils import convert_to_tensor
from .base import Distribution
from .utils import (assert_same_float_dtype, assert_dtype_is_int_or_float,
                    assert_dtype_in_dtypes, assert_rank_at_least,
                    broadcast_check, FLOATS, INTS)

__all__ = ["Normal", "Bernoulli", "Categorical", "Discrete"]


class Normal(Distribution):
    """univariate.py:43-184.  ``std`` xor ``logstd`` (ValueError otherwise)."""
    _group_sum_in_log_prob = True

    def __init__(self, mean=0., _sentinel=None, std=None, logstd=None,
                 group_ndims=0, is_reparameterized=True,
                 use_path_derivative=False, check_numerics=False, **kwargs):
        if _sentinel is not None:
            raise ValueError(
                "The order of logstd/std has changed to std/logstd since "
                "0.3.1. Please use named arguments: Normal(mean, std=..., "
                "...) or Normal(mean, logstd=..., ...).")
        self._mean = convert_to_tensor(mean)
        if (logstd is None) == (std is None):
            raise ValueError(
                "Either `std` or `logstd` should be passed. It is not allowed "
                "that both are specified or both are not.")
        elif logstd is None:
            self._std = convert_to_tensor(std, device=self._mean.device)
            dtype = assert_same_float_dtype([(self._mean, 'Normal.mean'),
                                             (self._std, 'Normal.std')])
            self._logstd = torch.log(self._std)              # :97
        else:
            self._logstd = convert_to_tensor(logstd, device=self._mean.device)
            dtype = assert_same_float_dtype(
                [(self._mean, 'Normal.mean'), (self._logstd, 'Normal.logstd')])
            self._std = torch.exp(self._logstd)              # :106
        broadcast_check(
            self._mean.shape, self._std.shape,
            "mean and std/logstd should be broadcastable to match each "
            "other. ({} vs. {})".format(tuple(self._mean.shape),
                                        tuple(self._std.shape)))
        self._check_numerics = check_numerics
        super(Normal, self).__init__(
            dtype=dtype, param_dtype=dtype, is_continuous=True,
            is_reparameterized=is_reparameterized,
            use_path_derivative=use_path_derivative, group_ndims=group_ndims,
            **kwargs)

    mean = property(lambda self: self._mean)
    logstd = property(lambda self: self._logstd)
    std = property(lambda self: self._std)

    def _get_value_shape(self):
        return torch.Size([])

    def _get_batch_shape(self):
        return torch.broadcast_shapes(self._mean.shape, self._std.shape)

    def _sample(self, n_samples, eps=None):
        mean, logstd = self._mean, self._logstd
        if not self.is_reparameterized:                      # :163-165
            mean, logstd = mean.detach(), logstd.detach()
        seed, it = self._next_rng()
        return ops.reparam_normal(mean, logstd, n_samples, eps=eps, seed=seed,
                                  it=it)

    def _log_prob(self, given):
        mean = self.path_param(self._mean)
        logstd = self.path_param(self._logstd)
        lp = ops.normal_log_prob(given, mean, logstd, self._group_ndims)
        if self._check_numerics and not bool(torch.isfinite(lp).all()):
            raise FloatingPointError("Normal.log_prob: precision has numeric "
                                     "errors")
        return lp


class Bernoulli(Distribution):
    """univariate.py:334-406."""
    _group_sum_in_log_prob = True

    def __init__(self, logits, dtype=torch.int32, group_ndims=0, **kwargs):
        self._logits = convert_to_tensor(logits)
        param_dtype = assert_same_float_dtype(
            [(self._logits, 'Bernoulli.logits')])
        assert_dtype_is_int_or_float(dtype)
        super(Bernoulli, self).__init__(
            dtype=dtype, param_dtype=param_dtype, is_continuous=False,
            is_reparameterized=False, group_ndims=group_ndims, **kwargs)

    logits = property(lambda self: self._logits)

    def _get_value_shape(self):
        return torch.Size([])

    def _get_batch_shape(self):
        return self._logits.shape

    def _sample(self, n_samples, u=None):
        seed, it = self._next_rng()
        return ops.sample_bernoulli(self._logits, n_samples, u=u, seed=seed,
                                    it=it, dtype=self.dtype)

    def _log_prob(self, given):
        return ops.bernoulli_log_prob(given, self._logits, self._group_ndims)


class Categorical(Distribution):
    """univariate.py:409-551."""
    _group_sum_in_log_prob = True

    def __init__(self, logits, dtype=torch.int32, group_ndims=0, **kwargs):
        self._logits = convert_to_tensor(logits)
        param_dtype = assert_same_float_dtype(
            [(self._logits, 'Categorical.logits')])
        assert_dtype_in_dtypes(dtype, INTS + FLOATS)
        assert_rank_at_least(self._logits, 1, 'Categorical.logits')
        self._n_categories = int(self._logits.shape[-1])
        super(Categorical, self).__init__(
            dtype=dtype, param_dtype=param_dtype, is_continuous=False,
            is_reparameterized=False, group_ndims=group_ndims, **kwargs)

    logits = property(lambda self: self._logits)
    n_categories = property(lambda self: self._n_categories)

    def _get_value_shape(self):
        return torch.Size([])

    def _get_batch_shape(self):
        return self._logits.shape[:-1]

    def _sample(self, n_samples, u=None):
        # tf.random.categorical (univariate.py:478-494) -> device sampler: inverse CDF of
        # softmax(logits), one Philox uniform per draw (``u``: injected uniforms for parity)
        seed, it = self._next_rng()
        out = ops.sample_categorical(self._logits, n_samples, u=u, seed=seed, it=it)
        return out if self.dtype == torch.int32 else out.to(self.dtype)

    def _log_prob(self, given):
        return ops.categorical_log_prob(given, self._logits,
                                        self._group_ndims)


Discrete = Categorical
