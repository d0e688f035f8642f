"""ExpConcrete / Concrete (Gumbel-softmax relaxations, multivariate.py:683-958)
and MatrixVariateNormalCholesky (multivariate.py:961-1160).

ExpConcrete and Concrete sample and score on the fused kernels of
csrc/concrete.cu (one pass per direction over the [S, *batch, C] tensor, the
gradients w.r.t. given, logits and temperature analytic) whenever the logits
and the temperature are float32 on one CUDA device, ``given`` is float32 and
1 <= C <= 1024.  Every other input takes the composition kept here: the
library's reduction kernels (log-sum-exp / sum over the category axis through
``ops.reduce_axes``) plus elementwise torch ops.  Both draw the same uniforms
from a given ``zs.random`` state.  The matrix-variate normal stays on torch's
triangular solves (cuBLAS: library code).
"""
import math

import torch

from .. import ops
from ..utils import convert_to_tensor
from .base import Distribution
from .utils import assert_same_float_dtype, assert_rank_at_least

__all__ = ["ExpConcrete", "ExpGumbelSoftmax", "Concrete", "GumbelSoftmax",
           "MatrixVariateNormalCholesky"]


class ExpConcrete(Distribution):
    """multivariate.py:683-815: log of a Concrete sample (values are
    log-probabilities on the simplex)."""
    _group_sum_in_log_prob = True
    _name = "ExpConcrete"
    _log_space = True

    def __init__(self, temperature, logits, group_ndims=0,
                 is_reparameterized=True, use_path_derivative=False,
                 check_numerics=False, **kwargs):
        self._logits = convert_to_tensor(logits)
        self._temperature = convert_to_tensor(temperature,
                                              device=self._logits.device)
        dtype = assert_same_float_dtype(
            [(self._logits, self._name + '.logits'),
             (self._temperature, self._name + '.temperature')])
        assert_rank_at_least(self._logits, 1, self._name + '.logits')
        if self._temperature.dim() != 0:
            raise ValueError(self._name + ".temperature should be a scalar "
                             "(0-D Tensor).")
        self._n_categories = int(self._logits.shape[-1])
        self._check_numerics = check_numerics
        super(ExpConcrete, self).__init__(
            dtype=dtype, param_dtype=dtype, is_continuous=True,
            is_reparameterized=is_reparameterized,
            use_path_derivative=use_path_derivative, group_ndims=group_ndims,
            **kwargs)

    temperature = property(lambda self: self._temperature)
    logits = property(lambda self: self._logits)
    n_categories = property(lambda self: self._n_categories)

    def _get_value_shape(self):
        return torch.Size([self._n_categories])

    def _get_batch_shape(self):
        return self._logits.shape[:-1]

    def _fused(self, given=None):
        """The kernels of csrc/concrete.cu take these inputs (decided from them alone)."""
        l, t = self._logits, self._temperature
        return (l.dtype == torch.float32 and t.dtype == torch.float32 and l.is_cuda
                and t.device == l.device
                and 1 <= self._n_categories <= ops.CONCRETE_MAX_CATEGORIES
                and (given is None or (given.dtype == torch.float32
                                       and given.device == l.device)))

    def _gumbel_logits(self, n_samples, u=None):
        logits, temperature = self._logits, self._temperature
        if not self.is_reparameterized:
            logits, temperature = logits.detach(), temperature.detach()
        rng = self._next_rng()
        if u is None:
            u = ops.base_noise(0, (int(n_samples),) + tuple(logits.shape), logits.device, *rng)
        u = u.clamp(1e-7, 1.0 - 1e-7)                 # open interval (0, 1)
        gumbel = -torch.log(-torch.log(u))
        return (logits + gumbel) / temperature

    def _sample(self, n_samples, u=None):
        """``u``: injected uniforms [n_samples] + logits.shape (clamped as drawn ones are)."""
        if self._fused():
            logits, temperature = self._logits, self._temperature
            if not self.is_reparameterized:
                logits, temperature = logits.detach(), temperature.detach()
            seed, it = self._next_rng()
            return ops.sample_concrete(logits, temperature, n_samples, self._log_space, u=u,
                                       seed=seed, it=it)
        a = self._gumbel_logits(n_samples, u)
        return torch.log_softmax(a, -1) if self._log_space else torch.softmax(a, -1)

    def _finish(self, lp):
        if self._check_numerics and not bool(torch.isfinite(lp).all()):
            raise FloatingPointError(self._name + ".log_prob has numeric errors")
        return ops.group_sum(lp, self._group_ndims)

    def _density_terms(self, temp, extra):
        """lgamma(n) + (n-1) log t + sum(temp + extra) - n * LSE(temp)."""
        n = float(self._n_categories)
        t = self.path_param(self._temperature)
        lp = math.lgamma(n) + (n - 1.0) * torch.log(t) + \
            ops.reduce_axes(temp + extra if extra is not None else temp,
                            ops.OP_SUM, -1) - \
            n * ops.reduce_axes(temp, ops.OP_LSE, -1)
        return self._finish(lp)

    def _log_prob(self, given):
        logits = self.path_param(self._logits)
        t = self.path_param(self._temperature)
        if self._fused(given):
            return self._finish(ops.concrete_log_prob(given, logits, t, self._log_space))
        if not self._log_space:
            log_given = torch.log(given)
            temp = (logits - t * log_given).contiguous()
            return self._density_terms(temp, -log_given)
        temp = (logits - t * given).contiguous()
        return self._density_terms(temp, None)


ExpGumbelSoftmax = ExpConcrete


class Concrete(ExpConcrete):
    """multivariate.py:820-958: the Gumbel-softmax relaxation on the simplex."""
    _name = "Concrete"
    _log_space = False


GumbelSoftmax = Concrete


class MatrixVariateNormalCholesky(Distribution):
    """multivariate.py:961-1160: X ~ MN(mean, U = Lu Lu^T, V = Lv Lv^T) with
    the row / column covariances given by their Cholesky factors."""
    _group_sum_in_log_prob = True

    def __init__(self, mean, u_tril, v_tril, group_ndims=0,
                 is_reparameterized=True, use_path_derivative=False,
                 check_numerics=False, **kwargs):
        self._mean = convert_to_tensor(mean)
        self._u_tril = convert_to_tensor(u_tril, device=self._mean.device)
        self._v_tril = convert_to_tensor(v_tril, device=self._mean.device)
        for t, nm in ((self._mean, 'mean'), (self._u_tril, 'u_tril'),
                      (self._v_tril, 'v_tril')):
            assert_rank_at_least(t, 2, 'MatrixVariateNormalCholesky.' + nm)
        self._n_row, self._n_col = int(self._mean.shape[-2]), \
            int(self._mean.shape[-1])
        batch = tuple(self._mean.shape[:-2])
        if tuple(self._u_tril.shape) != batch + (self._n_row, self._n_row):
            raise ValueError(
                "MatrixVariateNormalCholesky.u_tril should have compatible "
                "shape with mean. Expected {} got {}".format(
                    batch + (self._n_row, self._n_row),
                    tuple(self._u_tril.shape)))
        if tuple(self._v_tril.shape) != batch + (self._n_col, self._n_col):
            raise ValueError(
                "MatrixVariateNormalCholesky.v_tril should have compatible "
                "shape with mean. Expected {} got {}".format(
                    batch + (self._n_col, self._n_col),
                    tuple(self._v_tril.shape)))
        dtype = assert_same_float_dtype(
            [(self._mean, 'MatrixVariateNormalCholesky.mean'),
             (self._u_tril, 'MatrixVariateNormalCholesky.u_tril'),
             (self._v_tril, 'MatrixVariateNormalCholesky.v_tril')])
        self._check_numerics = check_numerics
        super(MatrixVariateNormalCholesky, self).__init__(
            dtype=dtype, param_dtype=dtype, is_continuous=True,
            is_reparameterized=is_reparameterized,
            use_path_derivative=use_path_derivative, group_ndims=group_ndims,
            **kwargs)

    mean = property(lambda self: self._mean)
    u_tril = property(lambda self: self._u_tril)
    v_tril = property(lambda self: self._v_tril)

    def _get_value_shape(self):
        return torch.Size([self._n_row, self._n_col])

    def _get_batch_shape(self):
        return self._mean.shape[:-2]

    def _sample(self, n_samples):
        mean, lu, lv = self._mean, self._u_tril, self._v_tril
        if not self.is_reparameterized:
            mean, lu, lv = mean.detach(), lu.detach(), lv.detach()
        from .. import ops
        noise = ops.base_noise(1, (int(n_samples),) + tuple(mean.shape), mean.device,
                               *self._next_rng())
        return mean + lu @ noise @ lv.transpose(-1, -2)

    def _log_prob(self, given):
        mean = self.path_param(self._mean)
        lu = self.path_param(self._u_tril)
        lv = self.path_param(self._v_tril)
        log_det_u = 2.0 * torch.log(torch.diagonal(lu, dim1=-2, dim2=-1)).sum(-1)
        log_det_v = 2.0 * torch.log(torch.diagonal(lv, dim1=-2, dim2=-1)).sum(-1)
        r, c = float(self._n_row), float(self._n_col)
        log_z = -(r * c) / 2.0 * math.log(2.0 * math.pi) - r / 2.0 * log_det_v \
            - c / 2.0 * log_det_u
        if self._check_numerics and not bool(torch.isfinite(log_z).all()):
            raise FloatingPointError("log[det(Cov)] has numeric errors")
        y = given - mean
        a = torch.linalg.solve_triangular(lu.expand(y.shape[:-2] + lu.shape[-2:]),
                                          y, upper=False)                 # Lu^-1 y
        x = torch.linalg.solve_triangular(lv.expand(y.shape[:-2] + lv.shape[-2:]),
                                          a.transpose(-1, -2), upper=False)
        lp = log_z - 0.5 * x.square().sum((-1, -2))
        return ops.group_sum(lp.contiguous(), self._group_ndims)
