"""zhusuan_b200 -- H100-native hot path of thu-ml/zhusuan.

``import zhusuan_b200 as zs`` exposes the same names as ``import zhusuan as
zs`` for the accelerated path: ``zs.HMC``, ``zs.SGLD/PSGLD/SGHMC/SGNHT``,
``zs.variational.elbo / iw_objective``, ``zs.is_loglikelihood``,
``zs.BayesianNet``, ``zs.meta_bayesian_net``, ``zs.distributions.*``,
``zs.log_mean_exp``.  All arithmetic runs in hand-written sm_90a kernels
(libzsb200.so, C ABI in include/zsb200.h); there is no CPU fallback.
"""
from . import distributions
from . import variational
from . import fused
from . import dist
from . import diagnostics
from . import ops
from .framework import *
from .framework import utils as _fw_utils
from .hmc import *
from .sgmcmc import *
from .evaluation import *
from .transform import *
from .utils import (TensorArithmeticMixin, log_mean_exp, log_sum_exp,
                    merge_dicts)
from .random import set_random_seed

__version__ = "0.1.0"
