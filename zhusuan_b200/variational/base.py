"""VariationalObjective -- the wiring contract of zhusuan/variational/base.py:24-196.

An objective ties together (i) a model, given as a MetaBayesianNet or as a
``log_joint(dict) -> Tensor`` callable, (ii) the observed values and (iii) the
variational family, either a sampled ``BayesianNet`` (``variational=``) or the
deprecated ``latent={name: [samples, log_q]}`` dictionary.  It exposes the two
terms every estimator is built from:

    log_joint term  log p(x, z) at the variational samples   (base.py:169-175)
    entropy term    - sum_z log q(z | x)                      (base.py:177-183)

and behaves like its ``.tensor`` in arithmetic and ``torch.*`` calls.
"""
import warnings

from ..framework.bn import BayesianNet, StochasticTensor
from ..utils import TensorArithmeticMixin, merge_dicts

__all__ = ['VariationalObjective']

_BOTH_OR_NEITHER = (
    "Either a {} `variational` representing "
    "the variational family or a dictionary `latent` "
    "representing the variational inputs should be passed. "
    "It is not allowed that both are specified or both are not.")
_LATENT_DEPRECATED = (
    "The `latent` argument has been deprecated and will be "
    "removed in the coming version (0.4.1), use the `variational` "
    "argument instead.")


def _from_variational_net(net):
    """Latent (un-observed stochastic) nodes of the variational BayesianNet:
    their samples become model observations, their cond_log_p is log q."""
    if not isinstance(net, BayesianNet):
        raise TypeError("`variational` should be a {} instance, got {}."
                        .format(BayesianNet.__name__, repr(net)))
    inputs, log_qs = {}, {}
    for name, node in net.nodes.items():
        if isinstance(node, StochasticTensor) and not node.is_observed():
            inputs[name] = node
            log_qs[name] = node.cond_log_p
    return inputs, log_qs


def _from_latent_dict(latent):
    warnings.warn(_LATENT_DEPRECATED, FutureWarning)
    inputs = {name: pair[0] for name, pair in latent.items()}
    log_qs = {name: pair[1] for name, pair in latent.items()}
    return inputs, log_qs


class VariationalObjective(TensorArithmeticMixin):
    def __init__(self, meta_bn, observed, latent=None, variational=None):
        is_fn = callable(meta_bn)
        self._meta_bn = None if is_fn else meta_bn
        if is_fn:
            self._log_joint = meta_bn
        if (variational is None) == (latent is None):
            raise ValueError(_BOTH_OR_NEITHER.format(BayesianNet))
        if variational is not None:
            self._v_inputs, self._v_log_probs = _from_variational_net(
                variational)
            self._variational = variational
        else:
            self._v_inputs, self._v_log_probs = _from_latent_dict(latent)
            self._variational = None
        self._observed = dict(observed)
        self._cache = {}

    # -- accessors ---------------------------------------------------------
    meta_bn = property(lambda self: self._meta_bn)
    variational = property(lambda self: self._variational)

    @property
    def bn(self):
        """The model observed at the variational samples (None for a plain
        log-joint callable); every stochastic node must end up observed."""
        if not self._meta_bn:
            return None
        if "bn" not in self._cache:
            net = self._meta_bn.observe(
                **merge_dicts(self._v_inputs, self._observed))
            for node in net.nodes.values():
                if isinstance(node, StochasticTensor) and \
                        not node.is_observed():
                    raise ValueError(
                        "Stochastic node '{}' in the model is neither "
                        "observed nor provided with a variational posterior."
                        .format(node.name))
            self._cache["bn"] = net
        return self._cache["bn"]

    @property
    def tensor(self):
        if "tensor" not in self._cache:
            self._cache["tensor"] = self._objective()
        return self._cache["tensor"]

    # -- the two terms -------------------------------------------------------
    def _log_joint_term(self):
        if self._meta_bn:
            return self.bn.log_joint()
        if "log_joint" not in self._cache:
            obs = merge_dicts(self._v_inputs, self._observed)
            # zs.fused.BNNRegressionLogJoint: value and gradient from one fused launch when
            # the shapes fit its kernel, else the callable under autograd
            f = getattr(self._log_joint, "_zsb_fused", None)
            obj = f.get("obj") if f is not None and \
                f.get("kind") == "bnn_regression" else None
            if obj is not None and obj.fused_inputs(obs) is not None:
                self._cache["log_joint"] = obj.fused_log_joint(obs)
            else:
                self._cache["log_joint"] = self._log_joint(obs)
        return self._cache["log_joint"]

    def _entropy_term(self):
        if "entropy" not in self._cache:
            terms = list(self._v_log_probs.values())
            self._cache["entropy"] = -sum(terms) if terms else None
        return self._cache["entropy"]

    def _objective(self):
        raise NotImplementedError()
