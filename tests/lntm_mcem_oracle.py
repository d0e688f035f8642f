"""Float64 NumPy restatement of the logistic-normal topic model of
examples/topic_models/lntm_mcem.py for the Monte-Carlo EM tests: ``oracle.models.LNTM`` (the E-step
objective) extended to any topic count, a subset of the corpus' documents, AIS's tempered log-joint
(evaluation.py:91-94 with the eta prior as proposal) and the M-step's log p(x | eta, beta) and its
gradient w.r.t. beta (:106-114).  Test oracle only."""
import numpy as np

from oracle import distributions as D
from oracle import models as OM

LOG_DELTA = 10.0


class LNTM(OM.LNTM):
    """x: the corpus [n_docs, V]; ``doc_ids`` selects the rows eta stands for (None: all).
    ``logp`` / ``grad`` are the E-step objective; ``logp_t`` / ``grad_t`` its tempered form,
    prior + t * likelihood."""

    def __init__(self, x, beta, eta_mean, eta_logstd, doc_ids=None, dtype=np.float64):
        x = np.asarray(x)
        if doc_ids is not None:
            x = x[np.asarray(doc_ids)]
        super().__init__(x, beta, eta_mean, eta_logstd, dtype)

    def log_prior(self, eta):
        return D.normal_log_prob(np.asarray(eta, self.dtype), self.mean, self.logstd, 1,
                                 self.dtype)

    def log_px(self, eta):
        """log p(x_d | eta_c, beta) [chains, docs] (cond_log_prob('x'))."""
        dw = self._theta(np.asarray(eta, self.dtype)) @ self.phi
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(self.x > 0, self.x * np.log(dw), 0).sum(-1)

    def logp_t(self, qs, t):
        return self.log_prior(qs[0]) + t * self.log_px(qs[0])

    def grad_t(self, qs, t):
        eta = np.asarray(qs[0], self.dtype)
        prior = -np.exp(-2.0 * self.logstd) * (eta - self.mean)
        return [prior + t * (self.grad(qs)[0] - prior)]

    def beta_grad(self, eta, g):
        """d/d beta of sum_{c,d} g[c, d] log_px[c, d]: [K, V]."""
        th = self._theta(np.asarray(eta, self.dtype))
        dw = th @ self.phi
        r = np.where(self.x > 0, self.x / dw, 0) * np.asarray(g, self.dtype)[..., None]
        gphi = np.einsum("cbk,cbv->kv", th, r)
        return self.phi * (gphi - (self.phi * gphi).sum(-1, keepdims=True))


def m_step_grad(x, beta, eta_mean, eta_logstd, eta, doc_ids=None):
    """-(log p(beta) + sum_d mean_c log p(x_d | eta_c, beta)) differentiated w.r.t. beta, and
    log_px = sum_d mean_c log p(x_d | eta_c, beta) (lntm_mcem.py:106-114)."""
    m = LNTM(x, beta, eta_mean, eta_logstd, doc_ids)
    C, B = np.shape(eta)[:2]
    beta = np.asarray(beta, np.float64)
    d_prior = -np.exp(-2.0 * LOG_DELTA) * beta
    grad = -(d_prior + m.beta_grad(eta, np.full((C, B), 1.0 / C)))
    return grad, m.log_px(eta).mean(0).sum()
