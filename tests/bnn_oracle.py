"""Float64 oracle of the BNN regression log-joint's outputs that SG-MCMC never needed: the gradient
w.r.t. y_logstd and the per-point predictions (bnn_vi.py:98-103).  Extends oracle/models.py::BNN,
whose logp / grad it reuses unchanged."""
import numpy as np

from oracle import distributions as D
from oracle import models as OM


class BNN(OM.BNN):
    def predictive(self, qs):
        """(y_mean [C, B], log N(y_b; y_mean, exp(y_logstd)) [C, B])."""
        d = self.dtype
        w0, w1 = (np.asarray(q, d) for q in qs)
        ym = self._fwd(w0, w1)[3]
        return ym, D.normal_log_prob(self.y[None, :], ym, d(self.Y_LOGSTD), 0, d).astype(d)

    def grad_y_logstd(self, qs):
        """d logp[c] / d y_logstd = n_train * mean_b (prec (y_b - y_mean)^2 - 1), [C]."""
        d = self.dtype
        ym, _ = self.predictive(qs)
        prec = np.exp(d(-2) * d(self.Y_LOGSTD))
        return (self.n_train * (prec * (self.y[None, :] - ym) ** 2 - 1).mean(1)).astype(d)
