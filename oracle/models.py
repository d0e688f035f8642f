"""Log-joints of the benchmark configs, as (logp, grad) NumPy callables
(TEST ORACLE ONLY).  Each follows the reference example that defines the
workload's shape (SURVEY.md section 8d):

  DiagGaussian   examples/toy_examples/gaussian.py:15-20  (Normal, group_ndims=1)
  DenseGaussian  config 2: log p(x) = -1/2 (x-mu)^T P (x-mu) - 1/2 log|2 pi Sigma|
                 (a callable log_joint with a shared precision matrix; the
                 reference's MultivariateNormalCholesky would broadcast L to
                 chains x D^2, multivariate.py:183-185, which is infeasible)
  DoubleWell     tests/test_mcmc.py:23-26 (2x^2 - x^4, optional injected noise)
  BNN            examples/bayesian_neural_nets/bnn_sgmcmc.py:19-35, 74-77
"""
import numpy as np

from . import distributions as D


class DiagGaussian(object):
    def __init__(self, mean, std, dtype=np.float32):
        self.dtype = dtype
        self.mean = np.asarray(mean, dtype)
        self.std = np.asarray(std, dtype)
        self.logstd = np.log(self.std).astype(dtype)   # univariate.py:97

    def logp(self, qs):
        return D.normal_log_prob(qs[0], self.mean, self.logstd, 1,
                                 self.dtype)

    def grad(self, qs):
        d = self.dtype
        prec = np.exp(d(-2) * self.logstd)
        return [(-(prec * (np.asarray(qs[0], d) - self.mean))).astype(d)]


class DenseGaussian(object):
    """P: precision [D, D] (symmetric), const = -1/2 log|2 pi Sigma|."""

    def __init__(self, precision, mean=None, const=0.0, dtype=np.float32):
        self.dtype = dtype
        self.P = np.asarray(precision, dtype)
        D_ = self.P.shape[0]
        self.mean = np.zeros(D_, dtype) if mean is None else np.asarray(
            mean, dtype)
        self.const = dtype(const)

    def _g(self, q):
        d = self.dtype
        return (-((np.asarray(q, d) - self.mean) @ self.P)).astype(d)

    def logp(self, qs):
        d = self.dtype
        x = np.asarray(qs[0], d) - self.mean
        g = self._g(qs[0])
        return (d(0.5) * (x * g).sum(-1, dtype=d) + self.const).astype(d)

    def grad(self, qs):
        return [self._g(qs[0])]


class DoubleWell(object):
    """tests/test_mcmc.py:23-26.  ``noise`` (optional) is a per-call list of
    injected N(0, 2^2) arrays consumed in call order (the reference's
    log-joint adds fresh noise on every evaluation; it has zero gradient)."""

    def __init__(self, dtype=np.float32):
        self.dtype = dtype

    def logp(self, qs):
        x = np.asarray(qs[0], self.dtype)
        return (self.dtype(2) * x ** 2 - x ** 4).astype(self.dtype)

    def grad(self, qs):
        x = np.asarray(qs[0], self.dtype)
        return [(self.dtype(4) * x - self.dtype(4) * x ** 3).astype(
            self.dtype)]


class BNN(object):
    """bnn_sgmcmc.py:19-35 with layer_sizes [n_in, n_hidden, 1]; per-chain
    weights w0 [C, H, n_in+1], w1 [C, 1, H+1]; prior N(0, exp(logstd));
    y ~ N(y_mean, exp(y_logstd)) (default -0.95); log_joint = sum log p(w) +
    mean_batch(log p(y|x,w)) * n_train  (bnn_sgmcmc.py:74-77).  logstd0 /
    logstd1 are scalars or arrays broadcasting against w0 / w1 (per weight,
    per hidden unit, per chain, ...)."""

    Y_LOGSTD = -0.95

    def __init__(self, x, y, n_train, logstd0=0.0, logstd1=0.0,
                 dtype=np.float64, y_logstd=None):
        self.dtype = dtype
        self.x = np.asarray(x, dtype)
        self.y = np.asarray(y, dtype)
        self.n_train = dtype(n_train)
        self.ls0, self.ls1 = np.asarray(logstd0, dtype), np.asarray(logstd1, dtype)
        if y_logstd is not None:
            self.Y_LOGSTD = y_logstd

    def _fwd(self, w0, w1):
        d = self.dtype
        x = self.x
        B, n_in = x.shape
        h0 = np.concatenate([x, np.ones((B, 1), d)], -1)           # [B, n_in+1]
        a1 = (h0 @ w0.transpose(0, 2, 1)) / np.sqrt(d(n_in + 1))        # [C,B,H]
        r1 = np.maximum(a1, 0)
        C = w0.shape[0]
        h1 = np.concatenate([r1, np.ones((C, B, 1), d)], -1)       # [C,B,H+1]
        H1 = h1.shape[-1]
        out = (h1 @ w1.transpose(0, 2, 1)) / np.sqrt(d(H1))
        return h0, a1, h1, out[..., 0]

    def logp(self, qs):
        d = self.dtype
        w0, w1 = (np.asarray(q, d) for q in qs)
        _, _, _, ym = self._fwd(w0, w1)
        lpw = (D.normal_log_prob(w0, 0, self.ls0, 2, d)
               + D.normal_log_prob(w1, 0, self.ls1, 2, d))
        lpy = D.normal_log_prob(self.y[None, :], ym, d(self.Y_LOGSTD), 0, d)
        return (lpw + lpy.mean(1) * self.n_train).astype(d)

    def grad(self, qs):
        d = self.dtype
        w0, w1 = (np.asarray(q, d) for q in qs)
        h0, a1, h1, ym = self._fwd(w0, w1)
        B = self.x.shape[0]
        n_in = self.x.shape[1]
        H1 = h1.shape[-1]
        prec_y = np.exp(d(-2) * d(self.Y_LOGSTD))
        dym = prec_y * (self.y[None, :] - ym) * (self.n_train / d(B))  # [C,B]
        dout = dym / np.sqrt(d(H1))
        gw1 = dout[:, None, :] @ h1                                  # [C,1,H+1]
        dh1 = dout[..., None] * w1[:, 0, None, :]                  # [C,B,H+1]
        da1 = dh1[..., :-1] * (a1 > 0) / np.sqrt(d(n_in + 1))
        gw0 = da1.transpose(0, 2, 1) @ h0                            # [C,H,n_in+1]
        gw0 = gw0 - np.exp(d(-2) * self.ls0) * w0
        gw1 = gw1 - np.exp(d(-2) * self.ls1) * w1
        return [gw0.astype(d), gw1.astype(d)]


class LNTM(object):
    """E-step objective of examples/topic_models/lntm_mcem.py:33-48 with log_joint = e_obj
    (:97-99): Normal prior on eta (group_ndims=1) + UnnormalizedMultinomial(log(softmax(eta) @
    softmax(beta)), normalize_logits=False).log_prob(x) (multivariate.py:435-443), dense.
    eta [chains, docs, K]; x [docs, V]; beta [K, V]."""

    def __init__(self, x, beta, eta_mean, eta_logstd, dtype=np.float64):
        self.dtype = dtype
        self.x = np.asarray(x, dtype)
        b = np.asarray(beta, np.float64)
        e = np.exp(b - b.max(-1, keepdims=True))
        self.phi = (e / e.sum(-1, keepdims=True)).astype(dtype)     # lntm_mcem.py:41
        self.mean = np.asarray(eta_mean, dtype)
        self.logstd = np.asarray(eta_logstd, dtype)

    def _theta(self, eta):
        e = np.exp(eta - eta.max(-1, keepdims=True))
        return e / e.sum(-1, keepdims=True)

    def logp(self, qs):
        d = self.dtype
        eta = np.asarray(qs[0], d)
        prior = D.normal_log_prob(eta, self.mean, self.logstd, 1, d)
        doc_word = self._theta(eta) @ self.phi                        # lntm_mcem.py:43-44
        with np.errstate(divide="ignore", invalid="ignore"):
            ll = np.where(self.x > 0, self.x * np.log(doc_word), 0).sum(-1)
        return (prior + ll).astype(d)

    def grad(self, qs):
        d = self.dtype
        eta = np.asarray(qs[0], d)
        th = self._theta(eta)
        doc_word = th @ self.phi
        ratio = np.where(self.x > 0, self.x / doc_word, 0)
        dth = ratio @ self.phi.T
        g = th * (dth - (th * dth).sum(-1, keepdims=True))
        g = g - np.exp(d(-2) * self.logstd) * (eta - self.mean)
        return [g.astype(d)]


def make_dense_gaussian_problem(D_, seed=2):
    """Config 2 synthetic target (SURVEY.md 8d): Sigma = A A^T / D + 0.1 I,
    rescaled to unit diagonal; P = Sigma^-1 computed in float64.
    Returns (P float64, const float64)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    A = rng.standard_normal((D_, D_))
    S = A @ A.T / D_ + 0.1 * np.eye(D_)
    s = 1.0 / np.sqrt(np.diag(S))
    S = S * s[:, None] * s[None, :]
    P = np.linalg.inv(S)
    P = 0.5 * (P + P.T)
    sign, logdet = np.linalg.slogdet(S)
    const = -0.5 * (D_ * np.log(2 * np.pi) + logdet)
    return P, const
