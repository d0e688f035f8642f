"""Float64 oracle of the L-layer BNN regression log-joint (build_bnn of bnn_vi.py:18-35 and
bnn_sgmcmc.py:19-35 at layer_sizes [n_0, ..., n_{L-1}, 1], log-joint bnn_vi.py:83-86): value,
gradient w.r.t. every layer and y_logstd, and the per-point predictions.  The same interface as
tests/bnn_oracle.py::BNN (logp / grad over a list of latents), so oracle/sgmcmc.py runs on it."""
import numpy as np

from oracle import distributions as D


class DeepBNN(object):
    def __init__(self, x, y, n_train, logstds, y_logstd=-0.95, dtype=np.float64):
        self.dtype = dtype
        self.x = np.asarray(x, dtype)
        self.y = np.asarray(y, dtype).reshape(-1)
        self.n_train = dtype(n_train)
        self.lss = [np.asarray(l, dtype) for l in logstds]
        self.Y_LOGSTD = y_logstd

    def _fwd(self, ws):
        """(inputs [h_i, 1] of every layer, their pre-activations, y_mean [C, B])."""
        d = self.dtype
        C, B = ws[0].shape[0], self.x.shape[0]
        h = np.broadcast_to(self.x, (C,) + self.x.shape)
        hs, zs = [], []
        for i, w in enumerate(ws):
            h = np.concatenate([h, np.ones((C, B, 1), d)], -1)
            hs.append(h)
            z = (h @ w.transpose(0, 2, 1)) / np.sqrt(d(h.shape[-1]))
            zs.append(z)
            h = np.maximum(z, 0) if i < len(ws) - 1 else z
        return hs, zs, h[..., 0]

    def logp(self, qs):
        d = self.dtype
        ws = [np.asarray(q, d) for q in qs]
        ym = self._fwd(ws)[2]
        lpw = sum(D.normal_log_prob(w, 0, ls, 2, d) for w, ls in zip(ws, self.lss))
        lpy = D.normal_log_prob(self.y[None, :], ym, d(self.Y_LOGSTD), 0, d)
        return (lpw + lpy.mean(1) * self.n_train).astype(d)

    def grad(self, qs):
        d = self.dtype
        ws = [np.asarray(q, d) for q in qs]
        hs, zs, ym = self._fwd(ws)
        B = self.x.shape[0]
        prec_y = np.exp(d(-2) * d(self.Y_LOGSTD))
        dz = (prec_y * (self.y[None, :] - ym) * (self.n_train / d(B)))[..., None]   # [C, B, 1]
        gs = [None] * len(ws)
        for i in range(len(ws) - 1, -1, -1):
            s = np.sqrt(d(hs[i].shape[-1]))
            gs[i] = (dz.transpose(0, 2, 1) @ hs[i]) / s - np.exp(d(-2) * self.lss[i]) * ws[i]
            if i:
                dz = (dz @ ws[i])[..., :-1] / s * (zs[i - 1] > 0)
        return [g.astype(d) for g in gs]

    def predictive(self, qs):
        """(y_mean [C, B], log N(y_b; y_mean, exp(y_logstd)) [C, B])."""
        d = self.dtype
        ym = self._fwd([np.asarray(q, d) for q in qs])[2]
        return ym, D.normal_log_prob(self.y[None, :], ym, d(self.Y_LOGSTD), 0, d).astype(d)

    def grad_y_logstd(self, qs):
        """d logp[c] / d y_logstd = n_train * mean_b (prec (y_b - y_mean)^2 - 1), [C]."""
        d = self.dtype
        ym, _ = self.predictive(qs)
        prec = np.exp(d(-2) * d(self.Y_LOGSTD))
        return (self.n_train * (prec * (self.y[None, :] - ym) ** 2 - 1).mean(1)).astype(d)

    def relu_ties(self, qs, rtol=3e-6):
        """[C] mask of the particles with a hidden pre-activation within rtol of its layer's
        largest one (per particle) of 0 on some row: float32 may take the other side of the ReLU
        there, which moves that row's contribution to every gradient upstream of the unit."""
        zs = self._fwd([np.asarray(q, self.dtype) for q in qs])[1]
        return np.any([(np.abs(z) < rtol * np.abs(z).max(axis=(1, 2), keepdims=True)).any((1, 2))
                       for z in zs[:-1]], axis=0)
