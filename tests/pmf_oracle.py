"""NumPy oracle of the chunked PMF log-joint (test helper, not a test module).

examples/probabilistic_matrix_factorization/pmf_hmc.py:19-31 with the log_joint override of
136-144, evaluated for every chunk of the sampled factor at once: the latent is
[K, n_chunks, chunk_size, D] and logp returns [K, n_chunks]; chunk c's value is the example's
log_pu + log_pv + log_pr for that chunk, where log_pv runs over the chunk's neighbour set (the
distinct columns its ratings touch, select_from_corpus at 34-60).  The gradient w.r.t. the latent
is derived by hand:
    d/du_i = -u_i / std^2 + sum_j (r_ij - s_ij) s_ij (1 - s_ij) / rating_std^2 v_j,
    s_ij = sigmoid(u_i . v_j).
"""
import numpy as np


class PMF(object):
    def __init__(self, rows, cols, ratings, fixed, n_rows, chunk_size, std, fixed_std, rating_std,
                 dtype=np.float64):
        d = dtype
        self.dtype = d
        self.rows = np.asarray(rows, np.int64)
        self.cols = np.asarray(cols, np.int64)
        self.r = np.asarray(ratings, np.float32).astype(d)
        fixed = np.asarray(fixed)
        self.K, self.D = fixed.shape[0], fixed.shape[-1]
        self.v = fixed.reshape(self.K, -1, self.D).astype(d)
        self.n_rows, self.chunk_size = int(n_rows), int(chunk_size)
        self.n_chunks = self.n_rows // self.chunk_size
        self.logstd = [d(np.log(np.float32(s))) for s in (std, fixed_std, rating_std)]
        self.chunk = self.rows // self.chunk_size
        nb = np.zeros((self.n_chunks, self.v.shape[1]), bool)
        nb[self.chunk, self.cols] = True
        self.nbr = nb                                   # [n_chunks, n_cols] neighbour mask

    def _normal(self, x, logstd):                       # Normal._log_prob (univariate.py)
        d = self.dtype
        return d(-0.5 * np.log(2 * np.pi)) - logstd - d(0.5) * np.exp(d(-2) * logstd) * x * x

    def _s(self, u):
        z = (u[:, self.rows] * self.v[:, self.cols]).sum(-1)       # [K, nnz]
        return 1.0 / (1.0 + np.exp(-z))

    def logp(self, qs):
        d = self.dtype
        u = np.asarray(qs[0], d).reshape(self.K, self.n_rows, self.D)
        out = self._normal(u, self.logstd[0]).sum(-1).reshape(
            self.K, self.n_chunks, self.chunk_size).sum(-1)
        pv = self._normal(self.v, self.logstd[1]).sum(-1)          # [K, n_cols]
        out = out + pv @ self.nbr.T.astype(d)
        lp_r = self._normal(self.r - self._s(u), self.logstd[2])
        for k in range(self.K):
            out[k] += np.bincount(self.chunk, lp_r[k], minlength=self.n_chunks)
        return out.astype(d)

    def grad(self, qs):
        d = self.dtype
        shape = np.shape(qs[0])
        u = np.asarray(qs[0], d).reshape(self.K, self.n_rows, self.D)
        s = self._s(u)
        coef = (self.r - s) * s * (1 - s) * np.exp(d(-2) * self.logstd[2])   # [K, nnz]
        g = -np.exp(d(-2) * self.logstd[0]) * u
        for k in range(self.K):
            np.add.at(g[k], self.rows, coef[k][:, None] * self.v[k, self.cols])
        return [g.reshape(shape).astype(d)]


def make_corpus(n_rows, n_cols, nnz, seed, pad_rows=0, heavy_row=None, heavy_n=0):
    """Synthetic ratings with skewed degrees: Zipf-like row and column popularity, the last
    ``pad_rows`` rows without ratings, and optionally one row with ``heavy_n`` ratings.
    Returns (rows, cols, normalised ratings in [0, 1]) with no duplicate (row, col) pair."""
    rng = np.random.RandomState(seed)
    live = n_rows - pad_rows
    pr = 1.0 / (1.0 + np.arange(live)) ** 0.8
    pc = 1.0 / (1.0 + np.arange(n_cols)) ** 0.8
    rows = rng.choice(live, size=nnz, p=pr / pr.sum())
    cols = rng.choice(n_cols, size=nnz, p=pc / pc.sum())
    if heavy_row is not None:
        rows = np.concatenate([rows, np.full(heavy_n, heavy_row)])
        cols = np.concatenate([cols, rng.randint(0, n_cols, heavy_n)])
    key = np.unique(rows * n_cols + cols)
    rng.shuffle(key)
    rows, cols = key // n_cols, key % n_cols
    ratings = ((rng.randint(1, 6, rows.size) - 1.0) / 4.0).astype(np.float32)
    return rows.astype(np.int64), cols.astype(np.int64), ratings
