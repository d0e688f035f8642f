"""Float64 torch restatement of gp_conditional and RBFKernel (examples/gaussian_process/utils.py:
10-90) and of the bound of examples/gaussian_process/svgp.py:49-139, with every draw injected.
Runs on whatever device its inputs are on."""
import math

import torch


def softplus(t):
    return torch.nn.functional.softplus(t)


def rbf(x, y, s):
    """utils.py:35-39: exp(-sum_j (x_j - y_j)^2 / s_j / 2) over [n_x, n_y]."""
    diff = x[:, None, :] - y[None, :, :]
    return torch.exp(-(diff * diff / s).sum(-1) / 2)


def gp_conditional(z, fz, x, s, full_cov=False, Kzz_chol=None):
    """utils.py:60-90 in the reference's own order (Kzz_inv = Li^T Li).  Returns (mean, std) for
    full_cov=False and (mean, cov_chol) for full_cov=True."""
    if Kzz_chol is None:
        Kzz_chol = torch.linalg.cholesky(rbf(z, z, s))
    eye = torch.eye(z.shape[0], dtype=z.dtype, device=z.device)
    Li = torch.linalg.solve_triangular(Kzz_chol, eye, upper=False)
    Kzz_inv = Li.t() @ Li
    Kxz = rbf(x, z, s)
    Kxziz = Kxz @ Kzz_inv
    mean = fz @ Kxziz.t()
    if full_cov:
        return mean, torch.linalg.cholesky(rbf(x, x, s) - Kxziz @ Kxz.t())
    return mean, torch.sqrt(1.0 - ((Kxz @ Li.t()) ** 2).sum(-1))


def moments_from_factors(x, z, s, Li, V):
    """The kernel's re-association: A = Kxz tril(Li)^T, mean = V A^T, std = sqrt(1 - |A_b|^2)."""
    A = rbf(x, z, s) @ torch.tril(Li).t()
    return V @ A.t(), torch.sqrt(1.0 - (A * A).sum(-1))


def moment_terms(x, z, s, Li, V):
    """Sums of the absolute terms of mean and var, for rounding bounds: each product and sum is
    taken over |.|, and each Kxz entry carries its exponent's own terms (1 + q / 2) Kxz."""
    diff = x[:, None, :] - z[None, :, :]
    q = (diff * diff / s).sum(-1)
    K = torch.exp(-q / 2)
    Ka = (1 + q / 2) * K
    La = torch.tril(Li).abs()
    A = K @ torch.tril(Li).t()
    Aa = Ka @ La.t()
    return V.abs() @ Aa.t(), 1.0 + 2.0 * (A.abs() * Aa).sum(-1)


def grad_terms(x, z, s, Li, V, A, std, g_mean, g_std):
    """Sums of the absolute terms of (dz, ds, dLi, dV), the hand-derived backward of
    moments_from_factors taken over |.|."""
    diff = x[:, None, :] - z[None, :, :]
    q = (diff * diff / s).sum(-1)
    K = torch.exp(-q / 2)
    Ka = (1 + q / 2) * K
    La = torch.tril(Li).abs()
    gm = torch.zeros(V.shape[0], x.shape[0], dtype=x.dtype, device=x.device) \
        if g_mean is None else g_mean.abs()
    c = torch.zeros_like(std) if g_std is None else (g_std / std).abs()
    dA = gm.t() @ V.abs() + c[:, None] * A.abs()
    G = (dA @ La) * Ka
    dz = (G[:, :, None] * diff.abs()).sum(0) / s
    ds = (G[:, :, None] * diff * diff).sum((0, 1)) / (2 * s * s)
    dLi = torch.tril(dA.t() @ Ka)
    dV = gm @ A.abs()
    return dz, ds, dLi, dV


def mvn_chol_log_prob(x, mean, L):
    """log N(x; mean, L L^T) over the last axis."""
    n = L.shape[-1]
    sol = torch.linalg.solve_triangular(L, (x - mean).unsqueeze(-1), upper=False).squeeze(-1)
    return -0.5 * (sol * sol).sum(-1) - torch.log(torch.diagonal(L)).sum() - \
        0.5 * n * math.log(2 * math.pi)


def normal_log_prob(x, mean, std):
    return -0.5 * ((x - mean) / std) ** 2 - torch.log(std) - 0.5 * math.log(2 * math.pi)


def svgp_bound(params, x, y, n_train, eps_fz, eps_fx):
    """svgp.py:49-139 with injected draws: fz = z_mean + eps_fz tril^T [K, M] (:75-85), the
    variational fx = mean + std eps_fx [K, B] (:86, its log-prob replaced by zeros, :133), and
    log_joint = log p(fz) + log p(y | fx) / B * n_train (:125-127).  Returns the per-particle
    objective [K]; the bound is its mean and the sgvb cost its negated mean."""
    s = softplus(params["k_raw_scale"])
    z_pos = params["z_pos"]
    raw = params["z_cov_raw"]
    tril = torch.tril(raw, -1) + torch.diag(softplus(torch.diagonal(raw)))
    fz = params["z_mean"] + eps_fz @ tril.t()
    log_qfz = mvn_chol_log_prob(fz, params["z_mean"], tril)
    mean, std = gp_conditional(z_pos, fz, x, s)
    fx = mean + std * eps_fx
    Kzz_chol = torch.linalg.cholesky(rbf(z_pos, z_pos, s))
    log_pfz = mvn_chol_log_prob(fz, torch.zeros_like(fz), Kzz_chol)
    noise = softplus(params["noise_level"])
    log_py = normal_log_prob(y, fx, noise).sum(-1)
    return log_pfz + log_py / x.shape[0] * n_train - log_qfz


def svgp_predict(params, x, y, std_y_train, eps_fz, eps_fx):
    """svgp.py:143-150: (log_likelihood, pred_mse) with the model observing the variational fx."""
    s = softplus(params["k_raw_scale"])
    raw = params["z_cov_raw"]
    tril = torch.tril(raw, -1) + torch.diag(softplus(torch.diagonal(raw)))
    fz = params["z_mean"] + eps_fz @ tril.t()
    mean, std = gp_conditional(params["z_pos"], fz, x, s)
    fx = mean + std * eps_fx
    noise = softplus(params["noise_level"])
    ll = normal_log_prob(y, fx, noise).sum(-1)
    ll = torch.logsumexp(ll, 0) - math.log(ll.shape[0])
    ll = ll / x.shape[0] - math.log(std_y_train)
    mse = ((fx.mean(0) - y) ** 2).mean() * std_y_train ** 2
    return ll, mse
