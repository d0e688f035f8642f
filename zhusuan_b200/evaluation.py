"""zhusuan/evaluation.py: importance-sampling and annealed-importance-sampling
marginal-likelihood estimators on the H100 kernels."""
import numpy as np
import torch

from .utils import merge_dicts
from .variational.monte_carlo import ImportanceWeightedObjective

__all__ = ["is_loglikelihood", "AIS"]


def is_loglikelihood(meta_bn, observed, latent=None, axis=None, proposal=None):
    """log p(x) >= log_mean_exp_axis(log p(x,z) - log q(z)); identical to
    ``ImportanceWeightedObjective.tensor`` (evaluation.py:22-54)."""
    return ImportanceWeightedObjective(
        meta_bn, observed, latent=latent, axis=axis,
        variational=proposal).tensor


class AIS(object):
    """Annealed importance sampling (evaluation.py:57-172) as a device-driven loop.

    Same schedule, adaptation phase and weight recursion as the reference, but nothing in the
    temperature loop touches the host: the whole sigmoid schedule (evaluation.py:107-112) is
    computed once into a device array, ``temperature`` -- the reference's placeholder -- is a
    0-d DEVICE tensor that each step overwrites with a device-to-device copy of the next
    schedule entry (the tempered log-joint multiplies by the tensor, so the same captured /
    enqueued work serves every temperature), the log-weights accumulate on the device
    (evaluation.py:155-158) and only the final bound is read back.  The reference performs
    ``n_temperatures`` ``sess.run`` round trips fetching three [chains] arrays each.

    ``run(noise=f)`` injects the HMC noise of step k as ``f(k)`` (k < n_adapt: adaptation
    iterations, then the temperature iterations) and ``init=[...]`` the two prior draws -- the
    parity surface against oracle/evaluation.py.
    """

    def __init__(self, meta_bn, proposal_meta_bn, hmc, observed, latent,
                 n_temperatures=1000, n_adapt=30, verbose=False):
        self._n_temperatures = n_temperatures
        self._n_adapt = n_adapt
        self._verbose = verbose
        if callable(meta_bn):
            log_joint = meta_bn
        else:
            log_joint = lambda obs: meta_bn.observe(**obs).log_joint()
        self._latent_k = list(latent.keys())
        self._latent_v = [latent[k] for k in self._latent_k]
        self._proposal = proposal_meta_bn
        log_prior = lambda obs: proposal_meta_bn.observe(**obs).log_joint()
        dev = self._latent_v[0].device
        # schedule[t] for t = 0..n_temperatures (float64 on the host once, as the reference's
        # NumPy arithmetic; evaluation.py:107-112), then float32 on the device
        t = np.arange(n_temperatures + 1, dtype=np.float64)
        self._schedule = torch.tensor(self._get_schedule_t(t), dtype=torch.float32, device=dev)
        self._temp = torch.zeros((), dtype=torch.float32, device=dev)

        def log_fn(obs):                                  # evaluation.py:91-94
            t = self._temp
            return log_prior(obs) * (1 - t) + log_joint(obs) * t
        self.log_fn = log_fn
        self._observed = dict(observed)
        self.sample_op, self.hmc_info = hmc.sample(log_fn, observed, latent)

    @property
    def temperature(self):
        return self._temp

    def _set_temperature(self, k):
        self._temp.copy_(self._schedule[k])               # device-to-device, no host sync

    def _init_latent(self, values=None):
        """evaluation.py:87, 100-101: z <- a fresh sample of the proposal."""
        if values is None:
            samples = self._proposal.observe().get(self._latent_k)   # as the reference
            values = [s.tensor if hasattr(s, "tensor") else s for s in samples]
        for z, s in zip(self._latent_v, values):
            z.copy_(torch.as_tensor(s, device=z.device))

    def _map_t(self, t):
        return 1. / (1. + np.exp(-4 * (2 * t / self._n_temperatures - 1)))

    def _get_schedule_t(self, t):
        return (self._map_t(t) - self._map_t(0)) / (
            self._map_t(self._n_temperatures) - self._map_t(0))

    def run(self, sess=None, feed_dict=None, noise=None, init=None):
        """evaluation.py:119-165.  ``sess`` is accepted for call-compatibility; observed tensors
        given in ``feed_dict`` by name replace the construction-time observations for the prior
        density AND the HMC transitions (``sess.run(..., feed_dict)`` feeds every op)."""
        obs_update = None
        if feed_dict:
            obs_update = {k: v for k, v in feed_dict.items() if isinstance(k, str)}
            self._observed.update(obs_update)
        step = 0

        def hmc_step():
            nonlocal step, obs_update
            kw = {}
            if noise is not None:
                kw["noise"] = noise(step)
            if obs_update:
                kw["observed"], obs_update = obs_update, None
            self.sample_op(**kw)
            step += 1
        adp_num_t = 2 if self._n_temperatures > 1 else 1
        self._init_latent(init[0] if init is not None else None)
        self._set_temperature(adp_num_t)
        for i in range(self._n_adapt):
            hmc_step()
            if self._verbose:
                print('Adapt iter {}, acc = {:.3f}'.format(
                    i, float(self.hmc_info.acceptance_rate.mean())))
        self._init_latent(init[1] if init is not None else None)
        self._set_temperature(0)
        with torch.no_grad():
            prior_density = self.log_fn(merge_dicts(
                self._observed, dict(zip(self._latent_k, self._latent_v))))
        log_weights = -prior_density.clone()
        for num_t in range(self._n_temperatures):
            self._set_temperature(num_t + 1)
            hmc_step()
            old_log_p = self.hmc_info.orig_log_prob
            new_log_p = self.hmc_info.log_prob
            if num_t + 1 < self._n_temperatures:
                log_weights += old_log_p - new_log_p
            else:
                log_weights += old_log_p
            if self._verbose:
                print('Finished step {}, Temperature = {:.4f}, acc = {:.3f}'
                      .format(num_t + 1, float(self._temp),
                              float(self.hmc_info.acceptance_rate.mean())))
        self.log_weights = log_weights
        return float(self._get_lower_bound(log_weights).mean())   # the ONE read-back

    @staticmethod
    def _get_lower_bound(log_weights):
        """evaluation.py:167-172: log_mean_exp over the chain axis (axis 0)."""
        from . import ops
        return ops.reduce_axes(log_weights.contiguous(), ops.OP_LME, 0)
