"""The logistic-normal topic model trained by Monte-Carlo EM (examples/topic_models/lntm_mcem.py:
148-194) and scored by AIS (:116-142, :208-219) on the GPU, in two arms over one
``zs.fused.LNTMLogJoint`` that holds the whole training corpus:

* ``fused``: HMC takes the E-step log-joint and its gradient from the sparse kernel (the object
  is HMC's provider), the M-step's log p(x | eta, beta) and its beta gradient come from
  ``cond_log_px``, and AIS runs on the tempered provider.
* ``generic``: HMC and AIS differentiate the dense torch restatement of the reference graph (the
  object wrapped in a plain callable), and the M-step forms the dense ``doc_word`` under autograd.

Both arms keep the example's state on the device: the persistent chains ``Eta [chains, docs, K]``
in corpus order (each batch copies its documents' rows in and out), one ``zs.HMC`` whose step-size
adaptation carries across batches, beta with TF's Adam (the restatement of tests/ssl_ais_models.py)
and the learning-rate schedule, the per-epoch ``Eta_mean`` / ``Eta_logstd`` update and the
perplexity.  The shuffle permutation and the HMC noise can be injected.  Imported by the GPU tests
and scripts/bench_lntm_mcem.py.
"""
import math

import torch

from ssl_ais_models import Adam

LOG_DELTA = 10.0


class MCEM(object):
    """x_train: [n_docs, V] counts, already zero-padded to a multiple of ``batch_size``;
    beta0: [K, V] float32 on the device."""

    def __init__(self, zs, x_train, beta0, n_chains=1, batch_size=100, fused=True,
                 num_e_steps=5, step_size=1e-3, n_leapfrogs=20, target_acceptance_rate=0.6,
                 learning_rate_0=1.0, t0=10):
        self.zs, self.fused = zs, fused
        dev = beta0.device
        self.x = torch.as_tensor(x_train, dtype=torch.float32, device=dev)
        n_docs = int(self.x.shape[0])
        K = int(beta0.shape[0])
        if n_docs % batch_size:
            raise ValueError("pad the corpus to a multiple of batch_size (lntm_mcem.py:71-74)")
        self.B, self.iters, self.num_e_steps = batch_size, n_docs // batch_size, num_e_steps
        self.learning_rate_0, self.t0, self.epoch = learning_rate_0, t0, 0
        self.beta = beta0.detach().clone().requires_grad_(True)
        self.opt = Adam({"beta": [self.beta]}, lr=learning_rate_0)
        self.Eta = torch.zeros(n_chains, n_docs, K, device=dev)
        self.lj = zs.fused.LNTMLogJoint(self.x, self.beta, torch.zeros(K, device=dev),
                                        torch.zeros(K, device=dev))
        self.order = torch.arange(n_docs, device=dev)     # corpus row of each shuffled position
        self.eta = torch.zeros(n_chains, batch_size, K, device=dev)
        self.lj.set_docs(self.order[:batch_size])
        self.hmc = zs.HMC(step_size=step_size, n_leapfrogs=n_leapfrogs, adapt_step_size=True,
                          target_acceptance_rate=target_acceptance_rate)
        target = self.lj if fused else (lambda obs: self.lj(obs))
        self.sample_op, self.hmc_info = self.hmc.sample(target, {}, {"eta": self.eta})

    def log_px(self):
        """sum_d mean_c log p(x_d | eta_c, beta) of the current batch (lntm_mcem.py:106-110)."""
        if self.fused:
            return self.lj.cond_log_px(self.eta, self.beta).mean(0).sum()
        x = self.lj.x.index_select(0, self.lj.doc_ids)
        K = self.beta.shape[0]
        doc_word = torch.softmax(self.eta, -1).reshape(-1, K) @ torch.softmax(self.beta, -1)
        doc_word = doc_word.reshape(self.eta.shape[:-1] + (-1,))
        return (x * torch.log(doc_word)).sum(-1).mean(0).sum()

    def batch(self, t, noise=None, record=None):
        """One batch: the E-step's HMC iterations, then the M-step and one Adam step.
        ``noise(j)`` gives the j-th E-step's HMC noise."""
        ids = self.order[t * self.B:(t + 1) * self.B]
        self.lj.set_docs(ids)
        self.eta.copy_(self.Eta[:, ids])
        for j in range(self.num_e_steps):
            self.sample_op(**({"noise": noise(j)} if noise is not None else {}))
            if record is not None:
                record["eta"].append(self.eta.clone())
                record["acc"].append(self.hmc_info.acceptance_rate.clone())
                record["step_size"].append(self.hmc_info.updated_step_size.clone())
        self.Eta[:, ids] = self.eta
        # M-step (lntm_mcem.py:106-114)
        log_p_beta = self.zs.distributions.Normal(
            torch.zeros_like(self.beta), logstd=LOG_DELTA, group_ndims=1).log_prob(self.beta).sum()
        log_px = self.log_px()
        grad, = torch.autograd.grad(-(log_p_beta + log_px), [self.beta])
        self.opt.step({"beta": [grad]})
        self.lj.set_beta(self.beta)
        if record is not None:
            record["log_px"].append(log_px.detach())
            record["grad_beta"].append(grad)
            record["beta"].append(self.beta.detach().clone())
        return log_px.detach()

    def run_epoch(self, perm=None, noise=None, record=None):
        """One epoch (lntm_mcem.py:149-194): shuffle, every batch, then the eta prior update.
        ``perm`` [n_docs] (device int64) is the epoch's shuffle; ``noise(t, j)`` the HMC noise.
        Returns the perplexity as a 0-d device tensor."""
        self.epoch += 1
        self.opt.lr = self.learning_rate_0 * (self.t0 / (self.t0 + self.epoch)) ** 2
        if perm is None:
            perm = torch.randperm(self.order.shape[0], device=self.order.device)
        self.order = self.order[perm]
        lls = []
        for t in range(self.iters):
            lls.append(self.batch(t, None if noise is None else (lambda j: noise(t, j)), record))
        Eta_mean = self.Eta.mean((0, 1))
        Eta_logstd = torch.log(self.Eta.std((0, 1), unbiased=False) + 1e-6)
        self.lj.eta_mean.copy_(Eta_mean)
        self.lj.eta_logstd.copy_(Eta_logstd)
        return torch.exp(-torch.stack(lls).sum() / self.x.sum())

    def ais(self, x_test, n_chains=25, n_temperatures=1000, n_adapt=30, step_size=0.01,
            n_leapfrogs=20, target_acceptance_rate=0.6, noise=None, init=None):
        """The test-set evaluation (lntm_mcem.py:116-142, 208-219): AIS from the eta prior to
        the posterior of every test document under the trained beta and eta prior.  Returns the
        ``zs.AIS`` object and the per-document lower bound."""
        zs, dev = self.zs, self.beta.device
        x_test = torch.as_tensor(x_test, dtype=torch.float32, device=dev)
        n_test = int(x_test.shape[0])
        mean, logstd = self.lj.eta_mean.clone(), self.lj.eta_logstd.clone()
        lj = zs.fused.LNTMLogJoint(x_test, self.beta.detach(), mean, logstd)

        @zs.meta_bayesian_net()
        def eta_prior():                                  # proposal: log_joint = log_prior
            bn = zs.BayesianNet()
            bn.normal("eta", mean.unsqueeze(0).expand(n_test, -1), logstd=logstd,
                      n_samples=n_chains, group_ndims=1)
            return bn
        eta = torch.zeros(n_chains, n_test, int(mean.shape[0]), device=dev)
        hmc = zs.HMC(step_size=step_size, n_leapfrogs=n_leapfrogs, adapt_step_size=True,
                     target_acceptance_rate=target_acceptance_rate)
        ais = zs.AIS(lj if self.fused else (lambda obs: lj(obs)), eta_prior(), hmc, observed={},
                     latent={"eta": eta}, n_temperatures=n_temperatures, n_adapt=n_adapt)
        bound = ais.run(noise=noise, init=init)
        return ais, bound


def perplexity_bound(bound, x_test):
    """lntm_mcem.py:219: exp(-ll_lb * n_docs_test / sum(X_test))."""
    return math.exp(-bound * x_test.shape[0] / float(x_test.sum()))
