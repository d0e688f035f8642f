"""CPU pins of tests/golden/ref_gan.npz, the DCGAN and Wasserstein GAN training step run on the
reference's own BayesianNet on the NumPy TF stand-in (tests/golden/make_ref_gan_golden.py): the
digests, the z draws (bn.uniform("z", -1, 1) = 2 u - 1), and the float64 restatement of
tests/gan_oracle.py reproducing the losses, every gradient (projected where the golden projects
it), the moving statistics after the step and the evaluation-mode generator."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import gan_oracle as GO

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "ref_gan.npz")
PROJ_K, PROJ_SEED = 8, 20261018


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLD))


def test_digests(g):
    with open(os.path.join(HERE, "golden", "ref_gan_digests.json")) as f:
        want = json.load(f)
    assert sorted(want) == sorted("ref_gan/" + k for k in g)
    for k, a in g.items():
        a = np.ascontiguousarray(a)
        assert want["ref_gan/" + k] == [str(a.dtype), list(a.shape),
                                        hashlib.sha256(a.tobytes()).hexdigest()], k


def proj(index, size):
    return np.random.default_rng([PROJ_SEED, index]).standard_normal((PROJ_K, size))


def grad_checks(g, kind, gen_names, disc_names, got_gen, got_disc):
    """(golden key, want, got) per gradient, projected as the golden stores it."""
    out = []
    k = 0
    for role, names, got in (("gen", gen_names, got_gen), ("disc", disc_names, got_disc)):
        for nm, a in zip(names, got):
            a = np.asarray(a, np.float64)             # dense kernels are [out, in] on both sides
            tail = nm.split("/", 2)[2]
            if a.size > 300:
                key = "%s/grad_proj_%s/%s" % (kind, role, tail)
                out.append((key, g[key], proj(k, a.size) @ a.ravel()))
            else:
                key = "%s/grad_%s/%s" % (kind, role, tail)
                out.append((key, g[key], a))
            k += 1
    return out


def trainable_names(g, kind, role):
    pre = "%s/%s/" % (kind, role)
    return sorted((k for k in g if k.startswith(pre)), key=lambda k: int(k[len(pre):].split("_")[0]))


def oracle_run(g, kind):
    D = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)       # noqa: E731
    gen = GO.params_from_golden(g, kind, "gen")
    disc = GO.params_from_golden(g, kind, "disc")

    def leaf(p):
        q = {}
        for k, v in p.items():
            if isinstance(v, dict):
                q[k] = {kk: D(vv).requires_grad_(kk in ("gamma", "beta")) for kk, vv in v.items()}
            else:
                q[k] = D(v).requires_grad_(True)
        return q
    gen, disc = leaf(gen), leaf(disc)
    z = D(2 * g[kind + "/u"].astype(np.float64) - 1)
    gl, dl, x_gen, gnew, dnew = GO.step(kind, gen, disc, D(g[kind + "/x"]), z)

    def by_name(p, names):
        out = []
        for nm in names:
            out.append(_lookup(p, nm, names))
        return out
    gn, dn = trainable_names(g, kind, "gen"), trainable_names(g, kind, "disc")
    gg = torch.autograd.grad(gl, by_name(gen, gn), retain_graph=True)
    dg = torch.autograd.grad(dl, by_name(disc, dn))
    x_eval, _ = GO.generator(kind, GO.with_stats(gen, gnew), D(2 * g[kind + "/u_eval"] - 1.0),
                             False)
    return dict(gen_loss=gl, disc_loss=dl, x_gen=x_gen, gnew=gnew, dnew=dnew, x_eval=x_eval,
                grads=grad_checks(g, kind, gn, dn, [t.numpy() for t in gg],
                                  [t.numpy() for t in dg]))


def _lookup(p, nm, names):
    """The tensor of golden parameter `nm` in the dict p of GO.params_from_golden."""
    i = names.index(nm)
    tail = nm.rsplit("_", 1)[1]
    seen_w, seen_bn, cur, role_disc = 0, -1, False, "/disc/" in nm
    for j, other in enumerate(names[:i + 1]):
        t = other.rsplit("_", 1)[1]
        if t == "kernel":
            is_dense = role_disc and j == len(names) - 2
            key = "Wd" if is_dense else "W%d" % seen_w
            if not is_dense:
                seen_w += 1
            cur = False
            if j == i:
                return p[key]
        elif t in ("gamma", "beta"):
            if not cur:
                seen_bn += 1
                cur = True
            if j == i:
                return p["bn%d" % seen_bn][tail]
        elif j == i:
            return p["bd" if role_disc else "b3"]
    raise KeyError(nm)


@pytest.mark.parametrize("kind", ["dcgan", "wgan"])
def test_oracle_reproduces_the_reference_step(g, kind):
    r = oracle_run(g, kind)
    np.testing.assert_allclose(2 * g[kind + "/u"] - 1, g[kind + "/z"], rtol=0, atol=1e-7)
    # the golden ran in float32 on the stand-in
    np.testing.assert_allclose(float(r["gen_loss"]), g[kind + "/gen_loss"], rtol=2e-5)
    np.testing.assert_allclose(float(r["disc_loss"]), g[kind + "/disc_loss"], rtol=2e-5)
    np.testing.assert_allclose(r["x_gen"].detach().numpy(), g[kind + "/x_gen"], rtol=1e-5,
                               atol=1e-6)
    for key, want, got in r["grads"]:
        np.testing.assert_allclose(got, want, rtol=1e-4,
                                   atol=1e-5 * max(1.0, float(np.abs(want).max())), err_msg=key)
    for role, new in (("gen", r["gnew"]), ("disc", r["dnew"])):
        for i, (m, v) in enumerate(new):
            np.testing.assert_allclose(m.detach().numpy(), g["%s/moving_mean_%s%d" % (kind, role, i)],
                                       rtol=1e-5, atol=1e-7)
            np.testing.assert_allclose(v.detach().numpy(),
                                       g["%s/moving_variance_%s%d" % (kind, role, i)], rtol=1e-5)
    np.testing.assert_allclose(r["x_eval"].detach().numpy(), g[kind + "/x_eval"], rtol=1e-5,
                               atol=1e-6)
