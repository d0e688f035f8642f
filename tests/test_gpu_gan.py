"""Both GAN examples (examples/generative_adversarial_nets/dcgan.py and wasserstein_gan.py) on the
fused layers (tests/gan_models.py) replay the reference's own training step of
tests/golden/ref_gan.npz: both losses, the gradient of each w.r.t. its own variable list, the
moving statistics after the step and the evaluation-mode generator, against the golden and against
the float64 restatement of tests/gan_oracle.py; the discriminator pass of gen_loss gives the bits
of the disc_loss pass.  Then a short training run of each on seeded synthetic images, z from the
prior, that stays finite and moves the losses."""
import os

import numpy as np
import pytest
import torch

import gan_models as GM
import gan_oracle as GO

pytestmark = pytest.mark.gpu


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_gan.npz")


def D64(t):
    return t.detach().double().cpu()


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _names(g, kind, role):
    pre = "%s/%s/" % (kind, role)
    return sorted((k for k in g if k.startswith(pre)), key=lambda k: int(k[len(pre):].split("_")[0]))


def _ordered(p):
    """The trainable tensors of a gan_models / gan_oracle parameter dict in the order the
    network reads them (the golden's order)."""
    out = []
    keys = sorted(k for k in p if k.startswith("W") and k != "Wd")
    for i, k in enumerate(keys):
        out.append(p[k])
        bnk = "bn%d" % i
        if bnk in p:
            out += [p[bnk][kk] for kk in ("gamma", "beta") if kk in p[bnk]]
    for k in ("Wd", "bd", "b3"):
        if k in p:
            out.append(p[k])
    return out


@pytest.mark.parametrize("kind", ["dcgan", "wgan"])
def test_port_replays_the_reference_step(gold, kind):
    """The fused port on the golden's parameters, images and z: both losses, each gradient w.r.t.
    its own list (projected as the golden stores it), the moving statistics after the step and
    the evaluation-mode generator, against the reference run and against float64."""
    g = gold
    gen = GM.params_from_golden(g, kind, "gen")
    disc = GM.params_from_golden(g, kind, "disc")
    x = torch.tensor(g[kind + "/x"], device="cuda")
    z = torch.tensor(2 * g[kind + "/u"] - 1, device="cuda")
    gen_loss, disc_loss, x_gen, fake, fake_g = GM.losses(kind, gen, disc, x, z)
    # the gen_loss pass (detached parameters, throwaway statistics) gives the same logits
    assert torch.equal(fake, fake_g)
    gg = torch.autograd.grad(gen_loss, _ordered(gen))
    dg = torch.autograd.grad(disc_loss, _ordered(disc))

    # float64 restatement on the same inputs
    g64 = {k: ({kk: D64(vv).requires_grad_(kk in ("gamma", "beta")) for kk, vv in v.items()}
               if isinstance(v, dict) else D64(v).requires_grad_(True))
           for k, v in GM.params_from_golden(g, kind, "gen").items()}
    d64 = {k: ({kk: D64(vv).requires_grad_(kk in ("gamma", "beta")) for kk, vv in v.items()}
               if isinstance(v, dict) else D64(v).requires_grad_(True))
           for k, v in GM.params_from_golden(g, kind, "disc").items()}
    gl64, dl64, xg64, gnew, dnew = GO.step(kind, g64, d64, D64(x), D64(z))
    want_g = torch.autograd.grad(gl64, _ordered(g64), retain_graph=True)
    want_d = torch.autograd.grad(dl64, _ordered(d64))

    for got, ref, gold_v in ((gen_loss, gl64, g[kind + "/gen_loss"]),
                             (disc_loss, dl64, g[kind + "/disc_loss"])):
        np.testing.assert_allclose(float(got.detach()), float(ref.detach()), rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(float(got.detach()), gold_v, rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(x_gen.detach().cpu().numpy(), g[kind + "/x_gen"], rtol=1e-5,
                               atol=1e-6)
    # gradients: against float64 at the bound of tests/test_gpu_blvae.py, and against the golden
    k = 0
    for role, got, want in (("gen", gg, want_g), ("disc", dg, want_d)):
        for nm, a, e in zip(_names(g, kind, role), got, want):
            a, e = D64(a), e.detach()
            err = float((a - e).abs().max())
            assert err <= 2e-4 * float(e.abs().max()) + 1e-6, (nm, err)
            tail = nm.split("/", 2)[2]
            if a.numel() > 300:
                gold_v = g["%s/grad_proj_%s/%s" % (kind, role, tail)]
                pr = np.random.default_rng([20261018, k]).standard_normal((8, a.numel()))
                a = pr @ a.numpy().ravel()
            else:
                gold_v, a = g["%s/grad_%s/%s" % (kind, role, tail)], a.numpy()
            np.testing.assert_allclose(a, gold_v, rtol=1e-3,
                                       atol=1e-4 * max(1.0, float(np.abs(gold_v).max())),
                                       err_msg=nm)
            k += 1
    # generator: one update; discriminator: two, on the real batch then on the fake one
    for role, p in (("gen", gen), ("disc", disc)):
        for i in range(3):
            key = "%s/moving_%%s_%s%d" % (kind, role, i)
            np.testing.assert_allclose(p["bn%d" % i]["mm"].cpu().numpy(), g[key % "mean"],
                                       rtol=1e-5, atol=1e-7, err_msg=key % "mean")
            np.testing.assert_allclose(p["bn%d" % i]["mv"].cpu().numpy(), g[key % "variance"],
                                       rtol=1e-5, atol=1e-7, err_msg=key % "variance")
    # evaluation-mode generator on the moved statistics, a second z
    ze = torch.tensor(2 * g[kind + "/u_eval"] - 1, device="cuda")
    G = GM.dcgan_generator if kind == "dcgan" else GM.wgan_generator
    with torch.no_grad():
        xe = G(gen, int(ze.shape[0]), False, ze)
    np.testing.assert_allclose(xe.cpu().numpy(), g[kind + "/x_eval"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind,steps", [("dcgan", 200), ("wgan", 200)])
def test_short_training_run(kind, steps):
    """A few hundred steps on seeded synthetic images (blurred blobs): finite, and the losses
    move."""
    torch.manual_seed(0)
    if kind == "dcgan":
        gen, disc = GM.dcgan_params(0, ngf=16, ndf=8)
        n, shape = 32, (32, 32, 3)
    else:
        gen, disc = GM.wgan_params(0, ngf=16, ndf=8)
        n, shape = 64, (28, 28, 1)
    opt_g, opt_d = GM.optimizers(kind, gen, disc)
    g = torch.Generator(device="cuda").manual_seed(1)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, shape[0], device="cuda"),
                            torch.linspace(-1, 1, shape[1], device="cuda"), indexing="ij")
    hist = []
    for step in range(steps):
        c = torch.rand((n, 2, 1, 1), generator=g, device="cuda") - 0.5
        img = torch.exp(-((yy - c[:, 0]) ** 2 + (xx - c[:, 1]) ** 2) * 6.0)
        x = img[..., None].expand(n, shape[0], shape[1], shape[2]).contiguous()
        hist.append(GM.train_step(kind, gen, disc, x, opt_g, opt_d))       # z from the prior
    h = np.array(hist)
    assert np.isfinite(h).all()
    assert abs(h[-20:, 0].mean() - h[:20, 0].mean()) > 1e-3
    assert abs(h[-20:, 1].mean() - h[:20, 1].mean()) > 1e-3
    for p in GM.trainable(gen) + GM.trainable(disc):
        assert torch.isfinite(p).all()
