"""Generates tests/golden/kwidth.npz by executing the unmodified reference on CPU: Generators and Discriminators whose
stride-4 convs and transposed convs have kernel widths other than 31.  Runs on its own, so the other fixtures stay
byte-identical:

    SEGAN_REFERENCE_ROOT=/path/to/segan_pytorch python tests/golden/make_golden_kwidth.py

Stored per Generator configuration <c> (kwidth, dec_kwidth; SEGAN+ otherwise: concat alpha skips, bias, z 1024):
  - the sha256 of the seeded state dict and its shapes;
  - the training-mode output of two seeded windows with a seeded z (sampled positions + norm);
  - 100 * L1 against a seeded clean batch and sampled gradients (idx / val / norm) of enc_blocks.0 / .4,
    dec_blocks.0 / .4 and alpha_0.
Stored per Discriminator configuration <c> (kwidth, norm_type bnorm | snorm; pool_type 'none', phase_shift 5):
  - the sha256 of the seeded state dict;
  - the training-mode logits of two seeded (B, 2, 16384) pairs after random.seed(99), and the five phase shifts that
    forward drew (python `random` right after the seeding, in the reference's order);
  - sampled gradients of logit.sum() w.r.t. the first and last tower conv and of the input.
Stored per SEGAN step configuration <c> (gkwidth, gdec_kwidth, dkwidth): one iteration of the reference's SEGAN.train
(batch 4, RMSprop) on the inputs of train_step_b4.npz (python random 99, z from torch seed 1234): the four losses and
sampled parameter updates (idx / delta / norm) of G enc_blocks.1 / dec_blocks.0 / dec_blocks.4 and D enc_blocks.0 /
enc_blocks.1."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_import import load_reference, quiet, reference_opts  # noqa: E402
from tests.golden.make_golden import SEED, sd_sha, seed_all, seeded_randn  # noqa: E402
from tests.golden.make_golden_gsnorm import Y_IDX, sample  # noqa: E402

G_CONFIGS = {"k15_11": (15, 11), "k20_32": (20, 32)}
D_CONFIGS = {"k11_bnorm": (11, "bnorm"), "k32_bnorm": (32, "bnorm"), "k11_snorm": (11, "snorm"),
             "k32_snorm": (32, "snorm")}
STEP_CONFIGS = {"k15_11_21": (15, 11, 21), "k20_32_11": (20, 32, 11)}
STEP_KEYS = ("G.enc_blocks.1.conv.weight", "G.dec_blocks.0.deconv.weight", "G.dec_blocks.4.deconv.weight",
             "D.enc_blocks.0.conv.weight", "D.enc_blocks.1.conv.weight")
G_GRAD_KEYS = ("enc_blocks.0.conv.weight", "enc_blocks.4.conv.weight", "dec_blocks.0.deconv.weight",
               "dec_blocks.4.deconv.weight", "alpha_0.skip_k")
FMAPS = [64, 128, 256, 512, 1024]


def build_generator(ref, kw, dkw):
    seed_all(SEED)
    with quiet():
        return ref.Generator(1, FMAPS, kw, [4] * 5, dec_kwidth=dkw, z_dim=1024, no_z=False, skip=True, bias=True,
                             skip_init="one", skip_type="alpha", skip_merge="concat")


def build_discriminator(ref, kw, norm):
    seed_all(SEED)
    with quiet():
        return ref.Discriminator(2, FMAPS, kw, [4] * 5, pool_type="none", pool_slen=16, norm_type=norm,
                                 phase_shift=5)


def inputs():
    x = 0.3 * seeded_randn(71, (2, 1, 16384))
    clean = (0.3 * seeded_randn(73, (2, 1, 16384))).clamp(-1, 1)
    z = seeded_randn(72, (2, 1024, 16))
    return x, clean, z


def golden_generators(ref, d):
    x, clean, z = inputs()
    for name, (kw, dkw) in G_CONFIGS.items():
        G = build_generator(ref, kw, dkw)
        sd = G.state_dict()
        d["sha_G.%s" % name] = np.array(sd_sha(sd))
        d["shapes.%s" % name] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()])
        G.train()
        y = G(x, z=z)
        d["y.%s" % name] = y.detach().reshape(-1)[torch.from_numpy(Y_IDX)].numpy()
        d["y_norm.%s" % name] = np.array(float(y.detach().double().norm()))
        loss = 100 * torch.nn.functional.l1_loss(y, clean)
        loss.backward()
        d["l1_loss.%s" % name] = np.array(float(loss.detach()))
        params = dict(G.named_parameters())
        for k in G_GRAD_KEYS:
            sample(d, "grad.%s.%s" % (name, k), params[k].grad)


def golden_discriminators(ref, d):
    x, clean, _ = inputs()
    pair = torch.cat((x, clean), 1).requires_grad_(True)
    for name, (kw, norm) in D_CONFIGS.items():
        D = build_discriminator(ref, kw, norm)
        d["sha_D.%s" % name] = np.array(sd_sha(D.state_dict()))
        D.train()
        random.seed(99)
        d["shifts.%s" % name] = np.array(draw_shifts())
        random.seed(99)
        pair.grad = None
        logit, _ = D(pair)
        logit.sum().backward()
        d["logit.%s" % name] = logit.detach().reshape(-1).numpy()
        sfx = "_orig" if norm == "snorm" else ""
        params = dict(D.named_parameters())
        for k in ("enc_blocks.0.conv.weight" + sfx, "enc_blocks.4.conv.weight" + sfx):
            sample(d, "grad.%s.%s" % (name, k), params[k].grad)
        sample(d, "grad.%s.input" % name, pair.grad)


def draw_shifts(n=5, phase_shift=5):
    """The reference's draw order (discriminator.py:161-163): randint(1, ps), then random() > 0.5 means right."""
    out = []
    for _ in range(n):
        shift = random.randint(1, phase_shift)
        out.append(shift if random.random() > 0.5 else -shift)
    return out


def golden_segan_steps(ref, d, B=4):
    for name, (gkw, gdkw, dkw) in STEP_CONFIGS.items():
        over = dict(batch_size=B, epoch=1, save_freq=10 ** 9, gkwidth=gkw, gdec_kwidth=gdkw, dkwidth=dkw)
        seed_all(SEED)
        with quiet():
            segan = ref.SEGAN(reference_opts(**over))
        d["step.sha_G.%s" % name] = np.array(sd_sha(segan.G.state_dict()))
        d["step.sha_D.%s" % name] = np.array(sd_sha(segan.D.state_dict()))
        pre = {("G." + k): v.detach().clone() for k, v in segan.G.state_dict().items()}
        pre.update({("D." + k): v.detach().clone() for k, v in segan.D.state_dict().items()})
        g = torch.Generator().manual_seed(SEED + 2)
        clean = (0.3 * torch.randn(B, 16384, generator=g)).clamp(-1, 1)
        noisy = (clean + 0.1 * torch.randn(B, 16384, generator=g)).clamp(-1, 1)
        dloader = [[["utt%d" % i for i in range(B)], clean.clone(), noisy.clone(), torch.zeros(B)]]
        losses = []
        crit = torch.nn.MSELoss()

        def criterion(a, b):
            l = crit(a, b)
            losses.append(float(l))
            return l
        genh = {}

        def _grab(m, i, o):
            genh.setdefault("y", o.detach().clone())
        segan.G.register_forward_hook(_grab)
        random.seed(99)
        torch.manual_seed(1234)
        with quiet():
            segan.train(reference_opts(**over), dloader, criterion, 100, 1e-5, 100, 10 ** 9, device="cpu")
        assert torch.equal(segan.G.z, seeded_randn(1234, segan.G.z.shape))
        for i, k in enumerate(("d_real_loss", "d_fake_loss", "g_adv_loss")):
            d["step.%s.%s" % (k, name)] = np.array(losses[i])
        d["step.g_l1_loss.%s" % name] = np.array(float(100 * torch.nn.functional.l1_loss(genh["y"],
                                                                                          clean.unsqueeze(1))))
        post = {("G." + k): v for k, v in segan.G.state_dict().items()}
        post.update({("D." + k): v for k, v in segan.D.state_dict().items()})
        for k in STEP_KEYS:
            sample(d, "step.delta.%s.%s" % (name, k), post[k] - pre[k])


def main():
    torch.set_num_threads(8)
    ref = load_reference()
    d = {}
    golden_generators(ref, d)
    golden_discriminators(ref, d)
    golden_segan_steps(ref, d)
    f = os.path.join(HERE, "kwidth.npz")
    np.savez_compressed(f, **d)
    print(f, os.path.getsize(f))


if __name__ == "__main__":
    main()
