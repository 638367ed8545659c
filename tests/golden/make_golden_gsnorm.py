"""Generates tests/golden/g_snorm.npz by executing the unmodified reference on CPU: spectrally normalised Generators
(Generator(..., norm_type='snorm')) in six configurations, plus one SEGAN(opts, generator=G_snorm) step.  Runs on
its own, so the other fixtures stay byte-identical:

    SEGAN_REFERENCE_ROOT=/path/to/segan_pytorch python tests/golden/make_golden_gsnorm.py

Stored per configuration <c>:
  - state-dict keys and shapes, the sha256 of the seeded state dict bare and after weights_init / wsegan_weights_init;
  - after ONE training-mode forward (torch.no_grad) on two seeded windows: every weight_u in full, weight_v sampled
    (idx / val / norm), sigma = u^T W v, and the output (sampled positions + norm);
  - the eval-mode output of the same windows;
  - after a further training-mode forward, sampled gradients (idx / val / norm) of 100 * L1 w.r.t. weight_orig of
    enc_blocks.0 / enc_blocks.4 / dec_blocks.0 / dec_blocks.4 and the first skip's alpha where present.
The SEGAN step (default configuration, batch 4) uses the inputs, z and python seed of train_step_b4.npz and stores its
four losses and the Generator's weight_u / weight_v afterwards."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_import import load_reference, quiet, reference_opts  # noqa: E402
from tests.golden.make_golden import SEED, arr_sha, hash_str, sd_sha, seed_all, seeded_randn  # noqa: E402

# name -> Generator keyword arguments over the SEGAN+ defaults (bias=True, skip_merge='concat', alpha skips)
CONFIGS = {
    "concat": dict(),
    "sum": dict(skip_merge="sum"),
    "conv": dict(skip_type="conv"),
    "no_z": dict(no_z=True),
    "no_skip": dict(skip=False),
    "no_bias": dict(bias=False),
}
N_SAMPLE = 256
Y_IDX = np.sort(np.random.RandomState(7).choice(2 * 16384, size=4096, replace=False)).astype(np.int64)
GRAD_KEYS = ("enc_blocks.0.conv.weight_orig", "enc_blocks.4.conv.weight_orig", "dec_blocks.0.deconv.weight_orig",
             "dec_blocks.4.deconv.weight_orig", "alpha_0.skip_k")


def generator_kwargs(name):
    kw = dict(z_dim=1024, no_z=False, skip=True, bias=True, skip_init="one", skip_type="alpha", skip_merge="concat",
              skip_kwidth=11, norm_type="snorm")
    kw.update(CONFIGS[name])
    return kw


def build_generator(ref, name):
    seed_all(SEED)
    with quiet():
        return ref.Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], **generator_kwargs(name))


def sample(d, tag, t):
    flat = t.detach().reshape(-1)
    idx = np.sort(np.random.RandomState(hash_str(tag) % (2 ** 31)).choice(
        flat.numel(), size=min(N_SAMPLE, flat.numel()), replace=False)).astype(np.int64)
    d["idx." + tag] = idx
    d["val." + tag] = flat[idx].numpy()
    d["norm." + tag] = np.array(float(flat.double().norm()))


def sn_prefixes(sd):
    return [k[:-len("weight_orig")] for k in sd if k.endswith("weight_orig")]


def store_vectors(d, tag, G):
    sd = G.state_dict()
    for p in sn_prefixes(sd):
        u, v = sd[p + "weight_u"], sd[p + "weight_v"]
        w = sd[p + "weight_orig"]
        wm = (w.transpose(0, 1) if ".deconv." in p else w).reshape(u.numel(), -1)
        d["u.%s.%s" % (tag, p)] = u.clone().numpy()          # a copy: the buffer is updated in place later
        sample(d, "v.%s.%s" % (tag, p), v)
        d["sigma.%s.%s" % (tag, p)] = np.array(float(torch.dot(u.double(), wm.double() @ v.double())))


def golden_generators(ref, d):
    raw = {}
    for k, seed, shape in (("xr", 71, (2, 1, 16384)), ("cr", 73, (2, 1, 16384)), ("zr", 72, (2, 1024, 16))):
        raw[k] = seeded_randn(seed, shape)
        d.update({k + ".seed": np.array(seed), k + ".shape": np.array(shape), k + ".sha256": np.array(arr_sha(raw[k]))})
    x, clean = 0.3 * raw["xr"], (0.3 * raw["cr"]).clamp(-1, 1)
    for name in CONFIGS:
        G = build_generator(ref, name)
        sd = G.state_dict()
        d["keys.%s" % name] = np.array(list(sd.keys()))
        d["shapes.%s" % name] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()])
        d["sha_G_init.%s" % name] = np.array(sd_sha(sd))
        for init_name in ("weights_init", "wsegan_weights_init"):
            Gi = build_generator(ref, name)
            torch.manual_seed(5)
            Gi.apply(getattr(ref, init_name))
            d["sha_%s.%s" % (init_name, name)] = np.array(sd_sha(Gi.state_dict()))
        z = None if generator_kwargs(name)["no_z"] else raw["zr"]
        G.train()
        with torch.no_grad():
            y = G(x, z=z)
        d["y_train.%s" % name] = y.reshape(-1)[torch.from_numpy(Y_IDX)].numpy()
        d["y_train_norm.%s" % name] = np.array(float(y.double().norm()))
        store_vectors(d, "train1.%s" % name, G)
        G.eval()
        with torch.no_grad():
            y = G(x, z=z)
        d["y_eval.%s" % name] = y.reshape(-1)[torch.from_numpy(Y_IDX)].numpy()
        d["y_eval_norm.%s" % name] = np.array(float(y.double().norm()))
        G.train()
        G.zero_grad()
        loss = 100 * torch.nn.functional.l1_loss(G(x, z=z), clean)
        loss.backward()
        d["l1_loss.%s" % name] = np.array(float(loss.detach()))
        params = dict(G.named_parameters())
        for k in GRAD_KEYS:
            if k in params:
                sample(d, "grad.%s.%s" % (name, k), params[k].grad)


def golden_segan_step(ref, d, B=4):
    """One iteration of the reference's SEGAN.train with a snorm Generator passed in (SEGAN(opts, generator=G)):
    the inputs of make_golden.golden_train_step (clean / noisy, python random 99, z from torch seed 1234)."""
    over = dict(batch_size=B, epoch=1, save_freq=10 ** 9)
    G = build_generator(ref, "concat")
    seed_all(SEED)
    with quiet():
        segan = ref.SEGAN(reference_opts(**over), generator=G)
    d["step.sha_G"] = np.array(sd_sha(segan.G.state_dict()))
    d["step.sha_D"] = np.array(sd_sha(segan.D.state_dict()))
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
    d["step.d_real_loss"] = np.array(losses[0])
    d["step.d_fake_loss"] = np.array(losses[1])
    d["step.g_adv_loss"] = np.array(losses[2])
    d["step.g_l1_loss"] = np.array(float(100 * torch.nn.functional.l1_loss(genh["y"], clean.unsqueeze(1))))
    store_vectors(d, "step", segan.G)


def main():
    torch.set_num_threads(8)
    ref = load_reference()
    d = {}
    golden_generators(ref, d)
    golden_segan_step(ref, d)
    f = os.path.join(HERE, "g_snorm.npz")
    np.savez_compressed(f, **d)
    print(f, os.path.getsize(f))


if __name__ == "__main__":
    main()
