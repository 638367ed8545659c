"""Generates tests/golden/g_topology.npz by executing the unmodified reference on CPU: Generators without z
(--no_z), without skip connections (--no_skip), with a narrower z (--z_dim 256) and the combinations below, plus
one SEGAN step with --reg_loss mse_loss.  Runs on its own, so the other fixtures of make_golden.py stay
byte-identical:

    SEGAN_REFERENCE_ROOT=/path/to/segan_pytorch python tests/golden/make_golden_gtopo.py

Stored per configuration <c>: state-dict keys and shapes, the sha256 of the seeded initial state dicts (bare
Generator, SEGAN's G after weights_init), the eval outputs for two seeded windows (4096 sampled positions and the
norm) and the `hall` keys, and sampled gradients (idx / val / norm) of 100 * L1 and 100 * MSE for dec_blocks.0, dec_blocks.4, enc_blocks.4 and, where
present, the first skip's alpha (or conv weight).  The SEGAN step uses the inputs, z and python seed of
train_step_b4.npz (make_golden.golden_train_step) and stores its four losses."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_import import load_reference, quiet, reference_opts  # noqa: E402
from tests.golden.make_golden import (SEED, arr_sha, build_reference_segan, hash_str, sd_sha, seed_all,
                                      seeded_randn)  # noqa: E402

# name -> train.py options over ckpt_segan+/train.opts
CONFIGS = {
    "no_z": dict(no_z=True),
    "no_skip": dict(no_skip=True),
    "no_z_no_skip": dict(no_z=True, no_skip=True),
    "z256": dict(z_dim=256),
    "no_z_sum": dict(no_z=True, skip_merge="sum"),
    "no_z_conv": dict(no_z=True, skip_type="conv"),
    "no_skip_no_bias": dict(no_skip=True, bias=False),
}
N_GRAD = 256
Y_IDX = np.sort(np.random.RandomState(7).choice(2 * 16384, size=4096, replace=False)).astype(np.int64)
GRAD_PREFIXES = ("dec_blocks.0.deconv.weight", "dec_blocks.4.deconv.weight", "enc_blocks.4.conv.weight",
                 "alpha_0.skip_k")


def generator_kwargs(over):
    """Generator constructor arguments of SEGAN.__init__ (model.py:82-96) for the options `over`."""
    o = reference_opts(**over)
    return dict(z_dim=o.z_dim, no_z=o.no_z, skip=not o.no_skip, bias=o.bias, skip_init=o.skip_init,
                skip_type=o.skip_type, skip_merge=o.skip_merge, skip_kwidth=o.skip_kwidth)


def build_generator(ref, over):
    seed_all(SEED)
    with quiet():
        return ref.Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], **generator_kwargs(over))


def grad_keys(G):
    names = [n for n, _ in G.named_parameters()]
    return [n for n in names if any(n == p or n == p + ".weight" for p in GRAD_PREFIXES)]


def golden_topologies(ref, d):
    raw = {}
    for k, seed, shape in (("xr", 71, (2, 1, 16384)), ("cr", 73, (2, 1, 16384))):
        raw[k] = seeded_randn(seed, shape)
        d.update({k + ".seed": np.array(seed), k + ".shape": np.array(shape), k + ".sha256": np.array(arr_sha(raw[k]))})
    x, clean = 0.3 * raw["xr"], (0.3 * raw["cr"]).clamp(-1, 1)
    for name, over in CONFIGS.items():
        G = build_generator(ref, over)
        sd = G.state_dict()
        d["keys.%s" % name] = np.array(list(sd.keys()))
        d["shapes.%s" % name] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()])
        d["sha_G_init.%s" % name] = np.array(sd_sha(sd))
        zdim = generator_kwargs(over)["z_dim"]
        no_z = generator_kwargs(over)["no_z"]
        # z as a seeded draw (absent with no_z: the reference ignores it and draws none)
        z = None
        if not no_z:
            z = seeded_randn(72, (2, zdim, 16))
            d.update({"zr.%s.seed" % name: np.array(72), "zr.%s.shape" % name: np.array(z.shape),
                      "zr.%s.sha256" % name: np.array(arr_sha(z))})
        G.eval()
        with torch.no_grad():
            y, hall = G(x, z=z, ret_hid=True)
        # outputs at a fixed sample of positions (the full outputs of seven configurations would not fit the
        # fixture's size budget) and the norm of the whole output
        d["y_idx.%s" % name] = Y_IDX
        d["y_val.%s" % name] = y.reshape(-1)[torch.from_numpy(Y_IDX)].numpy()
        d["y_norm.%s" % name] = np.array(float(y.double().norm()))
        d["hall_keys.%s" % name] = np.array(sorted(hall.keys()))
        d["has_z_attr.%s" % name] = np.array(hasattr(G, "z"))
        for loss_name, fn in (("l1", torch.nn.functional.l1_loss), ("mse", torch.nn.functional.mse_loss)):
            G.zero_grad()
            loss = 100 * fn(G(x, z=z), clean)
            loss.backward()
            d["%s_loss.%s" % (loss_name, name)] = np.array(float(loss.detach()))
            params = dict(G.named_parameters())
            for k in grad_keys(G):
                gr = params[k].grad.reshape(-1)
                idx = np.sort(np.random.RandomState(hash_str(k) % (2 ** 31)).choice(
                    gr.numel(), size=min(N_GRAD, gr.numel()), replace=False)).astype(np.int64)
                tag = "%s.%s.%s" % (loss_name, name, k)
                d["grad_idx." + tag] = idx
                d["grad_val." + tag] = gr[idx].numpy()
                d["grad_norm." + tag] = np.array(float(gr.double().norm()))
        segan = build_reference_segan(ref, **over)
        d["sha_segan_G.%s" % name] = np.array(sd_sha(segan.G.state_dict()))


def golden_mse_step(ref, d, B=4):
    """One iteration of the reference's SEGAN.train with reg_loss='mse_loss', on the inputs of
    make_golden.golden_train_step (same seeds: clean / noisy, python random 99, z from torch seed 1234)."""
    over = dict(batch_size=B, epoch=1, save_freq=10 ** 9, reg_loss="mse_loss")
    segan = build_reference_segan(ref, **over)
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
    d["mse_step.d_real_loss"] = np.array(losses[0])
    d["mse_step.d_fake_loss"] = np.array(losses[1])
    d["mse_step.g_adv_loss"] = np.array(losses[2])
    d["mse_step.g_reg_loss"] = np.array(float(100 * torch.nn.functional.mse_loss(genh["y"], clean.unsqueeze(1))))


def main():
    torch.set_num_threads(8)
    ref = load_reference()
    d = {}
    golden_topologies(ref, d)
    golden_mse_step(ref, d)
    f = os.path.join(HERE, "g_topology.npz")
    np.savez_compressed(f, **d)
    print(f, os.path.getsize(f))


if __name__ == "__main__":
    main()
