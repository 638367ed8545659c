"""Generates tests/golden/conv_skip_generator.npz by executing the unmodified reference on CPU: the Generator with
convolutional skip connections (skip_type='conv', skip_kwidth 11, bias on; seed 111).  Runs on its own, so the
other fixtures of make_golden.py stay byte-identical:

    SEGAN_REFERENCE_ROOT=/path/to/segan_pytorch python tests/golden/make_golden_conv_skip.py

Stored: the sha256 of the seeded initial state dicts (bare Generator, SEGAN's G after weights_init, and the keys /
shapes with --no_bias), the eval outputs for two seeded windows with skip_merge 'concat' and 'sum', and sampled
gradients of 100 * L1 (idx / val / norm) for the four skip convs and one encoder weight (concat)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_import import load_reference, quiet  # noqa: E402
from tests.golden.make_golden import (SEED, arr_sha, build_reference_segan, hash_str, sd_sha, seed_all,
                                      seeded_randn)  # noqa: E402

SKIP_KW = 11
GRAD_KEYS = tuple("alpha_%d.skip_k.%s" % (l, s) for l in range(4) for s in ("weight", "bias")) + \
    ("enc_blocks.2.conv.weight",)


def build_generator(ref, skip_merge, bias=True):
    seed_all(SEED)
    with quiet():
        return ref.Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], z_dim=1024, skip_merge=skip_merge,
                             skip_type='conv', skip_kwidth=SKIP_KW, bias=bias)


def golden_conv_skip_generator(ref, out):
    d = {}
    # inputs as seeded draws (tests/util.golden re-draws them and checks the sha256): x = 0.3 xr, z = zr,
    # clean = clamp(0.3 cr, -1, 1)
    raw = {}
    for k, seed, shape in (("xr", 61, (2, 1, 16384)), ("zr", 62, (2, 1024, 16)), ("cr", 63, (2, 1, 16384))):
        raw[k] = seeded_randn(seed, shape)
        d.update({k + ".seed": np.array(seed), k + ".shape": np.array(shape), k + ".sha256": np.array(arr_sha(raw[k]))})
    x, z, clean = 0.3 * raw["xr"], raw["zr"], (0.3 * raw["cr"]).clamp(-1, 1)
    for merge in ("concat", "sum"):
        G = build_generator(ref, merge)
        d["sha_G_init.%s" % merge] = np.array(sd_sha(G.state_dict()))
        G.eval()
        with torch.no_grad():
            d["y.%s" % merge] = G(x, z=z).numpy()
        if merge == "concat":
            d["keys"] = np.array(list(G.state_dict().keys()))
            G.zero_grad()
            loss = 100 * torch.nn.functional.l1_loss(G(x, z=z), clean)
            loss.backward()
            d["l1_loss"] = np.array(float(loss.detach()))
            params = dict(G.named_parameters())
            for k in GRAD_KEYS:
                gr = params[k].grad.reshape(-1)
                idx = np.sort(np.random.RandomState(hash_str(k) % (2 ** 31)).choice(
                    gr.numel(), size=min(1024, gr.numel()), replace=False)).astype(np.int64)
                d["grad_idx.%s" % k] = idx
                d["grad_val.%s" % k] = gr[idx].numpy()
                d["grad_norm.%s" % k] = np.array(float(gr.double().norm()))
    nb = build_generator(ref, "concat", bias=False)
    d["keys_no_bias"] = np.array(list(nb.state_dict().keys()))
    d["sha_G_init_no_bias"] = np.array(sd_sha(nb.state_dict()))
    # the full model: SEGAN(train.opts with skip_type conv) applies weights_init to G
    segan = build_reference_segan(ref, skip_type='conv')
    d["sha_segan_G"] = np.array(sd_sha(segan.G.state_dict()))
    d["shapes_segan_G"] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in segan.G.state_dict().values()])
    np.savez_compressed(os.path.join(out, "conv_skip_generator.npz"), **d)


def main():
    torch.set_num_threads(8)
    golden_conv_skip_generator(load_reference(), HERE)
    f = os.path.join(HERE, "conv_skip_generator.npz")
    print(f, os.path.getsize(f))


if __name__ == "__main__":
    main()
