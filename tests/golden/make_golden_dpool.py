"""Generates tests/golden/dpool_heads.npz by executing the unmodified reference on CPU: the Discriminator with the
pooled heads pool_type 'conv' / 'gmax' / 'gavg' / 'mlp' (discriminator.py:122-146), each with norm_type 'bnorm' and
'snorm' (seed 111, phase_shift 5).  Runs on its own, so the other fixtures stay byte-identical:

    SEGAN_REFERENCE_ROOT=/path/to/segan_pytorch python tests/golden/make_golden_dpool.py

Stored per head x norm (prefix "<head>.<norm>."): the state-dict keys and shapes; the sha256 of the seeded initial
state dicts of the bare Discriminator, of SEGAN's D (weights_init) and of WSEGAN's D (wsegan_weights_init); a
train-mode pass (python `random` seeded with 5 right before it) with its logits, int_act['avg_conv_h'] ('conv') and
sampled gradients (idx / val / norm) of  mse(logits, 1)  (a mean over all B * Lq logits for 'mlp') for every head
parameter and one tower weight; then an eval-mode pass (`random` seeded with 6) with its logits and avg_conv_h.  The
input is a seeded draw: x = 0.3 xr.  Also the error SEGAN's D loss raises on mlp's B * Lq logits (model.py:298:
criterion(d_real.view(-1), label) with B labels), as `segan_mlp_error`."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_import import load_reference, quiet, reference_opts  # noqa: E402
from tests.golden.make_golden import SEED, arr_sha, hash_str, sd_sha, seed_all, seeded_randn  # noqa: E402

HEADS = ("conv", "gmax", "gavg", "mlp")
NORMS = ("bnorm", "snorm")
FMAPS = [64, 128, 256, 512, 1024]
TRAIN_SEED, EVAL_SEED = 5, 6


def build_discriminator(ref, head, norm):
    seed_all(SEED)
    with quiet():
        return ref.Discriminator(2, FMAPS, 31, [4] * 5, pool_type=head, pool_slen=16, norm_type=norm, phase_shift=5)


def golden_dpool(ref, out):
    d = {}
    xr = seeded_randn(71, (3, 2, 16384))
    d.update({"xr.seed": np.array(71), "xr.shape": np.array((3, 2, 16384)), "xr.sha256": np.array(arr_sha(xr))})
    x = 0.3 * xr
    for head in HEADS:
        for norm in NORMS:
            p = "%s.%s." % (head, norm)
            D = build_discriminator(ref, head, norm)
            sd = D.state_dict()
            d[p + "keys"] = np.array(list(sd.keys()))
            d[p + "shapes"] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()])
            d[p + "sha_D"] = np.array(sd_sha(sd))
            seed_all(SEED)
            with quiet():
                segan = ref.SEGAN(reference_opts(dpool_type=head, dnorm_type=norm))
            d[p + "sha_segan_D"] = np.array(sd_sha(segan.D.state_dict()))
            seed_all(SEED)
            with quiet():
                wsegan = ref.WSEGAN(reference_opts(wsegan=True, misalign_pair=True, dpool_type=head, dnorm_type=norm))
            d[p + "sha_wsegan_D"] = np.array(sd_sha(wsegan.D.state_dict()))
            D.train()
            random.seed(TRAIN_SEED)
            y, act = D(x)
            d[p + "y_train"] = y.detach().numpy()
            if head == "conv":
                d[p + "avg_conv_h_train"] = act["avg_conv_h"].detach().numpy()
            D.zero_grad()
            loss = torch.nn.functional.mse_loss(y, torch.ones_like(y))
            loss.backward()
            d[p + "loss"] = np.array(float(loss.detach()))
            params = dict(D.named_parameters())
            keys = [k for k in params if not k.startswith("enc_blocks.")] + \
                ["enc_blocks.2.conv.weight" + ("_orig" if norm == "snorm" else "")]
            d[p + "grad_keys"] = np.array(keys)
            for k in keys:
                gr = params[k].grad.reshape(-1)
                idx = np.sort(np.random.RandomState(hash_str(k) % (2 ** 31)).choice(
                    gr.numel(), size=min(1024, gr.numel()), replace=False)).astype(np.int64)
                d[p + "grad_idx." + k] = idx
                d[p + "grad_val." + k] = gr[idx].numpy()
                d[p + "grad_norm." + k] = np.array(float(gr.double().norm()))
            D.eval()
            random.seed(EVAL_SEED)
            with torch.no_grad():
                y, act = D(x)
            d[p + "y_eval"] = y.numpy()
            if head == "conv":
                d[p + "avg_conv_h_eval"] = act["avg_conv_h"].numpy()
            if head == "mlp" and norm == "bnorm":
                try:
                    torch.nn.MSELoss()(y.view(-1), torch.ones(x.shape[0]))
                except RuntimeError as e:
                    d["segan_mlp_error"] = np.array(str(e))
    np.savez_compressed(os.path.join(out, "dpool_heads.npz"), **d)


def main():
    torch.set_num_threads(8)
    golden_dpool(load_reference(), HERE)
    f = os.path.join(HERE, "dpool_heads.npz")
    print(f, os.path.getsize(f))


if __name__ == "__main__":
    main()
