"""Oracle of the Generator with convolutional skip connections (GSkip skip_type='conv', generator.py:43-49,
63-64): the CPU restatement of oracle/segan_oracle.py extended by one branch.  A skip whose state dict carries
`alpha_<l>.skip_k.weight` is Conv1d(C, C, K, padding K//2) of the encoder's pre-activation; any other skip is the
alpha scale of the plain oracle.  Inputs, weights and output of the conv are rounded through the oracle's
operand-precision control like its other contractions.

`conv_skips()` routes the oracle's train steps (segan_train_step, wsegan_train_step) through this forward, so
they pick the skip type up from the state dict with no change to their signatures."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import segan_oracle as O

_plain_generator_forward = O.generator_forward


def skip_conv(sd, enc_idx, hj):
    """The conv skip of encoder level enc_idx applied to its pre-activation hj, or None for an alpha skip."""
    w = sd.get("alpha_%d.skip_k.weight" % enc_idx)
    if w is None:
        return None
    return O._q(F.conv1d(O._q(hj), O._q(w), sd.get("alpha_%d.skip_k.bias" % enc_idx), padding=w.shape[2] // 2))


def generator_forward(sd, x, z, ret_hid=False, skip_merge="concat"):
    """oracle.segan_oracle.generator_forward with conv skips (same arguments and results)."""
    n_enc = len([k for k in sd if k.startswith("enc_blocks.") and k.endswith("conv.weight")])
    n_dec = len([k for k in sd if k.startswith("dec_blocks.") and k.endswith("deconv.weight")])
    hall, skips = {}, {}
    hi = x
    for l in range(n_enc):
        a = O.gconv_linear(hi, sd["enc_blocks.%d.conv.weight" % l], sd.get("enc_blocks.%d.conv.bias" % l))
        hi = O.prelu(a, sd["enc_blocks.%d.act.weight" % l])
        if l < n_enc - 1:
            skips[l] = a                      # PRE-activation (generator.py:185,191)
        if ret_hid:
            hall["enc_%d" % l] = hi
    hi = torch.cat((z, hi), dim=1)
    if ret_hid:
        hall["enc_zc"] = hi
    enc_idx = n_enc - 1
    for l in range(n_dec):
        if enc_idx in skips:
            hj = skips[enc_idx]
            sk = skip_conv(sd, enc_idx, hj)
            if sk is None:
                alpha = sd["alpha_%d.skip_k" % enc_idx]
                sk = alpha.repeat(hj.size(0), 1, hj.size(2)) * hj
            hi = sk + hi if skip_merge == "sum" else torch.cat((hi, sk), dim=1)
        h = O.gdeconv_linear(hi, sd["dec_blocks.%d.deconv.weight" % l], sd["dec_blocks.%d.deconv.bias" % l])
        hi = torch.tanh(h) if l == n_dec - 1 else O.prelu(h, sd["dec_blocks.%d.act.weight" % l])
        enc_idx -= 1
        if ret_hid:
            hall["dec_%d" % l] = hi
    return (hi, hall) if ret_hid else hi


@contextlib.contextmanager
def conv_skips():
    """Inside the block the oracle's train steps use the conv-skip aware Generator forward."""
    O.generator_forward = generator_forward
    try:
        yield
    finally:
        O.generator_forward = _plain_generator_forward
