"""Oracle of the Generator topologies --no_z / --no_skip / --z_dim and of SEGAN's --reg_loss mse_loss: the CPU
restatement of oracle/segan_oracle.py's Generator forward, read off the state dict.
  - z width: dec_blocks.0 has zc + C input channels (zc = 0 with no_z: z is ignored, the reference's hall has no
    enc_zc);
  - skips: present when the state dict has alpha_<l> keys; conv skips go through conv_skip_oracle.skip_conv.
Contractions are rounded through the oracle's operand-precision control like the plain oracle's.

`gtopo(reg_loss)` routes the oracle's train steps through this forward and, with 'mse_loss', makes the SEGAN step's
regression term l1_weight * mse(Genh, clean) (model.py:79,318)."""
import contextlib
import types

import torch
import torch.nn.functional as F

from oracle import segan_oracle as O
from tests.conv_skip_oracle import skip_conv


def generator_forward(sd, x, z, ret_hid=False, skip_merge="concat"):
    """oracle.segan_oracle.generator_forward for any of the served topologies (same arguments and results)."""
    n_enc = len([k for k in sd if k.startswith("enc_blocks.") and k.endswith("conv.weight")])
    n_dec = len([k for k in sd if k.startswith("dec_blocks.") and k.endswith("deconv.weight")])
    zc = sd["dec_blocks.0.deconv.weight"].shape[0] - sd["enc_blocks.%d.conv.weight" % (n_enc - 1)].shape[0]
    has_skip = any(k.startswith("alpha_") for k in sd)
    hall, skips = {}, {}
    hi = x
    for l in range(n_enc):
        a = O.gconv_linear(hi, sd["enc_blocks.%d.conv.weight" % l], sd.get("enc_blocks.%d.conv.bias" % l))
        hi = O.prelu(a, sd["enc_blocks.%d.act.weight" % l])
        if has_skip and l < n_enc - 1:
            skips[l] = a                      # PRE-activation (generator.py:185,191)
        if ret_hid:
            hall["enc_%d" % l] = hi
    if zc > 0:
        assert z.shape[1] == zc, (z.shape, zc)
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


def _functional_with_l1_as(fn):
    """torch.nn.functional with l1_loss replaced (the oracle's SEGAN step calls F.l1_loss for its regression term)."""
    ns = {k: getattr(F, k) for k in dir(F) if not k.startswith("__")}
    ns["l1_loss"] = fn
    return types.SimpleNamespace(**ns)


@contextlib.contextmanager
def gtopo(reg_loss="l1_loss"):
    """Inside the block the oracle's train steps use this Generator forward and SEGAN's regression term is
    `reg_loss` ('l1_loss' | 'mse_loss'; use it for segan_train_step only: WSEGAN's terms stay L1)."""
    assert reg_loss in ("l1_loss", "mse_loss"), reg_loss
    plain_forward, plain_f = O.generator_forward, O.F
    O.generator_forward = generator_forward
    if reg_loss == "mse_loss":
        O.F = _functional_with_l1_as(F.mse_loss)
    try:
        yield
    finally:
        O.generator_forward, O.F = plain_forward, plain_f
