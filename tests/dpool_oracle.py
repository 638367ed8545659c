"""Oracle of the Discriminator with a pooled head (pool_type 'conv' / 'gmax' / 'gavg' / 'mlp', discriminator.py:122-146,
175-192): oracle/segan_oracle.py's discriminator_forward with the head chosen from the state dict -- `pool_conv.*`
keys: 'conv'; `mlp.*`: 'mlp'; `fc.0.*`: 'none' -- or, for the parameter-free poolings whose state dicts look alike,
from `pool_type`.  The tower is the plain oracle's own (it runs under a zero stand-in of the FC head and hands back
its last activation), so both heads share one tower.  The tower activation entering the head and mlp.0's input,
weight and output are rounded through the oracle's operand-precision control, as the kernels store them; the head's
small dots stay fp32, as in the kernels.

`pooled_heads(pool_type)` routes the oracle's train steps (segan_train_step, wsegan_train_step) through this forward,
so they pick the head up with no change to their signatures."""
import contextlib
import functools

import torch
import torch.nn.functional as F

from oracle import segan_oracle as O

_plain_discriminator_forward = O.discriminator_forward


def head_of(sd, pool_type=None):
    if "pool_conv.bias" in sd:
        return "conv"
    if "mlp.2.bias" in sd:
        return "mlp"
    if "fc.0.bias" in sd:
        return "none"
    if pool_type not in ("gmax", "gavg"):
        raise ValueError("a state dict with a bare `fc` head needs pool_type 'gmax' or 'gavg', got %r" % (pool_type,))
    return pool_type


def tower(sd, x, shifts, training=True):
    """The plain oracle's conv tower (BatchNorm statistics / power-iteration vectors in `sd` are updated in place):
    (last activation (B, C, Lq), acts).  The FC head it runs afterwards is a zero stand-in and is discarded."""
    n_enc = len([k for k in sd if k.startswith("enc_blocks.") and (k.endswith("conv.weight") or
                                                                   k.endswith("conv.weight_orig"))])
    c = sd["enc_blocks.%d.act.weight" % (n_enc - 1)].numel()
    kin = c * (x.shape[-1] // 4 ** n_enc)
    z = lambda *shape: torch.zeros(*shape, dtype=x.dtype)
    stand_in = {"fc.0.weight": z(256, kin), "fc.0.bias": z(256), "fc.1.weight": z(256), "fc.2.weight": z(128, 256),
                "fc.2.bias": z(128), "fc.3.weight": z(128), "fc.4.weight": z(1, 128), "fc.4.bias": z(1)}
    _, acts = _plain_discriminator_forward({**sd, **stand_in}, x, shifts, training=training, ret_act=True)
    del acts["logit"]
    return acts["h_%d" % (n_enc - 1)], acts


def discriminator_forward(sd, x, shifts, training=True, ret_act=False, pool_type=None):
    """oracle.segan_oracle.discriminator_forward with the pooled heads (same arguments and results; logits (B, 1),
    (B, 1, Lq) for 'mlp'; ret_act adds 'avg_conv_h' for the 'conv' head)."""
    head = head_of(sd, pool_type)
    if head == "none":
        return _plain_discriminator_forward(sd, x, shifts, training=training, ret_act=ret_act)
    h, acts = tower(sd, x, shifts, training)
    h = O._q(h)
    B = h.size(0)
    if head == "conv":
        a = F.conv1d(h, O._weight(sd, "pool_conv.", training), sd["pool_conv.bias"]).view(B, -1)
        acts["avg_conv_h"] = a
        y = F.linear(a, O._weight(sd, "fc.", training), sd["fc.bias"])
    elif head == "mlp":
        z = O._q(F.conv1d(h, O._q(O._weight(sd, "mlp.0.", training)), sd["mlp.0.bias"]))
        hm = O._q(F.prelu(z, O._weight(sd, "mlp.1.", training)))
        y = F.conv1d(hm, sd["mlp.2.weight"], sd["mlp.2.bias"])
    else:
        pooled = F.adaptive_max_pool1d(h, 1) if head == "gmax" else F.adaptive_avg_pool1d(h, 1)
        y = F.linear(pooled.view(B, -1), O._weight(sd, "fc.", training), sd["fc.bias"])
    acts["logit"] = y
    return (y, acts) if ret_act else y


@contextlib.contextmanager
def pooled_heads(pool_type):
    """Inside the block the oracle's train steps use the head-aware Discriminator forward for `pool_type`."""
    O.discriminator_forward = functools.partial(discriminator_forward, pool_type=pool_type)
    try:
        yield
    finally:
        O.discriminator_forward = _plain_discriminator_forward
