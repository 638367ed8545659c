"""Parameter containers with the reference's block names (segan/models/modules.py:73-141).

The blocks own ordinary nn.Conv1d / nn.ConvTranspose1d / nn.BatchNorm1d / nn.PReLU sub-modules so
that (i) state-dict keys are identical to the reference (SURVEY.md App. B) and (ii) construction
consumes the torch RNG in the reference's order.  Their arithmetic is NOT run through these
sub-modules: Generator / Discriminator drive the sm_90a kernels over whole networks
(segan_pytorch_b200.engine)."""
import torch.nn as nn


def build_norm_layer(norm_type, param=None, num_feats=None):
    if norm_type == 'bnorm':
        return nn.BatchNorm1d(num_feats)
    elif norm_type is None:
        return None
    elif norm_type == 'snorm':
        # the reference re-parametrises the conv in place and uses no norm layer (modules.py:12-14): the same torch
        # utility is applied to the container's nn.Conv1d so that the keys (weight_orig / weight_u / weight_v), the
        # RNG consumption of the u / v initialisation and the init quirks (xavier on the derived `weight` is lost)
        # are the reference's; the power iteration itself runs in the engine (sg_snorm_sigma)
        from torch.nn.utils import spectral_norm
        spectral_norm(param)
        return None
    raise TypeError('Unrecognized norm type: ', norm_type)


class GConv1DBlock(nn.Module):

    def __init__(self, ninp, fmaps, kwidth, stride=1, bias=True, norm_type=None):
        super().__init__()
        self.conv = nn.Conv1d(ninp, fmaps, kwidth, stride=stride, bias=bias)
        self.norm = build_norm_layer(norm_type, self.conv, fmaps)
        self.act = nn.PReLU(fmaps, init=0)
        self.kwidth = kwidth
        self.stride = stride

    def forward(self, x, ret_linear=False):
        raise NotImplementedError("blocks are parameter containers; call Generator / Discriminator")


class GDeconv1DBlock(nn.Module):

    def __init__(self, ninp, fmaps, kwidth, stride=4, bias=True, norm_type=None, act=None):
        super().__init__()
        pad = max(0, (stride - kwidth) // -2)
        # the reference ignores `bias` here: the transposed conv is always biased (modules.py:116-119)
        self.deconv = nn.ConvTranspose1d(ninp, fmaps, kwidth, stride=stride, padding=pad)
        self.norm = build_norm_layer(norm_type, self.deconv, fmaps)
        if act is not None:
            self.act = getattr(nn, act)()
        else:
            self.act = nn.PReLU(fmaps, init=0)
        self.kwidth = kwidth
        self.stride = stride

    def forward(self, x):
        raise NotImplementedError("blocks are parameter containers; call Generator / Discriminator")
