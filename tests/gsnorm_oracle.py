"""Oracle of the spectrally normalised Generator (norm_type='snorm'): torch.nn.utils.spectral_norm as
build_norm_layer applies it (modules.py:12-14) to every encoder Conv1d (dim 0) and decoder ConvTranspose1d (dim 1),
then the topology oracle's forward (tests/gtopo_oracle.py) on the normalised weights.  Skip convs and alphas are not
normalised.  Works in the dtype of the state dict (fp64 for the tests)."""
import torch
import torch.nn.functional as F

from tests import gtopo_oracle as TO


def sn_dim(key):
    """torch's default dim of spectral_norm: 1 for ConvTranspose1d, 0 otherwise."""
    return 1 if ".deconv." in key else 0


def sn_matrix(w, dim):
    """weight -> the [height][rest] matrix torch's spectral_norm iterates on."""
    if dim != 0:
        w = w.permute(dim, *[d for d in range(w.dim()) if d != dim])
    return w.reshape(w.shape[0], -1)


def normalised_state(sd, training):
    """(plain state dict with `<block>.weight` = weight_orig / sigma, {prefix: (u, v, sigma)}).  Training: one power
    iteration v = normalize(W^T u), u = normalize(W v), in place on the u / v tensors of `sd`, without grad; then
    sigma = u^T W v, differentiable w.r.t. weight_orig with u, v held constant (SpectralNorm.compute_weight)."""
    out, vec = {}, {}
    for k, t in sd.items():
        if k.endswith(("weight_u", "weight_v")):
            continue
        if not k.endswith("weight_orig"):
            out[k] = t
            continue
        p = k[:-len("weight_orig")]
        u, v = sd[p + "weight_u"], sd[p + "weight_v"]
        wm = sn_matrix(t, sn_dim(k))
        if training:
            with torch.no_grad():
                v.copy_(F.normalize(torch.mv(wm.detach().t(), u), dim=0, eps=1e-12))
                u.copy_(F.normalize(torch.mv(wm.detach(), v), dim=0, eps=1e-12))
        uc, vc = u.clone(), v.clone()
        sigma = torch.dot(uc, torch.mv(wm, vc))
        out[p + "weight"] = t / sigma
        vec[p] = (uc, vc, sigma)
    return out, vec


def generator_forward(sd, x, z, training=True, skip_merge="concat", ret_hid=False):
    """The snorm Generator's forward on the state dict `sd` (u / v advanced in place when training)."""
    plain, _ = normalised_state(sd, training)
    return TO.generator_forward(plain, x, z, ret_hid=ret_hid, skip_merge=skip_merge)
