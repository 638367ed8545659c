"""skip_type='conv' Generators (GSkip Conv1d skips, generator.py:43-49) on the CPU: the conv-skip oracle against
the reference's golden outputs and gradients (tests/golden/conv_skip_generator.npz), seeded construction of the
drop-in modules, the grouped tap-GEMM formulation the kernels run, and which configurations are served."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import segan_oracle as O
from segan_pytorch_b200 import engine as E
from segan_pytorch_b200.segan.models import Generator
from segan_pytorch_b200.segan.models.generator import GSkip
from tests import conv_skip_oracle as CO
from tests.util import build_segan, cpu_state, golden, max_abs, sd_sha, seed_all

GOLD = "conv_skip_generator.npz"


def conv_generator(skip_merge="concat", bias=True, skip_kwidth=11, seed=111):
    seed_all(seed)
    return Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], z_dim=1024, skip_merge=skip_merge,
                     skip_type='conv', skip_kwidth=skip_kwidth, bias=bias)


def golden_inputs(g):
    x = 0.3 * torch.from_numpy(g["xr"])
    return x, torch.from_numpy(g["zr"]), (0.3 * torch.from_numpy(g["cr"])).clamp(-1, 1)


@pytest.fixture(scope="module", autouse=True)
def _threads():
    torch.set_num_threads(max(1, min(8, torch.get_num_threads())))


@pytest.mark.parametrize("merge", ["concat", "sum"])
def test_seeded_generator_matches_reference_init(merge):
    g = golden(GOLD)
    G = conv_generator(merge)
    assert sd_sha(G.state_dict()) == str(g["sha_G_init.%s" % merge])
    assert G._served
    if merge == "concat":
        assert list(G.state_dict().keys()) == [str(k) for k in g["keys"]]
        assert tuple(G.state_dict()["alpha_2.skip_k.weight"].shape) == (256, 256, 11)
        assert tuple(G.state_dict()["alpha_2.skip_k.bias"].shape) == (256,)


def test_no_bias_generator_has_no_skip_bias():
    g = golden(GOLD)
    G = conv_generator(bias=False)
    assert list(G.state_dict().keys()) == [str(k) for k in g["keys_no_bias"]]
    assert not any(k.endswith("skip_k.bias") for k in G.state_dict())
    assert sd_sha(G.state_dict()) == str(g["sha_G_init_no_bias"])


def test_build_segan_conv_matches_reference_init():
    g = golden(GOLD)
    s = build_segan(skip_type="conv")
    sd = s.G.state_dict()
    assert sd_sha(sd) == str(g["sha_segan_G"])
    shapes = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()])
    assert np.array_equal(shapes, g["shapes_segan_G"])
    assert "GSkip" in repr(s.G.alpha_0) and "Conv1d" in repr(s.G.alpha_0)
    # module order: the skips sit between the encoder and the decoder (generator.py:123)
    names = [n for n, _ in s.G.named_parameters()]
    assert names.index("enc_blocks.4.act.weight") < names.index("alpha_0.skip_k.weight") < \
        names.index("dec_blocks.0.deconv.weight")


@pytest.mark.parametrize("merge", ["concat", "sum"])
def test_oracle_forward_vs_golden(merge):
    g = golden(GOLD)
    x, z, _ = golden_inputs(g)
    sd = cpu_state(conv_generator(merge))
    with O.oracle_mode(), torch.no_grad():
        y = CO.generator_forward(sd, x, z, skip_merge=merge)
    assert max_abs(y, g["y.%s" % merge]) <= 1e-5


def test_oracle_gradients_vs_golden():
    g = golden(GOLD)
    x, z, clean = golden_inputs(g)
    sd = cpu_state(conv_generator())
    keys = [k[len("grad_idx."):] for k in g if k.startswith("grad_idx.")]
    assert len(keys) == 9
    with O.oracle_mode():
        p = {k: sd[k].clone().requires_grad_(True) for k in keys}
        loss = 100 * F.l1_loss(CO.generator_forward({**sd, **p}, x, z), clean)
        grads = dict(zip(keys, torch.autograd.grad(loss, [p[k] for k in keys])))
    assert abs(float(loss.detach()) - float(g["l1_loss"])) <= 1e-5 * float(g["l1_loss"])
    for k in keys:
        got = grads[k].reshape(-1)[torch.from_numpy(g["grad_idx." + k])]
        ref = torch.from_numpy(g["grad_val." + k])
        assert float((got - ref).norm()) <= 1e-4 * float(ref.norm()) + 1e-7, k
        assert abs(float(grads[k].double().norm()) - float(g["grad_norm." + k])) <= 1e-4 * float(g["grad_norm." + k])


def test_oracle_routes_train_steps_through_conv_skips():
    sd = cpu_state(conv_generator())
    x, z = torch.zeros(1, 1, 4096), torch.zeros(1, 1024, 4)
    with pytest.raises(KeyError):
        O.generator_forward(sd, x, z)
    with CO.conv_skips():
        assert O.generator_forward is CO.generator_forward
        O.generator_forward(sd, x, z)
    assert O.generator_forward is not CO.generator_forward


@pytest.mark.parametrize("K", [1, 3, 11, 33])
def test_grouped_tap_gemm_equals_conv1d(K):
    torch.manual_seed(K)
    C, B, L = 64, 2, 64
    w = torch.randn(C, C, K, dtype=torch.float64)
    b = torch.randn(C, dtype=torch.float64)
    a = torch.randn(B, L, C, dtype=torch.float64)          # [B][L][C]: the engine's layout of the pre-activation
    ref = F.conv1d(a.transpose(1, 2), w, b, padding=K // 2).transpose(1, 2)
    wp = E.skipconv_pack_reference(w)
    D = (K // 2 + 3) // 4
    assert wp.shape == (2 * D + 1, 4 * C, 4 * C)
    got = E.skipconv_grouped_reference(a, wp, b)
    assert float((got - ref).abs().max()) <= 1e-10
    # the tap table covers every non-zero C x C block; the data-gradient table is the forward one mirrored
    d_lo, d_hi, tap0, fwd, dg = E.skipconv_geometry(C, K)
    assert (d_lo, d_hi, tap0) == (-D, D, 4 - D)
    needed = computed = 0
    for d in range(-D, D + 1):
        blk = wp[d + D].reshape(4, C, 4, C).abs().sum(dim=(1, 3))            # [po][pi]
        nz = blk.nonzero().tolist()
        needed += len(nz)
        for po, pi in nz:
            assert fwd[2][d + 4] <= po * C < fwd[3][d + 4] and fwd[0][d + 4] <= pi * C < fwd[1][d + 4]
        computed += (fwd[1][d + 4] - fwd[0][d + 4]) * (fwd[3][d + 4] - fwd[2][d + 4]) // (C * C)
        assert (dg[0][4 - d], dg[1][4 - d], dg[2][4 - d], dg[3][4 - d]) == \
            (fwd[2][d + 4], fwd[3][d + 4], fwd[0][d + 4], fwd[1][d + 4])
    assert needed == 4 * K
    if K == 11:
        assert computed == 50
        assert (fwd[0][2], fwd[1][2], fwd[2][2], fwd[3][2]) == (3 * C, 4 * C, 0, C)         # d = -2
        assert (fwd[0][6], fwd[1][6], fwd[2][6], fwd[3][6]) == (0, C, 3 * C, 4 * C)         # d = +2


@pytest.mark.parametrize("K", [1, 3, 5, 11, 31, 33])
def test_odd_widths_up_to_33_are_served(K):
    assert conv_generator(skip_kwidth=K)._served


@pytest.mark.parametrize("K", [2, 10, 12, 35, 37])
def test_unserved_widths_raise(K):
    with pytest.raises(NotImplementedError, match="odd skip_kwidth"):
        conv_generator(skip_kwidth=K)


def test_skip_dropout_raises():
    with pytest.raises(NotImplementedError, match="skip_dropout"):
        GSkip('conv', 64, 'one', skip_dropout=0.5, kwidth=11)
