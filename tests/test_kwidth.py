"""Kernel widths other than 31 without a GPU: which widths the Generator and Discriminator serve, the packed layouts and
tap tables at every width 4..32 (and unchanged at 31), and the reference fixture tests/golden/kwidth.npz pinned to the
seeded modules."""
import pytest
import torch

from segan_pytorch_b200 import engine as E
from segan_pytorch_b200.segan.models import Generator
from segan_pytorch_b200.segan.models.discriminator import Discriminator
from tests.util import golden, sd_sha, seed_all

FMAPS = [64, 128, 256, 512, 1024]


def kw_generator(kw, dkw, seed=111, **over):
    seed_all(seed)
    kw_args = dict(dec_kwidth=dkw, z_dim=1024, no_z=False, skip=True, bias=True, skip_init="one", skip_type="alpha",
                   skip_merge="concat")
    kw_args.update(over)
    return Generator(1, FMAPS, kw, [4] * 5, **kw_args)


def im2col_ref(v, off, k, reflect, roll):
    """col[b][t][ci*32 + j] = pad(v_ci)[4t + j - off] for j < k, else 0 (fp64; reflect: after the circular roll)."""
    B, L = v[0].shape
    col = torch.zeros(B, L // 4, 64, dtype=torch.float64)
    q = (4 * torch.arange(L // 4).view(-1, 1) + torch.arange(k).view(1, -1) - off)
    for ci, vc in enumerate(v):
        if reflect:
            r = q.abs()
            r = torch.where(r >= L, 2 * (L - 1) - r, r)
            vals = vc[:, (r - roll) % L]
        else:
            ok = (q >= 0) & (q < L)
            vals = vc[:, q.clamp(0, L - 1)] * ok
        col[:, :, ci * 32:ci * 32 + k] = vals
    return col


@pytest.mark.parametrize("k,served", [(3, False), (4, True), (11, True), (20, True), (31, True), (32, True),
                                      (33, False)])
def test_served_widths(k, served):
    G = kw_generator(k, 31)
    Gd = kw_generator(31, k)
    D = Discriminator(2, FMAPS, k, [4] * 5, pool_slen=16)
    for m in (G, Gd, D):
        assert m._served == served
        if not served:
            with pytest.raises(NotImplementedError, match="4-32"):
                m.engine


def test_per_layer_widths_served():
    assert kw_generator([15, 11, 31, 4, 32], [20, 5, 6, 32, 11])._served
    assert not kw_generator([15, 11, 31, 4, 33], 11)._served


@pytest.mark.parametrize("kind", [0, 1])
def test_pack_round_trip_and_tap_ranges_every_width(kind):
    """pack / unpack round trip at every width, and each tap table's ranges are exactly the non-zero blocks of the
    packed weight (data-gradient tables: of the transposed taps); tap_span bounds the non-empty taps."""
    c = 2
    for k in range(4, 33):
        w = torch.rand((c, c, k)) + 0.5
        m = E.pack_reference(kind, w, c, c, 0, k)
        assert torch.equal(E.unpack_reference(kind, m, c, c, 0, k), w)
        fwd, dg = ("conv_fwd", "conv_dgrad") if kind == 0 else ("deconv_fwd", "deconv_dgrad")
        # kind 0: M[t][co][p*c + ci] (phases along K); kind 1: M[t][r*c + co][ci] (phases along N)
        nz = m.view(9, c, 4, c).ne(0).any(3).any(1) if kind == 0 else m.view(9, 4, c, c).ne(0).any(3).any(2)
        for name, flip in ((fwd, False), (dg, True)):
            kc, nc = (4 * c, c) if (name in ("conv_fwd", "deconv_dgrad")) else (c, 4 * c)
            taps = E.tap_ranges(name, c, kc, nc, k)
            on_k = name in ("conv_fwd", "deconv_dgrad")
            lo, hi = (taps[0], taps[1]) if on_k else (taps[2], taps[3])
            for i in range(9):
                ph = nz[8 - i] if flip else nz[i]
                want = [p for p in range(4) if ph[p]]
                got = list(range(lo[i] // c, hi[i] // c))
                assert got == want, (k, name, i, got, want)
            d_lo, d_hi = E.tap_span(taps)
            live = [i - 4 for i in range(9) if (nz[8 - i] if flip else nz[i]).any()]
            assert (d_lo, d_hi) == (live[0], live[-1]) and live == list(range(d_lo, d_hi + 1))


def test_width_31_layouts_unchanged():
    """At k = 31 the tap tables and packed layouts are those of the fixed-width engine: tap -4 reads conv phases
    {2, 3} / deconv phases {0, 1}, tap +4 conv phase 0 / deconv phase 3, every other tap all phases; the packed
    layouts place W[.., 4d + p + 14] / W[.., -4d + r + 13]."""
    c = 64
    assert E.tap_ranges("conv_fwd", c, 4 * c, 128) == ([128] + [0] * 8, [256] * 8 + [64], [0] * 9, [128] * 9)
    assert E.tap_ranges("conv_dgrad", c, 128, 4 * c) == ([0] * 9, [128] * 9, [0] * 8 + [128], [64] + [256] * 8)
    assert E.tap_ranges("deconv_fwd", c, 256, 4 * c) == ([0] * 9, [256] * 9, [0] * 8 + [192], [128] + [256] * 8)
    assert E.tap_ranges("deconv_dgrad", c, 4 * c, 256) == ([192] + [0] * 8, [256] * 8 + [128], [0] * 9, [256] * 9)
    assert E.tap_span(E.tap_ranges("conv_fwd", c, 4 * c, 128)) == (-4, 4)
    w = torch.randn(3, 2, 31)
    m0, m1 = E.pack_reference(0, w, 3, 2, 0), E.pack_reference(1, w, 2, 3, 0)
    for d in range(-4, 5):
        for p in range(4):
            j0, j1 = 4 * d + p + 14, -4 * d + p + 13
            b0, b1 = m0[d + 4, :, p * 2:(p + 1) * 2], m1[d + 4, p * 2:(p + 1) * 2, :]
            assert torch.equal(b0, w[:, :, j0]) if 0 <= j0 < 31 else not b0.any()
            assert torch.equal(b1, w[:, :, j1].t()) if 0 <= j1 < 31 else not b1.any()
    assert E.dec_last_tap_index(torch.device("cpu")).tolist() == [
        (-4 * (jj // 4 - 4) + jj % 4 + 13) if jj < 36 and 0 <= -4 * (jj // 4 - 4) + jj % 4 + 13 < 31 else -1
        for jj in range(64)]


def test_deconv_geometry_gives_four_times_the_input():
    """The reference's padding max(0, (4 - k) // -2) and the trim of odd widths give exactly 4 * Lin samples for
    every served width, which is what the tap form computes."""
    for k in range(4, 33):
        out = (8 - 1) * 4 - 2 * E.deconv_padding(k) + k - (k % 2)
        assert out == 32, k
        assert E.deconv_padding(k) == (k - 4) // 2


def test_golden_pins_seeded_modules():
    """kwidth.npz was made from the reference's modules seeded as these are: same state-dict bytes."""
    d = golden("kwidth.npz")
    for name, (kw, dkw) in {"k15_11": (15, 11), "k20_32": (20, 32)}.items():
        sd = kw_generator(kw, dkw).state_dict()
        assert sd_sha(sd) == str(d["sha_G.%s" % name])
        assert [list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()] == d["shapes.%s" % name].tolist()
    for name, (kw, norm) in {"k11_bnorm": (11, "bnorm"), "k32_bnorm": (32, "bnorm"), "k11_snorm": (11, "snorm"),
                             "k32_snorm": (32, "snorm")}.items():
        seed_all(111)
        D = Discriminator(2, FMAPS, kw, [4] * 5, pool_type="none", pool_slen=16, norm_type=norm, phase_shift=5)
        assert sd_sha(D.state_dict()) == str(d["sha_D.%s" % name])


def test_im2col_reference_matches_conv_semantics():
    """The fp64 im2col the GPU test uses, times the width-k weight, is the reference's reflect-padded strided conv."""
    torch.manual_seed(0)
    L = 256
    v = torch.randn(1, L, dtype=torch.float64)
    for k in (4, 11, 20, 31, 32):
        w = torch.randn(1, 1, k, dtype=torch.float64)
        col = im2col_ref([v], E.conv_offset(k), k, 1, 0)
        got = col[0, :, :k] @ w[0, 0]
        xp = torch.nn.functional.pad(v.view(1, 1, L), (k // 2 - 1, k // 2), mode="reflect")
        ref = torch.nn.functional.conv1d(xp, w, stride=4).view(-1)
        assert torch.allclose(got, ref), k


# ---- the oracle against the reference fixture ---------------------------------------------------------------------
def _fixture_inputs():
    from tests.golden.make_golden import seeded_randn
    x = 0.3 * seeded_randn(71, (2, 1, 16384))
    clean = (0.3 * seeded_randn(73, (2, 1, 16384))).clamp(-1, 1)
    return x, clean, seeded_randn(72, (2, 1024, 16))


@pytest.mark.parametrize("name,kw,dkw", [("k15_11", 15, 11), ("k20_32", 20, 32)])
def test_oracle_generator_vs_reference(name, kw, dkw):
    """The oracle's Generator forward (widths read off the weights) reproduces the reference's output at non-31
    widths (fp32 on both sides: only the summation order differs)."""
    from oracle import segan_oracle as O
    from tests.golden.make_golden_gsnorm import Y_IDX
    d = golden("kwidth.npz")
    sd = {k: v.detach().clone() for k, v in kw_generator(kw, dkw).state_dict().items()}
    x, _, z = _fixture_inputs()
    with O.oracle_mode(), torch.no_grad():
        y = O.generator_forward(sd, x, z)
    err = float((y.reshape(-1)[torch.from_numpy(Y_IDX)].double() - torch.from_numpy(d["y.%s" % name]).double())
                .abs().max())
    assert err <= 1e-5, err


@pytest.mark.parametrize("name,kw,norm", [("k11_bnorm", 11, "bnorm"), ("k32_bnorm", 32, "bnorm"),
                                          ("k11_snorm", 11, "snorm"), ("k32_snorm", 32, "snorm")])
def test_oracle_discriminator_vs_reference(name, kw, norm):
    """The oracle's training-mode Discriminator reproduces the reference's logits with the phase shifts the reference
    drew, which the project's draw_phase_shifts reproduces from the same seed."""
    import random
    from oracle import segan_oracle as O
    from segan_pytorch_b200.segan.models.discriminator import draw_phase_shifts
    d = golden("kwidth.npz")
    random.seed(99)
    shifts = draw_phase_shifts(5, 5)
    assert shifts == d["shifts.%s" % name].tolist()
    seed_all(111)
    D = Discriminator(2, FMAPS, kw, [4] * 5, pool_type="none", pool_slen=16, norm_type=norm, phase_shift=5)
    sd = {k: v.detach().clone() for k, v in D.state_dict().items()}
    x, clean, _ = _fixture_inputs()
    with O.oracle_mode(), torch.no_grad():
        logit = O.discriminator_forward(sd, torch.cat((x, clean), 1), shifts, training=True)
    ref = torch.from_numpy(d["logit.%s" % name]).double()
    assert float((logit.reshape(-1).double() - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("name,gkw,gdkw,dkw", [("k15_11_21", 15, 11, 21), ("k20_32_11", 20, 32, 11)])
def test_oracle_segan_step_vs_reference(name, gkw, gdkw, dkw):
    """One oracle SEGAN step (RMSprop, batch 4) at non-31 widths against one iteration of the reference's SEGAN.train:
    the four losses and the sampled parameter updates of G and D."""
    import random
    from oracle import segan_oracle as O
    from segan_pytorch_b200.segan.models import SEGAN
    from tests.golden.make_golden import seeded_randn
    from tests.util import cpu_state, load_opts
    d = golden("kwidth.npz")
    B = 4
    seed_all(111)
    s = SEGAN(load_opts(batch_size=B, gkwidth=gkw, gdec_kwidth=gdkw, dkwidth=dkw))
    assert sd_sha(s.G.state_dict()) == str(d["step.sha_G.%s" % name])
    assert sd_sha(s.D.state_dict()) == str(d["step.sha_D.%s" % name])
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    pre = {**{"G." + k: v.clone() for k, v in sdG.items()}, **{"D." + k: v.clone() for k, v in sdD.items()}}
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    g = torch.Generator().manual_seed(111 + 2)
    clean = (0.3 * torch.randn(B, 16384, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 16384, generator=g)).clamp(-1, 1)
    random.seed(99)
    shifts3 = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    out = O.segan_train_step(sdG, sdD, sqG, sqD, clean.unsqueeze(1), noisy.unsqueeze(1), seeded_randn(1234, (B, 1024, 16)),
                             shifts3, l1_weight=100.0)
    for k in ("d_real_loss", "d_fake_loss", "g_adv_loss", "g_l1_loss"):
        ref = float(d["step.%s.%s" % (k, name)])
        assert abs(out[k] - ref) <= 1e-4 * max(1.0, abs(ref)), (k, out[k], ref)
    post = {**{"G." + k: v for k, v in sdG.items()}, **{"D." + k: v for k, v in sdD.items()}}
    for k in ("G.enc_blocks.1.conv.weight", "G.dec_blocks.0.deconv.weight", "G.dec_blocks.4.deconv.weight",
              "D.enc_blocks.0.conv.weight", "D.enc_blocks.1.conv.weight"):
        tag = "step.delta.%s.%s" % (name, k)
        got = (post[k] - pre[k]).reshape(-1)[torch.from_numpy(d["idx." + tag])].double()
        ref = torch.from_numpy(d["val." + tag]).double()
        # RMSprop's first step is -lr g / sqrt(0.01 g^2) = -10 lr sign(g): the update carries the gradient's sign only,
        # so elements whose gradient is within rounding of 0 may take either sign in two fp32 implementations
        agree = float((got.sign() == ref.sign()).double().mean())
        assert agree >= 0.95, (k, agree)
        # (and |g| near eps shortens the step: the magnitudes are bounded by 10 lr, not equal)
        assert float(got.abs().max()) <= 1.001 * float(ref.abs().max()), k
