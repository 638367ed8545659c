"""Spectrally normalised Generators (norm_type='snorm') on the CPU: the containers' keys, shapes and init quirks,
which configurations are served, and the layout identities the engine relies on, in fp64 against
torch.nn.utils.spectral_norm itself:
  - a decoder master M[9][4 Cout][Cin] is the same bytes as [36][Cout][Cin], on which the power iteration with
    u per output channel is spectral_norm(dim=1) of ConvTranspose1d's W[Cin][Cout][31];
  - weight_v packs as a kind-1 weight with one output channel, and unpacks back;
  - a tied (skip_merge='sum') master [W | W] iterated over one half gives W's sigma; over both it would give
    sigma * sqrt(2);
  - the packed weight_orig gradient is G / sigma - <G, W~> / sigma * u v^T on the [36][Cout][Cin] view."""
import math

import pytest
import torch
import torch.nn.functional as F

from segan_pytorch_b200 import engine as E
from segan_pytorch_b200.segan.models import Generator
from segan_pytorch_b200.segan.models.model import weights_init, wsegan_weights_init
from tests import gsnorm_oracle as GO
from tests.util import build_segan, seed_all

FM = [64, 128, 256, 512, 1024]
CONFIGS = {
    "concat": dict(skip_merge="concat"),
    "sum": dict(skip_merge="sum"),
    "conv": dict(skip_merge="concat", skip_type="conv"),
    "no_z": dict(skip_merge="concat", no_z=True),
    "no_skip": dict(skip=False),
    "no_bias": dict(skip_merge="concat", bias=False),
}


def snorm_generator(name, seed=111, fmaps=FM, **over):
    seed_all(seed)
    kw = dict(bias=True, norm_type="snorm")
    kw.update(CONFIGS[name])
    kw.update(over)
    return Generator(1, list(fmaps), 31, [4] * len(fmaps), **kw)


@pytest.fixture(scope="module", autouse=True)
def _threads():
    torch.set_num_threads(max(1, min(8, torch.get_num_threads())))


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_keys_and_shapes(name):
    G = snorm_generator(name)
    sd = G.state_dict()
    nl = len(FM)
    for l in range(nl):
        for blk, cout in (("enc_blocks.%d.conv." % l, FM[l]), ("dec_blocks.%d.deconv." % l, None)):
            assert blk + "weight" not in sd
            w = sd[blk + "weight_orig"]
            if blk.startswith("enc"):
                assert sd[blk + "weight_u"].shape == (w.shape[0],)                 # dim 0
                assert sd[blk + "weight_v"].shape == (w.shape[1] * 31,)
            else:
                assert sd[blk + "weight_u"].shape == (w.shape[1],)                 # ConvTranspose1d: dim 1
                assert sd[blk + "weight_v"].shape == (w.shape[0] * 31,)
    # skip convs and alphas are not normalised
    assert not any(k.startswith("alpha_") and k.endswith(("_orig", "_u", "_v")) for k in sd)
    assert G._served
    eng = E.GeneratorEngine(G)
    eng.layers = eng.packed_layers()
    assert all(pl.name.endswith("weight_orig") for pl in eng.layers)
    assert sorted(eng._sn_names()) == sorted(k for k in sd if k.endswith("weight_orig"))


@pytest.mark.parametrize("init", [weights_init, wsegan_weights_init])
def test_init_functions_reach_weight_orig(init):
    """weights_init / wsegan_weights_init write the derived `weight` attribute in place.  Until the first hooked
    forward, torch's spectral_norm leaves that attribute aliasing weight_orig's storage, so the init lands in
    weight_orig exactly as on a plain torch module; u and v keep their seeded values."""
    G = snorm_generator("concat")
    before = {k: v.clone() for k, v in G.state_dict().items()}
    torch.manual_seed(5)
    G.apply(init)
    after = G.state_dict()
    for l in range(len(FM)):
        for blk in ("enc_blocks.%d.conv" % l, "dec_blocks.%d.deconv" % l):
            m = G.get_submodule(blk)
            assert m.weight.data_ptr() == m.weight_orig.data_ptr()
            changed = not torch.equal(before[blk + ".weight_orig"], after[blk + ".weight_orig"])
            # weights_init matches class names containing 'Conv1d' only: ConvTranspose1d keeps torch's init
            assert changed == (blk.startswith("enc") or init is wsegan_weights_init), blk
            assert torch.equal(before[blk + ".weight_u"], after[blk + ".weight_u"])
            assert torch.equal(before[blk + ".weight_v"], after[blk + ".weight_v"])
    if init is weights_init:
        assert abs(float(after["enc_blocks.4.conv.weight_orig"].std()) - 0.02) < 1e-3


def test_served_configurations():
    for name in CONFIGS:
        assert snorm_generator(name, fmaps=[64, 128])._served, name
    assert snorm_generator("concat", fmaps=[64, 128], z_dim=256)._served
    G = snorm_generator("concat", fmaps=[64, 128], norm_type="bnorm")
    assert not G._served
    with pytest.raises(NotImplementedError, match="bnorm"):
        G.engine


def test_gnorm_type_is_ignored_by_segan_as_in_the_reference():
    """SEGAN(opts) never forwards gnorm_type to its Generator (model.py:82-96 of the reference): --gnorm_type snorm
    still trains an un-normalised G; the normalised one is reached through SEGAN(opts, generator=G)."""
    s = build_segan(gnorm_type="snorm")
    assert not any(k.endswith("weight_orig") for k in s.G.state_dict())
    assert s.G.norm_type is None
    from tests.util import load_opts
    from segan_pytorch_b200.segan.models import SEGAN
    G = snorm_generator("concat")
    s2 = SEGAN(load_opts(), generator=G)
    assert s2.G is G and any(k.endswith("weight_orig") for k in s2.G.state_dict())


def _deconv_case(cin, cout, seed, tied=False):
    g = torch.Generator().manual_seed(seed)
    w = 0.05 * torch.randn(cin, cout, 31, generator=g, dtype=torch.float64)
    u0 = F.normalize(torch.randn(cout, generator=g, dtype=torch.float64), dim=0)
    v0 = F.normalize(torch.randn(cin * 31, generator=g, dtype=torch.float64), dim=0)
    pl = E.PackedLayer("dec", 1, cout, 2 * cin if tied else cin, 0, "f", "d", tied=tied)
    return w, u0, v0, pl


def _torch_sn(mod, u0, v0):
    torch.nn.utils.spectral_norm(mod)
    mod.weight_u.copy_(u0)
    mod.weight_v.copy_(v0)
    hook = next(iter(mod._forward_pre_hooks.values()))
    with torch.no_grad():
        w_sn = hook.compute_weight(mod, do_power_iteration=True)
    u, v = mod.weight_u.clone(), mod.weight_v.clone()
    return u, v, float(torch.dot(u, GO.sn_matrix(mod.weight_orig.detach(), hook.dim) @ v)), w_sn


def _packed_iteration(m, T, nc, kc, ld, u0, vp0):
    """The kernels' iteration on M[t][n][k < kc] with rows ld apart, in fp64."""
    mm = m.reshape(T, nc, ld)[:, :, :kc]
    v = torch.einsum("tnk,n->tk", mm, u0)
    v = v / v.norm()
    u = torch.einsum("tnk,tk->n", mm, v)
    sigma = float(u.norm())
    return u / sigma, v.reshape(-1), sigma


@pytest.mark.parametrize("cin,cout", [(128, 64), (2048, 512), (64, 1)])
def test_decoder_master_is_spectral_norm_dim1(cin, cout):
    """[9][4 Cout][Cin] read as [36][Cout][Cin] (n_taps 36, nc = Cout, kc = Cin): u, v, sigma of the power iteration
    are torch's spectral_norm(dim=1) of the ConvTranspose1d, in fp64; the structural-zero taps keep v = 0."""
    w, u0, v0, pl = _deconv_case(cin, cout, cin + cout)
    T, nc, kc, ld = E.sn_geometry(pl)
    assert (T, nc, kc, ld) == (36, cout, cin, cin)
    m = E.pack_reference(1, w, cout, cin, 0)
    vp0 = E.sn_pack_v(pl, v0)
    assert vp0.numel() == 36 * cin
    u, vp, sigma = _packed_iteration(m, T, nc, kc, ld, u0, vp0)
    mod = torch.nn.ConvTranspose1d(cin, cout, 31, stride=4, padding=13).double()
    mod.weight.data.copy_(w)
    u_t, v_t, sig_t, _ = _torch_sn(mod, u0, v0)
    assert torch.allclose(u, u_t, rtol=0, atol=1e-12)
    assert torch.allclose(E.sn_unpack_v(pl, vp), v_t, rtol=0, atol=1e-12)
    assert abs(sigma - sig_t) <= 1e-12 * sig_t
    zero_slots = E.sn_pack_v(pl, torch.ones(cin * 31, dtype=torch.float64)) == 0
    assert int(zero_slots.sum()) == 5 * cin and float(vp[zero_slots].abs().max()) == 0.0


def test_decoder_master_over_dim0_is_wrong():
    """The same master iterated with u per packed row (4 Cout rows of 9 taps, what dim 0 of the packed layout would
    be) gives another sigma: the layout identity above is what makes the iteration torch's."""
    w, u0, v0, pl = _deconv_case(128, 64, 5)
    m = E.pack_reference(1, w, 64, 128, 0)
    mod = torch.nn.ConvTranspose1d(128, 64, 31, stride=4, padding=13).double()
    mod.weight.data.copy_(w)
    _, _, sig_t, _ = _torch_sn(mod, u0, v0)
    wrong = torch.linalg.matrix_norm(m.reshape(9, 256, 128).permute(1, 0, 2).reshape(256, -1), ord=2)
    assert abs(float(wrong) - sig_t) > 1e-3 * sig_t


def test_tied_master_iterates_one_half():
    """skip_merge='sum': the packed master holds [W | W] over 2 Cin columns.  With ld = 2 Cin and kc = Cin the
    iteration is W's; over the whole row it would give v = [v; v] / sqrt(2) and sigma * sqrt(2)."""
    w, u0, v0, pl = _deconv_case(256, 128, 9, tied=True)
    T, nc, kc, ld = E.sn_geometry(pl)
    assert (T, nc, kc, ld) == (36, 128, 256, 512)
    m = E.pack_reference(1, torch.cat((w, w), 0), 128, 512, 0)
    u, vp, sigma = _packed_iteration(m, T, nc, kc, ld, u0, E.sn_pack_v(pl, v0))
    mod = torch.nn.ConvTranspose1d(256, 128, 31, stride=4, padding=13).double()
    mod.weight.data.copy_(w)
    u_t, v_t, sig_t, _ = _torch_sn(mod, u0, v0)
    assert torch.allclose(u, u_t, rtol=0, atol=1e-12) and abs(sigma - sig_t) <= 1e-12 * sig_t
    assert torch.allclose(E.sn_unpack_v(pl, vp), v_t, rtol=0, atol=1e-12)
    _, _, sig_full = _packed_iteration(m, T, nc, 2 * kc, ld, u0, torch.cat(
        (E.sn_pack_v(pl, v0).view(36, 256), E.sn_pack_v(pl, v0).view(36, 256)), 1).reshape(-1))
    assert abs(sig_full - math.sqrt(2) * sig_t) <= 1e-9 * sig_t


@pytest.mark.parametrize("kind,tied", [(0, False), (1, False), (1, True)])
def test_weight_v_pack_unpack_round_trip(kind, tied):
    cin = 128
    pl = E.PackedLayer("x", kind, 64, 2 * cin if tied else cin, 0, "f", "d", tied=tied)
    v = torch.randn(cin * 31, dtype=torch.float64)
    vp = E.sn_pack_v(pl, v)
    T, nc, kc, ld = E.sn_geometry(pl)
    assert vp.numel() == T * kc
    assert torch.equal(E.sn_unpack_v(pl, vp), v)


@pytest.mark.parametrize("tied", [False, True])
def test_packed_weight_orig_gradient_formula(tied):
    """fp64: for L = <R, W~>, torch's gradient w.r.t. weight_orig, packed, equals the engine's
    G / sigma - (<G, W~> / sigma) u v^T formed on the packed layout (u per output channel, v in packed slots) --
    the sigma term applied to both copies of a tied master."""
    cin, cout = 128, 64
    w, u0, v0, pl = _deconv_case(cin, cout, 21, tied=tied)
    mod = torch.nn.ConvTranspose1d(cin, cout, 31, stride=4, padding=13).double()
    mod.weight.data.copy_(w)
    u, v, sigma, _ = _torch_sn(mod, u0, v0)
    hook = next(iter(mod._forward_pre_hooks.values()))
    r = torch.randn(cin, cout, 31, dtype=torch.float64)
    w_sn = hook.compute_weight(mod, do_power_iteration=False)
    (r * w_sn).sum().backward()
    ref = mod.weight_orig.grad
    T, nc, kc, ld = E.sn_geometry(pl)
    src = torch.cat((r, r), 0) if tied else r
    g = E.pack_reference(1, src, cout, src.shape[0], 0).reshape(T, nc, ld)
    coef = float((r * w_sn.detach()).sum()) / sigma
    corr = coef * torch.einsum("n,tk->tnk", u, E.sn_pack_v(pl, v).view(T, kc))
    d = g / sigma
    d[:, :, :kc] -= corr
    if tied:
        d[:, :, kc:] -= corr
        assert torch.equal(d[:, :, :kc], d[:, :, kc:])
    got = E.unpack_reference(1, d[:, :, :kc].reshape(9, 4 * cout, kc), cout, kc, 0)
    assert torch.allclose(got, ref, rtol=0, atol=1e-12 * float(ref.abs().max()))


def test_oracle_forward_matches_torch_modules():
    """tests/gsnorm_oracle.py's normalised weights are those torch's spectral_norm hooks compute on the containers
    (training: one power iteration; eval: the stored vectors)."""
    G = snorm_generator("concat", fmaps=[64, 128]).double()
    sd = {k: v.clone() for k, v in G.state_dict().items()}
    plain, vec = GO.normalised_state(sd, training=True)
    for blk in (G.enc_blocks[1].conv, G.dec_blocks[0].deconv, G.dec_blocks[1].deconv):
        hook = next(iter(blk._forward_pre_hooks.values()))
        with torch.no_grad():
            w = hook.compute_weight(blk, do_power_iteration=True)
        name = [k for k, m in G.named_modules() if m is blk][0]
        assert torch.allclose(plain[name + ".weight"], w, rtol=1e-13, atol=0)
        assert torch.allclose(sd[name + ".weight_u"], blk.weight_u, rtol=0, atol=1e-14)


# ---- pinned to the reference: tests/golden/g_snorm.npz (tests/golden/make_golden_gsnorm.py) ------------------------
GOLD = "g_snorm.npz"


def _golden_inputs(g):
    x = 0.3 * torch.from_numpy(g["xr"])
    return x, torch.from_numpy(g["zr"]), (0.3 * torch.from_numpy(g["cr"])).clamp(-1, 1)


def _vectors_vs_golden(g, tag, sd):
    """u in full, v at the sampled slots, sigma = u^T W v, each against the reference."""
    worst = 0.0
    for k in [k for k in sd if k.endswith("weight_orig")]:
        p = k[:-len("weight_orig")]
        u, v = sd[p + "weight_u"].double(), sd[p + "weight_v"].double()
        gu = torch.from_numpy(g["u.%s.%s" % (tag, p)]).double()
        idx = torch.from_numpy(g["idx.v.%s.%s" % (tag, p)])
        gv = torch.from_numpy(g["val.v.%s.%s" % (tag, p)]).double()
        wm = GO.sn_matrix(sd[k].double(), GO.sn_dim(k))
        sig = float(torch.dot(u, wm @ v))
        gs = float(g["sigma.%s.%s" % (tag, p)])
        worst = max(worst, float((u - gu).abs().max()), float((v[idx] - gv).abs().max()), abs(sig - gs) / abs(gs))
    return worst


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_containers_match_reference(name):
    """Keys, shapes and the seeded state dict, bare and after weights_init / wsegan_weights_init: the init lands in
    weight_orig exactly as in the reference."""
    from tests.util import golden, sd_sha
    g = golden(GOLD)
    G = snorm_generator(name)
    sd = G.state_dict()
    assert list(sd.keys()) == [str(k) for k in g["keys.%s" % name]]
    shapes = [list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()]
    assert shapes == g["shapes.%s" % name].tolist()
    assert sd_sha(sd) == str(g["sha_G_init.%s" % name])
    for init in (weights_init, wsegan_weights_init):
        Gi = snorm_generator(name)
        torch.manual_seed(5)
        Gi.apply(init)
        assert sd_sha(Gi.state_dict()) == str(g["sha_%s.%s" % (init.__name__, name)]), init.__name__


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oracle_matches_reference(name):
    """tests/gsnorm_oracle.py against the reference: u / v / sigma after one training forward, the training- and
    eval-mode outputs, and the 100 * L1 gradients after a second training forward."""
    from oracle import segan_oracle as O
    from tests.util import golden
    g = golden(GOLD)
    G = snorm_generator(name)
    sd = {k: v.detach().clone() for k, v in G.state_dict().items()}
    x, z, clean = _golden_inputs(g)
    z = None if G.no_z else z
    from tests.golden.make_golden_gsnorm import Y_IDX
    yi = torch.from_numpy(Y_IDX)
    with O.oracle_mode():
        with torch.no_grad():
            y_tr = GO.generator_forward(sd, x, z, training=True, skip_merge=G.skip_merge)
        assert _vectors_vs_golden(g, "train1.%s" % name, sd) <= 1e-5
        with torch.no_grad():
            y_ev = GO.generator_forward(sd, x, z, training=False, skip_merge=G.skip_merge)
        pG = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd)}
        loss = 100 * F.l1_loss(GO.generator_forward({**sd, **pG}, x, z, training=True, skip_merge=G.skip_merge), clean)
        grads = dict(zip(pG, torch.autograd.grad(loss, list(pG.values()))))
    assert float((y_tr.reshape(-1)[yi] - torch.from_numpy(g["y_train.%s" % name])).abs().max()) <= 1e-5
    assert float((y_ev.reshape(-1)[yi] - torch.from_numpy(g["y_eval.%s" % name])).abs().max()) <= 1e-5
    assert abs(float(loss.detach()) - float(g["l1_loss.%s" % name])) <= 1e-5 * float(g["l1_loss.%s" % name])
    for k in [k for k in g if k.startswith("idx.grad.%s." % name)]:
        key = k[len("idx.grad.%s." % name):]
        gi = torch.from_numpy(g[k])
        ref = torch.from_numpy(g["val.grad.%s.%s" % (name, key)])
        scale = float(g["norm.grad.%s.%s" % (name, key)]) / max(1.0, grads[key].numel()) ** 0.5
        assert float((grads[key].reshape(-1)[gi] - ref).abs().max()) <= 1e-3 * scale + 1e-9, key


def test_oracle_segan_step_matches_reference():
    """One SEGAN(opts, generator=G_snorm) step of the oracle (its Generator forward through tests/gsnorm_oracle.py)
    against the reference's: the four losses and the Generator's weight_u / weight_v afterwards."""
    import random
    from oracle import segan_oracle as O
    from segan_pytorch_b200.segan.models import SEGAN
    from tests.util import cpu_state, golden, load_opts, sd_sha
    g = golden(GOLD)
    t = golden("train_step_b4.npz")
    B = 4
    G = snorm_generator("concat")
    seed_all(111)
    s = SEGAN(load_opts(batch_size=B), generator=G)
    assert sd_sha(s.G.state_dict()) == str(g["step.sha_G"]) and sd_sha(s.D.state_dict()) == str(g["step.sha_D"])
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    random.seed(int(t["py_random_seed"]))
    shifts3 = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    torch.manual_seed(int(t["torch_seed_z"]))
    z = torch.randn(B, 1024, 16)
    clean = torch.from_numpy(t["clean"]).unsqueeze(1)
    noisy = torch.from_numpy(t["noisy"]).unsqueeze(1)
    plain = O.generator_forward
    O.generator_forward = lambda sd, x, z_, ret_hid=False, skip_merge="concat": GO.generator_forward(
        sd, x, z_, training=True, skip_merge=skip_merge, ret_hid=ret_hid)
    try:
        out = O.segan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts3, l1_weight=100.0)
    finally:
        O.generator_forward = plain
    for k in ("d_real_loss", "d_fake_loss", "g_adv_loss", "g_l1_loss"):
        assert abs(out[k] - float(g["step." + k])) <= 1e-4 * max(1.0, abs(float(g["step." + k]))), k
    assert _vectors_vs_golden(g, "step", sdG) <= 1e-4
