"""Kernel widths other than 31 on the H100: the width-taking entry points against fp64 (or exact copies) at every width
4..32 and bit for bit against the k = 31 entry points, Generators and Discriminators against the reference's outputs
and gradients (tests/golden/kwidth.npz), SEGAN steps against the oracle (pinned to the reference at these widths by
tests/test_kwidth.py) and under graph replay, every Generator topology and snorm against the oracle's
operand-precision control, a WSEGAN snorm step against the oracle, checkpoints and inference.
Run on an H100:  python -m pytest tests -m gpu"""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                             # noqa: E402
from segan_pytorch_b200._lib import SG_F16, SG_F32                            # noqa: E402
from segan_pytorch_b200.segan.models import SEGAN, WSEGAN                    # noqa: E402
from segan_pytorch_b200.segan.models.discriminator import Discriminator      # noqa: E402
from tests.test_gpu_parity_scale import LOSS_RTOL, WAVE_TOL                  # noqa: E402
from tests.test_kwidth import kw_generator, im2col_ref                       # noqa: E402
from tests.util import golden, load_opts, rel_err, sd_sha, seed_all          # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream
WIDTHS = list(range(4, 33))
# sampled single-pass gradients against the fp32 reference: PReLU's derivative jumps at 0 (slope 0.25 -> 1), so the
# ~1e-3 operand rounding of the 16-bit activations flips a few elements per layer (tests/test_gpu_parity_scale.py)
GRAD_REL = 0.1
LOGIT_REL = 2e-2


def _kind_shapes(kind):
    return (64, 32) if kind == 0 else (32, 64)          # (c_out, c_in): the pack kernels' 16 x 32 tile grid


# ---- entry points ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [0, 1])
def test_pack_unpack_kw_every_width(kind):
    """sg_pack_weights_kw (fp32 forward and data-gradient operands) and sg_unpack_wgrad_kw equal the tensor-algebra
    layouts exactly at every width; at k = 31 they equal sg_pack_weights / sg_unpack_wgrad bit for bit."""
    c_out, c_in = _kind_shapes(kind)
    g = torch.Generator().manual_seed(900 + kind)
    for k in WIDTHS:
        w = torch.randn((c_out, c_in, k) if kind == 0 else (c_in, c_out, k), generator=g)
        m = E.pack_reference(kind, w, c_out, c_in, 0, k)
        wd = w.to(DEV)
        f = torch.full(m.shape, 7.0, device=DEV)
        dg = torch.full((9, m.shape[2], m.shape[1]), 7.0, device=DEV)
        _lib.call("sg_pack_weights_kw", kind, _p(wd), c_out, c_in, 0, k, None, 0, _p(f), _p(dg), SG_F32, SG_F32,
                  _stream())
        back = torch.full_like(wd, 7.0)
        _lib.call("sg_unpack_wgrad_kw", kind, _p(f), c_out, c_in, 0, k, None, None, 0, _p(back), None, 0, _stream())
        torch.cuda.synchronize()
        assert torch.equal(f.cpu(), m), k
        assert torch.equal(dg.cpu(), m.flip(0).transpose(1, 2)), k
        assert torch.equal(back.cpu(), w), k
        if k == 31:
            f0, dg0, back0 = torch.zeros_like(f), torch.zeros_like(dg), torch.zeros_like(wd)
            _lib.call("sg_pack_weights", kind, _p(wd), c_out, c_in, 0, None, 0, _p(f0), _p(dg0), SG_F32, SG_F32,
                      _stream())
            _lib.call("sg_unpack_wgrad", kind, _p(f), c_out, c_in, 0, None, None, 0, _p(back0), None, 0, _stream())
            torch.cuda.synchronize()
            assert torch.equal(f0, f) and torch.equal(dg0, dg) and torch.equal(back0, back)
    with pytest.raises(_lib.SeganB200Error):
        _lib.call("sg_pack_weights_kw", kind, _p(wd), c_out, c_in, 0, 33, None, 0, _p(f), None, SG_F32, SG_F32,
                  _stream())


@pytest.mark.parametrize("cin,reflect", [(1, 1), (2, 1), (1, 0)])
def test_im2col_kw_every_width(cin, reflect):
    """sg_wave_im2col_kw is an exact copy: the fp16 matrix equals the fp64 im2col rounded once, with the D's two
    channels and a device-resident roll (reflect) or the zero padding of the last decoder's gradient."""
    B, L = 2, 4096
    g = torch.Generator().manual_seed(910 + cin)
    v = [torch.randn(B, L, generator=g).double() for _ in range(cin)]
    vd = [t.float().to(DEV) for t in v]
    roll = 3 if reflect else 0
    roll_dev = torch.tensor([roll], dtype=torch.int32, device=DEV)
    for k in WIDTHS:
        off = E.conv_offset(k) if reflect else E.deconv_padding(k)
        col = torch.full((B, L // 4, 64), 9.0, dtype=torch.float16, device=DEV)
        _lib.call("sg_wave_im2col_kw", _p(vd[0]), _p(vd[1]) if cin == 2 else None, cin, B, L, 0,
                  _p(roll_dev) if reflect else None, reflect, off, k, _p(col), None, _stream())
        torch.cuda.synchronize()
        ref = im2col_ref([t.float().double() for t in v], off, k, reflect, roll)
        assert torch.equal(col.cpu(), ref.half()), k
        if k == 31:
            col0 = torch.zeros_like(col)
            _lib.call("sg_wave_im2col", _p(vd[0]), _p(vd[1]) if cin == 2 else None, cin, B, L, 0,
                      _p(roll_dev) if reflect else None, reflect, off, _p(col0), None, _stream())
            torch.cuda.synchronize()
            assert torch.equal(col0, col)


def _fold_ref(P2, col0, L, k, roll):
    """gx[src(q)] += P2[t][col0 + j] for q = 4t + j - (k/2 - 1), j < k; src = un-roll(reflect(q)) (fp64)."""
    B, Lq, _ = P2.shape
    off = E.conv_offset(k)
    t = torch.arange(Lq).view(-1, 1)
    j = torch.arange(k).view(1, -1)
    q = (4 * t + j - off).reshape(-1)
    r = q.abs()
    r = torch.where(r >= L, 2 * (L - 1) - r, r)
    src = (r - roll) % L
    gx = torch.zeros(B, L, dtype=torch.float64)
    vals = P2[:, :, col0:col0 + k].double().reshape(B, -1)
    gx.index_add_(1, src, vals)
    return gx, (P2[:, :, col0:col0 + k].double().abs().reshape(B, -1))


@pytest.mark.parametrize("col0,roll", [(0, 0), (32, -4), (0, 5)])
def test_col2im_fold_kw_vs_fp64(col0, roll):
    """The D's input-gradient fold at every width against fp64, under non-zero rolls, within 8 fp32 roundings of the
    summed magnitudes; at k = 31 equal to sg_wave_col2im_fold (zero-filled destination: at most two atomic adds per
    sample, so the order does not matter)."""
    B, L = 2, 4096
    g = torch.Generator().manual_seed(920 + col0 + roll)
    P2 = torch.randn(B, L // 4, 64, generator=g).half()
    P2d = P2.to(DEV) if E.GS == SG_F16 else P2.to(E.GT).to(DEV)
    roll_dev = torch.tensor([roll], dtype=torch.int32, device=DEV)
    for k in WIDTHS:
        gx = torch.zeros(B, L, device=DEV)
        _lib.call("sg_wave_col2im_fold_kw", _p(P2d), col0, B, L, 0, _p(roll_dev), k, _p(gx), _stream())
        torch.cuda.synchronize()
        ref, mag = _fold_ref(P2d.float().cpu(), col0, L, k, roll)
        # a sample sums at most 2 x 8 terms in fp32
        assert float(((gx.cpu().double() - ref).abs()).max()) <= 16 * 2.0 ** -24 * 16 * float(mag.max()), k
        if k == 31:
            gx0 = torch.zeros_like(gx)
            _lib.call("sg_wave_col2im_fold", _p(P2d), col0, B, L, 0, _p(roll_dev), _p(gx0), _stream())
            torch.cuda.synchronize()
            assert torch.equal(gx0, gx)


@pytest.mark.parametrize("cin", [1, 2])
def test_wave_wgrad_fold_kw_every_width(cin):
    """dW[co][ci][j] += dwq[0][co][0][ci*32+j] + dwq[1][co][1][ci*32+j] for j < k, the blocks read cleared, the rest
    untouched; k = 31 equals sg_wave_wgrad_fold."""
    g = torch.Generator().manual_seed(930 + cin)
    for k in WIDTHS:
        dwq0 = torch.randn(2, 64, 2, 64, generator=g)
        dw0 = torch.randn(64, cin, k, generator=g)
        dwq, dw = dwq0.to(DEV), dw0.to(DEV)
        _lib.call("sg_wave_wgrad_fold_kw", _p(dwq), cin, k, _p(dw), _stream())
        torch.cuda.synchronize()
        blk = (dwq0[0, :, 0] + dwq0[1, :, 1]).view(64, 2, 32)[:, :cin, :k]
        assert torch.equal(dw.cpu(), dw0 + blk), k
        left = dwq0.clone()
        left.view(2, 64, 2, 2, 32)[0, :, 0, :cin, :k] = 0
        left.view(2, 64, 2, 2, 32)[1, :, 1, :cin, :k] = 0
        assert torch.equal(dwq.cpu(), left), k
        if k == 31:
            dwq1, dw1 = dwq0.to(DEV), dw0.to(DEV)
            _lib.call("sg_wave_wgrad_fold", _p(dwq1), cin, _p(dw1), _stream())
            torch.cuda.synchronize()
            assert torch.equal(dw1, dw) and torch.equal(dwq1, dwq)


@pytest.mark.parametrize("nsrc", [1, 2])
def test_last_deconv_wgrad_fold_kw_every_width(nsrc):
    """dWeff[src*half + c][j] = dwq[0][j][src][0][c] + dwq[1][j][src][1][c] (j < k): added to dW (times alpha on the
    skip half) with dalpha[c] += sum_j dWeff[half + c][j] * W[half + c][j] (fp64 within fp32 rounding); k = 31 equals
    sg_last_deconv_wgrad_fold(_1src)."""
    half = 64
    g = torch.Generator().manual_seed(940 + nsrc)
    for k in WIDTHS:
        dwq0 = torch.randn(2, 64, nsrc, 2, half, generator=g)
        w0 = torch.randn(nsrc * half, 1, k, generator=g)
        alpha0 = torch.rand(half, generator=g) + 0.5
        dw0 = torch.randn(nsrc * half, 1, k, generator=g)
        eff = (dwq0[0, :, :, 0] + dwq0[1, :, :, 1])[:k].permute(1, 2, 0).reshape(nsrc * half, 1, k)

        def run(name, kw_arg):
            dwq, dw, da = dwq0.to(DEV), dw0.to(DEV), torch.zeros(half, device=DEV)
            if nsrc == 2:
                _lib.call(name, _p(dwq), half, *kw_arg, _p(w0.to(DEV)), _p(alpha0.to(DEV)), _p(dw), _p(da), _stream())
            else:
                _lib.call(name, _p(dwq), half, *kw_arg, _p(dw), _stream())
            torch.cuda.synchronize()
            return dwq.cpu(), dw.cpu(), da.cpu()
        name, name_kw = (("sg_last_deconv_wgrad_fold", "sg_last_deconv_wgrad_fold_kw") if nsrc == 2 else
                         ("sg_last_deconv_wgrad_fold_1src", "sg_last_deconv_wgrad_fold_1src_kw"))
        dwq, dw, da = run(name_kw, (k,))
        exp = dw0.double() + eff.double()
        if nsrc == 2:
            exp[half:] = dw0[half:].double() + eff[half:].double() * alpha0.double().view(-1, 1, 1)
            exp_da = (eff[half:].double() * w0[half:].double()).sum((1, 2))
            assert float((da.double() - exp_da).abs().max()) <= 64 * 2.0 ** -24 * float(
                (eff[half:].double() * w0[half:].double()).abs().sum((1, 2)).max()), k
        assert float((dw.double() - exp).abs().max()) <= 2.0 ** -23 * float(exp.abs().max()), k
        assert float(dwq.view(2, 64, nsrc, 2, half)[0, :k, :, 0].abs().max()) == 0.0
        assert float(dwq.view(2, 64, nsrc, 2, half)[1, :k, :, 1].abs().max()) == 0.0
        if k == 31:
            dwq1, dw1, da1 = run(name, ())
            assert torch.equal(dw1, dw) and torch.equal(dwq1, dwq) and torch.equal(da1, da)


# ---- networks against the reference ----------------------------------------------------------------------------------
G_CONFIGS = {"k15_11": (15, 11), "k20_32": (20, 32)}
D_CONFIGS = {"k11_bnorm": (11, "bnorm"), "k32_bnorm": (32, "bnorm"), "k11_snorm": (11, "snorm"),
             "k32_snorm": (32, "snorm")}


def _inputs():
    from tests.golden.make_golden import seeded_randn
    x = 0.3 * seeded_randn(71, (2, 1, 16384))
    clean = (0.3 * seeded_randn(73, (2, 1, 16384))).clamp(-1, 1)
    return x, clean, seeded_randn(72, (2, 1024, 16))


def _sampled(d, tag, t):
    idx = torch.from_numpy(d["idx." + tag])
    return rel_err(t.detach().cpu().reshape(-1)[idx], d["val." + tag])


@pytest.mark.parametrize("name", list(G_CONFIGS))
def test_generator_vs_reference(name):
    """Training-mode output, 100 * L1 and sampled gradients against the reference at (encoder, decoder) widths
    (15, 11) and (20, 32)."""
    d = golden("kwidth.npz")
    kw, dkw = G_CONFIGS[name]
    G = kw_generator(kw, dkw)
    assert sd_sha(G.state_dict()) == str(d["sha_G.%s" % name])
    G = G.to(DEV).train()
    x, clean, z = _inputs()
    y = G(x.to(DEV), z=z.to(DEV))
    loss = 100 * torch.nn.functional.l1_loss(y, clean.to(DEV))
    loss.backward()
    from tests.golden.make_golden_gsnorm import Y_IDX
    err_y = float(np.abs(y.detach().cpu().reshape(-1).numpy()[Y_IDX] - d["y.%s" % name]).max())
    err_l = abs(loss.item() - float(d["l1_loss.%s" % name])) / abs(float(d["l1_loss.%s" % name]))
    params = dict(G.named_parameters())
    errs = {k: _sampled(d, "grad.%s.%s" % (name, k), params[k].grad)
            for k in ("enc_blocks.0.conv.weight", "enc_blocks.4.conv.weight", "dec_blocks.0.deconv.weight",
                      "dec_blocks.4.deconv.weight", "alpha_0.skip_k")}
    print("kwidth G %s: y max-abs %.2e, loss rel %.2e, grads %s" % (name, err_y, err_l,
                                                                   {k: round(v, 4) for k, v in errs.items()}))
    assert err_y <= WAVE_TOL and err_l <= LOSS_RTOL
    assert max(errs.values()) <= GRAD_REL, errs


def kw_discriminator(kw, norm):
    seed_all(111)
    return Discriminator(2, [64, 128, 256, 512, 1024], kw, [4] * 5, pool_type="none", pool_slen=16, norm_type=norm,
                         phase_shift=5)


@pytest.mark.parametrize("name", list(D_CONFIGS))
def test_discriminator_vs_reference(name):
    """Training-mode logits (phase shifts drawn after random.seed(99)) and sampled gradients of logit.sum() w.r.t. the
    first and last tower conv and the input pair, at widths 11 and 32 with BatchNorm and with spectral norm."""
    d = golden("kwidth.npz")
    kw, norm = D_CONFIGS[name]
    D = kw_discriminator(kw, norm)
    assert sd_sha(D.state_dict()) == str(d["sha_D.%s" % name])
    D = D.to(DEV).train()
    x, clean, _ = _inputs()
    pair = torch.cat((x, clean), 1).to(DEV).requires_grad_(True)
    random.seed(99)
    logit, _ = D(pair)
    logit.sum().backward()
    ref = torch.from_numpy(d["logit.%s" % name])
    err_l = float((logit.detach().cpu().reshape(-1).double() - ref.double()).abs().max()) / max(
        1.0, float(ref.abs().max()))
    sfx = "_orig" if norm == "snorm" else ""
    params = dict(D.named_parameters())
    errs = {k: _sampled(d, "grad.%s.%s" % (name, k), params[k].grad)
            for k in ("enc_blocks.0.conv.weight" + sfx, "enc_blocks.4.conv.weight" + sfx)}
    errs["input"] = _sampled(d, "grad.%s.input" % name, pair.grad)
    print("kwidth D %s: logit err %.2e, grads %s" % (name, err_l, {k: round(v, 4) for k, v in errs.items()}))
    assert err_l <= LOGIT_REL
    assert max(errs.values()) <= GRAD_REL, errs


# ---- steps, checkpoints, inference ------------------------------------------------------------------------------------
def _pairs(B, seed):
    g = torch.Generator().manual_seed(seed)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    return clean, noisy


def test_segan_steps_graph_replay_matches_eager():
    """SEGAN steps with widths (15, 11) and a D of width 21: eager twice (the noise floor) and graph-replayed; losses
    and G gradients of the replayed steps held to the floor."""
    B = 8
    clean, noisy = (t.to(DEV) for t in _pairs(B, 950))
    from oracle import segan_oracle as O
    random.seed(13)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(4)]
    prev_keep = E.KEEP_GRADS

    def run(graphs):
        prev = E.GRAPHS
        E.GRAPHS, E.KEEP_GRADS = graphs, True
        try:
            seed_all(111)
            opts = load_opts(batch_size=B, gkwidth=15, gdec_kwidth=11, dkwidth=21, g_lr=5e-7, d_lr=5e-7)
            s = SEGAN(opts).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(opts)
            out = []
            torch.manual_seed(99)
            for i in range(4):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, shifts3=shifts[i])
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad[:s.G.engine.flat.numel()].clone()))
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs
        finally:
            E.GRAPHS, E.KEEP_GRADS = prev, prev_keep

    (e1, n1), (e2, n2), (gr, n3) = run(False), run(False), run(True)
    assert n1 == 0 and n2 == 0 and n3 == 1
    for step in range(4):
        fl = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[step][0], e2[step][0]))
        fg = rel_err(e2[step][1], e1[step][1])
        el = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[step][0], gr[step][0]))
        eg = rel_err(gr[step][1], e1[step][1])
        print("kwidth SEGAN step %d: losses %s | floor loss %.2e grad %.2e | graph loss %.2e grad %.2e"
              % (step, [round(x, 4) for x in gr[step][0]], fl, fg, el, eg))
        assert all(x == x and abs(x) < 1e4 for x in gr[step][0])
        assert el <= 10 * fl + 2e-3 and eg <= 10 * fg + 5e-3


def test_checkpoint_round_trip_keeps_width(tmp_path):
    """state_dict shapes are [.., k]; a fresh Generator loading them gives the same outputs, and its packed masters
    are exactly the packed checkpoint weights (no value outside the k taps)."""
    x = _pairs(2, 953)[1].to(DEV)
    G1 = kw_generator(15, 11, seed=1).to(DEV).eval()
    sd = G1.state_dict()
    assert sd["enc_blocks.1.conv.weight"].shape == (128, 64, 15)
    assert sd["dec_blocks.0.deconv.weight"].shape == (2048, 512, 11)
    z = torch.randn(2, 1024, 16, device=DEV)
    with torch.no_grad():
        y1 = G1(x, z=z)
    path = str(tmp_path / "g.ckpt")
    torch.save(sd, path)
    G2 = kw_generator(15, 11, seed=2).to(DEV).eval()
    G2.load_state_dict(torch.load(path, map_location=DEV))
    with torch.no_grad():
        y2 = G2(x, z=z)
    assert torch.equal(y1, y2)
    for name, pl in ((n, l) for n, l in G2.engine.by_name.items()):
        m = G2.engine.mview(pl).view(pl.T, pl.nc, pl.kc).cpu()
        assert torch.equal(E.pack_reference(pl.kind, E.unpack_reference(pl.kind, m, pl.c_out, pl.c_in, 0, pl.kw),
                                            pl.c_out, pl.c_in, 0, pl.kw), m), name


def test_generate_and_clean_files_at_width_11(tmp_path):
    """generate and clean_files run a width-11 Generator: the same samples as G on the windows."""
    import os
    from scipy.io import wavfile
    from oracle import segan_oracle as O
    seed_all(111)
    s = SEGAN(load_opts(batch_size=2, gkwidth=11, no_z=True)).to(DEV)
    gen = torch.Generator().manual_seed(954)
    T = 40000
    wav = 0.3 * torch.randn(1, 1, T, generator=gen)
    out, _ = s.generate(wav)
    x = torch.zeros(3, 1, 16384)
    x.view(-1)[:T] = wav.view(-1)
    with torch.no_grad():
        y = s.G(x.to(DEV)).cpu().reshape(-1)[:T].numpy()
    assert float(np.abs(out - O.de_emphasize(y, 0.95)).max()) <= 1e-4
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    p = str(src / "u0.wav")
    wavfile.write(p, 16000, (np.random.RandomState(0).randn(T) * 3000).astype(np.int16))
    assert s.clean_files([p], str(dst), batch=2, group_windows=3) == 3
    from segan_pytorch_b200.segan.datasets import normalize_wave_minmax, pre_emphasize
    rate, w = wavfile.read(p)
    ref, _ = s.generate(torch.FloatTensor(pre_emphasize(normalize_wave_minmax(w), 0.95)).view(1, 1, -1))
    _, got = wavfile.read(str(dst / os.path.basename(p)))
    assert got.shape == ref.shape and float(np.abs(got - ref).max()) <= 2e-4


def test_cuda_core_route_refuses_other_widths(monkeypatch):
    """The CUDA-core waveform route serves k = 31 only: other widths raise NotImplementedError."""
    monkeypatch.setenv("SEGAN_B200_WAVE", "cuda")
    G = kw_generator(15, 11).to(DEV)
    with pytest.raises(NotImplementedError, match="tensor-core waveform route"):
        with torch.no_grad():
            G(torch.zeros(1, 1, 16384, device=DEV), z=torch.zeros(1, 1024, 16, device=DEV))
    D = kw_discriminator(11, "bnorm").to(DEV)
    with pytest.raises(NotImplementedError, match="tensor-core waveform route"):
        with torch.no_grad():
            D(torch.zeros(1, 2, 16384, device=DEV))


# ---- against the oracle (tests/test_kwidth.py pins it to the reference at these widths) -------------------------------
def _packed_masters_keep_their_zeros(eng):
    """Every packed master still has exactly the (tap, phase) blocks its width allows: re-packing its reference
    layout gives it back, so the optimiser wrote nothing into the structural zeros."""
    for name, pl in eng.by_name.items():
        if pl.kind == 2:
            continue
        m = eng.mview(pl).view(pl.T, pl.nc, pl.kc).cpu()
        ref = E.unpack_reference(pl.kind, m, pl.c_out, pl.c_in, 0, pl.kw)
        assert torch.equal(E.pack_reference(pl.kind, ref, pl.c_out, pl.c_in, 0, pl.kw), m), name


@pytest.mark.parametrize("gkw,gdkw,dkw", [(15, 11, 21), (20, 32, 11)])
def test_segan_step_batch16_vs_oracle(gkw, gdkw, dkw):
    """One fused SEGAN step at batch 16 against the oracle step and the oracle's operand-precision control, with the
    gates of the k = 31 step (tests/test_gpu_parity_scale.py); afterwards the RMSprop-updated packed masters keep the
    structural zeros of their widths."""
    from tests.test_gpu_parity_scale import GRAD_ABS, GRAD_VS_CONTROL, _loss_gate, _step_vs_oracle
    from tests.util import build_segan, cpu_state
    B = 16
    over = dict(batch_size=B, gkwidth=gkw, gdec_kwidth=gdkw, dkwidth=dkw)
    s = build_segan(**over)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 113, load_opts(**over),
                                                             "k %d/%d/%d B=16" % (gkw, gdkw, dkw))
    _loss_gate(lerr, cl, (0, 1, 3))
    assert lerr[2] <= max(1e-2, 3 * cl[2]), (losses, refl)
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS, (max(eD.values()), max(cD.values()))
    assert float(np.median(list(eD.values()))) <= GRAD_VS_CONTROL * float(np.median(list(cD.values()))) + GRAD_ABS
    assert max(eG.values()) <= GRAD_VS_CONTROL * max(cG.values()) + GRAD_ABS, (max(eG.values()), max(cG.values()))
    torch.cuda.synchronize()
    _packed_masters_keep_their_zeros(s.G.engine)
    _packed_masters_keep_their_zeros(s.D.engine)


TOPOLOGIES = {"no_skip": dict(no_skip=True), "sum": dict(skip_merge="sum"), "conv": dict(skip_type="conv"),
              "no_z": dict(no_z=True), "snorm": dict()}


@pytest.mark.parametrize("name", sorted(TOPOLOGIES))
def test_generator_topologies_vs_control(name):
    """Every Generator topology at encoder / decoder widths (15, 11): the output and the gradients of 100 * L1 of
    every parameter against the oracle, held to its operand-precision control (snorm: one power iteration, the
    spectral-norm oracle tests/gsnorm_oracle.py)."""
    import torch.nn.functional as F
    from oracle import segan_oracle as O
    from tests import gsnorm_oracle as GO
    from tests import gtopo_oracle as TO
    from tests.test_gpu_parity_scale import GRAD_ABS, GRAD_VS_CONTROL
    from tests.test_gtopo import generator_kwargs
    from tests.util import cpu_state
    B = 4
    snorm = name == "snorm"
    G = Generator_(generator_kwargs(TOPOLOGIES[name]), norm_type="snorm" if snorm else None)
    sdG = cpu_state(G)
    G = G.to(DEV).train()
    clean, noisy = _pairs(B, 960)
    z = None if G.no_z else torch.randn(B, 1024, 16, generator=torch.Generator().manual_seed(961))
    y = G(noisy.to(DEV), z=z.to(DEV) if z is not None else None)
    out = 100 * F.l1_loss(y, clean.to(DEV))
    out.backward()
    gG = {n: p.grad.detach().cpu() for n, p in G.named_parameters()}

    def fwd(sd, x):
        if snorm:
            return GO.generator_forward(sd, x, z, training=True, skip_merge=G.skip_merge)
        return TO.generator_forward(sd, x, z, skip_merge=G.skip_merge)

    def oracle():
        sd = {k: v.clone() for k, v in sdG.items()}
        pG = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd)}
        lo = 100 * F.l1_loss(fwd({**sd, **pG}, noisy), clean)
        return float(lo.detach()), dict(zip(pG.keys(), torch.autograd.grad(lo, list(pG.values()))))
    with O.oracle_mode():
        lo, go = oracle()
        with O.operand_precision(torch.float16):
            lc, gc = oracle()
    rep = {k: rel_err(gG[k], r) for k, r in go.items()}
    ctl = {k: rel_err(gc[k], r) for k, r in go.items()}
    print("kwidth G %s: loss %.5f vs %.5f | grads max %.3e (%s) | control max %.3e" % (
        name, float(out), lo, max(rep.values()), max(rep, key=rep.get), max(ctl.values())))
    assert abs(float(out) - lo) <= max(1e-3, 3 * abs(lc - lo)) * max(1.0, abs(lo))
    assert max(rep.values()) <= GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS


def Generator_(kwargs, norm_type=None):
    from segan_pytorch_b200.segan.models import Generator
    seed_all(111)
    return Generator(1, [64, 128, 256, 512, 1024], 15, [4] * 5, dec_kwidth=11, norm_type=norm_type, **kwargs)


def test_wsegan_snorm_step_vs_oracle():
    """The WSEGAN --misalign_pair step with a snorm G and a snorm D at widths 15 (G) / 21 (D), RMSprop: the four
    losses against the oracle step (both networks normalised), as the k = 31 recipe test does."""
    from oracle import segan_oracle as O
    from tests import gsnorm_oracle as GO
    from tests.util import cpu_state
    B = 3
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, dnorm_type="snorm", gkwidth=15, gdec_kwidth=15,
                     dkwidth=21)
    seed_all(111)
    G = kw_generator(15, 15, norm_type="snorm")
    s = WSEGAN(opts, generator=G)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    clean, noisy = _pairs(B, 962)
    z = torch.randn(B, 1024, 16, generator=torch.Generator().manual_seed(963))
    random.seed(6)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    Gopt, Dopt = s.build_optimizers(opts)
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, z=z.to(DEV), shifts=shifts,
                          perm=[2, 0, 1]).tolist()
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    plain_fwd = O.generator_forward
    O.generator_forward = lambda sd, x, z_, ret_hid=False, skip_merge="concat": GO.generator_forward(
        sd, x, z_, training=True, skip_merge=skip_merge, ret_hid=ret_hid)
    try:
        ref = O.wsegan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts, [2, 0, 1], pow_weight=0.001,
                                  l1_weight=100.0)
    finally:
        O.generator_forward = plain_fwd
    refl = [ref[k] for k in ("d_loss", "g_adv_loss", "pow_loss", "den_loss")]
    print("kwidth WSEGAN snorm: losses %s oracle %s" % (losses, refl))
    for got, want in zip(losses, refl):
        assert abs(got - want) <= 3e-2 * max(1.0, abs(want)), (losses, refl)
    torch.cuda.synchronize()
    _packed_masters_keep_their_zeros(s.G.engine)
    _packed_masters_keep_their_zeros(s.D.engine)
