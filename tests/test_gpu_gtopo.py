"""Generators without z (--no_z), without skips (--no_skip), with another z width (--z_dim) and SEGAN's --reg_loss
mse_loss on the H100: the MSE loss kernel and the one-source fold of the last decoder block against torch, the
Generator against the reference's golden outputs and the topology oracle (tests/gtopo_oracle.py), gradients against
the operand-precision control, full SEGAN / WSEGAN steps, graph replay, inference, checkpoints and the
command-line entry points.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import segan_oracle as O                                          # noqa: E402
from segan_pytorch_b200 import _lib, engine as E                             # noqa: E402
from tests import gtopo_oracle as TO                                         # noqa: E402
from tests import test_gpu_parity_scale as PS                                # noqa: E402
from tests.test_gpu_kernels import grad_dtype                                # noqa: E402,F401
from tests.test_gpu_parity_scale import GRAD_ABS, GRAD_VS_CONTROL, _loss_gate, _pairs, _step_vs_oracle  # noqa: E402
from tests.test_gtopo import CONFIGS, GOLD, generator_kwargs, golden_inputs, topo_generator  # noqa: E402
from tests.util import build_segan, cpu_state, golden, load_opts, max_abs, rel_err, seed_all  # noqa: E402

DEV = "cuda"
WAVE_TOL = 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _zdim(name):
    k = generator_kwargs(CONFIGS[name])
    return None if k["no_z"] else k["z_dim"]


# ---- kernel level ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("accumulate", [0, 1])
def test_mse_loss_kernel_vs_torch(accumulate):
    n = 300 * 16384 + 77                                # not a multiple of the block or the grid
    g = torch.Generator(device=DEV).manual_seed(5 + accumulate)
    y = torch.randn(n, device=DEV, generator=g)
    c = torch.randn(n, device=DEV, generator=g)
    gy0 = torch.randn(n, device=DEV, generator=g)
    w, scale = 100.0, 4.0

    def run(name):
        lo = torch.full((1,), 0.25, device=DEV)           # the loss is added to loss_out
        gy = gy0.clone()
        _lib.call(name, _p(y), _p(c), n, w, _p(lo), _p(gy), accumulate, scale, _st())
        torch.cuda.synchronize()
        return lo, gy
    lo, gy = run("sg_mse_loss_bwd")
    d = (y - c).double()
    ref_l = 0.25 + w * float((d * d).mean())
    ref_g = (gy0.double() if accumulate else 0) + scale * 2 * w * d / n
    print("mse kernel: loss %.7f vs %.7f, grad rel %.2e" % (float(lo), ref_l, rel_err(gy, ref_g)))
    assert abs(float(lo) - ref_l) <= 1e-5 * ref_l
    assert rel_err(gy, ref_g) <= 1e-6
    for name in ("sg_mse_loss_bwd", "sg_l1_loss_bwd"):      # the loss sum has a fixed order: same bits every run
        (l1, g1), (l2, g2) = run(name), run(name)
        assert torch.equal(l1, l2) and torch.equal(g1, g2), name


def test_one_source_last_deconv_fold():
    """dwq[2][64][2][cin] (s, k-slot, s', c): dW[c][0][k] += dwq[0][k][0][c] + dwq[1][k][1][c] for k < 31; the
    blocks read are cleared, the others left alone."""
    cin = 64
    g = torch.Generator(device=DEV).manual_seed(3)
    dwq = torch.randn(2, 64, 2, cin, device=DEV, generator=g)
    dwq0 = dwq.clone()
    dw = torch.full((cin, 1, 31), 0.5, device=DEV)
    _lib.call("sg_last_deconv_wgrad_fold_1src", _p(dwq), cin, _p(dw), _st())
    torch.cuda.synchronize()
    ref = 0.5 + (dwq0[0, :31, 0, :] + dwq0[1, :31, 1, :]).t().unsqueeze(1)
    assert max_abs(dw, ref) <= 1e-6
    cleared = dwq0.clone()
    cleared[0, :31, 0, :] = 0
    cleared[1, :31, 1, :] = 0
    assert torch.equal(dwq, cleared)
    with pytest.raises(_lib.SeganB200Error):
        _lib.call("sg_last_deconv_wgrad_fold_1src", _p(dwq), 0, _p(dw), _st())


def test_last_block_weight_gradient_vs_conv_transpose(grad_dtype):
    """The no-skip last decoder block's weight gradient through the engine (im2col of the tanh gradient, one-source
    position-pair GEMM, fold) against autograd of F.conv_transpose1d in fp32 on 16-bit-rounded operands."""
    B = 2
    G = topo_generator("no_z_no_skip").to(DEV).train()
    x = 0.3 * torch.randn(B, 1, 16384, generator=torch.Generator().manual_seed(4))
    y = G(x.to(DEV))
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    y.backward(gy)
    got = G.dec_blocks[4].deconv.weight.grad.detach().cpu()
    with torch.no_grad():
        hall = G(x.to(DEV), ret_hid=("dec_3",))[1]                  # no z: the same decoder input
    h = hall["dec_3"].cpu().to(E.GT).float().requires_grad_(True)        # the 16-bit operand the GEMM reads
    w = G.dec_blocks[4].deconv.weight.detach().cpu().clone().requires_grad_(True)
    out = F.conv_transpose1d(h, w, G.dec_blocks[4].deconv.bias.detach().cpu(), stride=4, padding=13)[..., :-1]
    yt = torch.tanh(out.detach())
    gpre = (gy.cpu() * (1 - yt ** 2) * E.LOSS_SCALE).to(E.GT).float() / E.LOSS_SCALE   # the gradient operand
    ref = torch.autograd.grad(out, w, gpre)[0]
    err = rel_err(got, ref)
    print("no-skip last block dW (%s): rel %.2e" % (E.GT, err))
    assert err <= 1e-2


# ---- Generator ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_generator_vs_reference_golden(name, mode):
    g = golden(GOLD)
    x, z, _ = golden_inputs(g, name)
    G = topo_generator(name).to(DEV)
    zz = z.to(DEV) if z is not None else None
    if mode == "eval":
        G.eval()
        with torch.no_grad():
            y, hall = G(x.to(DEV), z=zz, ret_hid=True)
    else:
        G.train()
        y, hall = G(x.to(DEV), z=zz, ret_hid=True)
        y = y.detach()
    yv = y.cpu().reshape(-1)[torch.from_numpy(g["y_idx.%s" % name])]
    err = max_abs(yv, g["y_val.%s" % name])
    print("G %s %s vs reference: max-abs %.3e" % (name, mode, err))
    assert err <= WAVE_TOL
    assert sorted(hall) == [str(k) for k in g["hall_keys.%s" % name]]
    if z is not None:
        assert hall["enc_zc"].shape[1] == z.shape[1] + 1024
    assert hasattr(G, "z") == bool(g["has_z_attr.%s" % name])


@pytest.mark.parametrize("name", ["no_z", "no_skip"])
def test_generator_forward_batch300_vs_oracle(name):
    """300 windows through the training configuration's G (SEGAN's weights_init), every output sample against the
    oracle, as for the default Generator (test_gpu_parity_scale.test_generator_forward_batch300)."""
    B = 300
    s = build_segan(batch_size=B, **CONFIGS[name])
    sd = cpu_state(s.G)
    G = s.G.to(DEV).eval()
    _, noisy, z = _pairs(B, 131)
    with torch.no_grad():
        y = G(noisy.to(DEV), z=z.to(DEV)).cpu()
    with O.oracle_mode(), torch.no_grad():
        ref = TO.generator_forward(sd, noisy, z)
        with O.operand_precision(torch.float16):
            ctl = TO.generator_forward(sd, noisy[:8], z[:8])
    err = max_abs(y, ref)
    print("G %s fwd B=300: max-abs %.3e (operand-precision control on 8 windows: %.3e)"
          % (name, err, max_abs(ctl, ref[:8])))
    assert err <= WAVE_TOL


@pytest.mark.parametrize("loss", ["l1", "mse"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_generator_gradients_vs_control(name, loss):
    """Gradients of 100 * L1 / 100 * MSE of every parameter, held to the oracle's operand-precision control."""
    B = 4
    s = build_segan(batch_size=B, **CONFIGS[name])
    sdG = cpu_state(s.G)
    G = s.G.to(DEV).train()
    clean, noisy, z = _pairs(B, 132)
    zd = _zdim(name)
    z = z[:, :zd].contiguous() if zd is not None else None
    fn = F.l1_loss if loss == "l1" else F.mse_loss
    y = G(noisy.to(DEV), z=z.to(DEV) if z is not None else None)
    out = 100 * fn(y, clean.to(DEV))
    out.backward()
    gG = {n: p.grad.detach().cpu() for n, p in G.named_parameters()}

    def oracle():
        pG = {k: sdG[k].clone().requires_grad_(True) for k in O._trainable(sdG)}
        lo = 100 * fn(TO.generator_forward({**sdG, **pG}, noisy, z, skip_merge=G.skip_merge), clean)
        return float(lo.detach()), dict(zip(pG.keys(), torch.autograd.grad(lo, list(pG.values()))))
    with O.oracle_mode():
        lo, go = oracle()
        with O.operand_precision(torch.float16):
            lc, gc = oracle()
    rep = {k: rel_err(gG[k], r) for k, r in go.items()}
    ctl = {k: rel_err(gc[k], r) for k, r in go.items()}
    print("G %s %s grads: loss %.5f vs %.5f | max %.3e (%s) | control max %.3e" % (
        name, loss, float(out), lo, max(rep.values()), max(rep, key=rep.get), max(ctl.values())))
    assert abs(float(out) - lo) <= max(1e-3, 3 * abs(lc - lo)) * max(1.0, abs(lo))
    assert max(rep.values()) <= GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS


# ---- train steps ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,reg_loss", [("no_z", "l1_loss"), ("no_skip", "l1_loss"), ("z256", "l1_loss"),
                                           ("default", "mse_loss")])
def test_train_step_batch16_vs_oracle(name, reg_loss, monkeypatch):
    B = 16
    over = dict(CONFIGS.get(name, {}), reg_loss=reg_loss)
    s = build_segan(batch_size=B, **over)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    if name == "z256":                                   # the shared step helper draws 1024-channel z
        pairs = PS._pairs
        monkeypatch.setattr(PS, "_pairs", lambda B_, seed: (lambda c, n, z: (c, n, z[:, :256].contiguous()))(
            *pairs(B_, seed)))
    with TO.gtopo(reg_loss):
        losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 133, load_opts(batch_size=B, **over),
                                                                 "%s %s B=16" % (name, reg_loss))
    _loss_gate(lerr, cl, (0, 1, 3))
    assert lerr[2] <= max(1e-2, 3 * cl[2]), (losses, refl)
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS
    assert float(np.median(list(eG.values()))) <= GRAD_VS_CONTROL * float(np.median(list(cG.values()))) + GRAD_ABS
    assert max(eG.values()) <= GRAD_VS_CONTROL * max(cG.values()) + GRAD_ABS


@pytest.mark.parametrize("name", ["no_z", "no_skip"])
def test_wsegan_misalign_step_vs_oracle(name):
    from segan_pytorch_b200.segan.models import WSEGAN
    B = 3
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, reg_loss="mse_loss", **CONFIGS[name])
    s = WSEGAN(opts)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    gen = torch.Generator().manual_seed(23)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1)
    z = torch.randn(B, 1024, 16, generator=gen)
    random.seed(6)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    Gopt, Dopt = s.build_optimizers(opts)
    # 'additive' windows: the masked denoising term runs, and stays L1 whatever reg_loss says (model.py:663)
    utt = ["a_additive", "b", "c_additive"]
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=utt, z=z.to(DEV),
                          shifts=shifts, perm=[2, 0, 1]).tolist()
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    mask = torch.tensor([1.0, 0.0, 1.0]).view(B, 1, 1).expand(B, 1, 16384).contiguous()
    with TO.gtopo():
        ref = O.wsegan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts, [2, 0, 1], pow_weight=0.001,
                                  l1_weight=100.0, additive_mask=mask)
    print("%s wsegan losses" % name, losses, [ref[k] for k in ("d_loss", "g_adv_loss", "pow_loss", "den_loss")])
    assert ref["den_loss"] > 0
    for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
        assert abs(got - ref[k]) <= 3e-2 * max(1.0, abs(ref[k])), (k, got, ref[k])
    rep = {k: rel_err(s.D.engine.grad_of(k).cpu(), g) for k, g in ref["gradsD"].items()
           if not (k.startswith("enc_blocks") and k.endswith("conv.bias"))}
    print("%s wsegan D grad rel errs (max): %.3e" % (name, max(rep.values())))
    assert max(rep.values()) <= 0.2, rep


@pytest.mark.parametrize("over", [dict(no_z=True), dict(no_skip=True, reg_loss="mse_loss")])
def test_graph_replayed_steps_match_eager_steps(over):
    """Four steps from the same state and inputs, z drawn by the step itself: eager vs eager gives the noise floor,
    the graph-replayed steps are held to it.  With no_z no step consumes torch CPU random numbers."""
    B = 4
    opts = load_opts(batch_size=B, g_lr=5e-7, d_lr=5e-7, **over)
    gen = torch.Generator().manual_seed(7)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1).to(DEV)
    noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1).to(DEV)
    random.seed(12)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(4)]
    no_z = bool(over.get("no_z"))

    def run(graphs):
        prev = E.GRAPHS
        E.GRAPHS = graphs
        try:
            s = build_segan(batch_size=B, **over).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(opts)
            out = []
            torch.manual_seed(99)
            for i in range(4):
                rng = torch.get_rng_state()
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, shifts3=shifts[i])
                torch.cuda.synchronize()
                if no_z:
                    assert torch.equal(torch.get_rng_state(), rng), i
                out.append((losses.tolist(), s.G.engine.grad.clone(), s.D.engine.grad.clone()))
            assert hasattr(s.G, "z") != no_z
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs
        finally:
            E.GRAPHS = prev

    (e1, n1), (e2, n2), (gr, n3) = run(False), run(False), run(True)
    assert n1 == 0 and n2 == 0 and n3 == 1
    floor_l = max(max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[i][0], e2[i][0])) for i in range(4))
    floor_g = max(max(rel_err(e2[i][1], e1[i][1]), rel_err(e2[i][2], e1[i][2])) for i in range(4))
    for step in range(4):
        (l0, gG0, gD0), (l2, gG2, gD2) = e1[step], gr[step]
        err_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l2))
        err_g = max(rel_err(gG2, gG0), rel_err(gD2, gD0))
        print("%s step %d: eager-vs-eager loss %.2e grad %.2e | graph-vs-eager loss %.2e grad %.2e"
              % (over, step, floor_l, floor_g, err_l, err_g))
        assert err_l <= 10 * floor_l + 2e-3, (step, l0, l2)
        assert err_g <= 10 * floor_g + 5e-3, (step, err_g, floor_g)


# ---- inference, checkpoints and entry points ------------------------------------------------------------------------
def test_no_z_inference_paths(tmp_path):
    """generate / generate_stream / clean_files with no_z: G on the same windows, no z drawn, G.z never set."""
    from scipy.io import wavfile
    from segan_pytorch_b200.segan.datasets import normalize_wave_minmax, pre_emphasize
    s = build_segan(no_z=True).to(DEV)
    gen = torch.Generator().manual_seed(14)
    T = 40000
    wav = 0.3 * torch.randn(1, 1, T, generator=gen)
    rng = torch.get_rng_state()
    out, _ = s.generate(wav, z=torch.randn(1, 1024, 16, generator=gen))
    x = torch.zeros(3, 1, 16384)
    x.view(-1)[:T] = wav.view(-1)
    with torch.no_grad():
        y = s.G(x.to(DEV)).cpu().reshape(-1)[:T].numpy()
    assert max_abs(out, O.de_emphasize(y, 0.95)) <= 1e-4
    batches = [(0.3 * torch.randn(3, 1, 16384, generator=gen)).pin_memory() for _ in range(3)]
    outs = [o.clone() for o in s.generate_stream(iter(batches))]
    with torch.no_grad():
        for hb, o in zip(batches, outs):
            assert max_abs(o, s.G(hb.to(DEV)).cpu()) <= 1e-6
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    paths = []
    for i, n in enumerate([40000, 9000]):
        p = str(src / ("u%d.wav" % i))
        wavfile.write(p, 16000, (np.random.RandomState(i).randn(n) * 3000).astype(np.int16))
        paths.append(p)
    assert s.clean_files(paths, str(dst), batch=2, group_windows=3) == 4
    assert torch.equal(torch.get_rng_state(), rng)
    assert not hasattr(s.G, "z")
    for p in paths:
        rate, w = wavfile.read(p)
        pw = torch.FloatTensor(pre_emphasize(normalize_wave_minmax(w), 0.95)).view(1, 1, -1)
        ref, _ = s.generate(pw)
        _, got = wavfile.read(str(dst / os.path.basename(p)))
        assert got.shape == ref.shape and max_abs(got, ref) <= 2e-4


@pytest.mark.parametrize("name", ["no_z_no_skip", "z256"])
def test_checkpoint_round_trip(name, tmp_path):
    B = 2
    s = build_segan(batch_size=B, **CONFIGS[name]).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B, **CONFIGS[name]))
    clean, noisy, z = [t.to(DEV) for t in _pairs(B, 134)]
    z = z[:, :_zdim(name)].contiguous() if _zdim(name) else None
    sd0 = {k: v.clone() for k, v in s.G.state_dict().items()}
    s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=z)
    sd1 = {k: v.clone() for k, v in s.G.state_dict().items()}
    assert list(sd1) == list(sd0)
    assert float((sd1["dec_blocks.4.deconv.weight"] - sd0["dec_blocks.4.deconv.weight"]).abs().max()) > 1e-6
    s.G.eval()
    with torch.no_grad():
        y1 = s.G(noisy, z=z).clone()
    s.G.save(str(tmp_path), 1)
    s2 = build_segan(seed=3, batch_size=B, **CONFIGS[name]).to(DEV)
    s2.G.load_pretrained(os.path.join(str(tmp_path), "weights_Generator-Generator-1.ckpt"), True)
    s2.G.eval()
    with torch.no_grad():
        assert max_abs(s2.G(noisy, z=z), y1) == 0.0


@pytest.mark.parametrize("flags", [["--no_z", "--no_skip", "--reg_loss", "mse_loss"], ["--z_dim", "256"]])
def test_train_and_clean_cli(flags, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    ck = str(tmp_path / "ckpt")
    subprocess.check_call([sys.executable, "train.py", "--save_path", ck, "--synthetic", "64", "--batch_size", "8",
                           "--epoch", "1", "--save_freq", "4", "--num_workers", "0"] + flags, cwd=ROOT, env=env)
    from scipy.io import wavfile
    wdir = tmp_path / "wavs"
    wdir.mkdir()
    rng = np.random.RandomState(0)
    lengths = {"a.wav": 40000, "b.wav": 16384}
    for n, T in lengths.items():
        wavfile.write(str(wdir / n), 16000, (rng.randn(T) * 3000).astype(np.int16))
    gck = sorted(f for f in os.listdir(ck) if "G" in f and f.endswith(".ckpt"))[0]
    subprocess.check_call([sys.executable, "clean.py", "--g_pretrained_ckpt", os.path.join(ck, gck), "--cfg_file",
                           os.path.join(ck, "train.opts"), "--test_files", str(wdir), "--synthesis_path",
                           str(tmp_path / "clean")], cwd=ROOT, env=env)
    for n, T in lengths.items():
        r, w = wavfile.read(str(tmp_path / "clean" / n))
        assert r == 16000 and w.shape[0] == T and np.isfinite(w).all(), (n, r, w.shape)


def test_refusals():
    with pytest.raises(NotImplementedError, match="positive multiple of 64"):
        build_segan(z_dim=100).to(DEV).G(torch.zeros(1, 1, 16384, device=DEV))
    s = build_segan(batch_size=2, reg_loss="smooth_l1_loss").to(DEV)
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=2))
    clean, noisy, z = [t.to(DEV) for t in _pairs(2, 135)]
    with pytest.raises(NotImplementedError, match="smooth_l1_loss"):
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=z)
