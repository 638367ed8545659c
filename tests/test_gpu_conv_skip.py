"""skip_type='conv' Generators on the H100: the grouped skip-conv tap-GEMMs and their emission / fold kernels against
torch, the Generator against the reference's golden outputs and the conv-skip oracle (tests/conv_skip_oracle.py),
full SEGAN / WSEGAN steps, checkpoints and the command-line entry points.
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
from segan_pytorch_b200._lib import SG_F16                                   # noqa: E402
from tests import conv_skip_oracle as CO                                     # noqa: E402
from tests.test_gpu_kernels import grad_dtype                                # noqa: E402,F401
from tests.test_gpu_parity_scale import (GRAD_ABS, GRAD_TOL_SMOOTH, GRAD_VS_CONTROL, _loss_gate, _pairs,  # noqa: E402
                                         _set_slopes, _step_vs_oracle)
from tests.test_conv_skip import GOLD, conv_generator, golden_inputs        # noqa: E402
from tests.util import build_segan, cpu_state, golden, load_opts, max_abs, rel_err, sd_sha, seed_all  # noqa: E402

DEV = "cuda"
WAVE_TOL = 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def exact_torch():
    """fp32 torch references without TF32."""
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr())


# ---- kernel level ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [4, 16, 1024])
@pytest.mark.parametrize("K", [1, 11, 33])
@pytest.mark.parametrize("C_", [64, 512])
def test_skip_conv_kernels_vs_torch(C_, K, rows, grad_dtype, exact_torch):
    """Forward, data gradient and weight gradient (+ fold) of the grouped skip conv: rows = L / 4 grouped rows per
    batch element (4 and 16: several batch elements per 128-row M tile; 1024: whole tiles)."""
    GT, GS = E.GT, E.GS
    B, L, P = (2 if rows == 1024 else 5), 4 * rows, K // 2
    g = torch.Generator(device=DEV).manual_seed(1000 * K + rows + C_)
    w = 0.05 * torch.randn(C_, C_, K, device=DEV, generator=g)
    b = 0.1 * torch.randn(C_, device=DEV, generator=g)
    a = torch.randn(B, L, C_, device=DEV, generator=g).half()
    gs = torch.randn(B, L, C_, device=DEV, generator=g).to(GT)
    D = (K // 2 + 3) // 4
    wf = torch.empty(2 * D + 1, 4 * C_, 4 * C_, dtype=torch.float16, device=DEV)
    wd = torch.empty(2 * D + 1, 4 * C_, 4 * C_, dtype=GT, device=DEV)
    _lib.call("sg_skipconv_emit", _p(w), C_, K, _p(wf), _p(wd), SG_F16, GS, _st())
    wp = E.skipconv_pack_reference(w)
    assert torch.equal(wf, wp.half())
    assert torch.equal(wd, wp.flip(0).transpose(1, 2).to(GT))
    d_lo, d_hi, tap0, taps, taps_dg = E.skipconv_geometry(C_, K)
    # forward (bias, fp16 out)
    out = torch.empty(B, L, C_, dtype=torch.float16, device=DEV)
    E.run_f(a, None, rows, 0, SG_F16, wf, SG_F16, 4 * C_, 4 * C_, taps, out, SG_F16, rows, 0, 0, rows, B, bias=b,
            bias_mod=C_, d_lo=d_lo, d_hi=d_hi, w_tap0=tap0)
    ref = F.conv1d(a.float().transpose(1, 2), w.half().float(), b, padding=P).transpose(1, 2)
    e_f = max_abs(out.float(), ref) / float(ref.abs().max())
    # data gradient (gradient dtype out)
    ga = torch.empty(B, L, C_, dtype=GT, device=DEV)
    E.run_f(gs, None, rows, 0, GS, wd, GS, 4 * C_, 4 * C_, taps_dg, ga, GS, rows, 0, 0, rows, B, d_lo=d_lo, d_hi=d_hi,
            w_tap0=tap0)
    ref_g = F.conv_transpose1d(gs.float().transpose(1, 2), w.to(GT).float(), padding=P).transpose(1, 2)
    e_d = max_abs(ga.float(), ref_g) / float(ref_g.abs().max())
    # weight gradient: both operands in the gradient format (wgmma needs one 16-bit type)
    a_op = a if GT == torch.float16 else a.to(GT)
    dwq = torch.zeros((2 * D + 1) * 16 * C_ * C_, dtype=torch.float32, device=DEV)
    E.run_w(gs, rows, GS, a_op, None, rows, 0, GS, 4 * C_, 4 * C_, taps, dwq, B, d_lo=d_lo, d_hi=d_hi, dw_tap0=tap0,
            ksplit=E.wgrad_ksplit(B * rows, 0, taps, 4 * C_, 4 * C_, d_lo, d_hi))
    dw = torch.full((C_, C_, K), 0.5, device=DEV)                      # the fold accumulates
    _lib.call("sg_skipconv_wgrad_fold", _p(dwq), C_, K, _p(dw), _st())
    ref_w = torch.nn.grad.conv1d_weight(a_op.float().transpose(1, 2), w.shape, gs.float().transpose(1, 2), padding=P)
    e_w = rel_err(dw - 0.5, ref_w)
    torch.cuda.synchronize()
    print("C=%d K=%d rows=%d %s: fwd %.2e dgrad %.2e wgrad %.2e" % (C_, K, rows, GT, e_f, e_d, e_w))
    assert e_f <= 2e-3
    assert e_d <= (2e-3 if GT == torch.float16 else 1e-2)
    assert e_w <= 1e-4
    assert int(torch.count_nonzero(dwq)) == 0                          # clear-on-read workspace


def test_skip_conv_entry_points_reject_unserved_shapes():
    t = torch.zeros(64 * 64 * 16, device=DEV)
    for c, k in ((64, 10), (64, 35), (96, 11), (64, 0)):
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_skipconv_emit", _p(t), c, k, _p(t), None, 0, 0, _st())
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_skipconv_wgrad_fold", _p(t), c, k, _p(t), _st())
    for dt_f, dt_d in ((7, SG_F16), (SG_F16, -1)):              # element types outside SG_F32 | SG_F16 | SG_BF16
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_skipconv_emit", _p(t), 64, 1, _p(t), _p(t), dt_f, dt_d, _st())


# ---- Generator ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("merge", ["concat", "sum"])
def test_generator_vs_reference_golden(merge, mode):
    """The reference's own conv-skip Generator output (2 windows).  train: the autograd path, whose forward keeps
    the pre-activations for backward (the fused-activation epilogue writes both)."""
    g = golden(GOLD)
    x, z, _ = golden_inputs(g)
    G = conv_generator(merge)
    assert sd_sha(G.state_dict()) == str(g["sha_G_init.%s" % merge])
    G = G.to(DEV)
    if mode == "eval":
        G.eval()
        with torch.no_grad():
            y = G(x.to(DEV), z=z.to(DEV))
    else:
        G.train()
        y = G(x.to(DEV), z=z.to(DEV)).detach()
    err = max_abs(y.cpu(), g["y.%s" % merge])
    print("conv-skip G %s %s vs reference: max-abs %.3e" % (merge, mode, err))
    assert err <= WAVE_TOL


def test_generator_forward_batch300_vs_oracle():
    B = 300
    G = conv_generator()
    sd = cpu_state(G)
    G = G.to(DEV).eval()
    _, noisy, z = _pairs(B, 121)
    with torch.no_grad():
        y = G(noisy.to(DEV), z=z.to(DEV)).cpu()
    with O.oracle_mode(), torch.no_grad():
        ref = CO.generator_forward(sd, noisy, z)
    err = max_abs(y, ref)
    print("conv-skip G fwd B=300: max-abs %.3e" % err)
    assert err <= WAVE_TOL


@pytest.mark.parametrize("slope", [None, 1.0])
def test_generator_l1_gradients_vs_oracle(slope, grad_dtype):
    """Gradients of 100 * L1(G(x), clean) for every parameter, the skip convs' weights and biases included."""
    B = 4
    s = build_segan(batch_size=B, skip_type="conv")
    if slope is not None:
        _set_slopes(s, slope)
    sdG = cpu_state(s.G)
    G = s.G.to(DEV).train()
    clean, noisy, z = _pairs(B, 122)
    y = G(noisy.to(DEV), z=z.to(DEV))
    loss = 100 * F.l1_loss(y, clean.to(DEV))
    loss.backward()
    gG = {n: p.grad.detach().cpu() for n, p in G.named_parameters()}

    def oracle():
        pG = {k: sdG[k].clone().requires_grad_(True) for k in O._trainable(sdG)}
        lo = 100 * F.l1_loss(CO.generator_forward({**sdG, **pG}, noisy, z), clean)
        return float(lo.detach()), dict(zip(pG.keys(), torch.autograd.grad(lo, list(pG.values()))))
    with O.oracle_mode():
        lo, go = oracle()
        with O.operand_precision(torch.float16):
            lc, gc = oracle()
    assert any(k.endswith("skip_k.weight") for k in go) and any(k.endswith("skip_k.bias") for k in go)
    rep = {k: rel_err(gG[k], r) for k, r in go.items()}
    ctl = {k: rel_err(gc[k], r) for k, r in go.items()}
    print("conv-skip G L1 grads, slopes %s, %s: loss %.5f vs %.5f | max %.3e (%s) | control max %.3e" % (
        slope, E.GT, float(loss), lo, max(rep.values()), max(rep, key=rep.get), max(ctl.values())))
    print("   skip convs:", {k: "%.2e/%.2e" % (v, ctl[k]) for k, v in rep.items() if "skip_k" in k})
    assert abs(float(loss) - lo) <= max(1e-3, 3 * abs(lc - lo)) * max(1.0, abs(lo))
    if slope is None:
        assert max(rep.values()) <= GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS
    else:
        # sign(G(x) - clean) still flips where |G(x) - clean| is below the operand error: as the control does
        assert max(rep.values()) <= max(GRAD_TOL_SMOOTH, GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS), \
            sorted(rep.items(), key=lambda kv: -kv[1])[:5]


# ---- train steps ----------------------------------------------------------------------------------------------------
def test_train_step_batch16_vs_oracle():
    B = 16
    s = build_segan(batch_size=B, skip_type="conv")
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    with CO.conv_skips():
        losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 123,
                                                                 load_opts(batch_size=B, skip_type="conv"), "conv B=16")
    print("   skip conv G grads:", {k: "%.2e/%.2e" % (v, cG[k]) for k, v in eG.items() if "skip_k" in k})
    _loss_gate(lerr, cl, (0, 1, 3))
    assert lerr[2] <= max(1e-2, 3 * cl[2]), (losses, refl)
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS
    assert float(np.median(list(eG.values()))) <= GRAD_VS_CONTROL * float(np.median(list(cG.values()))) + GRAD_ABS
    assert max(eG.values()) <= GRAD_VS_CONTROL * max(cG.values()) + GRAD_ABS


def test_graph_replayed_steps_match_eager_steps():
    """Four steps from the same state and inputs: eager vs eager gives the noise floor, the graph-replayed steps
    (capture after engine.GRAPH_WARMUP eager steps) are held to it.  At the reference's learning rate the first
    RMSprop step is 10 lr sign(g) on every weight and two eager runs already drift apart by tens of percent a step
    later; a 100x smaller rate keeps the trajectories close enough for the floor to mean something."""
    B = 4
    opts = load_opts(batch_size=B, skip_type="conv", g_lr=5e-7, d_lr=5e-7)
    gen = torch.Generator().manual_seed(7)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1).to(DEV)
    noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1).to(DEV)
    zs = [torch.randn(B, 1024, 16, generator=gen).to(DEV) for _ in range(4)]
    random.seed(12)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(4)]

    def run(graphs):
        prev = E.GRAPHS
        E.GRAPHS = graphs
        try:
            s = build_segan(batch_size=B, skip_type="conv").to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(opts)
            out = []
            for i in range(4):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=zs[i], shifts3=shifts[i])
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad.clone(), s.D.engine.grad.clone()))
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs
        finally:
            E.GRAPHS = prev

    (e1, n1), (e2, n2), (gr, n3) = run(False), run(False), run(True)
    assert n1 == 0 and n2 == 0 and n3 == 1
    # the floor is the spread of the two eager runs over the whole run: the order of the fp32 gradient atomics alone
    # moves a single step's gradients by 5e-4 .. 1e-2 (the D step's real / fake terms cancel), so one step's
    # eager-vs-eager distance can land far below what the next pair of runs shows
    floor_l = max(max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[i][0], e2[i][0])) for i in range(4))
    floor_g = max(max(rel_err(e2[i][1], e1[i][1]), rel_err(e2[i][2], e1[i][2])) for i in range(4))
    for step in range(4):
        (l0, gG0, gD0), (l2, gG2, gD2) = e1[step], gr[step]
        err_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l2))
        err_g = max(rel_err(gG2, gG0), rel_err(gD2, gD0))
        print("conv step %d: eager-vs-eager loss %.2e grad %.2e | graph-vs-eager loss %.2e grad %.2e"
              % (step, floor_l, floor_g, err_l, err_g))
        assert err_l <= 10 * floor_l + 2e-3, (step, l0, l2)
        assert err_g <= 10 * floor_g + 5e-3, (step, err_g, floor_g)


def test_wsegan_misalign_step_vs_oracle():
    from segan_pytorch_b200.segan.models import WSEGAN
    B = 3
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, skip_type="conv")
    s = WSEGAN(opts)
    assert s.G.skip_type == "conv"
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
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=["a", "b", "c"], z=z.to(DEV),
                          shifts=shifts, perm=[2, 0, 1]).tolist()
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    with CO.conv_skips():
        ref = O.wsegan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts, [2, 0, 1], pow_weight=0.001,
                                  l1_weight=100.0)
    print("conv wsegan losses", losses, [ref[k] for k in ("d_loss", "g_adv_loss", "pow_loss", "den_loss")])
    for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
        assert abs(got - ref[k]) <= 3e-2 * max(1.0, abs(ref[k])), (k, got, ref[k])
    rep = {k: rel_err(s.D.engine.grad_of(k).cpu(), g) for k, g in ref["gradsD"].items()
           if not (k.startswith("enc_blocks") and k.endswith("conv.bias"))}
    print("conv wsegan D grad rel errs (max):", max(rep.values()))
    assert max(rep.values()) <= 0.2, rep


# ---- checkpoints and entry points -----------------------------------------------------------------------------------
def test_checkpoint_round_trip_and_reference_state_dict(tmp_path):
    B = 2
    s = build_segan(batch_size=B, skip_type="conv").to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B, skip_type="conv"))
    clean, noisy, z = [t.to(DEV) for t in _pairs(B, 124)]
    sd0 = {k: v.clone() for k, v in s.G.state_dict().items()}
    s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=z)
    sd1 = {k: v.clone() for k, v in s.G.state_dict().items()}
    assert float((sd1["alpha_1.skip_k.weight"] - sd0["alpha_1.skip_k.weight"]).abs().max()) > 1e-4
    s.G.eval()
    with torch.no_grad():
        y1 = s.G(noisy, z=z).clone()
    s.G.save(str(tmp_path), 1)
    s2 = build_segan(seed=3, batch_size=B, skip_type="conv").to(DEV)
    s2.G.load_pretrained(os.path.join(str(tmp_path), "weights_Generator-Generator-1.ckpt"), True)
    s2.G.eval()
    with torch.no_grad():
        assert max_abs(s2.G(noisy, z=z), y1) == 0.0
    # a reference-layout state dict (the reference's own seeded init) loaded into another model
    g = golden(GOLD)
    x, zg, _ = golden_inputs(g)
    s2.G.load_state_dict(cpu_state(conv_generator()))
    with torch.no_grad():
        y = s2.G(x.to(DEV), z=zg.to(DEV)).cpu()
    assert max_abs(y, g["y.concat"]) <= WAVE_TOL


def test_train_and_clean_cli(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    ck = str(tmp_path / "ckpt")
    subprocess.check_call([sys.executable, "train.py", "--save_path", ck, "--synthetic", "64", "--batch_size", "8",
                           "--epoch", "1", "--save_freq", "4", "--skip_type", "conv", "--num_workers", "0"], cwd=ROOT, env=env)
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
