"""Parity at the BENCHMARKED shape and for the reference's canonical recipes (VERDICT round 1, items 1a / 1b):
  * G forward and D forward (train-mode BatchNorm) at batch 300 against the oracle on the host CPU
  * one full G+D step at batch 16 against the oracle step
  * --no_bias (run_segan+_train.sh), WSEGAN with Adam (run_wsegan_train.sh's optimiser)
  * WSEGAN.generate on lengths that are / are not multiples of 1024 against the unmodified reference's output
Every test prints, next to the kernels' error, the error of the oracle's own operand-precision control
(oracle.operand_precision(fp16): fp32 reference arithmetic with 16-bit operand rounding only): that is the part
of the distance to the fp32 reference that the operand FORMAT costs, independent of any kernel.
Run on an H100:  python -m pytest tests -m gpu"""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import segan_oracle as O                                         # noqa: E402
from tests.util import build_segan, cpu_state, golden, load_opts, max_abs, rel_err, sd_sha, seed_all  # noqa: E402

DEV = "cuda"
WAVE_TOL = 1e-3          # north_star: max-abs on fp32 waveforms
# SURVEY.md 8(d) gates
LOSS_RTOL = 1e-3
LOGIT_TOL = 1e-3
RUNSTAT_TOL = 1e-4
# Gradients (tools/parity_probe.py, tools/dgrad_probe.py take them apart): with the reference's PReLU slopes
# (init 0: the derivative jumps from 0 to 1 at 0) every parameter gradient of a train step is 5-7 % away from the
# fp32 oracle in relative L2 -- with bf16 AND with fp16 gradient tensors alike -- and the oracle's own operand-
# precision control (fp32 arithmetic, fp16-rounded operands, no kernel of ours involved) is just as far, tensor by
# tensor.  Two amplifiers of the ~1e-3 operand rounding of the forward activations: (i) the ~1e-3 of elements within
# that distance of 0 get the other side's derivative (100 % error there): sqrt(flipped fraction) ~ 3 % per layer,
# accumulating in quadrature and scaling with the jump (slopes 0.5 halve it); (ii) the D step adds the real and the
# fake pass, whose logit gradients 2(l - 1)/B and 2 l/B largely cancel at initialisation, so the relative error of
# the SUM is several times that of either pass (slopes 1, batch 8: each pass alone 0.2-0.5 %, the sum 6 % -- in the
# control exactly as in the kernels).  Train-step gradients are therefore held to the control:
# <= GRAD_VS_CONTROL x its error (+ GRAD_ABS); single-pass gradients with continuous activations to GRAD_TOL_SMOOTH.
GRAD_TOL_SMOOTH = 1e-2   # relative L2 per parameter tensor: one pass, continuous activation derivative
GRAD_VS_CONTROL = 1.5
GRAD_ABS = 5e-3


def _pairs(B, seed):
    g = torch.Generator().manual_seed(seed)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    z = torch.randn(B, 1024, 16, generator=g)
    return clean, noisy, z


def test_generator_forward_batch300():
    """BASELINE configs[1] shape: 300 windows through G (eval), every output sample against the oracle."""
    B = 300
    s = build_segan(batch_size=B)
    sdG = cpu_state(s.G)
    s = s.to(DEV)
    _, noisy, z = _pairs(B, 111)
    s.G.eval()
    with torch.no_grad():
        y = s.G(noisy.to(DEV), z=z.to(DEV)).cpu()
    with O.oracle_mode(), torch.no_grad():
        ref = O.generator_forward(sdG, noisy, z)
        with O.operand_precision(torch.float16):
            ctl = O.generator_forward(sdG, noisy[:8], z[:8])
    err = max_abs(y, ref)
    print("G fwd B=300: max-abs %.3e (operand-precision control on 8 windows: %.3e)" % (err, max_abs(ctl, ref[:8])))
    assert err <= WAVE_TOL


def test_discriminator_forward_batch300():
    """D forward in train mode at batch 300: BatchNorm statistics over 300 x L, logits and running statistics."""
    B = 300
    s = build_segan(batch_size=B)
    sdD = cpu_state(s.D)
    s = s.to(DEV)
    clean, noisy, _ = _pairs(B, 112)
    x = torch.cat((clean, noisy), 1)
    random.seed(5)
    shifts = O.draw_phase_shifts(5, 5)
    s.D.train()
    with torch.no_grad():
        y, _ = s.D(x.to(DEV), shifts=shifts)
    sd_ref = {k: v.clone() for k, v in sdD.items()}
    sd_ctl = {k: v.clone() for k, v in sdD.items()}
    with O.oracle_mode(), torch.no_grad():
        ref = O.discriminator_forward(sd_ref, x, shifts, training=True)
        with O.operand_precision(torch.float16):
            ctl = O.discriminator_forward(sd_ctl, x, shifts, training=True)
    rep, rep_ctl = {"logit": max_abs(y.cpu(), ref)}, {"logit": max_abs(ctl, ref)}
    for l in range(5):
        bn = s.D.enc_blocks[l].norm
        for nm, t in (("rm", bn.running_mean), ("rv", bn.running_var)):
            key = "enc_blocks.%d.norm.running_%s" % (l, "mean" if nm == "rm" else "var")
            rep[nm + str(l)] = max_abs(t.cpu(), sd_ref[key])
            rep_ctl[nm + str(l)] = max_abs(sd_ctl[key], sd_ref[key])
    print("D fwd B=300:", {k: "%.2e" % v for k, v in rep.items()})
    print("   control :", {k: "%.2e" % v for k, v in rep_ctl.items()})
    print("   logit scale: mean |logit| %.3f" % float(ref.abs().mean()))
    # held to the survey gate where the operand format allows it, else to 3x the control's own distance
    assert rep["logit"] <= max(LOGIT_TOL, 3 * rep_ctl["logit"]), rep
    for k, v in rep.items():
        if k != "logit":
            assert v <= max(RUNSTAT_TOL, 3 * rep_ctl[k]), (k, v, rep_ctl[k])


def _set_slopes(segan, value):
    """Every PReLU slope of G and D's conv tower := value (reference init: 0, modules.py:81,125)."""
    with torch.no_grad():
        for net in (segan.G, segan.D):
            for n, p in net.named_parameters():
                if n.endswith("act.weight"):
                    p.fill_(value)


def _step_vs_oracle(s, sdG, sdD, B, seed, opts, tag, control=True):
    """One fused train step vs the oracle step and vs the oracle's operand-precision control.
    Returns (losses, oracle losses, relative loss errors, eD, eG, control eD, control eG)."""
    clean, noisy, z = _pairs(B, seed)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(opts)
    random.seed(3)
    shifts3 = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, z=z.to(DEV), shifts3=shifts3).tolist()
    gD = {k: s.D.engine.grad_of(k).cpu() for k, _ in s.D.named_parameters()}
    gG = {k: s.G.engine.grad_of(k).cpu() for k, _ in s.G.named_parameters()}

    def oracle(sdG_, sdD_):
        sqG = {k: torch.zeros_like(sdG_[k]) for k in O._trainable(sdG_)}
        sqD = {k: torch.zeros_like(sdD_[k]) for k in O._trainable(sdD_)}
        return O.segan_train_step(sdG_, sdD_, sqG, sqD, clean, noisy, z, shifts3, l1_weight=100.0)
    clone = lambda sd: {k: v.clone() for k, v in sd.items()}
    ref = oracle(clone(sdG), clone(sdD))
    skip = lambda k: k.startswith("enc_blocks") and k.endswith("conv.bias")    # D: zero in exact arithmetic
    refl = [ref[k] for k in ("d_real_loss", "d_fake_loss", "g_adv_loss", "g_l1_loss")]
    lerr = [abs(a - b) / max(1.0, abs(b)) for a, b in zip(losses, refl)]
    eD = {k: rel_err(gD[k], g) for k, g in ref["gradsD"].items() if not skip(k)}
    eG = {k: rel_err(gG[k], g) for k, g in ref["gradsG"].items()}
    cD = cG = cl = None
    if control:
        with O.operand_precision(torch.float16):
            ctl = oracle(clone(sdG), clone(sdD))
        cD = {k: rel_err(ctl["gradsD"][k], g) for k, g in ref["gradsD"].items() if not skip(k)}
        cG = {k: rel_err(ctl["gradsG"][k], g) for k, g in ref["gradsG"].items()}
        cl = [abs(ctl[k] - b) / max(1.0, abs(b)) for k, b in
              zip(("d_real_loss", "d_fake_loss", "g_adv_loss", "g_l1_loss"), refl)]
    med = lambda d: float(np.median(list(d.values())))
    print("%s losses %s oracle %s rel %s%s" % (tag, ["%.5f" % v for v in losses], ["%.5f" % v for v in refl],
                                               ["%.1e" % v for v in lerr],
                                               (" control rel %s" % ["%.1e" % v for v in cl]) if cl else ""))
    print("%s D grads rel-L2: max %.3e (%s) median %.3e%s" % (
        tag, max(eD.values()), max(eD, key=eD.get), med(eD),
        (" | control max %.3e median %.3e" % (max(cD.values()), med(cD))) if cD else ""))
    print("%s G grads (through the UPDATED D) rel-L2: max %.3e median %.3e%s" % (
        tag, max(eG.values()), med(eG), (" | control max %.3e median %.3e" % (max(cG.values()), med(cG))) if cG else ""))
    return losses, refl, lerr, eD, eG, cD, cG, cl


def _loss_gate(lerr, cl, idx):
    """Losses: the survey's 1e-3, or what the operand format itself costs on this input (3x the control)."""
    for i in idx:
        assert lerr[i] <= max(LOSS_RTOL, 3 * cl[i]), (i, lerr, cl)


def test_train_step_batch16_vs_oracle():
    """One full G+D step at batch 16 (B >= 16: BatchNorm over a real batch) against the oracle step."""
    B = 16
    s = build_segan(batch_size=B)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 113, load_opts(batch_size=B), "B=16")
    # d_real / d_fake / g_l1; g_adv goes through the D that RMSprop's first, sign-like step (lr*sign(g) on 25.8 M
    # weights) produced and is compared loosely
    _loss_gate(lerr, cl, (0, 1, 3))
    assert lerr[2] <= max(1e-2, 3 * cl[2]), (losses, refl)
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS, (max(eD.values()), max(cD.values()))
    assert float(np.median(list(eD.values()))) <= GRAD_VS_CONTROL * float(np.median(list(cD.values()))) + GRAD_ABS


@pytest.mark.parametrize("slope", [1.0, 0.5])
def test_train_step_gradients_vs_control_other_slopes(slope):
    """The same step with every PReLU slope set to 0.5 / 1: the derivative jump halves / vanishes, the control's and
    the kernels' D-step errors move together (at slope 1 what is left is the cancellation between the real and the
    fake pass, see GRAD_TOL_SMOOTH's comment)."""
    B = 8
    s = build_segan(batch_size=B)
    _set_slopes(s, slope)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 117, load_opts(batch_size=B),
                                                             "slope=%g" % slope)
    if slope == 1.0:
        # identity activations: a BatchNorm shift that feeds the next conv + BatchNorm has zero gradient in exact
        # arithmetic (layers 0-3), like the conv biases
        drop = lambda d: {k: v for k, v in d.items() if not (k.endswith("norm.bias") and not k.startswith("enc_blocks.4"))}
        eD, cD = drop(eD), drop(cD)
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS, (max(eD.values()), max(cD.values()))
    assert float(np.median(list(eD.values()))) <= GRAD_VS_CONTROL * float(np.median(list(cD.values()))) + GRAD_ABS


def test_discriminator_single_pass_gradients_continuous_activation():
    """One D pass (LSGAN loss against target 1) with every PReLU slope at 1 -- no derivative jump, no second pass to
    cancel against: the backward kernels' own error, every parameter tensor within GRAD_TOL_SMOOTH of the oracle."""
    import ctypes as C
    B = 8
    s = build_segan(batch_size=B)
    _set_slopes(s, 1.0)
    sdD = cpu_state(s.D)
    s = s.to(DEV)
    s.D.train()
    clean, noisy, _ = _pairs(B, 118)
    shifts = [3, -1, 4, -2, 5]
    de = s.D.engine
    de.bind()
    de.zero_grad()
    loss = torch.zeros(1, device=DEV)
    _, cx = de.forward(clean.to(DEV), noisy.to(DEV), shifts, training=True)
    de.backward(cx, 1.0, 1.0, param_grads=True, loss_out=C.c_void_p(loss.data_ptr()))
    gD = {k: de.grad_of(k).cpu() for k, _ in s.D.named_parameters()}
    pD = {k: sdD[k].clone().requires_grad_(True) for k in O._trainable(sdD)}
    with O.oracle_mode():
        lo = O.discriminator_forward({**{k: v.clone() for k, v in sdD.items()}, **pD}, torch.cat((clean, noisy), 1), shifts)
        losso = torch.nn.functional.mse_loss(lo.view(-1), torch.ones(B))
        go = dict(zip(pD.keys(), torch.autograd.grad(losso, list(pD.values()))))
    zero_exact = lambda k: k.startswith("enc_blocks") and (k.endswith("conv.bias") or
                                                            (k.endswith("norm.bias") and not k.startswith("enc_blocks.4")))
    rep = {k: rel_err(gD[k], g) for k, g in go.items() if not zero_exact(k)}
    print("D single pass, slopes 1: loss %.5f vs %.5f, grads max %.3e (%s) median %.3e"
          % (float(loss), float(losso), max(rep.values()), max(rep, key=rep.get), float(np.median(list(rep.values())))))
    assert abs(float(loss) - float(losso)) <= 3e-3 * max(1.0, float(losso))
    assert max(rep.values()) <= GRAD_TOL_SMOOTH, sorted(rep.items(), key=lambda kv: -kv[1])[:5]


def test_generator_gradients_with_identical_discriminator():
    """G gradients of  MSE(D(G(x)), 1) + 100 L1  with the SAME D on both sides (no optimiser step in between), with
    the reference's slopes (vs the control) and with continuous activations (vs GRAD_TOL_SMOOTH)."""
    B = 8
    for slope in (None, 1.0):
        s = build_segan(batch_size=B)
        if slope is not None:
            _set_slopes(s, slope)
        sdG, sdD = cpu_state(s.G), cpu_state(s.D)
        s = s.to(DEV)
        s.G.train()
        s.D.train()
        clean, noisy, z = _pairs(B, 114)
        shifts = [2, -3, 1, -5, 4]
        y = s.G(noisy.to(DEV), z=z.to(DEV))
        logit, _ = s.D(torch.cat((y, noisy.to(DEV)), 1), shifts=shifts)
        loss = torch.nn.functional.mse_loss(logit.view(-1), torch.ones(B, device=DEV)) + \
            100 * torch.nn.functional.l1_loss(y, clean.to(DEV))
        loss.backward()
        gG = {n: p.grad.detach().cpu() for n, p in s.G.named_parameters()}

        def oracle_grads():
            pG = {k: sdG[k].clone().requires_grad_(True) for k in O._trainable(sdG)}
            yo = O.generator_forward({**sdG, **pG}, noisy, z)
            lo = O.discriminator_forward({k: v.clone() for k, v in sdD.items()}, torch.cat((yo, noisy), 1), shifts, training=True)
            losso = torch.nn.functional.mse_loss(lo.view(-1), torch.ones(B)) + 100 * torch.nn.functional.l1_loss(yo, clean)
            return float(losso), dict(zip(pG.keys(), torch.autograd.grad(losso, list(pG.values()))))
        with O.oracle_mode():
            losso, go = oracle_grads()
            with O.operand_precision(torch.float16):
                lossc, gc = oracle_grads()
        rep = {k: rel_err(gG[k], ref) for k, ref in go.items()}
        ctl = {k: rel_err(gc[k], ref) for k, ref in go.items()}
        print("G grads, identical D, slopes %s: max %.3e (%s) median %.3e | control max %.3e median %.3e; loss %.5f vs %.5f"
              % ("reference" if slope is None else slope, max(rep.values()), max(rep, key=rep.get),
                 float(np.median(list(rep.values()))), max(ctl.values()), float(np.median(list(ctl.values()))),
                 float(loss), losso))
        assert abs(float(loss) - losso) <= max(LOSS_RTOL, 3 * abs(lossc - losso) / max(1.0, abs(losso))) * max(1.0, abs(losso))
        if slope is None:
            assert max(rep.values()) <= GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS
        else:
            # even with continuous activations the 100 x L1 term keeps a discontinuity: sign(G(x) - clean) flips wherever
            # |G(x) - clean| is below the fp16 operand error of G(x) (~4e-4 of the samples, a few % of the gradient's L2
            # norm).  The control flips the same way: the gate is the smooth tolerance or the control's own error
            assert max(rep.values()) <= max(GRAD_TOL_SMOOTH, GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS), \
                sorted(rep.items(), key=lambda kv: -kv[1])[:5]


def test_no_bias_generator_step():
    """--no_bias (the reference's canonical SEGAN+ run, run_segan+_train.sh:7): encoder convs without bias."""
    B = 4
    s = build_segan(batch_size=B, bias=False)
    assert "enc_blocks.0.conv.bias" not in s.G.state_dict() and "dec_blocks.0.deconv.bias" in s.G.state_dict()
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    clean, noisy, z = _pairs(B, 115)
    s.G.eval()
    with torch.no_grad():
        y = s.G(noisy.to(DEV), z=z.to(DEV)).cpu()
    with O.oracle_mode(), torch.no_grad():
        ref = O.generator_forward(sdG, noisy, z)
    assert max_abs(y, ref) <= WAVE_TOL
    losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 115, load_opts(batch_size=B, bias=False), "no_bias")
    _loss_gate(lerr, cl, (0, 1, 3))
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS


def test_wsegan_adam_step_vs_oracle():
    """WSEGAN --misalign_pair with Adam(betas 0, 0.9) -- the optimiser of run_wsegan_train.sh -- one step:
    losses, D gradients (vs the control) and the post-step parameters against the oracle."""
    from segan_pytorch_b200.segan.models import WSEGAN
    B = 4
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, opt="adam")
    s = WSEGAN(opts)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    clean, noisy, z = _pairs(B, 116)
    random.seed(5)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    perm = [2, 0, 3, 1]
    Gopt, Dopt = s.build_optimizers(opts)
    assert Gopt.kind == "adam" and Gopt.betas == (0, 0.9)
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=["a"] * B, z=z.to(DEV),
                          shifts=shifts, perm=perm).tolist()
    gD = {k: s.D.engine.grad_of(k).cpu() for k, _ in s.D.named_parameters()}
    sdD0 = {k: v.clone() for k, v in sdD.items()}
    clone = lambda sd: {k: v.clone() for k, v in sd.items()}
    with O.operand_precision(torch.float16):
        ctl = O.wsegan_train_step(clone(sdG), clone(sdD), {}, {}, clean, noisy, z, shifts, perm, pow_weight=0.001,
                                  l1_weight=100.0, opt="adam")
    ref = O.wsegan_train_step(sdG, sdD, {}, {}, clean, noisy, z, shifts, perm, pow_weight=0.001, l1_weight=100.0,
                              opt="adam")
    for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
        assert abs(got - ref[k]) <= 1e-2 * max(1.0, abs(ref[k])), (k, got, ref[k])
    skip = lambda k: k.startswith("enc_blocks") and k.endswith("conv.bias")
    eD = {k: rel_err(gD[k], g) for k, g in ref["gradsD"].items() if not skip(k)}
    cD = {k: rel_err(ctl["gradsD"][k], g) for k, g in ref["gradsD"].items() if not skip(k)}
    print("wsegan/adam losses", losses, "D grads max rel-L2 %.3e | control %.3e" % (max(eD.values()), max(cD.values())))
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS
    # Adam's first step is lr * sign(g): the D update is +-lr wherever the gradient sign agrees
    post = s.D.state_dict()
    for k in ("enc_blocks.2.conv.weight", "fc.0.weight", "fc.2.weight"):
        d_got = (post[k].cpu() - sdD0[k]).reshape(-1)
        d_ref = (sdD[k] - sdD0[k]).reshape(-1)
        agree = float((torch.sign(d_got) == torch.sign(d_ref)).float().mean())
        assert float(d_got.abs().max()) <= 5.01e-5 and agree >= 0.95, (k, agree)


def test_wsegan_generate_vs_reference():
    """WSEGAN.generate (model.py:755-766, make_divN utils.py:26-38) against the unmodified reference's output on a
    20000-sample utterance (padded to 20480) and on a 4096-sample one (padded by a whole extra block)."""
    from segan_pytorch_b200.segan.models import WSEGAN
    g = golden("wsegan_generate.npz")
    seed_all(111)
    s = WSEGAN(load_opts(wsegan=True, misalign_pair=True))
    assert sd_sha(s.G.state_dict()) == str(g["sha_G"])
    s = s.to(DEV)
    out, hall = s.generate(torch.from_numpy(g["wav"]), z=torch.from_numpy(g["z"]).to(DEV))
    assert out.shape == g["out"].shape == (20000,)
    assert tuple(hall["enc_zc"].shape) == tuple(g["enc_zc_shape"])
    # de-emphasis integrates the waveform error (gain up to 1/(1-0.95) = 20)
    e1 = max_abs(out, g["out"])
    out2, _ = s.generate(torch.from_numpy(g["wav2"]), z=torch.from_numpy(g["z2"]).to(DEV))
    e2 = max_abs(out2, g["out2"])
    print("WSEGAN.generate max-abs (after de-emphasis): %.3e / %.3e" % (e1, e2))
    assert out2.shape == (4096,)
    assert e1 <= 20 * WAVE_TOL and e2 <= 20 * WAVE_TOL


def test_snorm_discriminator_vs_oracle():
    """norm_type='snorm' (run_wsegan_train.sh:8): D forward in train mode (two passes: the power iteration keeps
    moving u / v), eval mode, and the D-step gradients through W / sigma against the oracle (which is pinned against
    the reference's spectrally normalised Discriminator on the CPU, tests/test_oracle_pinned.py)."""
    from segan_pytorch_b200.segan.models import Discriminator
    B = 6
    seed_all(111)
    D = Discriminator(2, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], pool_type='none', pool_slen=16,
                      norm_type='snorm', phase_shift=5)
    sd = {k: v.detach().clone() for k, v in D.state_dict().items()}
    D = D.to(DEV)
    clean, noisy, _ = _pairs(B, 120)
    x = torch.cat((clean, noisy), 1)
    random.seed(9)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    D.train()
    for i in range(2):
        with torch.no_grad():
            y, _ = D(x.to(DEV), shifts=shifts[i])
        with O.oracle_mode(), torch.no_grad():
            ref = O.discriminator_forward(sd, x, shifts[i], training=True)
            with O.operand_precision(torch.float16):
                ctl = O.discriminator_forward({k: v.clone() for k, v in sd.items()}, x, shifts[i], training=True)
        e, c = max_abs(y.cpu(), ref), max_abs(ctl, ref)
        print("snorm D fwd pass %d: logits max-abs %.3e (control %.3e), |logit| %.3f" % (i, e, c, float(ref.abs().mean())))
        assert e <= max(LOGIT_TOL, 3 * c)
    got = D.state_dict()
    for k in ("enc_blocks.2.conv.weight_u", "enc_blocks.4.conv.weight_v", "fc.0.weight_v", "fc.3.weight_u", "enc_blocks.0.conv.weight_v"):
        assert max_abs(got[k].cpu(), sd[k]) <= 2e-4, (k, max_abs(got[k].cpu(), sd[k]))
    D.eval()
    with torch.no_grad():
        ye, _ = D(x.to(DEV), shifts=shifts[2])
    with O.oracle_mode(), torch.no_grad():
        re_ = O.discriminator_forward(sd, x, shifts[2], training=False)
    assert max_abs(ye.cpu(), re_) <= max(LOGIT_TOL, 3 * c)
    # gradients of a two-pass LSGAN D loss (real target 1, "fake" target 0 on swapped inputs): two power-iteration
    # states accumulate into one bucket
    D.train()
    de = D.engine
    de.zero_grad()
    losses = torch.zeros(2, device=DEV)
    import ctypes as C
    x2 = torch.cat((noisy, clean), 1)
    for i, (xx, tgt) in enumerate(((x, 1.0), (x2, 0.0))):
        _, cx = de.forward(xx[:, :1].to(DEV).contiguous(), xx[:, 1:].to(DEV).contiguous(), shifts[i], training=True)
        de.backward(cx, tgt, 1.0, param_grads=True, loss_out=C.c_void_p(losses.data_ptr() + 4 * i))
    gD = {k: de.grad_of(k).cpu() for k, _ in D.named_parameters()}
    pO = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd)}

    def oracle_loss(state):
        l1 = O.discriminator_forward(state, x, shifts[0], training=True)
        l2 = O.discriminator_forward(state, x2, shifts[1], training=True)
        return torch.nn.functional.mse_loss(l1.view(-1), torch.ones(B)) + torch.nn.functional.mse_loss(l2.view(-1), torch.zeros(B))
    with O.oracle_mode():
        lo = oracle_loss({**{k: v.clone() for k, v in sd.items()}, **pO})
        go = dict(zip(pO.keys(), torch.autograd.grad(lo, list(pO.values()))))
        pC = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd)}
        with O.operand_precision(torch.float16):
            lc = oracle_loss({**{k: v.clone() for k, v in sd.items()}, **pC})
        gc = dict(zip(pC.keys(), torch.autograd.grad(lc, list(pC.values()))))
    eD = {k: rel_err(gD[k], g) for k, g in go.items()}
    cD = {k: rel_err(gc[k], g) for k, g in go.items()}
    print("snorm D grads rel-L2: max %.3e (%s) median %.3e | control max %.3e; loss %.5f vs %.5f"
          % (max(eD.values()), max(eD, key=eD.get), float(np.median(list(eD.values()))), max(cD.values()),
             float(losses.sum()), float(lo)))
    assert abs(float(losses.sum()) - float(lo)) <= max(LOSS_RTOL, 3 * abs(float(lc) - float(lo))) * max(1.0, float(lo))
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS, sorted(eD.items(), key=lambda kv: -kv[1])[:5]


def test_wsegan_canonical_recipe_step():
    """run_wsegan_train.sh: --wsegan --gnorm_type snorm --dnorm_type snorm --opt adam --misalign_pair (gnorm_type is
    parsed but never reaches the Generator, SURVEY.md F5): one step against the oracle."""
    from segan_pytorch_b200.segan.models import WSEGAN
    B = 4
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, opt="adam", dnorm_type="snorm", gnorm_type="snorm")
    s = WSEGAN(opts)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    assert "enc_blocks.1.conv.weight_orig" in sdD and "enc_blocks.1.norm.weight" not in sdD
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    clean, noisy, z = _pairs(B, 121)
    random.seed(5)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    perm = [1, 3, 0, 2]
    Gopt, Dopt = s.build_optimizers(opts)
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=["a"] * B, z=z.to(DEV),
                          shifts=shifts, perm=perm).tolist()
    gD = {k: s.D.engine.grad_of(k).cpu() for k, _ in s.D.named_parameters()}
    clone = lambda sd: {k: v.clone() for k, v in sd.items()}
    with O.operand_precision(torch.float16):
        ctl = O.wsegan_train_step(clone(sdG), clone(sdD), {}, {}, clean, noisy, z, shifts, perm, pow_weight=0.001,
                                  l1_weight=100.0, opt="adam")
    sdD0 = clone(sdD)
    ref = O.wsegan_train_step(sdG, sdD, {}, {}, clean, noisy, z, shifts, perm, pow_weight=0.001, l1_weight=100.0,
                              opt="adam")
    for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
        tol = max(1e-2, 3 * abs(ctl[k] - ref[k]) / max(1.0, abs(ref[k])))
        assert abs(got - ref[k]) <= tol * max(1.0, abs(ref[k])), (k, got, ref[k], ctl[k])
    eD = {k: rel_err(gD[k], g) for k, g in ref["gradsD"].items()}
    cD = {k: rel_err(ctl["gradsD"][k], g) for k, g in ref["gradsD"].items()}
    print("canonical WSEGAN: losses", losses, "D grads max %.3e | control %.3e" % (max(eD.values()), max(cD.values())))
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS
    post = s.D.state_dict()
    for k in ("enc_blocks.3.conv.weight_orig", "fc.0.weight_orig", "enc_blocks.0.conv.weight_orig"):
        d_got = (post[k].cpu() - sdD0[k]).reshape(-1)
        d_ref = (sdD[k] - sdD0[k]).reshape(-1)
        agree = float((torch.sign(d_got) == torch.sign(d_ref)).float().mean())
        assert float(d_got.abs().max()) <= 5.01e-5 and agree >= 0.95, (k, agree)
    for k in ("enc_blocks.3.conv.weight_u", "fc.0.weight_v"):
        assert max_abs(post[k].cpu(), sdD[k]) <= 5e-4, k


def test_sum_merge_generator_vs_oracle():
    """skip_merge='sum' (generator.py:72-74): forward and parameter gradients of 100 * L1 against the oracle.  The
    engine runs it as the concat GEMM with tied weight halves; alphas are randomised so that they matter."""
    B = 4
    s = build_segan(batch_size=B, skip_merge="sum")
    g = torch.Generator().manual_seed(8)
    with torch.no_grad():
        for k, p in s.G.named_parameters():
            if k.endswith("skip_k"):
                p.copy_(0.5 + torch.rand(p.shape, generator=g))
            if k.endswith("act.weight"):
                p.fill_(1.0)                                  # continuous activations: see GRAD_TOL_SMOOTH
    sdG = cpu_state(s.G)
    assert sdG["dec_blocks.1.deconv.weight"].shape[0] == 512
    s = s.to(DEV)
    clean, noisy, z = _pairs(B, 122)
    s.G.train()
    y = s.G(noisy.to(DEV), z=z.to(DEV))
    loss = 100 * torch.nn.functional.l1_loss(y, clean.to(DEV))
    loss.backward()
    gG = {n: p.grad.detach().cpu() for n, p in s.G.named_parameters()}
    pG = {k: sdG[k].clone().requires_grad_(True) for k in O._trainable(sdG)}
    with O.oracle_mode():
        yo = O.generator_forward({**sdG, **pG}, noisy, z, skip_merge="sum")
        lo = 100 * torch.nn.functional.l1_loss(yo, clean)
        go = dict(zip(pG.keys(), torch.autograd.grad(lo, list(pG.values()))))
    assert max_abs(y.detach().cpu(), yo.detach()) <= WAVE_TOL
    rep = {k: rel_err(gG[k], v) for k, v in go.items()}
    print("sum-merge G: fwd max-abs %.2e, grads max %.3e (%s) median %.3e"
          % (max_abs(y.detach().cpu(), yo.detach()), max(rep.values()), max(rep, key=rep.get),
             float(np.median(list(rep.values())))))
    assert max(rep.values()) <= 2 * GRAD_TOL_SMOOTH, sorted(rep.items(), key=lambda kv: -kv[1])[:5]
    # the tied halves stay tied through an optimiser step and the exported weight is their common value
    eng = s.G.engine
    lay = eng.by_name["dec_blocks.2.deconv.weight"]
    Gopt, _ = s.build_optimizers(load_opts(batch_size=B, skip_merge="sum"))
    Gopt.step()
    m = eng.mview(lay).view(lay.T, lay.nc, 2, lay.kc // 2)
    assert torch.equal(m[:, :, 0], m[:, :, 1])
    w_new = s.G.state_dict()["dec_blocks.2.deconv.weight"].cpu()
    assert w_new.shape == sdG["dec_blocks.2.deconv.weight"].shape and float((w_new - sdG["dec_blocks.2.deconv.weight"]).abs().max()) > 0
