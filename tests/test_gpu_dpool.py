"""Discriminators with a pooled head (pool_type 'conv' / 'gmax' / 'gavg' / 'mlp') on the H100: the head kernels against fp32
torch, the Discriminator against the head-aware oracle (tests/dpool_oracle.py), SEGAN and WSEGAN steps, graph
replay, checkpoints and the command-line entry points.
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
from tests import dpool_oracle as DO                                         # noqa: E402
from tests.test_dpool import GOLD, HEADS, NORMS, pooled_discriminator        # noqa: E402
from tests.test_gpu_kernels import grad_dtype                                # noqa: E402,F401
from tests.test_gpu_parity_scale import (GRAD_ABS, GRAD_TOL_SMOOTH, GRAD_VS_CONTROL, LOGIT_TOL, _loss_gate,  # noqa: E402
                                         _pairs, _step_vs_oracle)
from tests.util import build_segan, cpu_state, golden, load_opts, max_abs, rel_err, seed_all  # noqa: E402

DEV = "cuda"
SEGAN_HEADS = ("conv", "gmax", "gavg")        # SEGAN cannot train mlp's per-position logits (the reference fails too)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _clone(sd):
    return {k: v.clone() for k, v in sd.items()}


# ---- kernel level ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("param_grads", [True, False])
@pytest.mark.parametrize("B", [1, 3, 300])
@pytest.mark.parametrize("head", HEADS)
def test_head_kernels_vs_torch(head, B, param_grads, grad_dtype):
    """sg_dhead_fwd / _bwd against fp32 torch autograd on the same fp16 activations.  param_grads: the fused MSE
    loss with parameter gradients (added to what the buffers hold); otherwise a given d loss / d logit and NULL
    parameter gradients (the G step, --vanilla_gan).  gmax: all-zero channels and channels whose maximum sits at two
    positions -- the gradient goes to the first.  mlp: mlp.2's per-position logits, loss over all B * Lq."""
    Lq, C_ = 16, 1024
    mlp = head == "mlp"
    conv, gmax = head in ("conv", "mlp"), head == "gmax"
    g = torch.Generator().manual_seed(17 * B + len(head) + (1000 if param_grads else 0))
    h = torch.randn(B, Lq, C_, generator=g).half()
    if gmax:
        h[:, :, :64] = 0
        top = (h[:, :, 64:128].float().abs().amax(dim=1) + 1.0).half()
        h[:, 3, 64:128] = top
        h[:, 9, 64:128] = top
    pw, pb = 0.05 * torch.randn(C_, generator=g), 0.1 * torch.randn(1, generator=g)
    fw, fb = 0.2 * torch.randn(Lq if conv else C_, generator=g), 0.1 * torch.randn(1, generator=g)
    kind = E.DHEAD_KINDS[head]
    hd = h.to(DEV)
    dpw, dpb, dfw, dfb = (t.to(DEV) for t in (pw, pb, fw, fb))
    pooled = None if mlp else torch.empty(B, Lq if conv else C_, device=DEV)
    argmax = torch.empty(B, C_, dtype=torch.int32, device=DEV) if gmax else None
    logit = torch.empty(B * Lq if mlp else B, device=DEV)
    _lib.call("sg_dhead_fwd", kind, _p(hd), B, Lq, C_, _p(dpw) if conv else None, _p(dpb) if conv else None,
              None if mlp else _p(dfw), None if mlp else _p(dfb), _p(pooled), _p(argmax), _p(logit), _st())
    # fp32 reference
    hr = h.float().permute(0, 2, 1).contiguous().requires_grad_(True)         # (B, C, Lq)
    pr = [t.clone().requires_grad_(True) for t in (pw, pb, fw, fb)]
    if conv:
        pool_ref = F.conv1d(hr, pr[0].view(1, C_, 1), pr[1]).view(B, Lq)
        idx_ref = None
    elif gmax:
        pool_ref, idx_ref = F.adaptive_max_pool1d(hr, 1, return_indices=True)
        pool_ref, idx_ref = pool_ref.view(B, C_), idx_ref.view(B, C_)
    else:
        pool_ref, idx_ref = F.adaptive_avg_pool1d(hr, 1).view(B, C_), None
    y = pool_ref.reshape(-1) if mlp else F.linear(pool_ref, pr[2].view(1, -1), pr[3]).view(-1)
    target, weight, LS = 1.0, 0.7, E.LOSS_SCALE
    if param_grads:
        loss_ref, g_in = weight * F.mse_loss(y, torch.full_like(y, target)), None
    else:
        g_in = torch.randn(y.numel(), generator=g)
        loss_ref = (y * g_in).sum()
    grads = torch.autograd.grad(loss_ref, [hr] + pr, allow_unused=True)       # gmax / gavg have no pool_conv
    g_h = torch.full((B, Lq, C_), float("nan"), dtype=E.GT, device=DEV)        # every element must be written
    pg = [torch.full_like(t, 0.5, device=DEV) for t in (pw, pb, fw, fb)] if param_grads else [None] * 4
    if not conv:
        pg[0] = pg[1] = None
    if mlp:
        pg[2] = pg[3] = None
    loss_out = torch.zeros(1, device=DEV)
    g_in_d = g_in.to(DEV) if g_in is not None else None
    _lib.call("sg_dhead_bwd", kind, _p(hd), B, Lq, C_, _p(dpw) if conv else None, None if mlp else _p(dfw),
              _p(pooled), _p(argmax),
              _p(logit), _p(g_in_d), target, weight,
              _p(loss_out) if param_grads else None, _p(g_h), *[_p(t) for t in pg], float(LS), _st())
    torch.cuda.synchronize()
    e_y = max_abs(logit.cpu(), y.detach()) / max(1.0, float(y.abs().max()))
    e_p = 0.0 if mlp else max_abs(pooled.cpu(), pool_ref.detach()) / max(1.0, float(pool_ref.abs().max()))
    gh_ref = grads[0].permute(0, 2, 1)
    assert not torch.isnan(g_h).any()
    e_h = max_abs(g_h.float().cpu() / LS, gh_ref) / float(gh_ref.abs().max())
    print("%s B=%d %s param_grads=%s: logit %.2e pooled %.2e g_h %.2e" % (head, B, E.GT, param_grads, e_y, e_p, e_h))
    assert e_y <= 1e-5 and e_p <= 1e-5
    assert e_h <= (2e-3 if E.GT == torch.float16 else 1e-2)
    if gmax:
        got_idx = argmax.cpu().long()
        assert torch.equal(got_idx, idx_ref)
        assert (got_idx[:, :64] == 0).all() and (got_idx[:, 64:128] == 3).all()
        off = torch.ones(B, Lq, C_, dtype=torch.bool)
        off.scatter_(1, got_idx.unsqueeze(1), False)
        assert (g_h.cpu()[off] == 0).all()                                  # exact zeros off the argmax
    if param_grads:
        assert abs(float(loss_out) - float(loss_ref)) <= 1e-5 * max(1.0, float(loss_ref))
        for got, ref, nm in zip(pg, grads[1:], ("pool_w", "pool_b", "fc_w", "fc_b")):
            if got is not None and ref is not None:
                assert rel_err((got.cpu() - 0.5) / LS, ref) <= 1e-4, nm
    # one more input: a given d loss / d logit with a NaN row and a row whose loss-scaled gradient is far past fp16's
    # range -- g_h must hold NaN there and +-65504 (fp16; bf16: the value), never inf or a NaN clipped to a number
    gx = torch.randn(B, y.numel() // B, generator=g)
    gx[0] = float("nan")
    if B > 1:
        gx[1] = 1e6
    hx = h.float().permute(0, 2, 1).contiguous().requires_grad_(True)
    if conv:
        px = F.conv1d(hx, pw.view(1, C_, 1), pb).view(B, Lq)
    else:
        px = (F.adaptive_max_pool1d if gmax else F.adaptive_avg_pool1d)(hx, 1).view(B, C_)
    yx = px.reshape(-1) if mlp else F.linear(px, fw.view(1, -1), fb).view(-1)
    ghx, = torch.autograd.grad((yx * gx.view(-1)).sum(), [hx])
    g_hx = torch.zeros(B, Lq, C_, dtype=E.GT, device=DEV)
    _lib.call("sg_dhead_bwd", kind, _p(hd), B, Lq, C_, _p(dpw) if conv else None, None if mlp else _p(dfw),
              _p(pooled), _p(argmax), _p(logit), _p(gx.view(-1).to(DEV)), target, weight, None, _p(g_hx),
              None, None, None, None, float(LS), _st())
    torch.cuda.synchronize()
    exp = ghx.permute(0, 2, 1) * LS
    if E.GT == torch.float16:
        exp = exp.clamp(-65504.0, 65504.0)
    got = g_hx.float().cpu()
    fin = ~torch.isnan(exp)
    assert torch.equal(torch.isnan(got), ~fin) and not torch.isinf(got).any()
    assert bool(((got[fin] - exp[fin]).abs() <= 8e-3 * exp[fin].abs() + 1e-4).all())


def test_head_entry_points_reject_bad_arguments():
    t = torch.zeros(4 * 16 * 1024, device=DEV)
    for kind, lq, c in ((0, 16, 1024), (5, 16, 1024), (1, 16, 96), (1, 0, 1024)):
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_dhead_fwd", kind, _p(t), 2, lq, c, _p(t), _p(t), _p(t), _p(t), _p(t), _p(t), _p(t), _st())
    with pytest.raises(_lib.SeganB200Error):          # gmax without an argmax buffer
        _lib.call("sg_dhead_fwd", E.DHEAD_KINDS["gmax"], _p(t), 2, 16, 1024, None, None, _p(t), _p(t), _p(t), None,
                  _p(t), _st())


# ---- Discriminator --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("head", HEADS)
def test_discriminator_forward_batch300_vs_oracle(head, norm):
    """Batch 300: a train-mode pass, then an eval-mode pass (running statistics / power-iteration vectors as the
    train pass left them) -- logits and avg_conv_h against the oracle, gated like test_discriminator_forward_batch300:
    LOGIT_TOL, or 3x the operand-precision control's own distance."""
    B = 300
    D = pooled_discriminator(head, norm)
    sd = cpu_state(D)
    D = D.to(DEV)
    clean, noisy, _ = _pairs(B, 131)
    x = torch.cat((clean, noisy), 1)
    sd_ref, sd_ctl = _clone(sd), _clone(sd)
    for mode, seed in (("train", 5), ("eval", 6)):
        training = mode == "train"
        D.train(training)
        random.seed(seed)
        shifts = O.draw_phase_shifts(5, 5)
        with torch.no_grad():
            y, act = D(x.to(DEV), shifts=shifts)
            got_a = act["avg_conv_h"].cpu() if head == "conv" else None
        with O.oracle_mode(), torch.no_grad():
            ref, ra = DO.discriminator_forward(sd_ref, x, shifts, training=training, ret_act=True, pool_type=head)
            with O.operand_precision(torch.float16):
                ctl, ca = DO.discriminator_forward(sd_ctl, x, shifts, training=training, ret_act=True, pool_type=head)
        assert tuple(y.shape) == ((B, 1, 16) if head == "mlp" else (B, 1))
        e, c = max_abs(y.cpu(), ref), max_abs(ctl, ref)
        print("%s/%s D fwd B=300 %s: logits max-abs %.3e (control %.3e), |logit| %.3f"
              % (head, norm, mode, e, c, float(ref.abs().mean())))
        assert e <= max(LOGIT_TOL, 3 * c)
        if head == "conv":
            ea, cc = max_abs(got_a, ra["avg_conv_h"]), max_abs(ca["avg_conv_h"], ra["avg_conv_h"])
            print("   avg_conv_h max-abs %.3e (control %.3e)" % (ea, cc))
            assert tuple(got_a.shape) == (B, 16) and ea <= max(LOGIT_TOL, 3 * cc)


@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("head", HEADS)
def test_single_pass_gradients_continuous_activation(head, norm):
    """One D pass (LSGAN loss against target 1) with every tower PReLU slope at 1: every parameter tensor within
    GRAD_TOL_SMOOTH of the oracle.  gmax keeps one discontinuity -- its argmax flips where the fp16 activations
    reorder a near tie -- and mlp another, its own PReLU(C) (init 0.25): the operand-precision control shows those
    flips as well, and for these two heads the gate also admits its error."""
    B = 8
    D = pooled_discriminator(head, norm)
    with torch.no_grad():
        for n, p in D.named_parameters():
            if n.endswith("act.weight"):
                p.fill_(1.0)
    sd = cpu_state(D)
    D = D.to(DEV).train()
    clean, noisy, _ = _pairs(B, 132)
    shifts = [3, -1, 4, -2, 5]
    de = D.engine
    de.bind()
    de.zero_grad()
    loss = torch.zeros(1, device=DEV)
    _, cx = de.forward(clean.to(DEV), noisy.to(DEV), shifts, training=True)
    de.backward(cx, 1.0, 1.0, param_grads=True, loss_out=C.c_void_p(loss.data_ptr()))
    gD = {k: de.grad_of(k).cpu() for k, _ in D.named_parameters()}
    x = torch.cat((clean, noisy), 1)

    def oracle():
        pD = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd)}
        lo = DO.discriminator_forward({**_clone(sd), **pD}, x, shifts, pool_type=head)
        lo = F.mse_loss(lo, torch.ones_like(lo))
        return float(lo), dict(zip(pD.keys(), torch.autograd.grad(lo, list(pD.values()))))
    with O.oracle_mode():
        losso, go = oracle()
        with O.operand_precision(torch.float16):
            _, gc = oracle()
    zero_exact = lambda k: norm == "bnorm" and k.startswith("enc_blocks") and (
        k.endswith("conv.bias") or (k.endswith("norm.bias") and not k.startswith("enc_blocks.4")))
    rep = {k: rel_err(gD[k], g) for k, g in go.items() if not zero_exact(k)}
    ctl = {k: rel_err(gc[k], g) for k, g in go.items() if not zero_exact(k)}
    print("%s/%s single pass, slopes 1: loss %.5f vs %.5f, grads max %.3e (%s) median %.3e | control max %.3e"
          % (head, norm, float(loss), losso, max(rep.values()), max(rep, key=rep.get),
             float(np.median(list(rep.values()))), max(ctl.values())))
    assert abs(float(loss) - losso) <= 3e-3 * max(1.0, losso)
    gate = GRAD_TOL_SMOOTH if head not in ("gmax", "mlp") else \
        max(GRAD_TOL_SMOOTH, GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS)
    assert max(rep.values()) <= gate, sorted(rep.items(), key=lambda kv: -kv[1])[:5]


# ---- train steps ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head", SEGAN_HEADS)
def test_train_step_batch16_vs_oracle(head):
    B = 16
    s = build_segan(batch_size=B, dpool_type=head)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    with DO.pooled_heads(head):
        losses, refl, lerr, eD, eG, cD, cG, cl = _step_vs_oracle(s, sdG, sdD, B, 133,
                                                                 load_opts(batch_size=B, dpool_type=head), head)
    print("   %s head D grads:" % head, {k: "%.2e/%.2e" % (v, cD[k]) for k, v in eD.items()
                                          if not k.startswith("enc_blocks")})
    _loss_gate(lerr, cl, (0, 1, 3))
    # g_adv goes through the D that RMSprop's first, sign-like step produced (compared loosely, as for 'none'); with
    # gmax every weight whose near-zero gradient took the other sign can also move a channel's argmax
    assert lerr[2] <= max(2e-2 if head == "gmax" else 1e-2, 3 * cl[2]), (losses, refl)
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS
    assert float(np.median(list(eD.values()))) <= GRAD_VS_CONTROL * float(np.median(list(cD.values()))) + GRAD_ABS
    assert max(eG.values()) <= GRAD_VS_CONTROL * max(cG.values()) + GRAD_ABS


@pytest.mark.parametrize("head", HEADS)
def test_wsegan_canonical_recipe_step(head):
    """run_wsegan_train.sh's recipe (--dnorm_type snorm --opt adam --misalign_pair) with a pooled head: one step
    against the oracle -- losses, every D gradient (vs the control) and the power-iteration vectors after the step.
    mlp: its B * Lq logits per pass are averaged by the LSGAN losses (model.py:581,590 size the targets like them)."""
    from segan_pytorch_b200.segan.models import WSEGAN
    B = 4
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, opt="adam", dnorm_type="snorm",
                     gnorm_type="snorm", dpool_type=head)
    s = WSEGAN(opts)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    assert ("mlp.0.weight_orig" if head == "mlp" else "fc.weight_orig") in sdD
    assert ("pool_conv.weight_orig" in sdD) == (head == "conv")
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    clean, noisy, z = _pairs(B, 134)
    random.seed(5)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    perm = [1, 3, 0, 2]
    Gopt, Dopt = s.build_optimizers(opts)
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=["a"] * B, z=z.to(DEV),
                          shifts=shifts, perm=perm).tolist()
    gD = {k: s.D.engine.grad_of(k).cpu() for k, _ in s.D.named_parameters()}
    with DO.pooled_heads(head):
        with O.operand_precision(torch.float16):
            ctl = O.wsegan_train_step(_clone(sdG), _clone(sdD), {}, {}, clean, noisy, z, shifts, perm,
                                      pow_weight=0.001, l1_weight=100.0, opt="adam")
        ref = O.wsegan_train_step(sdG, sdD, {}, {}, clean, noisy, z, shifts, perm, pow_weight=0.001, l1_weight=100.0,
                                  opt="adam")
    for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
        tol = max(1e-2, 3 * abs(ctl[k] - ref[k]) / max(1.0, abs(ref[k])))
        assert abs(got - ref[k]) <= tol * max(1.0, abs(ref[k])), (k, got, ref[k], ctl[k])
    eD = {k: rel_err(gD[k], g) for k, g in ref["gradsD"].items()}
    cD = {k: rel_err(ctl["gradsD"][k], g) for k, g in ref["gradsD"].items()}
    print("%s canonical WSEGAN: losses" % head, losses, "D grads max %.3e (%s) | control %.3e"
          % (max(eD.values()), max(eD, key=eD.get), max(cD.values())))
    assert max(eD.values()) <= GRAD_VS_CONTROL * max(cD.values()) + GRAD_ABS
    # the vectors of the pass after Adam's first (sign-like: +-lr) step, which near-zero gradients take either way
    post = s.D.state_dict()
    uv = ("mlp.0.weight_u", "mlp.1.weight_v") if head == "mlp" else ("fc.weight_u", "fc.weight_v")
    for k in ("enc_blocks.3.conv.weight_u",) + uv:
        assert max_abs(post[k].cpu(), sdD[k]) <= 1e-3, k


@pytest.mark.parametrize("head", SEGAN_HEADS)
def test_graph_replayed_steps_match_eager_steps(head):
    """Four SEGAN steps from the same state and inputs, graph-replayed vs eager, held to the noise floor of the eager
    schedule (two overlapped runs and the serial one, engine.OVERLAP off).  fp32 atomics (the weight-gradient GEMMs'
    red.add, the head's parameter gradients) add in whatever order the CTAs arrive; from a cold RMSprop state the
    first step is 10 lr sign(g), which turns last-bit differences of near-zero gradients into whole steps -- and
    whether two runs' atomics happen to arrive alike is luck (three eager runs can agree to 4e-7 and a fourth differ
    by 4e-2 one step later).  Every run therefore starts from a warm optimiser state (square_avg = 1: the step is
    ~lr g, linear in the gradient), and, as in the default head's test, a 100x smaller learning rate keeps the
    tower's slope-0 PReLU kinks from flipping under the updates; the trajectories then stay as close as their sums
    and a replay error shows."""
    B = 4
    opts = load_opts(batch_size=B, dpool_type=head, g_lr=5e-7, d_lr=5e-7)
    gen = torch.Generator().manual_seed(8)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1).to(DEV)
    noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1).to(DEV)
    zs = [torch.randn(B, 1024, 16, generator=gen).to(DEV) for _ in range(4)]
    random.seed(13)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(4)]

    def run(graphs, overlap=True):
        prev, prev_ov = E.GRAPHS, E.OVERLAP
        E.GRAPHS, E.OVERLAP = graphs, overlap
        try:
            s = build_segan(batch_size=B, dpool_type=head).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(opts)
            for opt in (Gopt, Dopt):
                opt._state()
                opt.s1.fill_(1.0)
            out = []
            for i in range(4):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=zs[i], shifts3=shifts[i])
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad.clone(), s.D.engine.grad.clone()))
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs
        finally:
            E.GRAPHS, E.OVERLAP = prev, prev_ov

    (e1, n1), (e2, n2), (es, ns), (gr, n3) = run(False), run(False), run(False, overlap=False), run(True)
    assert n1 == 0 and n2 == 0 and ns == 0 and n3 == 1
    floor_l = max(max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[i][0], o[i][0])) for i in range(4) for o in (e2, es))
    floor_g = max(max(rel_err(o[i][1], e1[i][1]), rel_err(o[i][2], e1[i][2])) for i in range(4) for o in (e2, es))
    for step in range(4):
        (l0, gG0, gD0), (l2, gG2, gD2) = e1[step], gr[step]
        err_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l2))
        err_g = max(rel_err(gG2, gG0), rel_err(gD2, gD0))
        print("%s step %d: eager-vs-eager loss %.2e grad %.2e | graph-vs-eager loss %.2e grad %.2e"
              % (head, step, floor_l, floor_g, err_l, err_g))
        assert err_l <= 10 * floor_l + 2e-3, (step, l0, l2)
        assert err_g <= 10 * floor_g + 5e-3, (step, err_g, floor_g)


# ---- checkpoints and entry points -----------------------------------------------------------------------------------
@pytest.mark.parametrize("head", SEGAN_HEADS)
def test_checkpoint_round_trip_keeps_reference_keys(head, tmp_path):
    g = golden(GOLD)
    B = 2
    s = build_segan(batch_size=B, dpool_type=head).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B, dpool_type=head))
    clean, noisy, z = [t.to(DEV) for t in _pairs(B, 135)]
    fc0 = s.D.state_dict()["fc.weight"].clone()
    s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=z)
    sd1 = s.D.state_dict()
    assert list(sd1.keys()) == [str(k) for k in g["%s.bnorm.keys" % head]]
    assert float((sd1["fc.weight"] - fc0).abs().max()) > 1e-6                 # the head was trained
    x = torch.cat((clean, noisy), 1)
    s.D.eval()
    with torch.no_grad():
        y1 = s.D(x, shifts=[1, -2, 3, -4, 5])[0].clone()
    s.D.save(str(tmp_path), 1)
    ck = [f for f in os.listdir(str(tmp_path)) if "Discriminator" in f and f.endswith(".ckpt")]
    assert len(ck) == 1, os.listdir(str(tmp_path))
    s2 = build_segan(seed=3, batch_size=B, dpool_type=head).to(DEV)
    s2.D.load_pretrained(os.path.join(str(tmp_path), ck[0]), True)
    s2.D.eval()
    with torch.no_grad():
        assert max_abs(s2.D(x, shifts=[1, -2, 3, -4, 5])[0], y1) == 0.0
    saved = torch.load(os.path.join(str(tmp_path), ck[0]), map_location="cpu")["state_dict"]
    assert list(saved.keys()) == [str(k) for k in g["%s.bnorm.keys" % head]]


def test_train_and_clean_cli(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    ck = str(tmp_path / "ckpt")
    subprocess.check_call([sys.executable, "train.py", "--save_path", ck, "--synthetic", "64", "--batch_size", "8",
                           "--epoch", "1", "--save_freq", "4", "--dpool_type", "conv", "--num_workers", "0"],
                          cwd=ROOT, env=env)
    ckw = str(tmp_path / "ckpt_w")
    subprocess.check_call([sys.executable, "train.py", "--save_path", ckw, "--synthetic", "32", "--batch_size", "4",
                           "--epoch", "1", "--save_freq", "4", "--wsegan", "--misalign_pair", "--opt", "adam",
                           "--dnorm_type", "snorm", "--dpool_type", "mlp", "--num_workers", "0"], cwd=ROOT, env=env)
    g = golden(GOLD)
    for d, key in ((ck, "conv.bnorm.keys"), (ckw, "mlp.snorm.keys")):
        dck = sorted(f for f in os.listdir(d) if "Discriminator" in f and f.endswith(".ckpt"))
        assert dck, os.listdir(d)
        sd = torch.load(os.path.join(d, dck[0]), map_location="cpu")["state_dict"]
        assert list(sd.keys()) == [str(k) for k in g[key]]
    from scipy.io import wavfile
    wdir = tmp_path / "wavs"
    wdir.mkdir()
    rng = np.random.RandomState(0)
    wavfile.write(str(wdir / "a.wav"), 16000, (rng.randn(40000) * 3000).astype(np.int16))
    gck = sorted(f for f in os.listdir(ck) if "G" in f and f.endswith(".ckpt"))[0]
    subprocess.check_call([sys.executable, "clean.py", "--g_pretrained_ckpt", os.path.join(ck, gck), "--cfg_file",
                           os.path.join(ck, "train.opts"), "--test_files", str(wdir), "--synthesis_path",
                           str(tmp_path / "clean")], cwd=ROOT, env=env)
    r, w = wavfile.read(str(tmp_path / "clean" / "a.wav"))
    assert r == 16000 and w.shape[0] == 40000 and np.isfinite(w).all()
