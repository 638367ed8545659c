"""CPU tests of tests/step_end_model.py: an fp32 evaluation of every kernel's formula (in two summation orders) passes
its fp64 gate with room to spare, and a planted defect of each kernel fails it by orders of magnitude, so the GPU
gates (tests/test_gpu_loss_end.py, tests/test_gpu_param_end.py) can tell a right kernel from a subtly wrong one.
Runs without a GPU."""
import math

import numpy as np
import pytest
import torch

from tests import step_end_model as M

C_PASS = 4.0                 # an fp32 evaluation's c: about 2, the long running sums up to ~3
C_FAIL = 100 * M.C_TOL       # a planted defect's c: orders of magnitude past the gate


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _sum32(t, dim, order):
    """fp32 sum along dim: 'fwd' = one running sum in index order, 'rev' = 16 interleaved running sums in reverse
    order added at the end (a strided warp's pattern)."""
    t = t.float().movedim(dim, -1)
    if order == "fwd":
        return t.cumsum(-1)[..., -1] if t.shape[-1] else t.sum(-1)
    t = t.flip(-1)
    n = t.shape[-1]
    pad = (-n) % 16
    t = torch.nn.functional.pad(t, (0, pad)).reshape(*t.shape[:-1], -1, 16)
    return t.cumsum(-2)[..., -1, :].sum(-1)


def _dot32(a, b, order):
    """fp32 a @ b^T (contraction over the last axis of both) with the products rounded, summed in `order`."""
    return _sum32((a.float()[..., :, None, :] * b.float()[None, :, :]), -1, order)


def _prelu32(z, s):
    return torch.where(z > 0, z, z.float() * s.float())


def _fails(c, what):
    print("planted defect %-48s c = %.3g" % (what, c))
    assert c > C_FAIL, (what, c)


ORDERS = ["fwd", "rev"]


# ------------------------------------------------------------------------------------------------------
# fc tail
# ------------------------------------------------------------------------------------------------------
def _fc_inputs(B, seed=1):
    g = _gen(seed)
    acc = torch.randn(B, 256, generator=g)
    acc[:, :8] = 0.0                                        # exact zeros: the z > 0 boundary (b0 = 0 there)
    b0 = 0.1 * torch.randn(256, generator=g)
    b0[:8] = 0.0
    s1 = torch.rand(256, generator=g)
    s1[:4], s1[4:8] = 0.0, 1.0
    w2 = 0.1 * torch.randn(128, 256, generator=g)
    b2 = 0.1 * torch.randn(128, generator=g)
    s3 = torch.rand(128, generator=g)
    s3[:2] = 0.0
    w4 = 0.1 * torch.randn(1, 128, generator=g)
    b4 = torch.tensor([0.02])
    return acc, b0, s1, w2, b2, s3, w4, b4


def _fc_fwd32(acc, b0, s1, w2, b2, s3, w4, b4, order, slope_bug=False):
    z1 = acc + b0
    sl = s1[:1].expand_as(s1) if slope_bug else s1
    h1 = _prelu32(z1, sl)
    z2 = _dot32(h1, w2, order) + b2
    h2 = _prelu32(z2, s3)
    logit = _dot32(h2, w4, order).reshape(-1) + b4
    return z1, z2, logit


@pytest.mark.parametrize("order", ORDERS)
def test_fc_tail_forward_fp32_passes(order):
    x = _fc_inputs(300)
    z1, z2, logit = _fc_fwd32(*x, order)
    acc, b0, s1, w2, b2, s3, w4, b4 = x
    c = [M.c_vec(z1, *M.fc_z1(acc, b0)), M.c_vec(z2, *M.fc_z2(z1, s1, w2, b2)), M.c_vec(logit, *M.fc_logit(z2, s3, w4, b4))]
    print("fc forward fp32 (%s): c z1 %.2f z2 %.2f logit %.2f" % (order, *c))
    assert all(v <= C_PASS for v in c)


def test_fc_tail_forward_defect_slope_index():
    acc, b0, s1, w2, b2, s3, w4, b4 = _fc_inputs(300)
    z1, z2, _ = _fc_fwd32(acc, b0, s1, w2, b2, s3, w4, b4, "fwd", slope_bug=True)
    _fails(M.c_vec(z2, *M.fc_z2(z1, s1, w2, b2)), "fc_tail_fwd: slope read as s1[0]")


def _fc_bwd32(z1, z2, logit, g_in, target, weight, s1, w2, s3, w4, B, gscale, order, bugs=()):
    """fp32 twin of fc_tail_bwd_rows_kernel + fc_tail_bwd_params_kernel (chunks of 16 rows)."""
    diff = logit - target
    gl = g_in * gscale if g_in is not None else 2.0 * diff / B * weight * gscale
    loss = _sum32(diff * diff / B * weight * (gscale if "loss_scaled" in bugs else 1.0), 0, order)
    gh2 = gl[:, None] * w4.reshape(1, -1)
    gz2 = torch.where(z2 > 0, gh2, gh2 * s3)
    gh1 = _dot32(gz2, w2.t().contiguous(), order)
    gz1 = torch.where(z1 > 0, gh1, gh1 * s1)
    rows = B - (B % 16 if "drop_tail" in bugs and B % 16 else 0)
    h1 = _prelu32(z1, s1)[:rows]
    h2 = _prelu32(z2, s3)[:rows]
    zs3 = h2 if "s3_from_h2" in bugs else z2[:rows]
    p = dict(w2=_dot32(gz2[:rows].t().contiguous(), h1.t().contiguous(), order), b0=_sum32(gz1[:rows], 0, order),
             s1=_sum32(torch.where(z1[:rows] <= 0, gh1[:rows] * z1[:rows], torch.zeros(())), 0, order),
             b2=_sum32(gz2[:rows], 0, order),
             s3=_sum32(torch.where(z2[:rows] <= 0, (gl[:rows, None] * w4.reshape(1, -1)) * zs3, torch.zeros(())), 0, order),
             w4=_sum32(gl[:rows, None] * h2, 0, order), b4=_sum32(gl[:rows], 0, order).reshape(1))
    return dict(gl=gl, loss=loss, gz2=gz2, gh1=gh1, gz1=gz1, params=p)


def _fc_bwd_case(B, g_in_path, seed=2):
    acc, b0, s1, w2, b2, s3, w4, b4 = _fc_inputs(B, seed)
    z1, z2, logit = _fc_fwd32(acc, b0, s1, w2, b2, s3, w4, b4, "fwd")
    g_in = torch.randn(B, generator=_gen(seed + 1)) if g_in_path else None
    return dict(z1=z1, z2=z2, logit=logit, g_in=g_in, s1=s1, w2=w2, s3=s3, w4=w4, B=B)


def _fc_bwd_c(k, out, target, weight, gscale, g0):
    B = k["B"]
    c = {}
    gl_ref = M.fc_g_logit(k["logit"], k["g_in"], target, weight, B, gscale)
    c["g_logit"] = M.c_vec(out["gl"], *gl_ref)
    c["loss"] = M.c_vec(out["loss"], *M.fc_loss(k["logit"], target, weight, B))
    c["g_z2"] = M.c_vec(out["gz2"], *M.fc_g_z2(k["z2"], out["gl"], k["s3"], k["w4"]))
    gh1, gz1 = M.fc_g_h1_z1(out["gz2"], k["z1"], k["s1"], k["w2"])
    c["g_h1"], c["g_z1"] = M.c_vec(out["gh1"], *gh1), M.c_vec(out["gz1"], *gz1)
    c["g_z1 f16"] = M.c_f(M.to16(out["gz1"], "f16"), *gz1, "f16")
    ref = M.fc_params(k["z1"], k["z2"], out["gl"], out["gz2"], out["gz1"], out["gh1"], k["s1"], k["s3"], k["w4"], g0)
    for name, (r, m) in ref.items():
        c["g_" + name] = M.c_vec(g0[name].reshape(r.shape) + out["params"][name].reshape(r.shape), r, m)
    return c


def _g0(seed=3):
    g = _gen(seed)
    return dict(b0=torch.randn(256, generator=g), s1=torch.randn(256, generator=g), w2=torch.randn(128, 256, generator=g),
                b2=torch.randn(128, generator=g), s3=torch.randn(128, generator=g), w4=torch.randn(128, generator=g),
                b4=torch.randn(1, generator=g))


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("B,g_in_path,target,gscale", [(300, False, 1.0, 1024.0), (17, True, 0.0, 1.0), (1, False, 0.0, 1.0)])
def test_fc_tail_backward_fp32_passes(B, g_in_path, target, gscale, order):
    k = _fc_bwd_case(B, g_in_path)
    g0 = _g0()
    out = _fc_bwd32(k["z1"], k["z2"], k["logit"], k["g_in"], target, 0.7, k["s1"], k["w2"], k["s3"], k["w4"], B,
                    gscale, order)
    c = _fc_bwd_c(k, out, target, 0.7, gscale, g0)
    print("fc backward fp32 B=%d (%s):" % (B, order), {n: round(v, 2) for n, v in c.items()})
    assert all(v <= C_PASS for v in c.values())


@pytest.mark.parametrize("bug,what", [("drop_tail", "fc_tail_bwd: last partial 16-row chunk dropped"),
                                      ("s3_from_h2", "fc_tail_bwd: g_s3 built from h2 instead of z2"),
                                      ("loss_scaled", "fc_tail_bwd: grad_scale applied to loss_out")])
def test_fc_tail_backward_defects(bug, what):
    B = 300
    k = _fc_bwd_case(B, False)
    # the random PReLU slopes (0 and 1 on a few channels) make h2 and z2 differ at z2 < 0, which every column has
    out = _fc_bwd32(k["z1"], k["z2"], k["logit"], None, 1.0, 0.7, k["s1"], k["w2"], k["s3"], k["w4"], B, 1024.0,
                    "fwd", bugs=(bug,))
    c = _fc_bwd_c(k, out, 1.0, 0.7, 1024.0, {n: torch.zeros_like(v) for n, v in _g0().items()})
    _fails(max(c.values()), what)


# ------------------------------------------------------------------------------------------------------
# regression losses
# ------------------------------------------------------------------------------------------------------
def _reg_inputs(n, seed=4):
    g = _gen(seed)
    y = torch.randn(n, generator=g)
    clean = torch.randn(n, generator=g)
    clean[::7] = y[::7]                                     # exact d = 0
    return y, clean


def _reg32(kind, y, clean, weight, gscale, gy0, order, bugs=()):
    n = y.numel()
    d = y - clean
    lscale = torch.tensor(weight, dtype=torch.float32) / n
    gs = lscale * gscale
    if kind == "l1":
        s = _sum32(d.abs(), 0, order)
        sg = torch.where(d >= 0, 1.0, -1.0) if "sign0" in bugs else torch.sign(d)
        g = sg * gs
    else:
        s = _sum32(d * d, 0, order)
        g = 2.0 * gs * d
    loss = s * lscale * (gscale if "loss_scaled" in bugs else 1.0)
    gy = g if (gy0 is None or "no_accumulate" in bugs) else gy0 + g
    return loss, gy


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("kind", ["l1", "mse"])
def test_reg_loss_fp32_passes(kind, order):
    y, clean = _reg_inputs(256 * 264 + 1)
    gy0 = torch.randn(y.numel(), generator=_gen(5))
    loss, gy = _reg32(kind, y, clean, 100.0, 1024.0, gy0, order)
    ref = M.reg_loss(kind, y, clean, 100.0, 1024.0, gy0)
    c = (M.c_vec(loss, *ref["loss"]), M.c_vec(gy, *ref["gy"]))
    print("%s fp32 (%s): c loss %.2f gy %.2f" % (kind, order, *c))
    assert all(v <= C_PASS for v in c)


@pytest.mark.parametrize("kind,bug,what", [("l1", "sign0", "l1_loss_bwd: sign(0) = +1"),
                                           ("mse", "no_accumulate", "mse_loss_bwd: accumulate ignored"),
                                           ("l1", "loss_scaled", "l1_loss_bwd: grad_scale applied to loss_out")])
def test_reg_loss_defects(kind, bug, what):
    y, clean = _reg_inputs(4099)
    gy0 = torch.randn(y.numel(), generator=_gen(5))
    loss, gy = _reg32(kind, y, clean, 100.0, 1024.0, gy0, "fwd", bugs=(bug,))
    ref = M.reg_loss(kind, y, clean, 100.0, 1024.0, gy0)
    _fails(max(M.c_vec(loss, *ref["loss"]), M.c_vec(gy, *ref["gy"])), what)


# ------------------------------------------------------------------------------------------------------
# optimisers
# ------------------------------------------------------------------------------------------------------
def _opt_inputs(n, seed=6):
    """Parameters with exact zeros (their new value is the update itself) and gradients spanning 1e-10 .. 1e2, so that
    eps and every factor of the update are visible."""
    g = _gen(seed)
    p = torch.randn(n, generator=g)
    p[::3] = 0.0
    mag = 10.0 ** (torch.rand(n, generator=g) * 12 - 10)
    gr = torch.sign(torch.randn(n, generator=g)) * mag
    return p, gr


def _rmsprop32(p, g, sq, lr, alpha, eps, gscale, bugs=()):
    gi = g * gscale
    if "scale_twice" in bugs:
        gi = gi * gscale
    s = alpha * sq + (1.0 - torch.tensor(alpha)) * gi * gi
    den = (s + eps).sqrt() if "eps_in_sqrt" in bugs else s.sqrt() + eps
    return p - lr * (gi / den), s


def _adam32(p, g, m, v, lr, b1, b2, eps, step, gscale, bugs=()):
    bc1 = np.float32(1.0) - np.float32(b1) ** np.float32(step)
    bc2 = np.float32(1.0) - np.float32(b2) ** np.float32(step)
    bc2s = float(np.sqrt(np.float32(bc2))) if "no_bc2" not in bugs else 1.0
    gi = g * gscale
    mi = b1 * m + (1.0 - torch.tensor(b1)) * gi
    vi = b2 * v + (1.0 - torch.tensor(b2)) * gi * gi
    return p - float(np.float32(lr) / bc1) * (mi / (vi.sqrt() / bc2s + eps)), mi, vi


@pytest.mark.parametrize("gscale", [1.0, 2.0 ** -10, 1.0 / (3 * 1024)])
def test_rmsprop_fp32_passes(gscale):
    p, g = _opt_inputs(10007)
    sq = torch.rand(p.numel(), generator=_gen(7)) * 1e-6
    sq[::5] = 0.0
    p1, s1 = _rmsprop32(p, g, sq, 5e-5, 0.99, 1e-8, gscale)
    ref = M.rmsprop_step(p, g, sq, 5e-5, 0.99, 1e-8, gscale)
    c = (M.c_vec(p1, *ref["p"]), M.c_vec(s1, *ref["sq"]))
    print("rmsprop fp32 grad_scale %.3g: c p %.2f sq %.2f" % (gscale, *c))
    assert all(v <= C_PASS for v in c)


@pytest.mark.parametrize("bug,what", [("eps_in_sqrt", "rmsprop_step: eps inside the sqrt"),
                                      ("scale_twice", "rmsprop_step: grad_scale applied twice")])
def test_rmsprop_defects(bug, what):
    p, g = _opt_inputs(10007)
    sq = torch.zeros(p.numel())
    p1, s1 = _rmsprop32(p, g, sq, 5e-5, 0.99, 1e-8, 2.0 ** -10, bugs=(bug,))
    ref = M.rmsprop_step(p, g, sq, 5e-5, 0.99, 1e-8, 2.0 ** -10)
    _fails(max(M.c_vec(p1, *ref["p"]), M.c_vec(s1, *ref["sq"])), what)


@pytest.mark.parametrize("betas,step", [((0.0, 0.9), 1), ((0.5, 0.999), 2), ((0.5, 0.999), 1000), ((0.0, 0.9), 3)])
def test_adam_fp32_passes(betas, step):
    p, g = _opt_inputs(10007)
    m = torch.randn(p.numel(), generator=_gen(8)) * 1e-3
    v = torch.rand(p.numel(), generator=_gen(9)) * 1e-6
    p1, m1, v1 = _adam32(p, g, m, v, 1e-4, *betas, 1e-8, step, 1.0 / (3 * 1024))
    ref = M.adam_step(p, g, m, v, 1e-4, *betas, 1e-8, step, 1.0 / (3 * 1024))
    c = (M.c_vec(p1, *ref["p"]), M.c_vec(m1, *ref["m"]), M.c_vec(v1, *ref["v"]))
    print("adam fp32 betas %s step %d: c p %.2f m %.2f v %.2f" % (betas, step, *c))
    assert all(v <= C_PASS for v in c)


def test_adam_defect_no_second_bias_correction():
    p, g = _opt_inputs(10007)
    z = torch.zeros(p.numel())
    p1, _, _ = _adam32(p, g, z, z, 1e-4, 0.5, 0.999, 1e-8, 2, 1.0, bugs=("no_bc2",))
    ref = M.adam_step(p, g, z, z, 1e-4, 0.5, 0.999, 1e-8, 2, 1.0)
    _fails(M.c_vec(p1, *ref["p"]), "adam_step: no second bias correction")


# ------------------------------------------------------------------------------------------------------
# packed masters
# ------------------------------------------------------------------------------------------------------
def test_emit_reference_matches_pack_reference_and_defect_fails():
    """emit's exact reference against engine.pack_reference (the layouts' tensor-algebra twin), and a Dg whose taps
    are not reversed differs."""
    from segan_pytorch_b200 import engine as E
    g = _gen(10)
    w = torch.randn(64, 32, 31, generator=g)
    m = E.pack_reference(0, w, 64, 32, 0)                  # [9][64][128]
    F, Dg = M.emit(m, 9, 64, 128, None, 0, None, "f32", "f32")
    assert torch.equal(F, m)
    assert torch.equal(Dg[2], m[6].t())
    bad = m.transpose(1, 2)                                 # tap t instead of T-1-t
    frac = float((bad != Dg).float().mean())
    print("planted defect %-48s %.0f%% of Dg differs" % ("emit_operands: Dg tap not reversed", 100 * frac))
    assert frac > 0.5


def test_alpha_grad_reference_and_defects():
    g = _gen(11)
    T, nc, kc, af = 9, 64, 256, 128
    dwp = torch.randn(T, nc, kc, generator=g)
    m = torch.randn(T, nc, kc, generator=g)
    alpha = 0.5 + torch.rand(kc - af, generator=g)
    d0 = torch.randn(kc - af, generator=g)
    D, (ra, ma) = M.alpha_grad(dwp, m, T, nc, kc, alpha, af, d0)
    assert torch.equal(D[..., :af], dwp[..., :af])
    for order in ORDERS:
        got = d0 + _sum32((dwp[..., af:] * m[..., af:]).reshape(-1, kc - af), 0, order)
        c = M.c_vec(got, ra, ma)
        print("alpha_grad fp32 (%s): c dalpha %.2f" % (order, c))
        assert c <= C_PASS
    bad = dwp.clone()
    bad[..., af - 32:] *= torch.cat((alpha[:32], alpha))    # alpha applied to 32 columns below alpha_from
    frac = float((bad != D).float().mean())
    print("planted defect %-48s %.1f%% of dW differs" % ("alpha_grad: alpha below alpha_from", 100 * frac))
    assert frac > 0.1


@pytest.mark.parametrize("order", ORDERS)
def test_folds_fp32_pass_and_defects(order):
    g = _gen(12)
    dwq = torch.randn(2, 64, 2, 64, generator=g)
    dw0 = torch.randn(64, 2, 31, generator=g)
    (r, m), after = M.wave_wgrad_fold(dwq, 2, dw0)
    q = dwq.reshape(2, 64, 2, 2, 32)[..., :31]
    got = dw0 + (q[0, :, 0] + q[1, :, 1]) if order == "fwd" else (dw0 + q[1, :, 1]) + q[0, :, 0]
    assert M.c_vec(got, r, m) <= C_PASS
    assert float(after.reshape(2, 64, 2, 2, 32)[0, :, 0, :, :31].abs().max()) == 0.0
    assert torch.equal(after.reshape(2, 64, 2, 2, 32)[0, :, 1], dwq.reshape(2, 64, 2, 2, 32)[0, :, 1])
    bad = dw0 + (q[0, :, 1] + q[1, :, 1])                   # an s != s' block read
    _fails(M.c_vec(bad, r, m), "wave_wgrad_fold: reads an s != s' block")
    half = 64
    dq = torch.randn(2, 64, 2, 2, half, generator=g)
    w = torch.randn(2 * half, 1, 31, generator=g)
    al = 0.5 + torch.rand(half, generator=g)
    d0, da0 = torch.randn(2 * half, 1, 31, generator=g), torch.randn(half, generator=g)
    (r, m), (ra, ma), _ = M.last_deconv_fold(dq, half, 2, w, al, d0, da0)
    eff = (dq[0, :31, :, 0] + dq[1, :31, :, 1]).permute(1, 2, 0).reshape(2 * half, 31)
    sc = torch.cat((torch.ones(half), al))[:, None]
    got = d0.reshape(2 * half, 31) + eff * sc
    dag = da0 + _sum32(eff[half:] * w.reshape(2 * half, 31)[half:], 1, order)
    assert M.c_vec(got, r, m) <= C_PASS and M.c_vec(dag, ra, ma) <= C_PASS
    bad = (dq[0, :31, :, 1] + dq[1, :31, :, 1]).permute(1, 2, 0).reshape(2 * half, 31)
    _fails(M.c_vec(d0.reshape(2 * half, 31) + bad * sc, r, m), "last_deconv_wgrad_fold: reads an s != s' block")


# ------------------------------------------------------------------------------------------------------
# STFT glue
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [1025, 16384 + 159])
def test_stft_frames_reference_and_defects(L):
    x = torch.randn(2, L, generator=_gen(13)).clamp(-1, 1)
    src = M.stft_src(L)
    assert src.min() >= 0 and src.max() < L and int(src[0, 0]) == 160 and int(src[1, 0]) == 0
    fr = M.stft_frames(x, "f16", False)
    assert torch.equal(fr[0, 3, 7].float(), x[0, 3 * 160 + 7 - 160].half().float())
    sp = M.stft_frames(x, "f16", True)
    hi, lo = sp[..., :320].double(), sp[..., 320:640].double()
    v = x.double()[:, src]
    assert float(((hi + lo) - v).abs().max()) <= 2.0 ** -22          # hi + lo carries ~22 bits of |x| <= 1
    s = torch.arange(320) - 160                                       # left reflect off by one: -s - 1
    off = torch.where(s < 0, -s - 1, s)
    frac = float((x[:, off].half() != fr[:, 0]).float().mean())
    print("planted defect %-48s %.0f%% of frame 0 differs" % ("stft_frames: left reflect off by one", 100 * frac))
    assert frac > 0.3
    lo16 = (v.float().half().float() - hi.float()).half()             # lo from the 16-bit value: all zero
    frac = float((lo16 != sp[..., 320:640]).float().mean())
    print("planted defect %-48s %.0f%% of lo differs" % ("stft_frames: lo computed in 16-bit", 100 * frac))
    assert frac > 0.5                                                 # (lo of a small |x| is below fp16's range)


def _spectra(rows, ld, bins, half, seed):
    g = _gen(seed)
    scale = 10.0 ** (torch.rand(rows, ld, generator=g) * 8 - 6)
    xg = torch.randn(rows, ld, generator=g) * scale
    xc = xg * (1 + 0.3 * torch.randn(rows, ld, generator=g))
    xc[:, :8] = xg[:, :8]                                             # identical bins: d = 0
    xc[:, half:half + 8] = xg[:, half:half + 8]
    xg[:, 8:12] = 0.0                                                 # zero power
    xg[:, half + 8:half + 12] = 0.0
    return xg, xc


def _logpow32(xg, xc, bins, half, weight, gscale, order, bugs=()):
    rows = xg.shape[0]
    re, im = xg[:, :bins], xg[:, half:half + bins]
    rc, ic = xc[:, :bins], xc[:, half:half + bins]
    pg, pc = re * re + im * im + 1e-19, rc * rc + ic * ic + 1e-19
    d = float(np.float32(4.342944819)) * (torch.log(pg) - torch.log(pc))
    wn = torch.tensor(weight, dtype=torch.float32) / (rows * bins)
    loss = _sum32(d.abs().reshape(-1), 0, order) * wn
    sg = torch.sign(d)
    if "flip_neg" in bugs:
        sg = sg.abs()
    s = sg * wn * gscale * 2.0 * float(np.float32(4.342944819)) / pg
    return loss, torch.stack((s * re, s * im), 1)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("fmt", ["f16", "bf16"])
def test_logpow_l1_fp32_passes(fmt, order):
    rows, bins, half, ld = 309, 1025, 1032, 2072
    xg, xc = _spectra(rows, ld, bins, half, 14)
    loss, gx = _logpow32(xg, xc, bins, half, 0.37, 8.0, order)
    ref = M.logpow_l1(xg, xc, bins, half, 0.37, 8.0)
    lr, (budget, mag) = ref["loss"]
    c = (M.c_budget(loss, lr, budget, mag), M.c_logpow_gx(M.to16(gx, fmt), ref["gx"], ref["d"], fmt))
    print("logpow_l1 fp32 %s (%s): c loss %.2f gx %.2f" % (fmt, order, *c))
    assert all(v <= C_PASS for v in c)


def test_logpow_l1_defect_sign_flip():
    rows, bins, half, ld = 309, 1025, 1032, 2072
    xg, xc = _spectra(rows, ld, bins, half, 14)
    _, gx = _logpow32(xg, xc, bins, half, 0.37, 8.0, "fwd", bugs=("flip_neg",))
    ref = M.logpow_l1(xg, xc, bins, half, 0.37, 8.0)
    _fails(M.c_logpow_gx(M.to16(gx, "bf16"), ref["gx"], ref["d"], "bf16"), "logpow_l1: sign flipped for d < 0")


def test_logf_bound():
    """The bound follows the documented __logf error: absolute on [0.5, 2], 3 ulp of the result elsewhere."""
    p = torch.tensor([0.5, 1.0, 2.0, 4.0, 1e-19, 1e6], dtype=torch.float64)
    e = M.logf_err(p)
    assert torch.all(e[:3] == M.LOGF_ABS)
    assert float(e[3]) == 3 * 2.0 ** -23 and float(e[4]) == 3 * 2.0 ** (5 - 23)
    assert math.isclose(float(e[5]), 3 * 2.0 ** (3 - 23))


@pytest.mark.parametrize("order", ORDERS)
def test_stft_fold_fp32_passes_and_defect(order):
    B, L = 3, 16384 + 159
    fr = 1 + L // 160
    gf = torch.randn(B, fr, 320, generator=_gen(15))
    g0 = torch.randn(B, L, generator=_gen(16))
    ref = M.stft_fold(gf, L, 0.37, g0)
    src = M.stft_src(L).reshape(-1)
    v = (0.37 * gf.reshape(B, -1))
    idx = torch.arange(src.numel()) if order == "fwd" else torch.arange(src.numel()).flip(0)
    got = g0.clone()
    got.index_add_(1, src[idx], v[:, idx])
    c = M.c_vec(got, *ref)
    print("stft_frames_fold fp32 (%s): c %.2f" % (order, c))
    assert c <= C_PASS
    bad = g0.clone()
    bad.index_add_(1, src, gf.reshape(B, -1))
    _fails(M.c_vec(bad, *ref), "stft_frames_fold: scale missing")


# ------------------------------------------------------------------------------------------------------
# the formulas are the reference's: the fp64 model against torch autograd / torch.optim
# ------------------------------------------------------------------------------------------------------
def _close(a, b, what):
    err = float((a.double() - b.double()).abs().max()) / max(1e-30, float(b.double().abs().max()))
    assert err <= 1e-12, (what, err)


@pytest.mark.parametrize("g_in_path", [False, True])
def test_fc_tail_model_is_the_autograd_derivative(g_in_path):
    """discriminator.py:111-117 (PReLU, Linear(256, 128), PReLU, Linear(128, 1)) with the LSGAN loss
    weight * mean((logit - target)^2) -- or a given d loss / d logit -- differentiated by autograd in fp64."""
    B, target, weight = 17, 1.0, 0.5
    x = [t.double() for t in _fc_inputs(B, 21)]
    x[0][:, :8] = 0.3                                       # no exact zeros: autograd's PReLU kink convention aside
    ps = [t.clone().requires_grad_(True) for t in x]
    acc, b0, s1, w2, b2, s3, w4, b4 = ps
    h1 = torch.nn.functional.prelu(acc + b0, s1)
    h2 = torch.nn.functional.prelu(torch.nn.functional.linear(h1, w2, b2), s3)
    logit = torch.nn.functional.linear(h2, w4, b4).view(-1)
    g_in = torch.randn(B, generator=_gen(22), dtype=torch.float64) if g_in_path else None
    loss = (logit * g_in).sum() if g_in_path else weight * ((logit - target) ** 2).mean()
    grads = torch.autograd.grad(loss, ps)
    z1, _ = M.fc_z1(x[0], x[1])
    z2, _ = M.fc_z2(z1, x[2], x[3], x[4])
    lg, _ = M.fc_logit(z2, x[5], x[6], x[7])
    _close(lg, logit.detach(), "logit")
    gl, _ = M.fc_g_logit(lg, g_in, target, weight, B, 1.0)
    gz2, _ = M.fc_g_z2(z2, gl, x[5], x[6])
    (gh1, _), (gz1, _) = M.fc_g_h1_z1(gz2, z1, x[2], x[3])
    _close(gz1, grads[0], "g_z1")
    names = ("b0", "s1", "w2", "b2", "s3", "w4", "b4")
    ref = M.fc_params(z1, z2, gl, gz2, gz1, gh1, x[2], x[5], x[6], {n: torch.zeros_like(t) for n, t in zip(names, x[1:])})
    for n, g in zip(names, grads[1:]):
        _close(ref[n][0], g.reshape(ref[n][0].shape), n)
    if not g_in_path:
        _close(M.fc_loss(lg, target, weight, B)[0], loss.detach(), "loss")


@pytest.mark.parametrize("kind", ["l1", "mse"])
def test_reg_loss_model_is_the_autograd_derivative(kind):
    y, clean = (t.double() for t in _reg_inputs(1001))
    yr = y.clone().requires_grad_(True)
    f = torch.nn.functional.l1_loss if kind == "l1" else torch.nn.functional.mse_loss
    loss = 100.0 * f(yr, clean)
    g, = torch.autograd.grad(loss, yr)                      # torch's L1 gradient at d = 0 is 0, as the kernel's
    ref = M.reg_loss(kind, y, clean, 100.0, 1.0)
    _close(ref["loss"][0], loss.detach(), "loss")
    _close(ref["gy"][0], g, "gy")


def test_logpow_model_is_the_autograd_derivative():
    """model.py:638-653's 10 log10(|X|^2 + 1e-19) L1 term, differentiated by autograd w.r.t. re and im of X_gen."""
    rows, bins, half, ld = 7, 65, 72, 150
    xg, xc = (t.double() for t in _spectra(rows, ld, bins, half, 23))
    xg[:, 8:12] = 0.5                                       # no zero-power / identical bins: autograd's |0|' aside
    xg[:, half + 8:half + 12] = 0.5
    xc[:, :8] *= 1.5
    xr = xg.clone().requires_grad_(True)
    eps = float(torch.tensor(1e-19, dtype=torch.float32))

    def lp(x):
        return 10 * torch.log10(x[:, :bins] ** 2 + x[:, half:half + bins] ** 2 + eps)
    loss = 0.375 * (lp(xr) - lp(xc)).abs().mean()
    g, = torch.autograd.grad(loss, xr)
    ref = M.logpow_l1(xg, xc, bins, half, 0.375, 1.0)
    _close(ref["loss"][0], loss.detach(), "loss")
    _close(ref["gx"][0], torch.stack((g[:, :bins], g[:, half:half + bins]), 1), "gx")


@pytest.mark.parametrize("kind", ["rmsprop", "adam"])
def test_optimizer_model_is_torch_optim(kind):
    """Three steps of the model, each on its own previous state, against torch.optim in fp64 (hyper-parameters as
    fp32 values, as the kernels receive them)."""
    n = 101
    g = _gen(24)
    p0 = torch.randn(n, generator=g, dtype=torch.float64)
    lr, eps = M.f32(2e-4), M.f32(1e-8)
    pr = p0.clone().requires_grad_(True)
    if kind == "rmsprop":
        a = M.f32(0.99)
        opt = torch.optim.RMSprop([pr], lr=lr, alpha=a, eps=eps)
    else:
        b1, b2 = M.f32(0.5), M.f32(0.999)
        opt = torch.optim.Adam([pr], lr=lr, betas=(b1, b2), eps=eps)
    p, s1, s2 = p0.clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for t in range(1, 4):
        gr = torch.randn(n, generator=g, dtype=torch.float64)
        pr.grad = gr.clone()
        opt.step()
        if kind == "rmsprop":
            r = M.rmsprop_step(p, gr, s1, 2e-4, 0.99, 1e-8, 1.0)
            p, s1 = r["p"][0], r["sq"][0]
        else:
            r = M.adam_step(p, gr, s1, s2, 2e-4, 0.5, 0.999, 1e-8, t, 1.0)
            p, s1, s2 = r["p"][0], r["m"][0], r["v"][0]
    _close(p - p0, pr.detach() - p0, kind)


def test_gates_fail_on_nan_and_unwritten_sentinels():
    """A NaN result, or a destination whose sentinel fill (a NaN pattern) was never overwritten, gives c = inf in
    every yardstick, also when other elements are right: no gate can pass it."""
    ref = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)
    mag = ref.abs()
    got = torch.tensor([1.0, float("nan"), 3.0])
    assert M.c_vec(got, ref, mag) == math.inf and M.c_budget(got, ref, 0 * mag, mag) == math.inf
    for fmt, dt in (("f16", torch.float16), ("bf16", torch.bfloat16)):
        _, unwritten = M.guarded((3,), dt, "cpu")
        assert M.is_sentinel(unwritten) and M.c_f(unwritten, ref, mag, fmt) == math.inf
        g = unwritten.reshape(1, 1, 3)
        d = (torch.ones(1, 3, dtype=torch.float64), torch.zeros(1, 3, dtype=torch.float64))
        assert M.c_logpow_gx(g, (ref.reshape(1, 1, 3), mag.reshape(1, 1, 3)), d, fmt) == math.inf
    _, w32 = M.guarded((3,), torch.float32, "cpu")
    assert M.c_vec(w32, ref, mag) == math.inf
