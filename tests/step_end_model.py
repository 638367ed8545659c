"""fp64 references and rounding-error yardsticks of the kernels at the two ends of a training step (not collected;
plain torch, runs on any device, no kernels):

  loss end       sg_fc_tail_fwd / sg_fc_tail_bwd (the Discriminator's fc tail), sg_l1_loss_bwd / sg_mse_loss_bwd,
                 and WSEGAN's spectral-loss glue sg_stft_frames / sg_logpow_l1 / sg_stft_frames_fold
  parameter end  sg_rmsprop_step / sg_adam_step, sg_emit_operands, sg_alpha_grad, sg_wave_wgrad_fold,
                 sg_last_deconv_wgrad_fold(_1src); sg_pack_weights / sg_unpack_wgrad in fp32 are engine.pack_reference /
                 unpack_reference

As in tests/bn_act_model.py, every arithmetic function evaluates its kernel's own formula on the kernel's own inputs
and returns (ref, mag): the fp64 value and the sum of the absolute values of the terms the kernel adds, so that an
fp32 evaluation in any summation order is within a small multiple of U * mag of ref (tapgemm_model.U, C_TOL; nvcc
contracts mul + add into FMA, so these kernels are never held to a torch fp32 emulation bit for bit).  Where a kernel
runs in stages (fc tail forward z1 -> z2 -> logit; backward rows -> parameter gradients) each stage is evaluated on
the kernel's own output of the stage before, so an error is caught where it is made.

Pure data movement (frames, emit without a scale, pack / unpack, the clearing by the folds) is exact: those
references are plain fp32 / 16-bit tensors to be compared bit for bit.  A single-rounding op (dW *= alpha, emit with
a scale) is exact as well: its reference is the same fp32 product, rounded once.

Bias corrections.  Adam's 1 - beta^step is computed on the host in fp32 and can cancel: at beta2 = 0.999, step 2 it
is 0.002 and one ulp of beta^step is 500 ulp of the difference.  adam_step therefore counts 1 and beta^step as the
correction's two terms (relative error U * (1 + beta^step) / (1 - beta^step)) and carries that into the update's mag.

__logf.  sg_logpow_l1 takes both logarithms with __logf, whose documented error (CUDA C Programming Guide, intrinsic
functions) is at most 2^-21.41 absolute for x in [0.5, 2] and 3 ulp of the result elsewhere.  logpow_l1 returns that
bound per bin (LOGF_ABS, logf_err), scaled by 10 / ln 10, plus the relative rounding of the power sums; a bin whose
fp64 |d| lies within it may take either gradient sign."""
import math

import torch

from tests import tapgemm_model as _tm
from tests.tapgemm_model import C_TOL, U, _ratio, half_ulp  # noqa: F401  (re-exported for the tests)

FC1, FC2, FC_CHUNK = 256, 128, 16          # elementwise.cu: fc tail widths, batch rows per parameter-gradient block
KW = 31
STFT_WIN, STFT_HOP = 320, 160
K10 = 10.0 / math.log(10.0)
LOGF_ABS = 2.0 ** -21.41                   # __logf on [0.5, 2]
LOGF_ULP = 3.0                             # __logf elsewhere, in ulp of the result


def _nan_is_inf(c):
    """A NaN c (a NaN output, or a sentinel that was never overwritten) fails every gate instead of slipping past
    comparisons, which are all False against NaN."""
    return math.inf if math.isnan(c) else c


def c_vec(got, ref, mag):
    """max |got - ref| / (U * mag); infinite where mag == 0 and got != ref, or where got is NaN.  got takes ref's
    shape (same numel)."""
    return _nan_is_inf(_ratio((got.double().reshape(ref.shape) - ref).abs(), U * mag))


def c_f(got16, ref, mag, fmt, trunc_stages=0):
    """tapgemm_model.c_f (a 16-bit store's error past half an ulp, fp16 saturating), infinite where got16 is NaN."""
    return _nan_is_inf(_tm.c_f(got16, ref, mag, fmt, trunc_stages))


def c_budget(got, ref, budget, mag):
    """Like c_vec after taking an absolute error budget off first (sg_logpow_l1's logarithms)."""
    err = ((got.double() - ref).abs() - budget).clamp_min(0.0)
    return _nan_is_inf(_ratio(err, U * mag))


def c_logpow_gx(got16, gx, d, fmt):
    """c_f of sg_logpow_l1's 16-bit gradient [rows][2][bins] (re | im halves gathered by the caller), where a bin
    whose |d| is within its bound may hold the gradient of either sign or 0."""
    ref, mag = gx
    dv, bound = d
    amb = (dv.abs() <= bound)[:, None, :].expand_as(ref)

    def err(t):
        tgt = t.clamp(-65504.0, 65504.0) if fmt == "f16" else t
        return ((got16.double() - tgt).abs() - half_ulp(tgt, fmt)).clamp_min(0.0)
    e = err(ref)
    e = torch.where(amb, torch.minimum(e, torch.minimum(err(-ref), got16.double().abs())), e)
    return _nan_is_inf(_ratio(e, U * mag))


def f32(v):
    """A Python float as the fp32 value a kernel argument holds."""
    return float(torch.tensor(v, dtype=torch.float32))


def to16(x, fmt):
    """fp32 -> 16-bit as the kernels store it: round to nearest, fp16 saturating at +-65504 (NaN stays NaN)."""
    if fmt == "f16":
        return x.float().clamp(-65504.0, 65504.0).half()
    return x.float().bfloat16()


# ------------------------------------------------------------------------------------------------------
# sentinel guard bands around a destination (the GPU tests)
# ------------------------------------------------------------------------------------------------------
GUARD = 4096
_SENT = {torch.float32: (torch.int32, 0x7FA5A5A5), torch.float16: (torch.int16, 0x7E5A),
         torch.bfloat16: (torch.int16, 0x7FA5)}          # NaN bit patterns no kernel writes


def guarded(shape, dtype, device, init=None):
    """(buf, view): `view` of `shape` sits between GUARD sentinel elements on each side of `buf`; it starts as
    `init` (copied) or as sentinels.  GUARD elements keep the view 16-byte aligned."""
    n = 1
    for d in shape:
        n *= d
    it, bits = _SENT[dtype]
    buf = torch.full((n + 2 * GUARD,), bits, dtype=it, device=device).view(dtype)
    view = buf[GUARD:GUARD + n].view(shape)
    if init is not None:
        view.copy_(init.reshape(shape))
    return buf, view


def guards_ok(buf):
    it, bits = _SENT[buf.dtype]
    b = buf.view(it)
    return bool((b[:GUARD] == bits).all()) and bool((b[-GUARD:] == bits).all())


def sentinel_mask(t):
    """The elements of t that still hold the guard-band sentinel (never written)."""
    it, bits = _SENT[t.dtype]
    return t.contiguous().view(it) == bits


def is_sentinel(t):
    """Every element of t still holds the guard-band sentinel (never written)."""
    return bool(sentinel_mask(t).all())


def bits_equal(a, b):
    """Bitwise equality (NaN-safe)."""
    it = torch.int32 if a.element_size() == 4 else torch.int16
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(it), b.contiguous().view(it))


def _prelu(z, s):
    return torch.where(z > 0, z, z * s)


# ------------------------------------------------------------------------------------------------------
# Discriminator fc tail (discriminator.py:111-117)
# ------------------------------------------------------------------------------------------------------
def fc_z1(acc, b0):
    """z1 = fc0_acc + b0: [B][256]."""
    a, b = acc.double(), b0.double()
    return a + b, a.abs() + b.abs()


def fc_z2(z1, s1, w2, b2):
    """z2 = W2 PReLU_s1(z1) + b2 on the kernel's z1: [B][128]."""
    h1 = _prelu(z1.double(), s1.double())
    W = w2.double()
    return h1 @ W.t() + b2.double(), h1.abs() @ W.abs().t() + b2.double().abs()


def fc_logit(z2, s3, w4, b4):
    """logit = w4 . PReLU_s3(z2) + b4 on the kernel's z2: [B]."""
    h2 = _prelu(z2.double(), s3.double())
    w = w4.double().reshape(-1)
    return h2 @ w + b4.double(), h2.abs() @ w.abs() + b4.double().abs()


def fc_g_logit(logit, g_logit_in, target, weight, batch, gscale):
    """d loss / d logit, loss-scaled: g_logit_in * gscale, or the fused MSE 2 (logit - target) / B * weight * gscale."""
    if g_logit_in is not None:
        g = g_logit_in.double().reshape(-1) * f32(gscale)
    else:
        g = 2.0 * (logit.double().reshape(-1) - f32(target)) / batch * f32(weight) * f32(gscale)
    return g, g.abs()


def fc_loss(logit, target, weight, batch):
    """sum_b (logit - target)^2 / B * weight (added to loss_out; grad_scale does not touch it)."""
    t = (logit.double().reshape(-1) - f32(target)) ** 2 / batch * f32(weight)
    return t.sum(), t.abs().sum()


def fc_g_z2(z2, g_logit, s3, w4):
    """First stage of the per-row backward, on the kernel's g_logit (its workspace): g_z2 = gl w4 [z2 > 0 | s3]
    [B][128]."""
    gl = g_logit.double().reshape(-1, 1)
    gh2 = gl * w4.double().reshape(1, -1)
    g = torch.where(z2.double() > 0, gh2, gh2 * s3.double())
    return g, g.abs()


def fc_g_h1_z1(g_z2, z1, s1, w2):
    """g_h1 = g_z2 W2 and g_z1 = g_h1 [z1 > 0 | s1] on the kernel's own g_z2: ((ref, mag), (ref, mag)) [B][256]."""
    G, W = g_z2.double(), w2.double()
    gh1, mh1 = G @ W, G.abs() @ W.abs()
    sl = torch.where(z1.double() > 0, torch.ones_like(gh1), s1.double().expand_as(gh1))
    return (gh1, mh1), (gh1 * sl, mh1 * sl.abs())


def fc_params(z1, z2, g_logit, g_z2, g_z1, g_h1, s1, s3, w4, g0):
    """Parameter gradients from the kernel's own row workspaces, added to the values the buffers held before (g0:
    dict b0, s1, w2, b2, s3, w4, b4) -> dict of (ref, mag):
      g_w2 += sum_b g_z2 h1^T       g_b0 += sum_b g_z1         g_s1 += sum_{b, z1 <= 0} g_h1 z1
      g_b2 += sum_b g_z2            g_s3 += sum_{b, z2 <= 0} gl w4 z2
      g_w4 += sum_b gl h2           g_b4 += sum_b gl"""
    Z1, Z2 = z1.double(), z2.double()
    gl = g_logit.double().reshape(-1)
    G2, G1, H1 = g_z2.double(), g_z1.double(), g_h1.double()
    h1, h2 = _prelu(Z1, s1.double()), _prelu(Z2, s3.double())
    w4d = w4.double().reshape(-1)
    terms = dict(
        w2=(G2.t() @ h1, G2.abs().t() @ h1.abs()),
        b0=(G1.sum(0), G1.abs().sum(0)),
        s1=(torch.where(Z1 <= 0, H1 * Z1, 0 * Z1).sum(0), torch.where(Z1 <= 0, (H1 * Z1).abs(), 0 * Z1).sum(0)),
        b2=(G2.sum(0), G2.abs().sum(0)),
        s3=(torch.where(Z2 <= 0, gl[:, None] * w4d * Z2, 0 * Z2).sum(0),
            torch.where(Z2 <= 0, (gl[:, None] * w4d * Z2).abs(), 0 * Z2).sum(0)),
        w4=(gl @ h2, gl.abs() @ h2.abs()),
        b4=(gl.sum().reshape(1), gl.abs().sum().reshape(1)),
    )
    out = {}
    for k, (r, m) in terms.items():
        p = g0[k].double().reshape(r.shape)
        out[k] = (p + r, p.abs() + m)
    return out


# ------------------------------------------------------------------------------------------------------
# regression losses (model.py:318): L1 and MSE
# ------------------------------------------------------------------------------------------------------
def reg_loss(kind, y, clean, weight, grad_scale, gy0=None):
    """kind 'l1' | 'mse' -> dict loss=(ref, mag) (the value added to loss_out), gy=(ref, mag) (gy0 + g, or g when
    gy0 is None).  The kernel forms d = y - clean in fp32: its sign is exact, so the L1 gradient is exactly
    +-w/n * grad_scale or 0."""
    n = y.numel()
    d = y.double() - clean.double()
    lscale = f32(weight) / n
    if kind == "l1":
        lt = d.abs() * lscale
        g = torch.sign(d) * lscale * f32(grad_scale)
    else:
        lt = d * d * lscale
        g = 2.0 * lscale * f32(grad_scale) * d
    gm = g.abs()
    if gy0 is not None:
        g, gm = gy0.double() + g, gy0.double().abs() + gm
    return dict(loss=(lt.sum(), lt.abs().sum()), gy=(g, gm))


# ------------------------------------------------------------------------------------------------------
# optimisers (torch.optim.RMSprop / Adam as model.py:221-225 use them)
# ------------------------------------------------------------------------------------------------------
def rmsprop_step(p, g, sq, lr, alpha, eps, grad_scale):
    """One step on the kernel's state: dict p=(ref, mag), sq=(ref, mag).
    gi = g * grad_scale ; sq' = alpha sq + (1 - alpha) gi^2 ; p' = p - lr gi / (sqrt(sq') + eps)."""
    a, lr, eps = f32(alpha), f32(lr), f32(eps)
    gi = g.double() * f32(grad_scale)
    s = a * sq.double() + (1.0 - a) * gi * gi
    sm = a * sq.double().abs() + (1.0 - a) * gi * gi
    den = s.sqrt() + eps
    upd = lr * gi / den
    P = p.double()
    return dict(p=(P - upd, P.abs() + upd.abs()), sq=(s, sm))


def adam_step(p, g, m, v, lr, beta1, beta2, eps, step, grad_scale):
    """One step on the kernel's state: dict p, m, v of (ref, mag).
    m' = b1 m + (1 - b1) gi ; v' = b2 v + (1 - b2) gi^2 ; p' = p - lr / bc1 * m' / (sqrt(v') / sqrt(bc2) + eps),
    bc = 1 - beta^step.  The update's mag carries the cancellation of the host's fp32 bias corrections (module
    docstring)."""
    b1, b2, lr, eps = f32(beta1), f32(beta2), f32(lr), f32(eps)
    gi = g.double() * f32(grad_scale)
    M = b1 * m.double() + (1.0 - b1) * gi
    Mm = b1 * m.double().abs() + (1.0 - b1) * gi.abs()
    V = b2 * v.double() + (1.0 - b2) * gi * gi
    Vm = b2 * v.double().abs() + (1.0 - b2) * gi * gi
    t1, t2 = b1 ** step, b2 ** step
    bc1, bc2 = 1.0 - t1, 1.0 - t2
    upd = lr / bc1 * M / (V.sqrt() / math.sqrt(bc2) + eps)
    amp = 1.0 + (1.0 + t1) / bc1 + 0.5 * (1.0 + t2) / bc2
    P = p.double()
    # the update inherits the relative error of m' (Mm / |M|) and of sqrt(v') (Vm / V / 2)
    rel = Mm / M.abs().clamp_min(1e-300) + 0.5 * Vm / V.clamp_min(1e-300)
    return dict(p=(P - upd, P.abs() + upd.abs() * (amp + rel)), m=(M, Mm), v=(V, Vm))


# ------------------------------------------------------------------------------------------------------
# packed masters: operands, alpha gradient, waveform-end folds
# ------------------------------------------------------------------------------------------------------
def colscale(kc, alpha, alpha_from, scale=None, device=None):
    """fp32 per-column factor the kernel multiplies by: alpha[k - alpha_from] for k >= alpha_from (else 1), times
    the device scalar `scale` (1/sigma), rounded once as the kernel forms it."""
    a = torch.ones(kc, dtype=torch.float32, device=device)
    if alpha is not None:
        a[alpha_from:] = alpha.float().to(a.device)
    if scale is not None:
        a = a * scale.float().to(a.device).reshape(())
    return a


def emit(m, n_taps, nc, kc, alpha, alpha_from, scale, fmt_f, fmt_dg):
    """sg_emit_operands, exact: (F [T][nc][kc], Dg [T][kc][nc]) in the destination formats ('f16' | 'bf16' | 'f32').
    F[t][n][k] = M[t][n][k] * a(k), Dg[t][k][n] = M[T-1-t][n][k] * a(k), one fp32 rounding of the product."""
    M = m.reshape(n_taps, nc, kc).float()
    v = M * colscale(kc, alpha, alpha_from, scale, M.device)
    F = v if fmt_f == "f32" else to16(v, fmt_f)
    Dg = v.flip(0).transpose(1, 2).contiguous()
    Dg = Dg if fmt_dg == "f32" else to16(Dg, fmt_dg)
    return F, Dg


def alpha_grad(dwp, m, n_taps, nc, kc, alpha, alpha_from, dalpha0=None):
    """sg_alpha_grad -> (dW exact fp32 [T][nc][kc], (ref, mag) of dalpha [kc - alpha_from] or None):
    dW[.., k] = dWp * alpha for k >= alpha_from (one rounding; the columns below keep their bits) and
    dalpha += sum_{t, n} dWp * M (before the scaling)."""
    D = dwp.reshape(n_taps, nc, kc).float().clone()
    M = m.reshape(n_taps, nc, kc)
    prod = (D[..., alpha_from:].double() * M[..., alpha_from:].double()).reshape(-1, kc - alpha_from)
    D[..., alpha_from:] = D[..., alpha_from:] * alpha.float()
    if dalpha0 is None:
        return D, None
    base = dalpha0.double()
    return D, (base + prod.sum(0), base.abs() + prod.abs().sum(0))


def wave_wgrad_fold(dwq, cin, dw0):
    """sg_wave_wgrad_fold: dwq [2][64][2][64] -> ((ref, mag) of dW [64][cin][31], dwq after the call (exact)).
    dW[co][ci][k] += dwq[0][co][0][ci*32 + k] + dwq[1][co][1][ci*32 + k]; the blocks read are cleared."""
    q = dwq.reshape(2, 64, 2, 64)
    p0 = q[0, :, 0].reshape(64, 2, 32)[:, :cin, :31].double()
    p1 = q[1, :, 1].reshape(64, 2, 32)[:, :cin, :31].double()
    base = dw0.double().reshape(64, cin, 31)
    after = q.clone()
    for s in (0, 1):
        blk = after[s, :, s].reshape(64, 2, 32)
        blk[:, :cin, :31] = 0
        after[s, :, s] = blk.reshape(64, 64)
    return (base + p0 + p1, base.abs() + p0.abs() + p1.abs()), after.reshape(dwq.shape)


def last_deconv_fold(dwq, half, nsrc, w, alpha, dw0, dalpha0=None):
    """sg_last_deconv_wgrad_fold (nsrc 2, alpha on the skip half) / _1src (nsrc 1): dwq [2][64][nsrc][2][half] ->
    ((ref, mag) of dW [nsrc*half][1][31], (ref, mag) of dalpha [half] or None, dwq after the call (exact)).
    dWeff[src*half + c][k] = dwq[0][k][src][0][c] + dwq[1][k][src][1][c]; dW += dWeff (* alpha[c] on src 1);
    dalpha[c] += sum_k dWeff[half + c][k] * W[half + c][k]."""
    q = dwq.reshape(2, 64, nsrc, 2, half)
    a = q[0, :KW, :, 0].double()                          # [k][src][c]
    b = q[1, :KW, :, 1].double()
    eff = (a + b).permute(1, 2, 0).reshape(nsrc * half, KW)
    effm = (a.abs() + b.abs()).permute(1, 2, 0).reshape(nsrc * half, KW)
    sc = torch.ones(nsrc * half, 1, dtype=torch.float64, device=dwq.device)
    if nsrc == 2:
        sc[half:, 0] = alpha.double()
    base = dw0.double().reshape(nsrc * half, KW)
    dW = (base + eff * sc, base.abs() + effm * sc.abs())
    da = None
    if nsrc == 2 and dalpha0 is not None:
        W = w.double().reshape(2 * half, KW)[half:]
        da = (dalpha0.double() + (eff[half:] * W).sum(1), dalpha0.double().abs() + (effm[half:] * W.abs()).sum(1))
    after = q.clone()
    after[0, :KW, :, 0] = 0
    after[1, :KW, :, 1] = 0
    return dW, da, after.reshape(dwq.shape)



# ------------------------------------------------------------------------------------------------------
# WSEGAN spectral loss glue (model.py:638-653)
# ------------------------------------------------------------------------------------------------------
def stft_src(L, device=None):
    """Source sample of every frame element: [1 + L/160][320] indices of reflect(160 t + n - 160) onto [0, L)."""
    fr = 1 + L // STFT_HOP
    s = (torch.arange(fr, device=device)[:, None] * STFT_HOP + torch.arange(STFT_WIN, device=device)[None, :]
         - STFT_HOP)
    s = torch.where(s < 0, -s, s)
    return torch.where(s >= L, 2 * (L - 1) - s, s)


def stft_frames(x, fmt, split):
    """sg_stft_frames, exact: [B][frames][320] 16-bit, or with split rows of 960 = hi | lo | hi, hi = x rounded to
    16 bits, lo = (x - hi) rounded (x - hi is exact in fp32)."""
    B, L = x.shape
    v = x.float()[:, stft_src(L, x.device)]
    if not split:
        return to16(v, fmt)
    hi = to16(v, fmt)
    lo = to16(v - hi.float(), fmt)
    return torch.cat((hi, lo, hi), -1)


def ulp32(v):
    """Spacing of fp32 at |v| (normal range)."""
    e = torch.frexp(v.double().abs().clamp_min(2.0 ** -126))[1]
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 24)


def logf_err(p):
    """Documented bound of __logf(p) against ln(p) (fp64 p as the kernel's fp32 argument)."""
    lp = torch.log(p)
    return torch.where((p >= 0.5) & (p <= 2.0), torch.full_like(lp, LOGF_ABS), LOGF_ULP * ulp32(lp))


def logpow_l1(xg, xc, bins, half, weight, grad_scale):
    """sg_logpow_l1 on X_gen, X_clean [rows][ld] fp32 (re at column f, im at half + f) -> dict
      d     = (10 log10 pg - 10 log10 pc, bound) per bin [rows][bins]: bound = the kernel's worst error on d
      loss  = (wn sum |d|, (wn sum bound, wn sum |d|)): what loss_out gains and its error budget (a per-bin absolute
              part from the logarithms plus summation rounding, U * mag)
      gx    = (ref, mag) [rows][2][bins] of sign(d) wn grad_scale (20 / ln 10) (re, im) / pg,  wn = weight / (rows bins);
              where |d| <= bound the kernel may take either sign (or 0); mag is the unsigned size."""
    rows = xg.shape[0]
    re, im = xg[:, :bins].double(), xg[:, half:half + bins].double()
    rc, ic = xc[:, :bins].double(), xc[:, half:half + bins].double()
    eps = float(torch.tensor(1e-19, dtype=torch.float32))
    pg, pc = re * re + im * im + eps, rc * rc + ic * ic + eps
    d = K10 * (torch.log(pg) - torch.log(pc))
    # __logf of each argument, 3 U of each power sum (two products and two adds, all terms positive), and the two
    # roundings of the difference and its product with 10 / ln 10
    bound = K10 * (logf_err(pg) + logf_err(pc) + 6 * U) + 3 * U * d.abs()
    wn = f32(weight) / (rows * bins)
    g = wn * f32(grad_scale) * 2.0 * K10 / pg
    gx = torch.stack((g * re, g * im), 1)
    sg = torch.sign(d)[:, None, :]
    # mag: the size of the gradient of either sign, so that a bin within the bound may take any of them
    return dict(d=(d, bound), loss=(wn * d.abs().sum(), (wn * bound.sum(), wn * d.abs().sum())),
                gx=(sg * gx, gx.abs()))


def stft_fold(gf, L, scale, g0):
    """sg_stft_frames_fold: g_wave [B][L] = g0 + scale * overlap-add of g_frames [B][frames][320] through the
    frames' reflect map -> (ref, mag)."""
    B = gf.shape[0]
    src = stft_src(L, gf.device).reshape(-1)
    v = gf.double().reshape(B, -1) * f32(scale)
    ref = g0.double().clone().reshape(B, L)
    mag = ref.abs()
    ref.index_add_(1, src, v)
    mag.index_add_(1, src, v.abs())
    return ref, mag
