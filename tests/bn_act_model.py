"""fp64 references and rounding-error yardsticks of the BatchNorm / PReLU streaming kernels (not collected; plain
torch, runs on any device, no kernels): sg_bn_stats, sg_bn_finalize, sg_act_fwd, sg_act_bwd_reduce (pass 0),
sg_act_bwd_apply (pass 1), sg_stat_grads, and the BatchNorm statistics of the tap-GEMM epilogue.

Every function is evaluated on the kernel's own 16-bit inputs and fp32 per-channel constants and returns
(ref, mag): the fp64 value and the sum of the absolute values of the terms the kernel actually adds.  An fp32
evaluation is then within a small multiple of U * mag of ref, whatever its summation order (tapgemm_model.U,
C_TOL; a 16-bit store adds half an output ulp, which tapgemm_model.c_f takes off first).

Long fp32 runs.  A sum that one fp32 partial accumulates over n additions can be off by up to n * U * mag (each
addition rounds the running sum, which is bounded by mag); its rounding errors have random signs, so the observed
error grows like sqrt(n) at worst.  The kernels' per-thread partials run over up to ~200 rows (bn_stats at D enc0,
batch 300) and the tap-GEMM epilogue's shared-memory `colstat` over up to ~150 warp partials per CTA; measured on an
H100 the worst c of any such sum is 3.7 (DESIGN.md section 3), so the sums are held to C_TOL with no run-length
allowance.

Centring of red2.  The tiled and TMA-staged backward kernels accumulate sum(g_pre * x) in fp32 and centre it in
double at the flush: red2 = is * (sum(g_pre * x) - mu * sum(g_pre)).  Its error is therefore bounded by
U * is * sum|g_pre| * (|x| + |mu|), not by the per-element centred U * is * sum|g_pre| * |x - mu| the generic
kernel's arithmetic would allow: with |mu| = 8 sigma the honest yardstick is ~9x looser than the generic one.
bwd_pass0 returns the looser one for every kernel."""
import torch

from tests.tapgemm_model import C_TOL, U, _ratio, c_f, half_ulp  # noqa: F401  (re-exported for the tests)

SLICES = 8                  # SG_STAT_SLICES


def c_vec(got, ref, mag):
    """max |got - ref| / (U * mag); infinite where mag == 0 and got != ref."""
    return _ratio((got.double() - ref).abs(), U * mag)


def reflect_src(L, H, roll, device=None):
    """Exact row l feeding consumer row qh in [0, L + 2H): q = qh - H reflected onto [0, L) (F.pad mode='reflect'),
    then un-rolled: the consumer view is roll(y, roll) along time, so l = (reflect(q) - roll) mod L."""
    q = torch.arange(-H, L + H, device=device)
    q = torch.where(q < 0, -q, q)
    q = torch.where(q >= L, 2 * (L - 1) - q, q)
    return torch.remainder(q - roll, L)


def _consts(C, ss, mi, slope, device):
    one = torch.ones(C, dtype=torch.float64, device=device)
    sc = ss[0].double() if ss is not None else one
    sh = ss[1].double() if ss is not None else one * 0
    mu = mi[0].double() if mi is not None else one * 0
    inv = mi[1].double() if mi is not None else one
    sl = slope.double() if slope is not None else None
    return sc, sh, mu, inv, sl


# ------------------------------------------------------------------------------------------------------
# statistics and finalize
# ------------------------------------------------------------------------------------------------------
def stats(x):
    """x [..., C] 16-bit -> (ref, mag) [2][C]: sum x and sum x^2 per channel; mag = sum|x| and sum x^2."""
    x = x.reshape(-1, x.shape[-1]).double()
    sq = (x * x).sum(0)
    return torch.stack((x.sum(0), sq)), torch.stack((x.abs().sum(0), sq))


def finalize(st, count, gamma, beta, eps, momentum, rmean=None, rvar=None):
    """st [S][2][C] fp64 slices (summed here), fp32 gamma / beta / running buffers -> {name: (ref, mag)} for
    mean, invstd, sc, sh (gate in units of |beta| + |mean * sc|), rmean, rvar (running update with the unbiased
    factor n / (n - 1), 1 when n == 1)."""
    s = st.double().sum(0)
    n = float(count)
    mean = s[0] / n
    var = (s[1] / n - mean * mean).clamp_min(0.0)
    invstd = 1.0 / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))
    g, b = gamma.double(), beta.double()
    sc = g * invstd
    sh = b - mean * sc
    out = dict(mean=(mean, mean.abs()), invstd=(invstd, invstd), sc=(sc, sc.abs()),
               sh=(sh, b.abs() + (mean * sc).abs()))
    if rmean is not None:
        m = float(torch.tensor(momentum, dtype=torch.float32))
        unb = var * (n / (n - 1.0)) if n > 1 else var
        rm0, rv0 = rmean.double(), rvar.double()
        out["rmean"] = ((1 - m) * rm0 + m * mean, (1 - m) * rm0.abs() + m * mean.abs())
        out["rvar"] = ((1 - m) * rv0 + m * unb, (1 - m) * rv0.abs() + m * unb)
    return out


# ------------------------------------------------------------------------------------------------------
# forward: h[b][H + q] = act(x * sc + sh) at q = (l + roll) mod L, reflect halo
# ------------------------------------------------------------------------------------------------------
def pre_act(a, ss):
    """(y, ymag) = (x * sc + sh, |x * sc| + |sh|) in fp64 on a [B][L][C] (sc = 1, sh = 0 without ss)."""
    C = a.shape[-1]
    sc, sh, _, _, _ = _consts(C, ss, None, None, a.device)
    x = a.double()
    return x * sc + sh, (x * sc).abs() + sh.abs()


def act_fwd(a, ss, slope, roll, H):
    """a [B][L][C] 16-bit, ss [2][C] fp32 or None, slope [C] fp32 or None (identity) -> (ref, mag)
    [B][L + 2H][C]: the pre-rounding value of every h row, halo rows included."""
    B, L, C = a.shape
    y, ym = pre_act(a, ss)
    if slope is not None:
        sl = slope.double()
        neg = y <= 0
        y = torch.where(neg, y * sl, y)
        ym = torch.where(neg, ym * sl.abs(), ym)
    src = reflect_src(L, H, roll, a.device)
    return y[:, src], ym[:, src]


# ------------------------------------------------------------------------------------------------------
# backward pass 0: g_pre and the reductions
# ------------------------------------------------------------------------------------------------------
def fold_grad(g_h, L, H, roll):
    """Consumer-view gradient g_h [B][L + 2H][C] -> (g, gmag) [B][L][C] at exact positions: the adjoint of
    act_fwd's row map (every consumer row adds into the exact row it was read from)."""
    B, _, C = g_h.shape
    src = reflect_src(L, H, roll, g_h.device)
    gd = g_h.double()
    g = torch.zeros(B, L, C, dtype=torch.float64, device=g_h.device)
    gm = torch.zeros_like(g)
    g.index_add_(1, src, gd)
    gm.index_add_(1, src, gd.abs())
    return g, gm


def bwd_pass0(g_h, g_add, a, ss, mi, slope, roll, H):
    """-> dict gpre=(ref, mag) [B][L][C], red=(ref, mag) [3][C]:
    g_pre = g * (y <= 0 ? slope : 1) + g_add (the skip gradient joins after the activation derivative);
    red0 = sum_{y <= 0} g * y, red1 = sum g_pre, red2 = is * sum g_pre * (x - mu); red2's mag is the centred-at-
    the-flush bound is * sum|g_pre| * (|x| + |mu|) (module docstring)."""
    B, L, C = a.shape
    sc, sh, mu, inv, sl = _consts(C, ss, mi, slope, a.device)
    g, gm = fold_grad(g_h, L, H, roll)
    y, ym = pre_act(a, ss)
    x = a.double()
    zero = torch.zeros_like(g)
    if sl is not None:
        neg = y <= 0
        red0 = torch.where(neg, g * y, zero).sum((0, 1))
        mag0 = torch.where(neg, gm * ym, zero).sum((0, 1))
        gp = torch.where(neg, g * sl, g)
        gpm = torch.where(neg, gm * sl.abs(), gm)
    else:
        red0 = mag0 = zero.sum((0, 1))
        gp, gpm = g, gm
    if g_add is not None:
        gp = gp + g_add.double()
        gpm = gpm + g_add.double().abs()
    red1, mag1 = gp.sum((0, 1)), gpm.sum((0, 1))
    red2 = inv * (gp * (x - mu)).sum((0, 1))
    mag2 = inv.abs() * (gpm * (x.abs() + mu.abs())).sum((0, 1))
    return dict(gpre=(gp, gpm), red=(torch.stack((red0, red1, red2)), torch.stack((mag0, mag1, mag2))))


def bwd_pass1(gpre, a, ss, mi, red, use_bn=True):
    """gpre = (ref, mag) of pass 0, red [S][3][C] fp64 slices -> (ref, mag) [B][L][C] of the BN-backward output
    out = sc * g_pre - sc * r1 - sc * is * r2 * (x - mu), with r1, r2 the slice sums over B * L rounded to fp32 as
    the kernels do; without BN the output is g_pre itself."""
    gp, gpm = gpre
    if not use_bn:
        return gp, gpm
    B, L, C = a.shape
    sc, _, mu, inv, _ = _consts(C, ss, mi, None, a.device)
    rs = red.double().sum(0)
    n = float(B * L)
    r1 = (rs[1] / n).float().double()
    r2 = (rs[2] / n).float().double()
    x = a.double()
    ref = sc * gp - sc * r1 - sc * inv * r2 * (x - mu)
    mag = sc.abs() * (gpm + r1.abs() + (inv * r2).abs() * (x.abs() + mu.abs()))
    return ref, mag


def stat_grads(red, n_stats, g0):
    """red [S][n_stats][C] fp64 slices, g0 = list of the fp32 targets' values before the call (None: skipped) ->
    list of (ref, mag) or None: g_s + sum over slices of red[slice][s]."""
    out = []
    for s in range(3):
        if s >= n_stats or g0[s] is None:
            out.append(None)
            continue
        r = red[:, s].double()
        out.append((g0[s].double() + r.sum(0), g0[s].double().abs() + r.abs().sum(0)))
    return out
