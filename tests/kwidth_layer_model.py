"""fp64 references of the hidden stride-4 layers at kernel width k (not collected; plain torch, runs on any device, no
kernels).  Each is written from the reference modules' semantics -- F.conv1d on the reflect-padded input, the
ConvTranspose1d of GDeconv1DBlock -- and never from the engine's tap tables or packed layouts, so a table or packing
error cannot cancel out of a comparison with them.

Activations are in the engine's row layout: a tensor of positions [B][C][4R] is stored as rows [B][R][4C], element
(row m, phase p, channel c) = position 4m + p (rows_to_ncl / ncl_to_rows).  Every function takes its operands as they
are (the caller rounds them to the launch's 16-bit format first) and returns (value, magnitude) in float64: the
magnitude is the same operation applied to |operands|, the sum of the absolute values of the terms that make up each
element, which scales the rounding-error gates of tests/tapgemm_model.py.

  encoder / D conv      y = conv1d(xp[16 - (k//2 - 1) : 16 + L + k//2], W, stride 4)
                        xp: L positions between two 16-position halos (sg_act_fwd writes them as reflections)
  conv data gradient    d y / d xp over all L + 32 positions: zero where the conv never reads
  deconv                y = conv_transpose1d(x, W, stride 4, padding (k - 4)//2), its last sample dropped for odd k
                        (GDeconv1DBlock's padding max(0, (4 - k) // -2) and the trim of santi-pdp/segan_pytorch
                        segan/models/modules.py:137-138)
  weight gradients      d y / d W in the reference layouts W[cout][cin][k] (conv) and W[cin][cout][k] (deconv)"""
import torch
import torch.nn.functional as F

HALO = 16            # positions of reflect halo on each side of an encoder activation
WIDTHS = list(range(4, 33))


def rows_to_ncl(a, c):
    """[B][R][4c] -> [B][c][4R]"""
    B, R, _ = a.shape
    return a.reshape(B, R, 4, c).permute(0, 3, 1, 2).reshape(B, c, 4 * R)


def ncl_to_rows(x):
    """[B][c][4R] -> [B][R][4c]"""
    B, c, P = x.shape
    return x.reshape(B, c, P // 4, 4).permute(0, 2, 3, 1).reshape(B, P // 4, 4 * c)


def _pair(fn, *ops):
    """(fn(ops), fn(|ops|)) in float64."""
    ops = [None if t is None else t.double() for t in ops]
    return fn(*ops), fn(*[None if t is None else t.abs() for t in ops])


def _conv(xp, w, k):
    L = xp.shape[-1] - 2 * HALO
    return F.conv1d(xp[..., HALO - (k // 2 - 1):HALO + L + k // 2], w, stride=4)


def _deconv(x, w, k):
    y = F.conv_transpose1d(x, w, stride=4, padding=(k - 4) // 2)
    return y[..., :-1] if k % 2 else y


def _grad(fn, wrt, gy, *ops):
    """d <fn(ops), gy> / d ops[wrt]: the layer is linear in each operand, so the value of ops[wrt] does not matter."""
    ops = list(ops)
    ops[wrt] = torch.zeros_like(ops[wrt]).requires_grad_(True)
    return torch.autograd.grad(fn(*ops), ops[wrt], gy)[0]


def conv_fwd(xp, w, k, bias=None):
    """xp [B][cin][L + 32], w [cout][cin][k], bias [cout] -> [B][cout][L/4]"""
    def f(x_, w_, b_):
        y = _conv(x_, w_, k)
        return y if b_ is None else y + b_.view(1, -1, 1)
    return _pair(f, xp, w, bias)


def conv_dgrad(gy, w, k):
    """gy [B][cout][Lq], w [cout][cin][k] -> d / d xp: [B][cin][4 Lq + 32]"""
    B, _, Lq = gy.shape

    def f(g_, w_):
        xp = torch.zeros(B, w_.shape[1], 4 * Lq + 2 * HALO, dtype=g_.dtype, device=g_.device)
        return _grad(lambda x, ww: _conv(x, ww, k), 0, g_, xp, w_)
    return _pair(f, gy, w)


def conv_wgrad(xp, gy, k):
    """xp [B][cin][4 Lq + 32], gy [B][cout][Lq] -> d / d W: [cout][cin][k]"""
    def f(x_, g_):
        w = torch.zeros(g_.shape[1], x_.shape[1], k, dtype=g_.dtype, device=g_.device)
        return _grad(lambda ww, x: _conv(x, ww, k), 0, g_, w, x_)
    return _pair(f, xp, gy)


def deconv_fwd(x, w, k, bias=None):
    """x [B][cin][Lin], w [cin][cout][k], bias [cout] -> [B][cout][4 Lin]"""
    def f(x_, w_, b_):
        y = _deconv(x_, w_, k)
        return y if b_ is None else y + b_.view(1, -1, 1)
    return _pair(f, x, w, bias)


def deconv_dgrad(gy, w, k):
    """gy [B][cout][4 Lin], w [cin][cout][k] -> d / d x: [B][cin][Lin]"""
    B, _, P = gy.shape

    def f(g_, w_):
        x = torch.zeros(B, w_.shape[0], P // 4, dtype=g_.dtype, device=g_.device)
        return _grad(lambda xx, ww: _deconv(xx, ww, k), 0, g_, x, w_)
    return _pair(f, gy, w)


def deconv_wgrad(x, gy, k):
    """x [B][cin][Lin], gy [B][cout][4 Lin] -> d / d W: [cin][cout][k]"""
    def f(x_, g_):
        w = torch.zeros(x_.shape[1], g_.shape[1], k, dtype=g_.dtype, device=g_.device)
        return _grad(lambda ww, xx: _deconv(xx, ww, k), 0, g_, w, x_)
    return _pair(f, x, gy)


def packed_live(kind, k, c_out, c_in, device=None):
    """bool [9][nc][kc]: the elements of a packed master M[d + 4][nc][kc] that hold a weight of a width-k layer, from
    the modules' index arithmetic.  Conv (kind 0): M[d+4][co][p*cin + ci] = W[co][ci][j], j = 4d + p + (k//2 - 1),
    the input position 4(m + d) + p that output m reads at tap j.  Deconv (kind 1): M[d+4][r*cout + co][ci] =
    W[ci][co][j], j = -4d + r + (k - 4)//2, the tap that carries input row m + d to output position 4m + r.  Every
    other element is a structural zero."""
    d = torch.arange(-4, 5, device=device).view(9, 1)
    p = torch.arange(4, device=device).view(1, 4)
    if kind == 0:
        j = 4 * d + p + (k // 2 - 1)
        ok = (j >= 0) & (j < k)                                       # [9][phase]
        return ok.view(9, 1, 4, 1).expand(9, c_out, 4, c_in).reshape(9, c_out, 4 * c_in)
    j = -4 * d + p + (k - 4) // 2
    ok = (j >= 0) & (j < k)
    return ok.view(9, 4, 1, 1).expand(9, 4, c_out, c_in).reshape(9, 4 * c_out, c_in)
