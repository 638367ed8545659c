"""fp64 references and the rounding-error yardstick of the two tap-GEMM forms (not collected; plain torch, runs on
any device, no kernels).

Both forms multiply 16-bit operands exactly and accumulate in fp32, so whatever the summation order an output
element is off by a small multiple of U * mag, U = 2^-24 and mag = the same sum over the absolute values of its
terms (plus, on the tensor cores, the accumulator's truncation: see c_w).  c_w / c_f express an observed error in
those units; the GPU tests gate them at C_TOL.  A 16-bit store adds half an ulp of the output format, which c_f
takes off first.

  form W:  dW[d][n][kc] += sum_{b,m} G[b][m][n] * A[b][m + d][kc]         (rows outside A's buffer read as zero)
  form F:  out[b][m][n]  = bias[n % bias_mod] + sum_d sum_kc A[b][m + d][kc] * W[d + 4 - w_tap0][n][kc]
Only the (n, kc) box of a tap's table entry is live; everything else is structurally zero."""
import torch

U = 2.0 ** -24
C_TOL = 16.0          # gate on c_w / c_f
MANT = {"f16": 11, "bf16": 8}       # significant bits


def shifted_rows(a, a_halo, d, rows, m_lo=0):
    """a [B][R + 2 a_halo][C] -> [B][rows][C]: buffer rows m_lo + d .. m_lo + d + rows of every batch element's OWN
    buffer, zeros where that leaves the buffer."""
    B, RH, C = a.shape
    lo = a_halo + m_lo + d
    clo, chi = max(lo, 0), min(lo + rows, RH)
    out = a.new_zeros(B, rows, C)
    if chi > clo:
        out[:, clo - lo:chi - lo] = a[:, clo:chi]
    return out


def _cat(a0, a1):
    return a0 if a1 is None else torch.cat((a0, a1), -1)


def ref_w(g, a0, a1, a_halo, taps, d_lo=-4, d_hi=4):
    """(ref, mag), float64 [d_hi - d_lo + 1][nc][kc] on g's device; zero outside each tap's live (n, kc) box."""
    B, R, nc = g.shape
    kc = a0.shape[-1] + (a1.shape[-1] if a1 is not None else 0)
    G = g.double().reshape(B * R, nc).t().contiguous()
    Gabs = G.abs()
    ref = torch.zeros(d_hi - d_lo + 1, nc, kc, dtype=torch.float64, device=g.device)
    mag = torch.zeros_like(ref)
    for d in range(d_lo, d_hi + 1):
        i = d + 4
        k0, k1, n0, n1 = taps[0][i], taps[1][i], taps[2][i], taps[3][i]
        A = torch.cat([shifted_rows(a, a_halo, d, R)[..., max(k0 - c0, 0):max(k1 - c0, 0)]
                       for a, c0 in ((a0, 0), (a1, a0.shape[-1])) if a is not None], -1)
        A = A.double().reshape(B * R, k1 - k0)
        ref[d - d_lo, n0:n1, k0:k1] = G[n0:n1] @ A
        mag[d - d_lo, n0:n1, k0:k1] = Gabs[n0:n1] @ A.abs()
    return ref, mag


def ref_f(a0, a1, a_halo, w, taps, m_lo, m_hi, d_lo=-4, d_hi=4, w_tap0=0, bias=None):
    """(ref, mag), float64 [B][m_hi - m_lo][nc] on a0's device.  w [slots][nc][kc]; only each tap's live box of it
    is read.  bias [bias_mod]: channel n adds bias[n % bias_mod]."""
    a = _cat(a0, a1)
    B, nc = a.shape[0], w.shape[1]
    rows = m_hi - m_lo
    ref = torch.zeros(B, rows, nc, dtype=torch.float64, device=a.device)
    mag = torch.zeros_like(ref)
    for d in range(d_lo, d_hi + 1):
        i = d + 4
        k0, k1, n0, n1 = taps[0][i], taps[1][i], taps[2][i], taps[3][i]
        A = shifted_rows(a, a_halo, d, rows, m_lo)[..., k0:k1].double()
        Wt = w[i - w_tap0, n0:n1, k0:k1].double().t()
        ref[..., n0:n1] += A @ Wt
        mag[..., n0:n1] += A.abs() @ Wt.abs()
    if bias is not None:
        b = bias.double()[torch.arange(nc, device=bias.device) % bias.numel()]
        ref += b
        mag += b.abs()
    return ref, mag


def prelu_ref(ref, mag, slope):
    """PReLU applied to the fp32 value before the one rounding: (act, mag_act).  slope [slope_mod] repeats over n."""
    s = slope.double()[torch.arange(ref.shape[-1], device=slope.device) % slope.numel()]
    act = torch.where(ref > 0, ref, ref * s)
    return act, torch.where(ref > 0, mag, mag * s.abs() + act.abs())


def sign_safe(ref, mag):
    """Elements whose sign no fp32 summation order can flip (PReLU picks its branch by it)."""
    return ref.abs() > C_TOL * U * mag


def _ratio(err, den):
    r = torch.where(den > 0, err / den.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return float(r.max()) if r.numel() else 0.0


TRUNC_PER_STAGE = 1.0 / 32     # x C_TOL = U * mag / 2 per 64-position stage


def c_w(got, ref, mag, scale=1.0, trunc_stages=0):
    """max |got - scale * ref| / (U * |scale| * mag).  Where mag == 0 any difference is infinite.
    trunc_stages: wgmma adds every 16-position block into its fp32 accumulator with truncation, not rounding to
    nearest, so a tensor-core sum loses up to an ulp of the running sum per block, always towards zero: the error
    grows with the number of 64-position stages one accumulator walks instead of averaging out (measured on an
    H100: the result shrinks by 1.1 * U of itself per stage on average; an element's error follows the size of its
    partial sums, not of its final value).  The gate allows U * mag / 2 per stage on top of C_TOL * U * mag."""
    den = mag * (1.0 + TRUNC_PER_STAGE * trunc_stages)
    return _ratio((got.double() - scale * ref).abs(), U * abs(scale) * den)


def half_ulp(v, fmt):
    """Half the spacing of the 16-bit format at v (fp16: subnormal spacing 2^-24 below 2^-14)."""
    p = MANT[fmt]
    e = torch.frexp(v.double().abs())[1]                   # |v| = m * 2^e, m in [0.5, 1)
    e = e.clamp_min(-13 if fmt == "f16" else -125)
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - p - 1)


def c_f(got16, ref, mag, fmt, trunc_stages=0):
    """The error of a 16-bit store in excess of half an output ulp, over U * mag.  fp16 stores saturate at +-65504.
    trunc_stages: as in c_w (the same accumulator), a number or a tensor that broadcasts against ref (per column)."""
    tgt = ref.clamp(-65504.0, 65504.0) if fmt == "f16" else ref
    err = (got16.double() - tgt).abs() - half_ulp(tgt, fmt)
    return _ratio(err.clamp_min(0.0), U * mag * (1.0 + TRUNC_PER_STAGE * trunc_stages))


def c_pair(got_a, got_b, mag, fmt=None, trunc_stages=0):
    """Distance between two results of the same launch in the units of c_f / c_w: each may be off the fp64 value by
    C_TOL (and, stored in a 16-bit format, by half an ulp of itself), so two correct ones stay within 2 C_TOL."""
    err = (got_a.double() - got_b.double()).abs()
    if fmt is not None:
        err = (err - half_ulp(got_a, fmt) - half_ulp(got_b, fmt)).clamp_min(0.0)
    return _ratio(err, U * mag * (1.0 + TRUNC_PER_STAGE * trunc_stages))


def f_stages(taps, d_lo, d_hi, n0, n1, split=1):
    """64-channel k-steps one form-F tensor-core accumulator walks for the tile of columns [n0, n1): every live tap
    whose N range overlaps the tile contributes its K range; a tile split `split` ways (stream-K pieces, interleaved
    fp32 k-split) gives each piece at most ceil(steps / split), and the pieces are added in fp32 with rounding."""
    steps = sum((taps[1][d + 4] - taps[0][d + 4]) // 64 for d in range(d_lo, d_hi + 1)
                if taps[2][d + 4] < n1 and taps[3][d + 4] > n0)
    return -(-steps // max(1, split))
