"""The waveform-end glue of the tensor-core route (sg_wave_shiftadd_tanh, sg_wave_col2im_fold, sg_wave_im2col in
its zero-padded mode, sg_tanh_bwd) and the layout / reduction kernels (sg_ncl_to_nlc, sg_nlc_to_ncl, sg_colsum,
sg_convert_f32_rows, sg_deemphasis_segments), each against an fp64 evaluation of its own formula on the 16-bit
operands it reads.  Tolerances follow the rounding of each operation: data movement is bit-exact, a 16-bit store is
one rounding, and an fp32 sum must satisfy |err| <= c * 2^-24 * sum|terms| per output (U below).
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E          # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, SG_F32, BACKEND_TCGEN05  # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream
U = 2.0 ** -24
TDT = {SG_F16: torch.float16, SG_BF16: torch.bfloat16}


@pytest.fixture(params=["f16", "bf16"])
def grad_dtype(request):
    """Runs a test once per 16-bit gradient format (sg_set_grad_dtype)."""
    prev = "bf16" if E.GS == SG_BF16 else "f16"
    E.set_grad_dtype(request.param)
    yield request.param
    E.set_grad_dtype(prev)


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _ratio(err, scale):
    """max over outputs of |err| / (2^-24 * scale): the c of the fp32 reduction bound."""
    return float((err.abs() / (U * scale.clamp_min(1e-300))).max())


def _phase_roll(x, s):
    """discriminator.py:165-172 on the last axis: +s rolls right."""
    return torch.roll(x, shifts=s, dims=-1)


# ------------------------------------------------------------------------------------------------------
# last decoder block: shift-add + bias + tanh
# ------------------------------------------------------------------------------------------------------
def _shiftadd_ref(P, bias):
    """y[b][4m + r] = tanh(bias + sum_{d=-4..4, 0 <= m+d < Lin} P[b][m+d][(d+4)*4 + r]) in fp64, and the sum of
    |terms| of every output."""
    B, Lin, _ = P.shape
    Pd = P.double()
    s = torch.zeros(B, Lin, 4, dtype=torch.float64, device=P.device)
    a = torch.zeros_like(s)
    for d in range(-4, 5):
        blk = Pd[:, :, (d + 4) * 4:(d + 4) * 4 + 4]               # [B][m + d][r]
        lo, hi = max(0, -d), min(Lin, Lin - d)                     # rows m with 0 <= m + d < Lin
        if lo < hi:
            s[:, lo:hi] += blk[:, lo + d:hi + d]
            a[:, lo:hi] += blk[:, lo + d:hi + d].abs()
    b = 0.0 if bias is None else float(bias[0])
    return torch.tanh(s + b).reshape(B, 4 * Lin), (a + abs(b)).reshape(B, 4 * Lin)


@pytest.mark.parametrize("B,Lin,with_bias", [(300, 4096, True), (7, 1000, True), (3, 1000, False), (300, 5, True),
                                             (2, 5, False)])
def test_wave_shiftadd_tanh_vs_index_formula(B, Lin, with_bias):
    """Every output, the rows m < 4 and m >= Lin - 4 whose taps fall off the ends included: within
    c = 8 units of 2^-24 * (|bias| + sum|P|) + tanhf's own error (folded into the same c via |y|)."""
    g = _gen(101)
    P = torch.randn(B, Lin, 64, generator=g).to(DEV)
    P[:, :, 36:] = 1e4                  # columns 36..63 are never read (the GEMM's padding columns)
    bias = torch.tensor([0.3], device=DEV) if with_bias else None
    y = torch.full((B, 4 * Lin), 7.0, device=DEV)
    _lib.call("sg_wave_shiftadd_tanh", _p(P), B, Lin, _p(bias), _p(y), _stream())
    ref, asum = _shiftadd_ref(P, bias)
    torch.cuda.synchronize()
    err = y.double() - ref
    c = _ratio(err, asum + ref.abs())
    edge = torch.cat((err[:, :16], err[:, -16:]), 1).abs().max()
    print("shiftadd_tanh B=%d Lin=%d: max |err| %.3e (edges %.3e), c = %.2f (tol 8)" % (B, Lin, float(err.abs().max()),
                                                                                       float(edge), c))
    assert c <= 8.0


def test_wave_last_block_gemm_plus_shiftadd_vs_transposed_conv():
    """The default waveform route of G's last block: the W2_last GEMM (engine.run_f, column jj = (d+4)*4 + r holds
    tap k = -4d + r + 13) followed by sg_wave_shiftadd_tanh, against tanh(ConvTranspose1d(k 31, s 4, p 13)[:-1])
    in fp64 on the same fp16 operands (modules.py:135-141), two sources as the skip concat reads them."""
    g = _gen(102)
    B, Lin, c0, c1 = 5, 1024, 64, 64
    x0 = torch.randn(B, Lin, c0, generator=g).to(torch.float16).to(DEV)
    x1 = torch.randn(B, Lin, c1, generator=g).to(torch.float16).to(DEV)
    weff = (0.05 * torch.randn(c0 + c1, 31, generator=g)).to(DEV)
    bias = torch.tensor([0.05], device=DEV)
    kidx = E.dec_last_tap_index(torch.device(DEV))
    w2 = (weff.t()[kidx.clamp(min=0)] * (kidx >= 0).float().unsqueeze(1)).half().contiguous()   # [64][cin]
    P = torch.zeros(B, Lin, 64, device=DEV)
    E.run_f(x0, x1, Lin, 0, SG_F16, w2, SG_F16, c0 + c1, 64, E.tap_ranges("full", 0, c0 + c1, 64), P, SG_F32, Lin, 0,
            0, Lin, B, d_lo=0, d_hi=0, w_tap0=4, a0_c=c0, a1_c=c1, backend=BACKEND_TCGEN05)
    y = torch.empty(B, 4 * Lin, device=DEV)
    _lib.call("sg_wave_shiftadd_tanh", _p(P), B, Lin, _p(bias), _p(y), _stream())
    x = torch.cat((x0, x1), -1).double().permute(0, 2, 1)
    w = weff.half().double().view(c0 + c1, 1, 31)
    pre = F.conv_transpose1d(x, w, bias.double(), stride=4, padding=13)[:, 0, :-1]
    asum = F.conv_transpose1d(x.abs(), w.abs(), None, stride=4, padding=13)[:, 0, :-1] + abs(float(bias))
    ref = torch.tanh(pre)
    torch.cuda.synchronize()
    err = y.double() - ref
    c = _ratio(err, asum + ref.abs())
    print("last block GEMM + shiftadd: max |err| %.3e, c = %.2f (tol 16)" % (float(err.abs().max()), c))
    assert c <= 16.0


# ------------------------------------------------------------------------------------------------------
# D input gradient: reflect fold + phase un-roll (the adjoint of sg_wave_im2col, reflect, off 14)
# ------------------------------------------------------------------------------------------------------
def _im2col_reflect64(x, roll):
    """[B][L] fp64 -> [B][L/4][31]: pad(shift(x))[4t + k - 14], reflect padding (14, 15)."""
    xp = F.pad(_phase_roll(x, roll).unsqueeze(1), (14, 15), mode="reflect").squeeze(1)
    return xp.unfold(1, 31, 4)


@pytest.mark.parametrize("col0", [0, 32])
@pytest.mark.parametrize("roll,roll_on_device", [(0, False), (3, False), (-5, False), (4, True), (-2, True)])
def test_wave_col2im_fold_is_the_adjoint_of_im2col(col0, roll, roll_on_device, grad_dtype):
    """gx += fold(P2) must be im2col^T P2: against the fp64 autograd adjoint of the reflect im2col per sample
    (c = 4 on the fold's fp32 sums and the accumulation onto a nonzero gx), and as the identity
    <im2col(x), P2> = <x, fold(P2)> with the kernel's own im2col (x exactly representable in 16 bits).
    Columns 31 and 63 and the other channel's half of P2 hold garbage that must not be read."""
    g = _gen(103)
    B, L = 3, 4096
    Lq = L // 4
    gt = TDT[E.GS]
    P2 = torch.randn(B, Lq, 64, generator=g).to(gt)
    P2[:, :, 31] = 3e3
    P2[:, :, 63] = -3e3
    other = 32 - col0
    P2[:, :, other:other + 31] *= 1e3
    P2 = P2.to(DEV)
    gx0 = torch.randn(B, L, generator=g).to(DEV)
    gx = gx0.clone()
    rdev = torch.tensor([9, roll], dtype=torch.int32, device=DEV)
    rptr = C.c_void_p(rdev.data_ptr() + 4) if roll_on_device else None
    _lib.call("sg_wave_col2im_fold", _p(P2), col0, B, L, 0 if roll_on_device else roll, rptr, _p(gx), _stream())
    # fp64 adjoint
    x64 = torch.zeros(B, L, dtype=torch.float64, device=DEV, requires_grad=True)
    p = P2[:, :, col0:col0 + 31].double()
    (_im2col_reflect64(x64, roll) * p).sum().backward()
    ref = x64.grad
    xa = torch.zeros(B, L, dtype=torch.float64, device=DEV, requires_grad=True)
    (_im2col_reflect64(xa, roll) * p.abs()).sum().backward()
    torch.cuda.synchronize()
    err = gx.double() - gx0.double() - ref
    c = _ratio(err, xa.grad + gx0.double().abs() + ref.abs())
    print("col2im_fold %s col0=%d roll=%d dev=%s: max |err| %.3e, c = %.2f (tol 4)"
          % (grad_dtype, col0, roll, roll_on_device, float(err.abs().max()), c))
    assert c <= 4.0
    # <im2col(x), P2> = <x, fold(P2)> with the kernel's im2col; x = k / 64, |k| < 256: exact in fp16 and bf16
    x = (torch.randint(-255, 256, (B, L), generator=g).double() / 64).float().to(DEV)
    col = torch.zeros(B, Lq, 64, dtype=gt, device=DEV)
    cols = (_p(col), None) if gt == torch.float16 else (None, _p(col))
    _lib.call("sg_wave_im2col", _p(x), _p(x), 2, B, L, roll, None, 1, 14, cols[0], cols[1], _stream())
    fold = torch.zeros(B, L, device=DEV)
    _lib.call("sg_wave_col2im_fold", _p(P2), col0, B, L, roll, None, _p(fold), _stream())
    torch.cuda.synchronize()
    lhs = float((col[:, :, col0:col0 + 31].double() * p).sum())
    rhs = float((x.double() * fold.double()).sum())
    bound = 4 * U * float((x.double().abs() * xa.grad).sum())
    assert abs(lhs - rhs) <= bound, (lhs, rhs, bound)


@pytest.mark.parametrize("which", ["f16", "bf16"])
@pytest.mark.parametrize("L", [16384, 4096, 1280])
def test_wave_im2col_zero_padding_mode(L, which):
    """The mode G's backward uses on d loss / d pre-tanh (engine.py: reflect 0, off 13, one 16-bit copy only):
    col[b][t][k] = zero-pad(x)[4t + k - 13] for k < 31, columns 31..63 zero; bit-exact against F.pad(...).unfold."""
    g = _gen(104)
    B = 3
    x = torch.randn(B, L, generator=g).to(DEV)
    tdt = torch.float16 if which == "f16" else torch.bfloat16
    col = torch.full((B, L // 4, 64), 7.0, dtype=tdt, device=DEV)
    cols = (_p(col), None) if which == "f16" else (None, _p(col))
    _lib.call("sg_wave_im2col", _p(x), None, 1, B, L, 0, None, 0, 13, cols[0], cols[1], _stream())
    ref = torch.zeros(B, L // 4, 64, dtype=tdt, device=DEV)
    ref[:, :, :31] = F.pad(x, (13, 14)).unfold(1, 31, 4).to(tdt)
    torch.cuda.synchronize()
    assert torch.equal(col, ref)


@pytest.mark.parametrize("n,with_bias", [(100003, True), (300 * 16384, True), (300 * 16384, False), (77, True)])
def test_tanh_bwd(n, with_bias):
    """gpre = gy * (1 - y^2) per element (c = 3 of 2^-24 * |gy| * (1 + y^2)); dbias accumulates sum(gpre) onto its
    nonzero value (c = 8 of 2^-24 * (sum|gpre| + |dbias0|)); dbias = NULL writes gpre alone."""
    g = _gen(105)
    gy = torch.randn(n, generator=g).to(DEV)
    y = torch.tanh(2 * torch.randn(n, generator=g)).to(DEV)
    gpre = torch.full((n,), 7.0, device=DEV)
    db0 = 3.0
    db = torch.tensor([db0], device=DEV) if with_bias else None
    _lib.call("sg_tanh_bwd", _p(gy), _p(y), n, _p(gpre), _p(db), _stream())
    gy64, y64 = gy.double(), y.double()
    ref = gy64 * (1 - y64 * y64)
    torch.cuda.synchronize()
    c = _ratio(gpre.double() - ref, gy64.abs() * (1 + y64 * y64))
    print("tanh_bwd n=%d: gpre c = %.2f (tol 3)" % (n, c))
    assert c <= 3.0
    if with_bias:
        e = float(db) - (db0 + float(ref.sum()))
        cb = abs(e) / (U * (float(ref.abs().sum()) + db0))
        print("tanh_bwd n=%d: dbias err %.3e, c = %.2f (tol 8)" % (n, e, cb))
        assert cb <= 8.0


# ------------------------------------------------------------------------------------------------------
# layout and reductions
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [SG_F16, SG_BF16])
@pytest.mark.parametrize("B,Cc,L", [(3, 100, 37), (2, 37, 100), (4, 1024, 16), (1, 64, 64)])
def test_ncl_nlc_layout_bit_exact(B, Cc, L, dtype):
    """fp32 NCL -> 16-bit NLC (the z input) and 16-bit NLC -> fp32 NCL (hall outputs): pure layout plus one
    round-to-nearest, bit for bit, with C and L not multiples of the 32 x 32 tile."""
    g = _gen(106)
    tdt = TDT[dtype]
    src = torch.randn(B, Cc, L, generator=g).to(DEV)
    dst = torch.full((B, L, Cc), 7.0, dtype=tdt, device=DEV)
    _lib.call("sg_ncl_to_nlc", _p(src), B, Cc, L, _p(dst), dtype, _stream())
    s16 = torch.randn(B, L, Cc, generator=g).to(tdt).to(DEV)
    back = torch.full((B, Cc, L), 7.0, device=DEV)
    _lib.call("sg_nlc_to_ncl", _p(s16), dtype, B, Cc, L, _p(back), _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst, src.permute(0, 2, 1).to(tdt))
    assert torch.equal(back, s16.permute(0, 2, 1).float())


@pytest.mark.parametrize("dtype", [SG_F16, SG_BF16])
@pytest.mark.parametrize("rows,Cc,mod,accumulate", [(20011, 64, 64, 0), (20011, 64, 64, 1), (1003, 256, 64, 1),
                                                    (4097, 1024, 1024, 0), (300 * 16, 1024, 256, 1), (7, 512, 128, 0)])
def test_colsum_vs_fp64(rows, Cc, mod, accumulate, dtype):
    """out[m] (= out[m] +) sum over rows and channels c = m (mod `mod`): c = 8 of 2^-24 * (sum|terms| + |out0|)."""
    g = _gen(107)
    tdt = TDT[dtype]
    a = torch.randn(rows, Cc, generator=g).to(tdt).to(DEV)
    out0 = torch.randn(mod, generator=g).to(DEV)
    out = out0.clone()
    tmp = torch.full((8 * Cc,), 5.0, dtype=torch.float64, device=DEV)     # the kernel clears its workspace
    _lib.call("sg_colsum", _p(a), dtype, rows, Cc, mod, _p(out), accumulate, _p(tmp), _stream())
    a64 = a.double()
    ref = a64.sum(0).view(Cc // mod, mod).sum(0)
    asum = a64.abs().sum(0).view(Cc // mod, mod).sum(0)
    if accumulate:
        ref = ref + out0.double()
        asum = asum + out0.double().abs()
    torch.cuda.synchronize()
    c = _ratio(out.double() - ref, asum)
    print("colsum rows=%d C=%d mod=%d acc=%d: c = %.2f (tol 8)" % (rows, Cc, mod, accumulate, c))
    assert c <= 8.0


@pytest.mark.parametrize("dtype", [SG_F16, SG_BF16])
def test_convert_f32_rows_subrange_and_saturation(dtype):
    """out[r][col0 + c] = 16-bit(ws[r][col0 + c]) for c < ncols, ld > ncols: the columns outside the range keep
    their bits; fp16 saturates to +-65504 like the tap-GEMM epilogue (cvt.rn.satfinite), bf16 rounds to nearest."""
    g = _gen(108)
    tdt = TDT[dtype]
    rows, ld, col0, ncols = 37, 96, 16, 48
    ws = torch.randn(rows, ld, generator=g) * 3e4           # |x| up to ~1.5e5: many fp16 overflows
    ws[0, col0:col0 + 8] = torch.tensor([65504.0, 65519.0, 65520.0, 1e30, -65520.0, -1e30, 6e-8, -0.0])
    ws = ws.to(DEV)
    out0 = torch.randn(rows, ld, generator=g).to(tdt).to(DEV)
    out = out0.clone()
    _lib.call("sg_convert_f32_rows", _p(ws), _p(out), dtype, rows, ld, col0, ncols, _stream())
    sl = slice(col0, col0 + ncols)
    exp = ws[:, sl].clamp(-65504.0, 65504.0).half() if dtype == SG_F16 else ws[:, sl].bfloat16()
    torch.cuda.synchronize()
    assert torch.equal(out[:, sl], exp)
    assert torch.equal(out[:, :col0], out0[:, :col0]) and torch.equal(out[:, col0 + ncols:], out0[:, col0 + ncols:])
    if dtype == SG_F16:
        assert bool(torch.isfinite(out.float()).all())


def test_convert_f32_rows_matches_direct_16bit_epilogue(monkeypatch):
    """The split-K tail stores fp32 sums and converts them with sg_convert_f32_rows; the direct launch rounds in
    its epilogue.  On the same accumulators the two must store the same bits, saturated values included."""
    monkeypatch.setattr(E, "STREAM_K", False)          # one schedule for both launches: identical fp32 accumulators
    g = _gen(109)
    B, cin, cout, R, halo = 3, 64, 128, 160, 4
    kc, nc = 4 * cin, cout
    taps = E.tap_ranges("conv_fwd", cin, kc, nc)
    w = torch.randn(9, nc, kc, generator=g) * 2000.0       # outputs ~1e5: about half of them saturate
    for i in range(9):
        mask = torch.zeros(nc, kc)
        mask[taps[2][i]:taps[3][i], taps[0][i]:taps[1][i]] = 1
        w[i] *= mask
    w = w.to(torch.float16).to(DEV)
    a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    bias = torch.randn(nc, generator=g).to(DEV)
    direct = torch.zeros(B, R, nc, dtype=torch.float16, device=DEV)
    E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, nc, taps, direct, SG_F16, R, 0, 0, R, B, bias=bias, bias_mod=nc,
            backend=BACKEND_TCGEN05)
    acc = torch.zeros(B, R, nc, device=DEV)
    E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, nc, taps, acc, SG_F32, R, 0, 0, R, B, bias=bias, bias_mod=nc,
            backend=BACKEND_TCGEN05)
    conv = torch.zeros_like(direct)
    _lib.call("sg_convert_f32_rows", _p(acc), _p(conv), SG_F16, B * R, nc, 0, nc, _stream())
    torch.cuda.synchronize()
    sat = float((acc.abs() > 65504).float().mean())
    print("direct vs fp32 + convert: %.1f %% of the outputs saturate" % (100 * sat))
    assert sat > 0.05
    assert torch.equal(conv, direct)


def test_deemphasis_segments_vs_iir():
    """clean.py's batched de-emphasis: every segment filtered from a zero state (lengths 1, 4096, 5000, 4097 and
    170000 > 10 s at 16 kHz), against scipy's fp64 IIR x[n] = c x[n-1] + y[n]: c = 32 of 2^-24 times the same
    filter applied to |y|.  Samples between segments are left untouched."""
    from scipy.signal import lfilter
    coef = 0.95
    g = np.random.default_rng(110)
    lens = [1, 4096, 5000, 4097, 170000]
    gaps = [3, 0, 11, 1, 5]
    segs, off = [], 0
    for n, gap in zip(lens, gaps):
        off += gap
        segs.append((off, n))
        off += n
    total = off + 7
    y = (0.3 * g.standard_normal(total)).astype(np.float32)
    y[segs[-1][0]:segs[-1][0] + 1000] += 0.8           # a DC step: the state carries across 1024 x 4 chunks
    yd = torch.from_numpy(y).to(DEV)
    x = torch.full((total,), 7.0, device=DEV)
    seg = torch.tensor([v for s in segs for v in s], dtype=torch.int64, device=DEV)
    _lib.call("sg_deemphasis_segments", _p(yd), _p(seg), len(segs), coef, _p(x), _stream())
    torch.cuda.synchronize()
    xs = x.cpu().numpy().astype(np.float64)
    inside = np.zeros(total, dtype=bool)
    worst = 0.0
    for o, n in segs:
        yy = y[o:o + n].astype(np.float64)
        ref = lfilter([1.0], [1.0, -coef], yy)
        scale = lfilter([1.0], [1.0, -coef], np.abs(yy))
        worst = max(worst, float(np.max(np.abs(xs[o:o + n] - ref) / (U * scale + 1e-300))))
        inside[o:o + n] = True
    print("deemphasis_segments: c = %.2f (tol 32)" % worst)
    assert worst <= 32.0
    assert np.all(xs[~inside] == 7.0)
