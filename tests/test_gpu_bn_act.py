"""The BatchNorm / PReLU streaming kernels (sg_bn_stats, sg_bn_finalize, sg_act_fwd, sg_act_bwd_reduce,
sg_act_bwd_apply, sg_stat_grads) and the BatchNorm statistics of the tap-GEMM epilogue (TapGemmF.bn_stats), each
against the fp64 evaluation of its own formula on the 16-bit operands it reads (tests/bn_act_model.py), at rounding-
level gates: c <= C_TOL = 16 in units of 2^-24 * sum|terms| (half an output ulp taken off 16-bit stores; sums of long
fp32 runs included: `adds` in the printed tags is the longest run one fp32 partial makes).  Every output sits between
guard bands that must keep their bits; the statistics targets start non-zero and the kernels must add to them.  The pointwise outputs must
have the same bits (+0 and -0 equal) under every variant (sg_set_ew_variant: vec, unroll, cap) -- "every variant
computes identical values" (elementwise.cu).

Which kernel each variant reaches (elementwise.cu sg_bn_stats .. sg_act_bwd_apply; _fwd_kernel / _bwd_kernel below
mirror the rules and test_every_instantiation_is_reached checks the tables cover all 24):
  bn_stats   vec 16 -> bn_stats_bulk; (vec, unroll) -> bn_stats_kernel<vec, unroll>           (STATS_VARIANTS, all)
  act_fwd    vec 16 -> act_fwd_bulk if no bf16 twins and (H == 0 or L >= 2H + 3), else act_fwd_kernel<8, 4>;
             (vec, unroll) -> act_fwd_kernel<vec, unroll>                                      (FWD_VARIANTS, all)
  act_bwd    vec 16 and g_h (and g_add) contiguous -> act_bwd_bulk<MODE>; vec >= 8 and ldh, lda % 8 == 0 ->
             act_bwd_tiled_kernel<MODE, unroll >= 4 ? 4 : 2>; otherwise act_bwd_kernel<MODE, 4, unroll>

  forward case           C     B    L     H   roll   a     reaches with FWD_VARIANTS
  c64_L35_min_rollLm1    64    3    35    16  34     f16   bulk, <4,2|4|8>, <8,2|4>
  c128_L20_fallback      128   3    20    16  -5     bf16  <8,4> (vec 16: H < L < 2H + 3), <4,2|4|8>, <8,2|4>
  c256_L37_twins         256   17   37    16  1      f16   <8,4> (vec 16: bf16 twins), <4,2|4|8>, <8,2|4>
  c512_L1000_noH_roll1mL 512   3    1000  0   -999   bf16  bulk, <4,2|4|8>, <8,2|4>
  c1024_L100_none        1024  1    100   16  5      f16   (act NONE) bulk, <4,2|4|8>, <8,2|4>
  c64_L4096_tilewrap     64    3    4096  16  512    f16   bulk (wrap on a 256-row tile boundary), registers
  c128_L1024_tilewrap    128   3    1024  16  -256   bf16  bulk (wrap on a 128-row tile boundary), registers
  c256_L256_saturate     256   3    256   16  -1     f16   bulk, registers; |x * sc + sh| up to ~1e5
  c1024_L16_last         1024  17   16    0   0      f16   bulk, registers
  c512_L64_twins_sat     512   3    64    16  -5     f16   <8,4> (twins), registers; saturating fp16 h

  backward case          C     B    L     H   roll   a     g_h / g_add          BN   reaches with BWD_VARIANTS
  c64_L35_bn_rollLm1     64    3    35    16  34     f16   contiguous           yes  bulk, tiled<2|4>, <4,2|4|8>
  c128_L37_skip_strided  128   17   37    16  -1     f16   ldh zc+C, lda 2C     no   tiled<2|4> (vec 16 too), <4,..>
  c256_L100_bn_ldh4      256   3    100   16  5      bf16  ldh C + 4            yes  <4,2|4|8> only (every variant)
  c1024_L1000_bn_noH     1024  1    1000  0   -999   f16   contiguous           yes  bulk, tiled<2|4>, <4,2|4|8>
  c512_L64_bn            512   3    64    16  -5     bf16  contiguous           yes  bulk, tiled<2|4>, <4,2|4|8>
  c64_L1024_skip_sat     64    3    1024  16  256    f16   contiguous + g_add   no   bulk (3 tensors), tiled, generic;
                                                                                     |g_pre| up to ~1.2e5
  c128_L4096_bn_tilewrap 128   1    4096  16  -640   f16   contiguous           yes  bulk (wrap on a 64-row tile)
  c1024_L16_last_zc      1024  17   16    0   0      f16   ldh zc + C           no   tiled<2|4>, <4,..>
The D chain (batch 300, five layers) and the fused statistics (D conv layers 1-4 at batch 300) run at the default
variants and at one non-default set each.
Run on an H100:  python -m pytest tests/test_gpu_bn_act.py -m gpu"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E          # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, SG_F32, BACKEND_TCGEN05  # noqa: E402
from tests import bn_act_model as M                        # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream
ACT_NONE, ACT_PRELU = 0, 1
SL = M.SLICES
NUM_SMS = 132
SENT = 0x7E5A                       # guard-band bits (an fp16 NaN)
TDT = {SG_F16: torch.float16, SG_BF16: torch.bfloat16}
FMT = {SG_F16: "f16", SG_BF16: "bf16"}

EW_DEFAULT = {1: (16, 4, 2), 2: (4, 8, 3), 3: (16, 4, 2), 4: (16, 4, 2)}    # elementwise.cu g_ew
EW_REGISTER = {1: (8, 4, 2), 2: (4, 4, 3), 3: (8, 2, 2), 4: (8, 2, 4)}    # the non-default set of the batch-300 runs
STATS_VARIANTS = [(16, 4, 2), (4, 2, 32), (4, 4, 1), (4, 8, 3), (8, 2, 1), (8, 4, 32)]
FWD_VARIANTS = [(16, 4, 2), (4, 2, 1), (4, 4, 32), (4, 8, 3), (8, 2, 32), (8, 4, 1)]
BWD_VARIANTS = [(16, 4, 2), (16, 2, 1), (8, 2, 1), (8, 4, 32), (4, 2, 32), (4, 4, 1), (4, 8, 3)]


@pytest.fixture(autouse=True)
def _restore_globals():
    """sg_set_ew_variant and sg_set_grad_dtype are process-global: every test leaves the defaults behind."""
    prev = "bf16" if E.GS == SG_BF16 else "f16"
    yield
    for kind, v in EW_DEFAULT.items():
        assert _lib.load().sg_set_ew_variant(kind, *v) == 0
    E.set_grad_dtype(prev)


@pytest.fixture(params=["f16", "bf16"])
def grad_dtype(request):
    """Runs a test once per 16-bit gradient format (sg_set_grad_dtype)."""
    E.set_grad_dtype(request.param)
    yield request.param


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _cdiv(a, b):
    return -(-a // b)


def _set(kind, v):
    assert _lib.load().sg_set_ew_variant(kind, *v) == 0


# ------------------------------------------------------------------------------------------------------
# the dispatch rules, mirrored (case tables in the module docstring) and the fp32 run length per partial
# ------------------------------------------------------------------------------------------------------
def _stats_kernel(v):
    return "bn_stats_bulk" if v[0] == 16 else "bn_stats_kernel<%d,%d>" % v[:2]


def _fwd_kernel(v, L, H, twins):
    if v[0] == 16:
        return "act_fwd_bulk" if not twins and (H == 0 or L >= 2 * H + 3) else "act_fwd_kernel<8,4>"
    return "act_fwd_kernel<%d,%d>" % v[:2]


def _bwd_kernel(mode, v, C_, ldh, lda):
    vec, unr, _ = v
    if vec == 16 and ldh == C_ and lda == C_:
        return "act_bwd_bulk<%d>" % mode
    if vec >= 8 and ldh % 8 == 0 and lda % 8 == 0:
        return "act_bwd_tiled_kernel<%d,%d>" % (mode, 4 if unr >= 4 else 2)
    return "act_bwd_kernel<%d,4,%d>" % (mode, unr)


def _stats_adds(v, rows, C_):
    vec, unr, cap = v
    if vec == 16:
        tiles = _cdiv(rows, 8 * (256 // (C_ // 8)))
        return _cdiv(tiles, max(1, min(tiles, 2 * NUM_SMS))) * 8
    rpb = 256 // (C_ // vec)
    grid = max(1, min(_cdiv(rows, rpb * 2 * unr), cap * NUM_SMS))
    return _cdiv(rows, grid * rpb)


def _bwd_adds(v, B, L, C_, ldh, lda):
    name = _bwd_kernel(0, v, C_, ldh, lda)
    vec, unr, cap = v
    if name.startswith("act_bwd_bulk"):
        tiles = B * (_cdiv(L, 4 * (256 // (C_ // 8))) + 1)
        return _cdiv(tiles, min(tiles, 2 * NUM_SMS)) * 4
    if name.startswith("act_bwd_tiled"):
        U = 4 if unr >= 4 else 2
        total = B * _cdiv(L, (256 // (C_ // 8)) * U)
        return _cdiv(total, min(total, cap * NUM_SMS)) * U
    rpb = 256 // (C_ // 4)
    grid = max(1, min(_cdiv(B * L, rpb * unr), cap * NUM_SMS))
    return _cdiv(B * L, grid * rpb)


# ------------------------------------------------------------------------------------------------------
# guarded buffers
# ------------------------------------------------------------------------------------------------------
class Guarded16:
    """A 16-bit tensor of `shape` inside a flat buffer with `guard` sentinel elements on either side."""

    def __init__(self, shape, dtype, guard):
        self.n, self.guard = math.prod(shape), guard
        self.flat = torch.empty(self.n + 2 * guard, dtype=dtype, device=DEV)
        self.flat.view(torch.int16).fill_(SENT)
        self.t = self.flat[guard:guard + self.n].view(shape)

    def guard_ok(self):
        bits = self.flat.view(torch.int16)
        return bool((bits[:self.guard] == SENT).all()) and bool((bits[self.guard + self.n:] == SENT).all())


class Slices:
    """[SL][k][C] fp64 statistics target, pre-filled non-zero, between two guard slices."""

    def __init__(self, k, C_, g, zero=False):
        self.buf = torch.randn(SL + 2, k, C_, generator=g, dtype=torch.float64).to(DEV)
        if zero:
            self.buf[1:SL + 1].zero_()
        self.init = self.buf.clone()
        self.t = self.buf[1:SL + 1]

    def added(self):
        """The sum over slices of what the kernels added (fp64)."""
        return (self.t - self.init[1:SL + 1]).sum(0)

    def guard_ok(self):
        return torch.equal(self.buf[0], self.init[0]) and torch.equal(self.buf[SL + 1], self.init[SL + 1])


def _same(x, y):
    """Bit identity of two 16-bit tensors, +0 and -0 compared equal (no NaN is expected in either)."""
    return torch.equal(x.float(), y.float())


def _roll_dev(roll):
    """A device int32 holding `roll`, and a different host value that the device value must override."""
    t = torch.tensor([12345, roll], dtype=torch.int32, device=DEV)
    return C.c_void_p(t.data_ptr() + 4), t, (-roll if roll else 1)


# ------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------
def _act_operands(B, L, C_, dt, g, zeros=True, saturate=False, bn=True):
    """a [B][L][C] 16-bit ~ N(0, 2); ss = (sc, sh) fp32 with exact zeros of x * sc + sh planted (channels c % 5 == 0:
    sc a power of two, sh = -0.75 sc, a = 0.75 at l % 3 == 0) and, with `saturate`, sc = 3e4 on channels c % 7 == 3;
    slope fp32 of either sign."""
    a = 2 * torch.randn(B, L, C_, generator=g)
    sc = 1 + 0.3 * torch.randn(C_, generator=g)
    sh = 0.3 * torch.randn(C_, generator=g)
    if zeros:
        z = torch.arange(C_) % 5 == 0
        sc[z] = torch.tensor([0.5, 1.0, 2.0])[torch.arange(int(z.sum())) % 3]
        sh[z] = -0.75 * sc[z]
        a[:, ::3, z] = 0.75
    if saturate:
        sc[torch.arange(C_) % 7 == 3] = 3e4
    if not bn:
        sc.fill_(1.0)
        sh.zero_()
        if zeros:
            a[:, ::3, ::5] = 0.0
    slope = 0.3 * torch.randn(C_, generator=g)
    return a.to(TDT[dt]).to(DEV), torch.stack((sc, sh)).to(DEV), slope.to(DEV)


def _gate(tag, c, tol=M.C_TOL):
    print("%-60s c = %.3g (tol %g)" % (tag, c, tol))
    assert c <= tol, (tag, c)


# ------------------------------------------------------------------------------------------------------
# statistics and finalize
# ------------------------------------------------------------------------------------------------------
STATS_CASES = [(64, 3 * 37, SG_F16), (128, 17 * 100, SG_BF16), (256, 1 * 1000, SG_F16), (512, 3 * 35, SG_BF16),
               (1024, 17 * 16, SG_F16), (64, 4 * 4096 + 3, SG_F16)]


@pytest.mark.parametrize("C_,rows,dt", STATS_CASES)
def test_bn_stats_vs_fp64(C_, rows, dt):
    """sum x and sum x^2 per channel with |mu| = 8 sigma on half the channels, added onto pre-filled slices, under
    every variant (all six instantiations); the two guard slices keep their bits."""
    g = _gen(201)
    mu = torch.where(torch.arange(C_) % 2 == 0, 8.0, -0.1) * (1 + torch.rand(C_, generator=g))
    sig = 1 + torch.rand(C_, generator=g)
    a = (mu + sig * torch.randn(rows, C_, generator=g)).to(TDT[dt]).to(DEV)
    ref, mag = M.stats(a)
    for v in STATS_VARIANTS:
        _set(2, v)
        st = Slices(2, C_, g)
        _lib.call("sg_bn_stats", _p(a), dt, rows, C_, _p(st.t), _stream())
        torch.cuda.synchronize()
        n = _stats_adds(v, rows, C_)
        _gate("bn_stats %s C=%d rows=%d adds=%d" % (_stats_kernel(v), C_, rows, n),
              M.c_vec(st.added(), ref, mag))
        assert st.guard_ok()


@pytest.mark.parametrize("case", ["random", "n1", "var_clamped", "no_running"])
def test_bn_finalize_vs_fp64(case):
    """mean, biased var clamped at 0, invstd, sc = gamma * invstd, sh = beta - mean * sc (c in units of |beta| +
    |mean * sc|) and the running update with n / (n - 1) (1 at n = 1), each within a couple of fp32 ulps of fp64;
    the outputs' neighbours keep their bits."""
    g = _gen(202)
    C_ = 256
    n = {"random": 300 * 1024, "n1": 1, "var_clamped": 17, "no_running": 4096}[case]
    mean = 8 * torch.randn(C_, generator=g, dtype=torch.float64)
    var = torch.rand(C_, generator=g, dtype=torch.float64) + 1e-3
    s = torch.stack((mean * n, (var + mean * mean) * n))
    if case == "n1":
        s[1] = mean * mean                     # one sample: var = 0 up to fp64 rounding
    if case == "var_clamped":
        s[1, ::2] = (mean[::2] * mean[::2] * (1 - 1e-12)) * n     # sum x^2 / n < mean^2: var must clamp to 0
    w = torch.rand(SL, 1, C_, generator=g, dtype=torch.float64)
    st = (s.unsqueeze(0) * w / w.sum(0)).to(DEV)
    gamma = (1 + 0.3 * torch.randn(C_, generator=g)).to(DEV)
    beta = (0.5 * torch.randn(C_, generator=g)).to(DEV)
    rm0, rv0 = torch.randn(C_, generator=g).to(DEV), (torch.rand(C_, generator=g) + 0.5).to(DEV)
    out = torch.full((4 * C_ + 64,), 1234.5, device=DEV)          # ss | guard | mi | guard
    ss, mi = out[:2 * C_], out[2 * C_ + 32:4 * C_ + 32]
    running = case != "no_running"
    rm, rv = rm0.clone(), rv0.clone()
    eps, mom = 1e-5, 0.1
    _lib.call("sg_bn_finalize", _p(st), n, C_, _p(gamma), _p(beta), eps, mom, _p(rm) if running else None,
              _p(rv) if running else None, _p(ss), _p(mi), _stream())
    ref = M.finalize(st, n, gamma, beta, eps, mom, rm0, rv0)
    torch.cuda.synchronize()
    got = dict(mean=mi[:C_], invstd=mi[C_:], sc=ss[:C_], sh=ss[C_:], rmean=rm, rvar=rv)
    tol = dict(mean=2, invstd=2, sc=4, sh=8, rmean=8, rvar=8)
    for k in ("mean", "invstd", "sc", "sh") + (("rmean", "rvar") if running else ()):
        _gate("bn_finalize %s %s" % (case, k), M.c_vec(got[k], *ref[k]), tol[k])
    if not running:
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0)
    assert bool((out[2 * C_:2 * C_ + 32] == 1234.5).all()) and bool((out[4 * C_ + 32:] == 1234.5).all())


# ------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------
FWD_CASES = {
    # id: (C, B, L, H, roll, a dtype, twins, act, saturate)
    "c64_L35_min_rollLm1": (64, 3, 35, 16, 34, SG_F16, False, ACT_PRELU, False),
    "c128_L20_fallback": (128, 3, 20, 16, -5, SG_BF16, False, ACT_PRELU, False),
    "c256_L37_twins": (256, 17, 37, 16, 1, SG_F16, True, ACT_PRELU, False),
    "c512_L1000_noH_roll1mL": (512, 3, 1000, 0, -999, SG_BF16, False, ACT_PRELU, False),
    "c1024_L100_none": (1024, 1, 100, 16, 5, SG_F16, False, ACT_NONE, False),
    "c64_L4096_tilewrap": (64, 3, 4096, 16, 512, SG_F16, False, ACT_PRELU, False),
    "c128_L1024_tilewrap": (128, 3, 1024, 16, -256, SG_BF16, False, ACT_PRELU, False),
    "c256_L256_saturate": (256, 3, 256, 16, -1, SG_F16, False, ACT_PRELU, True),
    "c1024_L16_last": (1024, 17, 16, 0, 0, SG_F16, False, ACT_PRELU, False),
    "c512_L64_twins_sat": (512, 3, 64, 16, -5, SG_F16, True, ACT_PRELU, True),
}


def _run_fwd(a, dt, ss, slope, act, roll, rdev, H, twins):
    B, L, C_ = a.shape
    Lh = L + 2 * H
    h = Guarded16((B, Lh, C_), TDT[dt], 3 * C_)
    hb = Guarded16((B, Lh, C_), torch.bfloat16, 3 * C_) if twins else None
    ab = Guarded16((B, L, C_), torch.bfloat16, 3 * C_) if twins else None
    _lib.call("sg_act_fwd", _p(a), dt, B, L, C_, _p(ss), _p(slope) if act == ACT_PRELU else None, act, roll, rdev, H,
              _p(h.t), _p(hb.t) if twins else None, _p(ab.t) if twins else None, _stream())
    return h, hb, ab


@pytest.mark.parametrize("case", list(FWD_CASES))
def test_act_fwd_vs_fp64_every_variant(case):
    """h = act(x * sc + sh) at the rolled row and its reflect mirror, within C_TOL of fp64 (fp16 saturating at
    +-65504), under every variant; the bf16 twins h_bf16 (same gate in bf16) and a_bf16 (bit-equal to a in bf16,
    written from interior rows only); the same launch with the shift in device memory and a different host shift
    gives the same bits; and every variant stores the same bits as every other."""
    C_, B, L, H, roll, dt, twins, act, sat = FWD_CASES[case]
    g = _gen(203)
    a, ss, slope = _act_operands(B, L, C_, dt, g, saturate=sat)
    ref, mag = M.act_fwd(a, ss, slope if act == ACT_PRELU else None, roll, H)
    if sat:
        assert float(ref.abs().max()) > 65504
    first = None
    for v in FWD_VARIANTS:
        _set(1, v)
        name = _fwd_kernel(v, L, H, twins)
        h, hb, ab = _run_fwd(a, dt, ss, slope, act, roll, None, H, twins)
        rptr, _keep, host = _roll_dev(roll)
        hd, _, _ = _run_fwd(a, dt, ss, slope, act, host, rptr, H, twins)
        torch.cuda.synchronize()
        _gate("act_fwd %s %s h" % (case, name), M.c_f(h.t, ref, mag, FMT[dt]))
        assert h.guard_ok(), (case, name)
        assert torch.equal(hd.t.view(torch.int16), h.t.view(torch.int16)) and hd.guard_ok(), (case, name, "roll_dev")
        if twins:
            _gate("act_fwd %s %s h_bf16" % (case, name), M.c_f(hb.t, ref, mag, "bf16"))
            assert torch.equal(ab.t.view(torch.int16), a.to(torch.bfloat16).view(torch.int16)), (case, name)
            assert hb.guard_ok() and ab.guard_ok(), (case, name)
        if first is None:
            first = (name, h.t, hb.t if twins else None)
        else:
            assert _same(h.t, first[1]), (case, name, "differs from", first[0])
            if twins:
                assert _same(hb.t, first[2]), (case, name, "h_bf16 differs from", first[0])


# ------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------
BWD_CASES = {
    # id: (C, B, L, H, roll, a dtype, mode, ldh extra columns (zc) or ldh, skip, saturate)
    "c64_L35_bn_rollLm1": (64, 3, 35, 16, 34, SG_F16, "bn", 0, False, False),
    "c128_L37_skip_strided": (128, 17, 37, 16, -1, SG_F16, "nobn", 64, True, False),
    "c256_L100_bn_ldh4": (256, 3, 100, 16, 5, SG_BF16, "bn", 4, False, False),
    "c1024_L1000_bn_noH": (1024, 1, 1000, 0, -999, SG_F16, "bn", 0, False, False),
    "c512_L64_bn": (512, 3, 64, 16, -5, SG_BF16, "bn", 0, False, False),
    "c64_L1024_skip_sat": (64, 3, 1024, 16, 256, SG_F16, "nobn", 0, False, True),
    "c128_L4096_bn_tilewrap": (128, 1, 4096, 16, -640, SG_F16, "bn", 0, False, False),
    "c1024_L16_last_zc": (1024, 17, 16, 0, 0, SG_F16, "nobn", 1024, False, False),
}


class BwdOperands:
    """g_h in the consumer view [B][L + 2H][ldh] (the layer's gradient at column zc when ldh = zc + C, as the G's
    last encoder layer reads it; ldh = C + 4 when zc == 4), g_add [B][L][2C] read at column C (lda = 2C, the G's
    skip gradient) or contiguous, the activation a, BN constants with |mu| ~ 8 sigma on some channels."""

    def __init__(self, case, g):
        C_, B, L, H, roll, dt, mode, zc, strided_skip, sat = BWD_CASES[case]
        self.C, self.B, self.L, self.H, self.roll, self.dt = C_, B, L, H, roll, dt
        self.bn = mode == "bn"
        gt = E.GT
        self.a, ss, self.slope = _act_operands(B, L, C_, dt, g, bn=self.bn)
        self.ss = ss if self.bn else None
        if self.bn:
            mu = self.a.double().mean((0, 1))
            sd = (self.a.double() - mu).pow(2).mean((0, 1)).sqrt()
            self.mi = torch.stack((mu, 1.0 / sd)).float()
        else:
            self.mi = None
        self.ldh = C_ + zc
        self.zc = 0 if zc == 4 else zc
        gh = torch.randn(B, L + 2 * H, self.ldh, generator=g)
        if sat:
            gh[..., 3::7] *= 3e4                   # |g| ~ 6e4 on channels c % 7 == 3: the mirror fold overflows fp16
            gh[..., 3::7] = gh[..., 3::7].clamp(-6e4, 6e4)
        self.gh_buf = gh.to(gt).to(DEV)
        self.gh = self.gh_buf[..., self.zc:self.zc + C_]
        self.gh_ptr = C.c_void_p(self.gh_buf.data_ptr() + 2 * self.zc)
        self.gadd, self.gadd_ptr, self.lda = None, None, 0
        if strided_skip:
            buf = torch.randn(B, L, 2 * C_, generator=g).to(gt).to(DEV)
            self.gadd_buf, self.gadd, self.lda = buf, buf[..., C_:], 2 * C_
            self.gadd_ptr = C.c_void_p(buf.data_ptr() + 2 * C_)
        elif mode == "nobn" and case.endswith("_sat"):
            self.gadd = torch.randn(B, L, C_, generator=g).to(gt).to(DEV)
            self.gadd_ptr, self.lda = _p(self.gadd), C_
        self.lda_eff = self.lda if self.lda else C_

    def kernel(self, mode, v):
        return _bwd_kernel(mode, v, self.C, self.ldh, self.lda_eff)

    def reduce(self, red, g_a, roll, rdev):
        _lib.call("sg_act_bwd_reduce", self.gh_ptr, self.ldh, self.H, roll, rdev, self.gadd_ptr, self.lda, _p(self.a),
                  self.dt, self.B, self.L, self.C, _p(self.ss), _p(self.mi), _p(self.slope), ACT_PRELU, _p(red),
                  _p(g_a), _stream())

    def apply(self, red, use_bn, g_a, roll, rdev):
        _lib.call("sg_act_bwd_apply", self.gh_ptr, self.ldh, self.H, roll, rdev, self.gadd_ptr, self.lda, _p(self.a),
                  self.dt, self.B, self.L, self.C, _p(self.ss), _p(self.mi), _p(self.slope), ACT_PRELU, _p(red),
                  use_bn, _p(g_a), _stream())


@pytest.mark.parametrize("case", list(BWD_CASES))
def test_act_bwd_vs_fp64_every_variant(case, grad_dtype):
    """Pass 0 (sg_act_bwd_reduce): red0..red2 added onto pre-filled slices within C_TOL, and, without BN, g_a
    = g_pre within C_TOL (fp16 saturating); pass 1 (sg_act_bwd_apply) on a red the test builds itself, within C_TOL
    of fp64, and with use_bn = 0 the same bits as pass 0's g_a.  Under every variant: guard bands keep their bits,
    the device shift overrides a different host shift with identical results, and the pointwise outputs have the
    same bits as under the first variant."""
    g = _gen(204)
    op = BwdOperands(case, g)
    B, L, C_, H, roll = op.B, op.L, op.C, op.H, op.roll
    gt = E.GT
    fmt = FMT[E.GS]
    p0 = M.bwd_pass0(op.gh, op.gadd, op.a, op.ss, op.mi, op.slope, roll, H)
    rref, rmag = p0["red"]
    if case.endswith("_sat") and fmt == "f16":
        assert float(p0["gpre"][0].abs().max()) > 65504
    # pass 1 input: the fp64 reductions split unevenly over the slices
    w = torch.rand(SL, 1, 1, generator=g, dtype=torch.float64).to(DEV)
    red_in = rref.unsqueeze(0) * (w / w.sum(0))
    p1 = M.bwd_pass1(p0["gpre"], op.a, op.ss, op.mi, red_in, use_bn=op.bn)
    first0 = first1 = None
    for v in BWD_VARIANTS:
        _set(3, v)
        _set(4, v)
        k0, k1 = op.kernel(0, v), op.kernel(1, v)
        n = _bwd_adds(v, B, L, C_, op.ldh, op.lda_eff)
        rptr, _keep, host = _roll_dev(roll)
        red, red_d = Slices(3, C_, g), Slices(3, C_, g)
        ga0 = None if op.bn else Guarded16((B, L, C_), gt, 3 * C_)
        ga0d = None if op.bn else Guarded16((B, L, C_), gt, 3 * C_)
        op.reduce(red.t, ga0.t if ga0 else None, roll, None)
        op.reduce(red_d.t, ga0d.t if ga0d else None, host, rptr)
        ga1, ga1d = Guarded16((B, L, C_), gt, 3 * C_), Guarded16((B, L, C_), gt, 3 * C_)
        op.apply(red_in, int(op.bn), ga1.t, roll, None)
        op.apply(red_in, int(op.bn), ga1d.t, host, rptr)
        torch.cuda.synchronize()
        for s in range(3):
            for tag, r in (("", red), (" roll_dev", red_d)):
                _gate("act_bwd %s %s %s red%d%s adds=%d" % (case, fmt, k0, s, tag, n),
                      M.c_vec(r.added()[s], rref[s], rmag[s]))
        assert red.guard_ok() and red_d.guard_ok(), (case, k0)
        if ga0 is not None:
            _gate("act_bwd %s %s %s g_a (pass 0)" % (case, fmt, k0), M.c_f(ga0.t, *p0["gpre"], fmt))
            assert ga0.guard_ok() and ga0d.guard_ok(), (case, k0)
            assert torch.equal(ga0.t.view(torch.int16), ga0d.t.view(torch.int16)), (case, k0, "roll_dev")
            assert _same(ga1.t, ga0.t), (case, k1, "use_bn = 0 differs from pass 0")
            if first0 is None:
                first0 = (k0, ga0.t)
            else:
                assert _same(ga0.t, first0[1]), (case, k0, "differs from", first0[0])
        _gate("act_bwd %s %s %s g_a (pass 1)" % (case, fmt, k1), M.c_f(ga1.t, *p1, fmt))
        assert ga1.guard_ok() and ga1d.guard_ok(), (case, k1)
        assert torch.equal(ga1.t.view(torch.int16), ga1d.t.view(torch.int16)), (case, k1, "roll_dev")
        if first1 is None:
            first1 = (k1, ga1.t)
        else:
            assert _same(ga1.t, first1[1]), (case, k1, "differs from", first1[0])


@pytest.mark.parametrize("n_stats,targets", [(3, (1, 1, 1)), (3, (1, 1, 0)), (2, (1, 1, 0)), (1, (1, 0, 0)),
                                             (3, (0, 1, 1))])
def test_stat_grads_vs_fp64(n_stats, targets):
    """g_s[c] += sum over slices of red[slice][s][c] at slice stride n_stats; null targets are skipped and every
    target's neighbours keep their bits."""
    g = _gen(205)
    C_ = 512
    red = (1e3 * torch.randn(SL, n_stats, C_, generator=g, dtype=torch.float64)).to(DEV)
    buf = torch.full((3, C_ + 64), 1234.5, device=DEV)
    g0 = [torch.randn(C_, generator=g).to(DEV) for _ in range(3)]
    views = []
    for s in range(3):
        buf[s, 32:32 + C_] = g0[s]
        views.append(buf[s, 32:32 + C_] if targets[s] else None)
    _lib.call("sg_stat_grads", _p(red), C_, n_stats, _p(views[0]), _p(views[1]), _p(views[2]), _stream())
    ref = M.stat_grads(red, n_stats, [g0[s] if targets[s] else None for s in range(3)])
    torch.cuda.synchronize()
    for s in range(3):
        if ref[s] is not None:
            _gate("stat_grads n=%d g%d" % (n_stats, s), M.c_vec(views[s], *ref[s]), 4)
        else:
            assert torch.equal(buf[s, 32:32 + C_], g0[s])
    assert bool((buf[:, :32] == 1234.5).all()) and bool((buf[:, 32 + C_:] == 1234.5).all())


# ------------------------------------------------------------------------------------------------------
# the D's BatchNorm chain and the G encoder's pass 0 at batch 300
# ------------------------------------------------------------------------------------------------------
D_LAYERS = [(64, 4096, 16, 3), (128, 1024, 16, -5), (256, 256, 16, 5), (512, 64, 16, -1), (1024, 16, 0, 0)]


@pytest.mark.parametrize("variants", ["default", "register"])
def test_d_chain_batch300(variants):
    """Each of the D's five BN layers at batch 300: bn_stats -> bn_finalize -> act_fwd -> act_bwd_reduce ->
    act_bwd_apply -> stat_grads, every stage gated against fp64 on the previous stage's kernel outputs."""
    for kind, v in (EW_DEFAULT if variants == "default" else EW_REGISTER).items():
        _set(kind, v)
    B = 300
    g = _gen(206)
    fmt = FMT[E.GS]
    for C_, L, H, roll in D_LAYERS:
        tag = "D chain %s C=%d L=%d" % (variants, C_, L)
        mu = torch.where(torch.arange(C_) % 4 == 0, 8.0, 0.3) * torch.randn(C_, generator=g).sign()
        a = (mu + torch.randn(B, L, C_, generator=g)).half().to(DEV)
        stats = torch.zeros(SL, 2, C_, dtype=torch.float64, device=DEV)
        _lib.call("sg_bn_stats", _p(a), SG_F16, B * L, C_, _p(stats), _stream())
        gamma = (1 + 0.2 * torch.randn(C_, generator=g)).to(DEV)
        beta = (0.2 * torch.randn(C_, generator=g)).to(DEV)
        rm0, rv0 = (0.1 * torch.randn(C_, generator=g)).to(DEV), (1 + torch.rand(C_, generator=g)).to(DEV)
        rm, rv = rm0.clone(), rv0.clone()
        ss, mi = torch.empty(2, C_, device=DEV), torch.empty(2, C_, device=DEV)
        _lib.call("sg_bn_finalize", _p(stats), B * L, C_, _p(gamma), _p(beta), 1e-5, 0.1, _p(rm), _p(rv), _p(ss),
                  _p(mi), _stream())
        slope = (0.25 * torch.rand(C_, generator=g)).to(DEV)
        h = torch.empty(B, L + 2 * H, C_, dtype=torch.float16, device=DEV)
        _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(slope), ACT_PRELU, roll, None, H, _p(h), None, None,
                  _stream())
        gh = (0.5 * torch.randn(B, L + 2 * H, C_, generator=g)).to(E.GT).to(DEV)
        red = torch.zeros(SL, 3, C_, dtype=torch.float64, device=DEV)
        _lib.call("sg_act_bwd_reduce", _p(gh), C_, H, roll, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
                  _p(slope), ACT_PRELU, _p(red), None, _stream())
        ga = torch.empty(B, L, C_, dtype=E.GT, device=DEV)
        _lib.call("sg_act_bwd_apply", _p(gh), C_, H, roll, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
                  _p(slope), ACT_PRELU, _p(red), 1, _p(ga), _stream())
        gp0 = [torch.randn(C_, generator=g).to(DEV) for _ in range(3)]
        gp = [t.clone() for t in gp0]
        _lib.call("sg_stat_grads", _p(red), C_, 3, _p(gp[0]), _p(gp[1]), _p(gp[2]), _stream())
        torch.cuda.synchronize()
        ref, mag = M.stats(a)
        n = _stats_adds((EW_DEFAULT if variants == "default" else EW_REGISTER)[2], B * L, C_)
        for s in range(2):
            _gate("%s bn_stats s%d adds=%d" % (tag, s, n), M.c_vec(stats.sum(0)[s], ref[s], mag[s]))
        fin = M.finalize(stats, B * L, gamma, beta, 1e-5, 0.1, rm0, rv0)
        got = dict(mean=mi[0], invstd=mi[1], sc=ss[0], sh=ss[1], rmean=rm, rvar=rv)
        for k, tol in (("mean", 2), ("invstd", 2), ("sc", 4), ("sh", 8), ("rmean", 8), ("rvar", 8)):
            _gate("%s bn_finalize %s" % (tag, k), M.c_vec(got[k], *fin[k]), tol)
        _gate("%s act_fwd" % tag, M.c_f(h, *M.act_fwd(a, ss, slope, roll, H), "f16"))
        p0 = M.bwd_pass0(gh, None, a, ss, mi, slope, roll, H)
        v3 = (EW_DEFAULT if variants == "default" else EW_REGISTER)[3]
        n = _bwd_adds(v3, B, L, C_, C_, C_)
        rs = red.sum(0)
        for s in range(3):
            _gate("%s act_bwd_reduce red%d adds=%d" % (tag, s, n), M.c_vec(rs[s], p0["red"][0][s], p0["red"][1][s]))
        _gate("%s act_bwd_apply (%s)" % (tag, fmt), M.c_f(ga, *M.bwd_pass1(p0["gpre"], a, ss, mi, red), fmt))
        for s, r in enumerate(M.stat_grads(red, 3, gp0)):
            _gate("%s stat_grads g%d" % (tag, s), M.c_vec(gp[s], *r), 4)


@pytest.mark.parametrize("variants", ["default", "register"])
def test_g_encoder_pass0_batch300(variants):
    """The G encoder's backward without BN (one pass writes g_pre): layer 0 (C 64, L 4096, halo 16) with the skip
    gradient read at column C of a [B][L][2C] tensor, and the last layer (C 1024, L 16, no halo) whose gradient is
    read at column zc = 1024 of the [B][L][zc + C] input gradient."""
    for kind, v in (EW_DEFAULT if variants == "default" else EW_REGISTER).items():
        _set(kind, v)
    B = 300
    g = _gen(207)
    fmt = FMT[E.GS]
    for C_, L, H, zc, skip in ((64, 4096, 16, 0, True), (1024, 16, 0, 1024, False)):
        a = torch.randn(B, L, C_, generator=g).half().to(DEV)
        a[:, ::3, ::5] = 0.0
        slope = (0.25 * torch.rand(C_, generator=g)).to(DEV)
        ghb = (0.5 * torch.randn(B, L + 2 * H, zc + C_, generator=g)).to(E.GT).to(DEV)
        gh = ghb[..., zc:]
        gadd, gptr, lda = None, None, 0
        if skip:
            gsk = (0.5 * torch.randn(B, L, 2 * C_, generator=g)).to(E.GT).to(DEV)
            gadd, gptr, lda = gsk[..., C_:], C.c_void_p(gsk.data_ptr() + 2 * C_), 2 * C_
        red = torch.zeros(SL, 3, C_, dtype=torch.float64, device=DEV)
        ga = Guarded16((B, L, C_), E.GT, 3 * C_)
        _lib.call("sg_act_bwd_reduce", C.c_void_p(ghb.data_ptr() + 2 * zc), zc + C_, H, 0, None, gptr, lda, _p(a),
                  SG_F16, B, L, C_, None, None, _p(slope), ACT_PRELU, _p(red), _p(ga.t), _stream())
        torch.cuda.synchronize()
        p0 = M.bwd_pass0(gh, gadd, a, None, None, slope, 0, H)
        v3 = (EW_DEFAULT if variants == "default" else EW_REGISTER)[3]
        kname = _bwd_kernel(0, v3, C_, zc + C_, lda or C_)
        n = _bwd_adds(v3, B, L, C_, zc + C_, lda or C_)
        tag = "G enc %s C=%d L=%d %s" % (variants, C_, L, kname)
        rs = red.sum(0)
        for s in range(3):
            _gate("%s red%d adds=%d" % (tag, s, n), M.c_vec(rs[s], p0["red"][0][s], p0["red"][1][s]))
        _gate("%s g_a (%s)" % (tag, fmt), M.c_f(ga.t, *p0["gpre"], fmt))
        assert ga.guard_ok()


# ------------------------------------------------------------------------------------------------------
# BatchNorm statistics in the tap-GEMM epilogue
# ------------------------------------------------------------------------------------------------------
def _conv_weights(cin, cout, g):
    kc, nc = 4 * cin, cout
    taps = E.tap_ranges("conv_fwd", cin, kc, nc)
    w = torch.randn(9, nc, kc, generator=g) * (0.5 / math.sqrt(31 * cin))
    for i in range(9):
        mask = torch.zeros(nc, kc)
        mask[taps[2][i]:taps[3][i], taps[0][i]:taps[1][i]] = 1
        w[i] *= mask
    return w.half().to(DEV), taps


def _colstat_adds(B, R, nc):
    """Longest run of one shared-memory colstat float: 8 warp partials (16 rows each) per 128-row tile, every tile
    of one CTA (tapgemm_tc.cu: TR / TB / TN and a grid of min(132, tiles))."""
    TR, TB = (128, 1) if R >= 128 else (R, min(128 // R, B))
    tiles = _cdiv(R, TR) * _cdiv(B, TB) * (nc // (256 if nc % 256 == 0 else (128 if nc % 128 == 0 else 64)))
    return 8 * _cdiv(tiles, min(NUM_SMS, tiles))


FUSED_CASES = [(300, 64, 128, 1024, SG_F16), (300, 128, 256, 256, SG_F16), (300, 256, 512, 64, SG_BF16),
               (300, 512, 1024, 16, SG_F16), (3, 64, 128, 37, SG_F16), (5, 128, 64, 160, SG_BF16),
               (33, 128, 512, 16, SG_BF16), (7, 64, 256, 100, SG_F16)]


@pytest.mark.parametrize("B,cin,cout,R,odt", FUSED_CASES)
def test_tapgemm_fused_bn_stats_vs_fp64(B, cin, cout, R, odt):
    """TapGemmF.bn_stats (the D's fused statistics, SEGAN_B200_FUSE_BN_STATS=1): sum and sum of squares per channel of
    the stored 16-bit output, added onto pre-filled slices, within C_TOL; the guard slices keep their bits.
    The D conv shapes of layers 1-4 at batch 300 and ragged batches / rows."""
    g = _gen(208)
    w, taps = _conv_weights(cin, cout, g)
    kc, halo = 4 * cin, 4
    a0 = torch.randn(B, R + 2 * halo, kc, generator=g).half().to(DEV)
    bias = (4 * torch.randn(cout, generator=g)).to(DEV)
    out = torch.empty(B, R, cout, dtype=TDT[odt], device=DEV)
    st = Slices(2, cout, g)
    E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, cout, taps, out, odt, R, 0, 0, R, B, bias=bias, bias_mod=cout,
            backend=BACKEND_TCGEN05, stats=st.t)
    torch.cuda.synchronize()
    ref, mag = M.stats(out)
    n = _colstat_adds(B, R, cout)
    for s in range(2):
        _gate("fused bn_stats B=%d C=%d R=%d %s s%d adds=%d" % (B, cout, R, FMT[odt], s, n),
              M.c_vec(st.added()[s], ref[s], mag[s]))
    assert st.guard_ok()


def test_tapgemm_fused_bn_stats_refusals():
    """The host refuses fused statistics with a k-split, an fp32 output or a partial n range."""
    g = _gen(209)
    B, cin, cout, R, halo = 3, 64, 128, 64, 4
    w, taps = _conv_weights(cin, cout, g)
    a0 = torch.randn(B, R + 2 * halo, 4 * cin, generator=g).half().to(DEV)
    st = torch.zeros(SL, 2, cout, dtype=torch.float64, device=DEV)
    out16 = torch.zeros(B, R, cout, dtype=torch.float16, device=DEV)
    out32 = torch.zeros(B, R, cout, device=DEV)
    for kw in (dict(out=out16, out_dtype=SG_F16, ksplit=2), dict(out=out32, out_dtype=SG_F32),
               dict(out=out16, out_dtype=SG_F16, n_lo=0, n_hi=64)):
        with pytest.raises(_lib.SeganB200Error):
            E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, 4 * cin, cout, taps, kw.pop("out"), kw.pop("out_dtype"), R,
                    0, 0, R, B, backend=BACKEND_TCGEN05, stats=st, **kw)
    torch.cuda.synchronize()
    assert float(st.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------
# host refusals and coverage
# ------------------------------------------------------------------------------------------------------
def test_host_refusals():
    """Arguments the host refuses before any launch (every pointer is a real allocation sized for the call)."""
    lib = _lib.load()
    err = _lib.SeganB200Error
    for C_ in (32, 96, 2048):
        B, L, H = 1, 35, 16
        a = torch.zeros(B, L, C_, dtype=torch.float16, device=DEV)
        h = torch.zeros(B, L + 2 * H, C_, dtype=torch.float16, device=DEV)
        ss = torch.ones(2, C_, device=DEV)
        sl = torch.ones(C_, device=DEV)
        red = torch.zeros(SL, 3, C_, dtype=torch.float64, device=DEV)
        ga = torch.zeros(B, L, C_, dtype=E.GT, device=DEV)
        with pytest.raises(err):
            _lib.call("sg_bn_stats", _p(a), SG_F16, B * L, C_, _p(red), _stream())
        with pytest.raises(err):
            _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(sl), ACT_PRELU, 0, None, H, _p(h), None, None,
                      _stream())
        with pytest.raises(err):
            _lib.call("sg_act_bwd_reduce", _p(h), C_, H, 0, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(ss),
                      _p(sl), ACT_PRELU, _p(red), None, _stream())
        with pytest.raises(err):
            _lib.call("sg_act_bwd_apply", _p(h), C_, H, 0, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(ss),
                      _p(sl), ACT_PRELU, _p(red), 1, _p(ga), _stream())
    C_, B, H = 64, 2, 16
    ss, sl = torch.ones(2, C_, device=DEV), torch.ones(C_, device=DEV)
    red = torch.zeros(SL, 3, C_, dtype=torch.float64, device=DEV)
    for L in (20, 34):                         # L < 2H + 3: the backward's single-mirror fold does not hold
        a = torch.zeros(B, L, C_, dtype=torch.float16, device=DEV)
        gh = torch.zeros(B, L + 2 * H, C_, dtype=E.GT, device=DEV)
        ga = torch.zeros(B, L, C_, dtype=E.GT, device=DEV)
        with pytest.raises(err):
            _lib.call("sg_act_bwd_reduce", _p(gh), C_, H, 0, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(ss),
                      _p(sl), ACT_PRELU, _p(red), None, _stream())
        with pytest.raises(err):
            _lib.call("sg_act_bwd_apply", _p(gh), C_, H, 0, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(ss),
                      _p(sl), ACT_PRELU, _p(red), 1, _p(ga), _stream())
    for L in (16, 8):                          # L <= H: reflect padding needs pad < L
        a = torch.zeros(B, L, C_, dtype=torch.float16, device=DEV)
        h = torch.zeros(B, L + 2 * H, C_, dtype=torch.float16, device=DEV)
        with pytest.raises(err):
            _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(sl), ACT_PRELU, 0, None, H, _p(h), None, None,
                      _stream())
    a = torch.zeros(B, 64, C_, dtype=torch.float16, device=DEV)
    h = torch.zeros(B, 64 + 2 * H, C_, dtype=torch.float16, device=DEV)
    with pytest.raises(err):                   # PReLU without a slope
        _lib.call("sg_act_fwd", _p(a), SG_F16, B, 64, C_, _p(ss), None, ACT_PRELU, 0, None, H, _p(h), None, None,
                  _stream())
    gs = torch.zeros(3, C_, device=DEV)
    for n_stats in (0, 4):
        with pytest.raises(err):
            _lib.call("sg_stat_grads", _p(red), C_, n_stats, _p(gs[0]), _p(gs[1]), _p(gs[2]), _stream())
    for bad in ((0, 4, 2, 3), (5, 4, 2, 3), (1, 3, 2, 3), (1, 4, 3, 3), (1, 8, 8, 3), (3, 8, 8, 2), (1, 4, 2, 0),
                (1, 4, 2, 33), (3, 16, 4, 0), (4, 16, 4, 33)):
        assert lib.sg_set_ew_variant(*bad) != 0, bad
    torch.cuda.synchronize()
    assert float(red.abs().max()) == 0.0 and float(gs.abs().max()) == 0.0


def test_every_instantiation_is_reached():
    """The case tables above reach all 24 instantiations of the six entry points' streaming kernels."""
    reached = {_stats_kernel(v) for v in STATS_VARIANTS}
    for C_, B, L, H, roll, dt, twins, act, sat in FWD_CASES.values():
        reached |= {_fwd_kernel(v, L, H, twins) for v in FWD_VARIANTS}
    for case in BWD_CASES:
        C_, zc = BWD_CASES[case][0], BWD_CASES[case][7]
        skip = BWD_CASES[case][8]
        lda = 2 * C_ if skip else C_
        reached |= {_bwd_kernel(m, v, C_, C_ + zc, lda) for v in BWD_VARIANTS for m in (0, 1)}
    want = {"bn_stats_bulk", "act_fwd_bulk", "act_bwd_bulk<0>", "act_bwd_bulk<1>"}
    for vec, unr in ((4, 2), (4, 4), (4, 8), (8, 2), (8, 4)):
        want |= {"bn_stats_kernel<%d,%d>" % (vec, unr), "act_fwd_kernel<%d,%d>" % (vec, unr)}
    for m in (0, 1):
        want |= {"act_bwd_tiled_kernel<%d,%d>" % (m, u) for u in (2, 4)}
        want |= {"act_bwd_kernel<%d,4,%d>" % (m, u) for u in (2, 4, 8)}
    assert len(want) == 24 and reached == want, sorted(want ^ reached)
