"""Kernel-level GPU tests: every C-ABI kernel against a plain fp32 torch evaluation of the same
formula on the same (16-bit-rounded) operands, and the wgmma tap-GEMMs against the FFMA ones.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E          # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, SG_F32, BACKEND_FFMA, BACKEND_TCGEN05  # noqa: E402
from oracle import segan_oracle as O                       # noqa: E402
from tests.util import max_abs, rel_err                    # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream


@pytest.fixture(params=["f16", "bf16"])
def grad_dtype(request):
    """Runs a test once per 16-bit gradient format (sg_set_grad_dtype): fp16 (default) and round 1's bf16."""
    prev = "bf16" if E.GS == SG_BF16 else "f16"
    E.set_grad_dtype(request.param)
    yield request.param
    E.set_grad_dtype(prev)


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _packed_random(kind, c, kc, nc, g, dtype, scale=0.05):
    taps = E.tap_ranges(kind, c, kc, nc)
    w = torch.randn(9, nc, kc, generator=g) * scale
    for i in range(9):
        mask = torch.zeros(nc, kc)
        mask[taps[2][i]:taps[3][i], taps[0][i]:taps[1][i]] = 1
        w[i] *= mask
    return w.to(dtype).to(DEV), taps


def _ref_f(a_pad, halo, w, m_lo, m_hi, d_lo=-4, d_hi=4, w_tap0=0):
    """a_pad: (B, R+2H, Kc) float32 with zero rows already in place; returns (B, m_hi-m_lo, Nc)."""
    B, RH, Kc = a_pad.shape
    R = RH - 2 * halo
    ext = 16
    ap = F.pad(a_pad, (0, 0, ext, ext))
    out = 0
    for d in range(d_lo, d_hi + 1):
        rows = ap[:, ext + halo + m_lo + d: ext + halo + m_hi + d, :]
        out = out + rows @ w[d + 4 - w_tap0].float().t()
    return out


EW_DEFAULT_REG = {1: (8, 4, 2), 2: (4, 4, 3), 3: (8, 2, 2), 4: (8, 2, 4)}  # the best register-staged variants
EW_DEFAULT = {1: (16, 4, 2), 2: (4, 8, 3), 3: (16, 4, 2), 4: (16, 4, 2)}    # elementwise.cu g_ew


@pytest.fixture(autouse=True)
def _restore_cta_pair():
    yield
    _lib.load().sg_set_cta_pair(1)
    for kind, v in EW_DEFAULT.items():
        _lib.load().sg_set_ew_variant(kind, *v)


F_CASES = ["conv_fwd", "conv_dgrad", "deconv_fwd_cat", "deconv_dgrad", "small_rows", "fc"]


def _f_case(case):
    """The operands and geometry of one test_tapgemm_f case, as a dict of its local names."""
    g = _gen(1)
    B = 3
    bias = None
    a1 = None
    a1_c = 0
    n_lo, n_hi = 0, None
    d_lo, d_hi, w_tap0, ksplit = -4, 4, 0, 1
    out_dtype, tdt = SG_F16, torch.float16
    if case == "conv_fwd":
        cin, cout, R, halo = 64, 128, 160, 4
        kc, nc = 4 * cin, cout
        w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
        a0 = (torch.randn(B, R + 2 * halo, kc, generator=g)).to(torch.float16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        bias = torch.randn(nc, generator=g).to(DEV)
        adt, wdt = SG_F16, SG_F16
    elif case == "conv_dgrad":
        cin, cout, R, halo = 64, 128, 96, 0
        kc, nc = cout, 4 * cin
        w, taps = _packed_random("conv_dgrad", cin, kc, nc, g, torch.bfloat16)
        a0 = torch.randn(B, R, kc, generator=g).to(torch.bfloat16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = -4, R + 4, R, 4
        adt, wdt, out_dtype, tdt = SG_BF16, SG_BF16, SG_BF16, torch.bfloat16
    elif case == "deconv_fwd_cat":
        cin, cout, R, halo = 256, 64, 64, 0
        kc, nc = cin, 4 * cout
        w, taps = _packed_random("deconv_fwd", cout, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1_c = 128
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        bias = torch.randn(cout, generator=g).to(DEV)
        adt, wdt = SG_F16, SG_F16
    elif case == "deconv_dgrad":
        cin, cout, R, halo = 256, 64, 64, 0
        kc, nc = 4 * cout, cin
        w, taps = _packed_random("deconv_dgrad", cout, kc, nc, g, torch.bfloat16)
        a0 = torch.randn(B, R, kc, generator=g).to(torch.bfloat16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        n_lo, n_hi = 128, 256
        adt, wdt, out_dtype, tdt = SG_BF16, SG_BF16, SG_BF16, torch.bfloat16
    elif case == "small_rows":
        B = 11
        cin, cout, R, halo = 128, 256, 16, 4
        kc, nc = 4 * cin, cout
        w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        adt, wdt = SG_F16, SG_F16
    else:  # fc: one tap, rows = 1, split-K into fp32
        B = 70
        kc, nc, R, halo = 2048, 256, 1, 0
        taps = E.tap_ranges("full", 0, kc, nc)
        w = (torch.randn(1, nc, kc, generator=g) * 0.05).to(torch.float16).to(DEV)
        a0 = torch.randn(B, 1, kc, generator=g).to(torch.float16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, 1, 1, 0
        d_lo = d_hi = 0
        w_tap0, ksplit = 4, 4
        adt, wdt, out_dtype, tdt = SG_F16, SG_F16, SG_F32, torch.float32
    return dict(locals())


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05, 2])
@pytest.mark.parametrize("case", F_CASES)
def test_tapgemm_f(backend, case):
    """backend 1 = tensor cores with sg_set_cta_pair(0), 2 = tensor cores with sg_set_cta_pair(1)."""
    _lib.load().sg_set_cta_pair(1 if backend == 2 else 0)
    if backend == 2:
        backend = BACKEND_TCGEN05
    c = _f_case(case)
    B, R, halo, kc, nc, taps, w, a0, a1, a1_c, bias = (c[k] for k in ("B", "R", "halo", "kc", "nc", "taps", "w", "a0", "a1",
                                                                       "a1_c", "bias"))
    m_lo, m_hi, out_rows, out_halo, n_lo, n_hi = (c[k] for k in ("m_lo", "m_hi", "out_rows", "out_halo", "n_lo", "n_hi"))
    d_lo, d_hi, w_tap0, ksplit = (c[k] for k in ("d_lo", "d_hi", "w_tap0", "ksplit"))
    adt, wdt, out_dtype, tdt = (c[k] for k in ("adt", "wdt", "out_dtype", "tdt"))
    nhi = nc if n_hi is None else n_hi
    out = torch.zeros(B, out_rows + 2 * out_halo, nc, dtype=tdt, device=DEV)
    E.run_f(a0, a1, R, halo, adt, w, wdt, kc, nc, taps, out, out_dtype, out_rows, out_halo, m_lo, m_hi, B,
            bias=bias, bias_mod=(bias.numel() if bias is not None else 0), n_lo=n_lo, n_hi=n_hi,
            d_lo=d_lo, d_hi=d_hi, w_tap0=w_tap0, ksplit=ksplit, backend=backend,
            a0_c=a0.shape[-1], a1_c=a1_c)
    torch.cuda.synchronize()
    a_full = a0.float() if a1 is None else torch.cat((a0.float(), a1.float()), -1)
    ref = _ref_f(a_full, halo, w, m_lo, m_hi, d_lo, d_hi, w_tap0)
    if bias is not None:
        ref = ref + bias.repeat(nc // bias.numel())
    got = out[:, out_halo + m_lo: out_halo + m_hi, n_lo:nhi].float()
    ref = ref[:, :, n_lo:nhi]
    err = max_abs(got, ref)
    tol = 3e-2 if tdt != torch.float32 else 2e-3
    assert err <= tol * max(1.0, float(ref.abs().max())), (case, backend, err, float(ref.abs().max()))
    if n_lo > 0:   # untouched columns stay zero
        assert float(out[:, :, :n_lo].abs().max()) == 0.0


F_REUSE_CASES = ["conv_fwd", "conv_fwd_n512", "deconv_cat", "conv_dgrad_halo", "deconv_dgrad_sub", "taps3"]


def _f_reuse_case(case):
    """The operands and geometry of one test_tapgemm_f_a_reuse case, as a dict of its local names."""
    g = _gen(8)
    B = 5
    a1, a1_c, bias = None, 0, None
    n_lo, n_hi, d_lo, d_hi = 0, None, -4, 4
    adt, odt, tdt = SG_F16, SG_F16, torch.float16
    if case in ("conv_fwd", "conv_fwd_n512", "taps3"):
        cin, cout, R, halo = (64, 128, 328, 4) if case != "conv_fwd_n512" else (128, 512, 136, 4)
        kc, nc = 4 * cin, cout
        w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        bias = torch.randn(nc, generator=g).to(DEV)
        if case == "taps3":
            d_lo, d_hi = -1, 1
    elif case == "deconv_cat":
        cout, R, halo = 64, 256, 0
        kc, nc = 256, 4 * cout
        w, taps = _packed_random("deconv_fwd", cout, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1_c = 128
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        bias = torch.randn(cout, generator=g).to(DEV)
    elif case == "conv_dgrad_halo":
        cin, cout, R, halo = 64, 128, 256, 0
        kc, nc = cout, 4 * cin
        w, taps = _packed_random("conv_dgrad", cin, kc, nc, g, torch.bfloat16)
        a0 = torch.randn(B, R, kc, generator=g).to(torch.bfloat16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = -4, R + 4, R, 4
        adt, odt, tdt = SG_BF16, SG_BF16, torch.bfloat16
    else:   # deconv dgrad, upper half of the columns only (z gets no gradient)
        cin, cout, R, halo = 512, 64, 192, 0
        kc, nc = 4 * cout, cin
        w, taps = _packed_random("deconv_dgrad", cout, kc, nc, g, torch.bfloat16)
        a0 = torch.randn(B, R, kc, generator=g).to(torch.bfloat16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        n_lo, n_hi = 256, 512
        adt, odt, tdt = SG_BF16, SG_BF16, torch.bfloat16
    return dict(locals())


@pytest.mark.parametrize("case", F_REUSE_CASES)
def test_tapgemm_f_a_reuse(case):
    """sg_set_cta_pair(2) (the activation-reuse schedule's setting; the sm_90a kernels run one schedule for every
    setting).  Shapes with >= 128 rows per batch element,
    a partial last M tile, an odd number of M tiles, two K sources, halo'd outputs and N sub-ranges."""
    _lib.load().sg_set_cta_pair(2)
    c = _f_reuse_case(case)
    B, R, halo, kc, nc, taps, w, a0, a1, a1_c, bias = (c[k] for k in ("B", "R", "halo", "kc", "nc", "taps", "w", "a0", "a1",
                                                                       "a1_c", "bias"))
    m_lo, m_hi, out_rows, out_halo, n_lo, n_hi = (c[k] for k in ("m_lo", "m_hi", "out_rows", "out_halo", "n_lo", "n_hi"))
    d_lo, d_hi, adt, odt, tdt = (c[k] for k in ("d_lo", "d_hi", "adt", "odt", "tdt"))
    nhi = nc if n_hi is None else n_hi
    out = torch.zeros(B, out_rows + 2 * out_halo, nc, dtype=tdt, device=DEV)
    E.run_f(a0, a1, R, halo, adt, w, adt, kc, nc, taps, out, odt, out_rows, out_halo, m_lo, m_hi, B,
            bias=bias, bias_mod=(bias.numel() if bias is not None else 0), n_lo=n_lo, n_hi=n_hi, d_lo=d_lo, d_hi=d_hi,
            backend=BACKEND_TCGEN05, a0_c=a0.shape[-1], a1_c=a1_c)
    torch.cuda.synchronize()
    a_full = a0.float() if a1 is None else torch.cat((a0.float(), a1.float()), -1)
    ref = _ref_f(a_full, halo, w, m_lo, m_hi, d_lo, d_hi)
    if bias is not None:
        ref = ref + bias.repeat(nc // bias.numel())
    got = out[:, out_halo + m_lo: out_halo + m_hi, n_lo:nhi].float()
    ref = ref[:, :, n_lo:nhi]
    err = max_abs(got, ref)
    assert err <= 3e-2 * max(1.0, float(ref.abs().max())), (case, err, float(ref.abs().max()))
    if n_lo > 0:
        assert float(out[:, :, :n_lo].abs().max()) == 0.0


@pytest.mark.parametrize("case", ["conv_fwd", "small_rows_two_ntiles", "wave_single_tap"])
def test_tapgemm_f_fused_bn_stats(case):
    """sg_tapgemm_f.bn_stats: the tensor-core kernel's epilogue accumulates per-column sum / sum of squares of the
    stored fp16 outputs (BatchNorm1d batch statistics) -- against the same statistics computed from the output."""
    g = _gen(9)
    d_lo, d_hi, w_tap0 = -4, 4, 0
    if case == "conv_fwd":
        B, cin, cout, R, halo = 5, 64, 128, 160, 4
        kc, nc = 4 * cin, cout
        w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    elif case == "small_rows_two_ntiles":
        B, cin, cout, R, halo = 33, 128, 512, 16, 4
        kc, nc = 4 * cin, cout
        w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    else:
        B, R, halo, kc, nc = 3, 512, 0, 64, 64
        taps = E.tap_ranges("full", 0, kc, nc)
        w = (torch.randn(1, nc, kc, generator=g) * 0.2).to(torch.float16).to(DEV)
        a0 = torch.randn(B, R, kc, generator=g).to(torch.float16).to(DEV)
        d_lo = d_hi = 0
        w_tap0 = 4
    bias = torch.randn(nc, generator=g).to(DEV)
    out = torch.zeros(B, R, nc, dtype=torch.float16, device=DEV)
    stats = torch.zeros(8, 2, nc, dtype=torch.float64, device=DEV)
    E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, nc, taps, out, SG_F16, R, 0, 0, R, B, bias=bias, bias_mod=nc,
            d_lo=d_lo, d_hi=d_hi, w_tap0=w_tap0, backend=BACKEND_TCGEN05, stats=stats)
    ref_stats = torch.zeros(8, 2, nc, dtype=torch.float64, device=DEV)
    _lib.call("sg_bn_stats", _p(out), SG_F16, B * R, nc, _p(ref_stats), _stream())
    torch.cuda.synchronize()
    o64 = out.double().reshape(-1, nc)
    got = stats.sum(0)
    assert rel_err(got[0], o64.sum(0)) <= 1e-5 and rel_err(got[1], (o64 * o64).sum(0)) <= 1e-5
    assert rel_err(got, ref_stats.sum(0)) <= 1e-5
    # and the output itself is what the un-fused launch writes
    out2 = torch.zeros_like(out)
    E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, nc, taps, out2, SG_F16, R, 0, 0, R, B, bias=bias, bias_mod=nc,
            d_lo=d_lo, d_hi=d_hi, w_tap0=w_tap0, backend=BACKEND_TCGEN05)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("mode", ["narrow", "splitk"])
@pytest.mark.parametrize("sms,case,B", [(8, "deconv_cat", 17), (8, "deconv_cat", 21), (8, "small_rows", 33),
                                        (8, "dgrad_halo", 9), (8, "dgrad_halo", 10)])
def test_tapgemm_f_wave_split(monkeypatch, sms, case, B, mode):
    """engine.run_f splits a launch whose tile count is just over a multiple of the CTA pairs into whole
    waves of full-width tiles plus a tail of narrow tiles on a batch sub-range (pointer offsets, tile_n
    hint).  The SM count is patched down so that small test shapes take that path."""
    monkeypatch.setattr(E, "NUM_SMS", sms)
    monkeypatch.setattr(E, "SPLIT_WAVES", mode == "narrow")
    monkeypatch.setattr(E, "SPLITK_TAIL", mode == "splitk")     # tail = split-K into fp32 + convert kernel
    g = _gen(4)
    a1, a1_c, bias = None, 0, None
    if case == "deconv_cat":
        cout, R, halo = 64, 64, 0
        kc, nc = 256, 4 * cout
        w, taps = _packed_random("deconv_fwd", cout, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1_c = 128
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        bias = torch.randn(cout, generator=g).to(DEV)
        adt, odt, tdt = SG_F16, SG_F16, torch.float16
    elif case == "small_rows":
        cin, cout, R, halo = 128, 512, 16, 4
        kc, nc = 4 * cin, cout
        w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = 0, R, R, 0
        adt, odt, tdt = SG_F16, SG_F16, torch.float16
    else:   # conv dgrad into a halo'd consumer view, bf16
        cin, cout, R, halo = 64, 128, 160, 0
        kc, nc = cout, 4 * cin
        w, taps = _packed_random("conv_dgrad", cin, kc, nc, g, torch.bfloat16)
        a0 = torch.randn(B, R, kc, generator=g).to(torch.bfloat16).to(DEV)
        m_lo, m_hi, out_rows, out_halo = -4, R + 4, R, 4
        adt, odt, tdt = SG_BF16, SG_BF16, torch.bfloat16
    if mode == "narrow":
        b1, tn = E._plan_f_split(m_hi - m_lo, B, nc)
    else:
        ksteps = sum((taps[1][i] - taps[0][i]) // 64 for i in range(9))
        b1, tn = E._plan_f_tail_splitk(m_hi - m_lo, B, nc, ksteps)
        if not (0 < b1 < B):
            pytest.skip("no split-K tail for this shape")
    assert 0 < b1 < B, (b1, tn)                       # the split path is what this test exercises
    out = torch.zeros(B, out_rows + 2 * out_halo, nc, dtype=tdt, device=DEV)
    E.run_f(a0, a1, R, halo, adt, w, adt, kc, nc, taps, out, odt, out_rows, out_halo, m_lo, m_hi, B,
            bias=bias, bias_mod=(bias.numel() if bias is not None else 0), backend=BACKEND_TCGEN05,
            a0_c=a0.shape[-1], a1_c=a1_c)
    torch.cuda.synchronize()
    a_full = a0.float() if a1 is None else torch.cat((a0.float(), a1.float()), -1)
    ref = _ref_f(a_full, halo, w, m_lo, m_hi)
    if bias is not None:
        ref = ref + bias.repeat(nc // bias.numel())
    got = out[:, out_halo + m_lo: out_halo + m_hi, :].float()
    err = max_abs(got, ref)
    assert err <= 3e-2 * max(1.0, float(ref.abs().max())), (case, sms, b1, tn, err)


def test_wgrad_split_plan_fills_whole_waves():
    """The weight-gradient split count is chosen from the exact number of non-empty (tap, n, kc) tiles."""
    fm = [64, 128, 256, 512, 1024]
    for l in range(1, 5):
        cin, cout, Lq = fm[l - 1], fm[l], 16384 // 4 ** (l + 1)
        taps = E.tap_ranges("conv_fwd", cin, 4 * cin, cout)
        ks = E.wgrad_ksplit(300 * Lq, 0, taps, 4 * cin, cout)
        tk = 256 if 4 * cin >= 256 else 4 * cin
        valid = sum(1 for d in range(9) for n0 in range(0, cout, 128) for k0 in range(0, 4 * cin, tk)
                    if not (n0 + 128 <= taps[2][d] or n0 >= taps[3][d] or k0 + tk <= taps[0][d] or k0 >= taps[1][d]))
        tiles = valid * ks
        assert tiles / float(-(-tiles // E.NUM_SMS) * E.NUM_SMS) >= 0.8, (l, ks, tiles)


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05])
@pytest.mark.parametrize("case", ["conv", "deconv_cat", "small_rows", "conv_wide", "fc"])
def test_tapgemm_w(backend, case):
    g = _gen(2)
    a1, a1_c = None, 0
    d_lo, d_hi, tap0, ksplit = -4, 4, 0, 3
    if case == "conv":
        B, cin, cout, R, halo = 3, 64, 128, 128, 4
        kc, nc = 4 * cin, cout
        taps = E.tap_ranges("conv_fwd", cin, kc, nc)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    elif case == "deconv_cat":
        B, cin, cout, R, halo = 2, 256, 64, 64, 0
        kc, nc = cin, 4 * cout
        taps = E.tap_ranges("deconv_fwd", cout, kc, nc)
        a0 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1 = torch.randn(B, R, 128, generator=g).to(torch.float16).to(DEV)
        a1_c = 128
    elif case == "small_rows":
        B, cin, cout, R, halo = 9, 128, 128, 16, 4
        kc, nc = 4 * cin, cout
        taps = E.tap_ranges("conv_fwd", cin, kc, nc)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    elif case == "conv_wide":           # 2 x 2 blocks of 256 x 256 per tap
        B, cin, cout, R, halo = 5, 128, 512, 64, 4
        kc, nc = 4 * cin, cout
        taps = E.tap_ranges("conv_fwd", cin, kc, nc)
        a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    else:
        B, kc, nc, R, halo = 70, 1024, 256, 1, 0
        taps = E.tap_ranges("full", 0, kc, nc)
        a0 = torch.randn(B, 1, kc, generator=g).to(torch.float16).to(DEV)
        d_lo = d_hi = 0
        tap0, ksplit = 4, 1
    gg = (torch.randn(B, R, nc, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    slots = d_hi + 4 - tap0 + 1
    dw = torch.zeros(slots, nc, kc, dtype=torch.float32, device=DEV)
    a0 = a0.to(torch.bfloat16)
    a1 = a1.to(torch.bfloat16) if a1 is not None else None
    E.run_w(gg, R, SG_BF16, a0, a1, R, halo, SG_BF16, kc, nc, taps, dw, B, d_lo=d_lo, d_hi=d_hi, dw_tap0=tap0,
            ksplit=ksplit, backend=backend, a0_c=a0.shape[-1], a1_c=a1_c)
    torch.cuda.synchronize()
    a_full = a0.float() if a1 is None else torch.cat((a0.float(), a1.float()), -1)
    ap = F.pad(a_full, (0, 0, 16, 16))
    for d in range(d_lo, d_hi + 1):
        rows = ap[:, 16 + halo + d: 16 + halo + d + R, :]
        ref = torch.einsum("bmn,bmk->nk", gg.float(), rows)
        mask = torch.zeros(nc, kc, device=DEV)
        mask[taps[2][d + 4]:taps[3][d + 4], taps[0][d + 4]:taps[1][d + 4]] = 1
        got = dw[d + 4 - tap0]
        err = max_abs(got * mask, ref * mask)
        assert err <= 2e-3 * max(1.0, float(ref.abs().max())), (case, backend, d, err)
        assert float((got * (1 - mask)).abs().max()) == 0.0, (case, d, "structural zeros written")


def test_pack_and_unpack_roundtrip():
    g = _gen(3)
    for kind, (co, ci) in ((0, (128, 64)), (1, (64, 256))):
        shape = (co, ci, 31) if kind == 0 else (ci, co, 31)
        w = (torch.randn(*shape, generator=g) * 0.1).to(DEV)
        alpha = (torch.rand(ci // 2, generator=g) + 0.5).to(DEV) if kind == 1 else None
        if kind == 0:
            wf = torch.zeros(9, co, 4 * ci, dtype=torch.float16, device=DEV)
            wd = torch.zeros(9, 4 * ci, co, dtype=torch.bfloat16, device=DEV)
        else:
            wf = torch.zeros(9, 4 * co, ci, dtype=torch.float16, device=DEV)
            wd = torch.zeros(9, ci, 4 * co, dtype=torch.bfloat16, device=DEV)
        _lib.call("sg_pack_weights", kind, _p(w), co, ci, 0, _p(alpha), ci // 2, _p(wf), _p(wd), SG_F16, SG_BF16,
                  _stream())
        # semantic check: tap-GEMM on the packed weights == the reference op on the fp32 weights
        B, R = 2, 32
        if kind == 0:
            x = torch.randn(B, ci, 4 * R, generator=g).to(DEV)                # NCL input, L = 4R
            ref = O.gconv_linear(x.cpu(), w.cpu().half().float(), None)       # (B, co, R)
            xp = F.pad(x, (16, 16), mode="reflect")                          # 16-position halo
            a = xp.permute(0, 2, 1).contiguous().view(B, R + 8, 4 * ci).half()
            out = torch.zeros(B, R, co, dtype=torch.float16, device=DEV)
            E.run_f(a, None, R, 4, SG_F16, wf, SG_F16, 4 * ci, co, E.tap_ranges("conv_fwd", ci, 4 * ci, co), out,
                    SG_F16, R, 0, 0, R, B, backend=BACKEND_FFMA)
            got = out.float().permute(0, 2, 1).cpu()
            ref = O.gconv_linear(x.half().float().cpu(), w.cpu().half().float(), None)
        else:
            x = torch.randn(B, ci, R, generator=g).to(DEV)
            weff = w.clone()
            weff[ci // 2:] *= alpha.view(-1, 1, 1)
            ref = O.gdeconv_linear(x.half().float().cpu(), weff.cpu().half().float(), torch.zeros(co))
            a = x.permute(0, 2, 1).contiguous().half()
            out = torch.zeros(B, R, 4 * co, dtype=torch.float16, device=DEV)
            E.run_f(a, None, R, 0, SG_F16, wf, SG_F16, ci, 4 * co, E.tap_ranges("deconv_fwd", co, ci, 4 * co), out,
                    SG_F16, R, 0, 0, R, B, backend=BACKEND_FFMA)
            got = out.float().view(B, 4 * R, co).permute(0, 2, 1).cpu()
        torch.cuda.synchronize()
        assert max_abs(got, ref) <= 2e-2 * max(1.0, float(ref.abs().max())), kind
        # unpack(pack-layout gradient) restores the reference layout
        dwp = wf.float().contiguous()
        dw = torch.zeros_like(w)
        dalpha = torch.zeros(ci // 2, device=DEV) if kind == 1 else None
        _lib.call("sg_unpack_wgrad", kind, _p(dwp), co, ci, 0, _p(w), _p(alpha), ci // 2, _p(dw), _p(dalpha), 0,
                  _stream())
        torch.cuda.synchronize()
        if kind == 0:
            assert max_abs(dw, w.half().float()) == 0.0
        else:
            weff16 = (weff.half().float())
            exp = weff16.clone()
            exp[ci // 2:] *= alpha.view(-1, 1, 1)
            assert max_abs(dw, exp) <= 1e-6
            assert max_abs(dalpha, (weff16[ci // 2:] * w[ci // 2:]).sum((1, 2))) <= 1e-3


def test_wave_conv_fwd_and_grads(grad_dtype):
    g = _gen(4)
    B, L, roll = 3, 4096, -3
    x0 = (0.3 * torch.randn(B, L, generator=g)).to(DEV)
    x1 = (0.3 * torch.randn(B, L, generator=g)).to(DEV)
    w = (0.05 * torch.randn(64, 2, 31, generator=g)).to(DEV)
    bias = (0.1 * torch.randn(64, generator=g)).to(DEV)
    a = torch.zeros(B, L // 4, 64, dtype=torch.float16, device=DEV)
    _lib.call("sg_wave_conv_fwd", _p(x0), _p(x1), 2, B, L, roll, _p(w), _p(bias), 64, _p(a), None, None, _stream())
    xin = torch.stack((x0, x1), 1).cpu()
    ref = O.gconv_linear(O.phase_roll(xin, roll), w.cpu(), bias.cpu())
    torch.cuda.synchronize()
    assert max_abs(a.float().permute(0, 2, 1).cpu(), ref) <= 2e-3 * float(ref.abs().max())
    # G variant: 1 channel, PReLU + reflect halo
    slope = (0.2 * torch.rand(64, generator=g)).to(DEV)
    hp = torch.zeros(B, L // 4 + 32, 64, dtype=torch.float16, device=DEV)
    w1 = w[:, :1].contiguous()
    _lib.call("sg_wave_conv_fwd", _p(x0), None, 1, B, L, 0, _p(w1), None, 64, _p(a), _p(slope), _p(hp), _stream())
    ref1 = O.gconv_linear(x0.cpu().unsqueeze(1), w1.cpu(), None)
    h_ref = F.pad(F.prelu(ref1, slope.cpu()), (16, 16), mode="reflect")
    torch.cuda.synchronize()
    assert max_abs(hp.float().permute(0, 2, 1).cpu(), h_ref) <= 2e-3 * float(h_ref.abs().max())
    # gradients of the 2-channel rolled conv
    ga = (0.1 * torch.randn(B, L // 4, 64, generator=g)).to(E.GT).to(DEV)
    dw = torch.zeros_like(w)
    db = torch.zeros(64, device=DEV)
    _lib.call("sg_wave_conv_wgrad", _p(x0), _p(x1), 2, B, L, roll, _p(ga), 64, _p(dw), _p(db), _stream())
    gx0 = torch.zeros(B, L, device=DEV)
    _lib.call("sg_wave_conv_dgrad", _p(ga), B, L, roll, _p(w), 2, 64, _p(gx0), 0, _stream())
    xin_r = xin.clone().requires_grad_(True)
    wr = w.cpu().clone().requires_grad_(True)
    out = O.gconv_linear(O.phase_roll(xin_r, roll), wr, bias.cpu())
    out.backward(ga.float().permute(0, 2, 1).cpu())
    torch.cuda.synchronize()
    assert rel_err(dw.cpu(), wr.grad) <= 1e-4
    assert rel_err(db.cpu(), ga.float().sum((0, 1)).cpu()) <= 1e-4
    assert rel_err(gx0.cpu(), xin_r.grad[:, 0]) <= 1e-4


def test_wave_deconv_fwd_and_bwd(grad_dtype):
    g = _gen(5)
    B, Lin = 2, 1024
    x0 = (torch.randn(B, Lin, 64, generator=g)).to(torch.float16).to(DEV)
    x1 = (torch.randn(B, Lin, 64, generator=g)).to(torch.float16).to(DEV)
    w = (0.05 * torch.randn(128, 31, generator=g)).to(DEV)
    bias = torch.tensor([0.05], device=DEV)
    y = torch.zeros(B, 4 * Lin, device=DEV)
    _lib.call("sg_wave_deconv_fwd", _p(x0), 64, _p(x1), 64, B, Lin, _p(w), _p(bias), _p(y), _stream())
    xin = torch.cat((x0, x1), -1).float().permute(0, 2, 1).cpu().requires_grad_(True)
    wr = w.cpu().view(128, 1, 31).clone().requires_grad_(True)
    br = bias.cpu().clone().requires_grad_(True)
    ref = torch.tanh(O.gdeconv_linear(xin, wr, br))
    torch.cuda.synchronize()
    assert max_abs(y.cpu(), ref[:, 0].detach()) <= 1e-4
    gy = (torch.randn(B, 4 * Lin, generator=g)).to(DEV)
    gpre = torch.zeros_like(gy)
    gx = torch.zeros(B, Lin, 128, dtype=E.GT, device=DEV)
    dw = torch.zeros_like(w)
    db = torch.zeros(1, device=DEV)
    _lib.call("sg_wave_deconv_bwd", _p(x0), 64, _p(x1), 64, B, Lin, _p(w), _p(gy), _p(y), _p(gpre), _p(gx),
              _p(dw), _p(db), _stream())
    ref.backward(gy.cpu().unsqueeze(1))
    torch.cuda.synchronize()
    assert rel_err(dw.cpu(), wr.grad[:, 0]) <= 1e-3
    assert rel_err(db.cpu(), br.grad) <= 1e-3
    assert rel_err(gx.float().permute(0, 2, 1).cpu(), xin.grad) <= 1e-2      # bf16 output


@pytest.mark.parametrize("variant", [(4, 2, 3), (4, 4, 16), (4, 8, 2), (8, 2, 8), (8, 4, 1), (16, 2, 2)])
@pytest.mark.parametrize("C_,L,roll,halo", [(64, 256, 2, 16), (256, 64, -5, 16), (1024, 16, 0, 0), (128, 96, 4, 16)])
def test_bn_act_fwd_bwd(C_, L, roll, halo, variant, grad_dtype):
    """Every streaming-kernel variant (channels/thread, rows in flight, grid cap; for the backward
    kernels vec 8 = the tiled kernel, vec 4 = the generic one; vec 16 = the TMA-staged kernels of stream_ew.cu)
    against fp32 torch."""
    lib = _lib.load()
    for kind in (1, 2, 3, 4):
        v = variant if not (kind >= 3 and variant == (4, 8, 2)) else (4, 4, 2)
        assert lib.sg_set_ew_variant(kind, *v) == 0
    assert lib.sg_set_ew_variant(1, 3, 2, 3) != 0 and lib.sg_set_ew_variant(9, 4, 2, 3) != 0   # rejected
    g = _gen(6)
    B = 4
    a = torch.randn(B, L, C_, generator=g).to(torch.float16).to(DEV)
    gamma = (1 + 0.1 * torch.randn(C_, generator=g)).to(DEV)
    beta = (0.1 * torch.randn(C_, generator=g)).to(DEV)
    slope = (0.2 * torch.rand(C_, generator=g)).to(DEV)
    rm, rv = torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV)
    stats = torch.zeros(8, 2, C_, dtype=torch.float64, device=DEV)
    ss = torch.zeros(2, C_, device=DEV)
    mi = torch.zeros(2, C_, device=DEV)
    _lib.call("sg_bn_stats", _p(a), SG_F16, B * L, C_, _p(stats), _stream())
    _lib.call("sg_bn_finalize", _p(stats), B * L, C_, _p(gamma), _p(beta), 1e-5, 0.1, _p(rm), _p(rv), _p(ss),
              _p(mi), _stream())
    h = torch.zeros(B, L + 2 * halo, C_, dtype=torch.float16, device=DEV)
    hb = torch.zeros(B, L + 2 * halo, C_, dtype=torch.bfloat16, device=DEV)
    abf = torch.zeros(B, L, C_, dtype=torch.bfloat16, device=DEV)
    _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(slope), 1, roll, None, halo, _p(h), _p(hb), _p(abf),
              _stream())
    # the same launch with the shift read from device memory (CUDA-graph mode): identical result
    roll_dev = torch.tensor([7, roll], dtype=torch.int32, device=DEV)
    rptr = C.c_void_p(roll_dev.data_ptr() + 4)
    h_d = torch.zeros_like(h)
    _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(slope), 1, 0, rptr, halo, _p(h_d), None, None,
              _stream())
    assert torch.equal(h_d, h)
    # reference: NCL fp32
    an = a.float().permute(0, 2, 1).cpu().requires_grad_(True)
    gm, bt, sl = (t.cpu().clone().requires_grad_(True) for t in (gamma, beta, slope))
    rm_r, rv_r = torch.zeros(C_), torch.ones(C_)
    y = F.prelu(O.batchnorm_train(an, gm, bt, rm_r, rv_r), sl)
    yr = O.phase_roll(y, roll)
    if halo:
        yr = F.pad(yr, (halo, halo), mode="reflect")
    torch.cuda.synchronize()
    e_h = max_abs(h.float().permute(0, 2, 1).cpu(), yr.detach())
    assert e_h <= 1e-2, ("act_fwd", e_h)
    assert max_abs(hb.float(), h.float()) <= 4e-2 and max_abs(abf.float(), a.float()) <= 4e-2
    assert max_abs(rm.cpu(), rm_r) <= 1e-5 and max_abs(rv.cpu(), rv_r) <= 1e-4
    # backward: gradient arrives in the consumer view (incl. halo)
    gh = (torch.randn(B, L + 2 * halo, C_, generator=g)).to(E.GT).to(DEV)
    yr.backward(gh.float().permute(0, 2, 1).cpu())
    red = torch.zeros(8, 3, C_, dtype=torch.float64, device=DEV)
    ga = torch.zeros(B, L, C_, dtype=E.GT, device=DEV)
    _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, roll, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
              _p(slope), 1, _p(red), None, _stream())
    # no-BN variant with a skip gradient on the pre-activation (Generator encoder), strided sources
    gsk = (torch.randn(B, L, 2 * C_, generator=g)).to(E.GT).to(DEV)
    a2 = a.float().permute(0, 2, 1).cpu().requires_grad_(True)
    sl2 = slope.cpu().clone().requires_grad_(True)
    y2 = F.prelu(a2, sl2)
    y2p = F.pad(y2, (halo, halo), mode="reflect") if halo else y2
    (y2p * gh.float().permute(0, 2, 1).cpu()).sum().add((a2 * gsk[:, :, C_:].float().permute(0, 2, 1).cpu()).sum()).backward()
    red2 = torch.zeros(8, 3, C_, dtype=torch.float64, device=DEV)
    ga2 = torch.zeros(B, L, C_, dtype=E.GT, device=DEV)
    gadd_ptr = C.c_void_p(gsk.data_ptr() + 2 * C_)
    _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, 0, None, gadd_ptr, 2 * C_, _p(a), SG_F16, B, L, C_, None, None,
              _p(slope), 1, _p(red2), _p(ga2), _stream())
    torch.cuda.synchronize()
    assert rel_err(ga2.float().permute(0, 2, 1).cpu(), a2.grad) <= 1e-2
    rs2 = red2.sum(0)
    assert rel_err(rs2[0].float().cpu(), sl2.grad) <= 2e-3
    assert rel_err(rs2[1].float().cpu(), a2.grad.sum((0, 2))) <= 2e-3
    _lib.call("sg_act_bwd_apply", _p(gh), C_, halo, roll, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
              _p(slope), 1, _p(red), 1, _p(ga), _stream())
    ga_d = torch.zeros_like(ga)
    _lib.call("sg_act_bwd_apply", _p(gh), C_, halo, 0, rptr, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
              _p(slope), 1, _p(red), 1, _p(ga_d), _stream())
    red_d = torch.zeros_like(red)
    _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, 0, rptr, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
              _p(slope), 1, _p(red_d), None, _stream())
    gp = torch.ones(3, C_, device=DEV)
    _lib.call("sg_stat_grads", _p(red), C_, 3, _p(gp[0]), None, _p(gp[2]), _stream())
    torch.cuda.synchronize()
    rs = red.sum(0)
    assert torch.equal(ga_d, ga) and rel_err(red_d.sum(0), rs) <= 1e-6
    assert rel_err(gp[0] - 1, rs[0].float()) <= 1e-6 and rel_err(gp[2] - 1, rs[2].float()) <= 1e-6
    assert float((gp[1] - 1).abs().max()) == 0.0
    assert rel_err(rs[0].float().cpu(), sl.grad) <= 2e-3
    assert rel_err(rs[1].float().cpu(), bt.grad) <= 2e-3
    assert rel_err(rs[2].float().cpu(), gm.grad) <= 2e-3
    assert rel_err(ga.float().permute(0, 2, 1).cpu(), an.grad) <= 1e-2


def test_deemphasis_and_preemphasis():
    g = _gen(8)
    y = (0.1 * torch.randn(50001, generator=g))
    x = torch.zeros_like(y).to(DEV)
    _lib.call("sg_deemphasis", _p(y.to(DEV)), y.numel(), 0.95, _p(x), _stream())
    torch.cuda.synchronize()
    ref = O.de_emphasize(y.numpy(), 0.95)
    assert max_abs(x.cpu(), torch.from_numpy(ref)) <= 2e-5
    back = torch.zeros_like(x)
    _lib.call("sg_preemphasis", _p(x), y.numel(), 0.95, _p(back), _stream())
    torch.cuda.synchronize()
    assert max_abs(back.cpu(), y) <= 1e-5


def test_cpu_tensor_rejected_loudly():
    from tests.util import build_segan
    s = build_segan()
    with pytest.raises(RuntimeError):
        s.G(torch.zeros(1, 1, 16384))


# ------------------------------------------------------------------------------------------------------
# round 2: stream-K over the last partial wave and the fused PReLU (+ reflect halo) output of the tensor-core
# forward-form kernel
# ------------------------------------------------------------------------------------------------------
def _sk_case(case, g):
    """Shapes with MORE tiles than the 132 CTAs of an H100 and a ragged last wave."""
    if case == "conv_fwd":          # 1024 rows x 12 batches = 96 M tiles x 2 N tiles = 192 = 132 + 60
        B, cin, cout, R, halo = 12, 64, 512, 1024, 4
        kc, nc, kind, c = 4 * cin, cout, "conv_fwd", cin
        m_lo, m_hi, out_halo = 0, R, 0
    elif case == "deconv_fwd":      # tap-dependent N ranges: tiles of different N have different k-step counts
        B, cin, cout, R, halo = 41, 128, 128, 256, 0       # 82 M tiles x 2 N tiles = 164 = 132 + 32
        kc, nc, kind, c = cin, 4 * cout, "deconv_fwd", cout
        m_lo, m_hi, out_halo = 0, R, 0
    else:                           # conv_dgrad into a halo'd view, two M tiles per batch element (the second one short)
        B, cin, cout, R, halo = 77, 64, 128, 128, 0        # rows -4..132 = 136 -> 2 M tiles x 77 = 154 = 132 + 22
        kc, nc, kind, c = cout, 4 * cin, "conv_dgrad", cin
        m_lo, m_hi, out_halo = -4, R + 4, 4
    w, taps = _packed_random(kind, c, kc, nc, g, torch.float16)
    a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.float16).to(DEV)
    return B, kc, nc, R, halo, m_lo, m_hi, out_halo, w, taps, a0


@pytest.mark.parametrize("case", ["conv_fwd", "deconv_fwd", "conv_dgrad"])
def test_tapgemm_f_stream_k(case):
    """The leftover tiles of the last wave are split along K over several CTAs (fp32 partial sums in per-CTA
    workspace slots, summed in slot order by the warp that counts the last contribution): same result as the
    unsplit schedule up to the fp32 summation order, counters left zeroed, bitwise repeatable."""
    g = _gen(21)
    B, kc, nc, R, halo, m_lo, m_hi, out_halo, w, taps, a0 = _sk_case(case, g)
    bias = torch.randn(nc, generator=g).to(DEV)
    outs = []
    ws = E.sk_workspace(DEV)
    assert ws is not None and int(ws[:8192].count_nonzero()) == 0     # counters; the slots keep stale partial sums
    ws[8192:].zero_()
    lib = _lib.load()
    for sk in (False, True, True):
        prev = E.STREAM_K
        E.STREAM_K = sk
        lib.sg_set_stream_k(16, 1e-6)          # force the split whatever the cost model says about this shape
        try:
            out = torch.zeros(B, R + 2 * out_halo, nc, dtype=torch.float16, device=DEV)
            E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, nc, taps, out, SG_F16, R, out_halo, m_lo, m_hi, B,
                    bias=bias, bias_mod=nc, backend=BACKEND_TCGEN05)
            torch.cuda.synchronize()
            outs.append(out.float().cpu())
        finally:
            E.STREAM_K = prev
            lib.sg_set_stream_k(16, 2.5)
    assert int(ws[:8192].count_nonzero()) == 0, "the split-K counters must be left zeroed"
    assert int(ws[8192:].count_nonzero()) > 0, "the split path did not run"
    ref = _ref_f(F.pad(a0.float().cpu(), (0, 0, 0, 0)), halo, w.cpu(), m_lo, m_hi) + bias.cpu()
    lo = out_halo + m_lo
    for o in outs:
        assert rel_err(o[:, lo:lo + (m_hi - m_lo)], ref) <= 2e-3
    # split vs unsplit: only the fp32 summation order of the split tiles differs (then one fp16 rounding)
    assert max_abs(outs[1], outs[0]) <= 4e-3 * float(ref.abs().max())
    # the partial sums are added in slot order by whichever warp finishes the tile: bitwise repeatable
    assert torch.equal(outs[1], outs[2])


@pytest.mark.parametrize("halo", [16, 0])
@pytest.mark.parametrize("inplace", [False, True])
def test_tapgemm_f_fused_prelu_output(halo, inplace):
    """sg_tapgemm_f.out2 / .slope: PReLU(out) written by the epilogue, with the reflect halo of the next conv
    (modules.py:92-101), next to the raw output -- or into the only output (inference decoder) -- also on tiles
    finished through the stream-K path."""
    if inplace and halo:
        pytest.skip("in-place activation has no halo")
    g = _gen(22)
    B, cin, cout, R = 12, 64, 512, 1024            # 192 tiles on 132 CTAs: 60 of them take the stream-K path
    kc, nc = 4 * cin, cout
    w, taps = _packed_random("conv_fwd", cin, kc, nc, g, torch.float16)
    a0 = torch.randn(B, R + 8, kc, generator=g).to(torch.float16).to(DEV)
    bias = torch.randn(nc, generator=g).to(DEV)
    slope = (0.3 * torch.rand(128, generator=g)).to(DEV)        # slope index = n % 128
    out = torch.zeros(B, R, nc, dtype=torch.float16, device=DEV)
    out2 = torch.zeros(B, R + 2 * halo, nc, dtype=torch.float16, device=DEV)
    _lib.load().sg_set_stream_k(16, 1e-6)      # force the split of the 22 leftover tiles
    if inplace:
        E.run_f(a0, None, R, 4, SG_F16, w, SG_F16, kc, nc, taps, out, SG_F16, R, 0, 0, R, B, bias=bias, bias_mod=nc,
                backend=BACKEND_TCGEN05, slope=slope, slope_mod=128)
    else:
        E.run_f(a0, None, R, 4, SG_F16, w, SG_F16, kc, nc, taps, out, SG_F16, R, 0, 0, R, B, bias=bias, bias_mod=nc,
                backend=BACKEND_TCGEN05, out2=out2, out2_halo=halo, slope=slope, slope_mod=128)
    torch.cuda.synchronize()
    _lib.load().sg_set_stream_k(16, 2.5)
    ref = _ref_f(a0.float().cpu(), 4, w.cpu(), 0, R) + bias.cpu()                       # (B, R, nc)
    sl = slope.cpu().repeat(nc // 128)
    act = torch.where(ref > 0, ref, ref * sl)
    if inplace:
        assert rel_err(out.float().cpu(), act) <= 2e-3
        return
    assert rel_err(out.float().cpu(), ref) <= 2e-3
    if halo:
        act = F.pad(act.permute(0, 2, 1), (halo, halo), mode="reflect").permute(0, 2, 1)
    assert rel_err(out2.float().cpu(), act) <= 2e-3
    # the halo rows are bit-copies of their mirror positions
    if halo:
        o2 = out2.cpu()
        assert torch.equal(o2[:, 0], o2[:, 2 * halo]) and torch.equal(o2[:, halo + R + halo - 1], o2[:, halo + R - 1 - halo])


def test_generator_forward_fused_vs_unfused_activation():
    """Generator forward with the activation in the GEMM epilogue vs the separate sg_act_fwd pass: the fused path
    rounds PReLU(fp32 accumulator) once, the separate pass rounds the pre-activation first -- one fp16 ulp apart."""
    from tests.util import build_segan
    s = build_segan().to(DEV)
    g = _gen(23)
    x = (0.3 * torch.randn(5, 1, 16384, generator=g)).to(DEV)
    z = torch.randn(5, 1024, 16, generator=g).to(DEV)
    s.G.eval()
    outs = []
    for fuse in (True, False):
        prev = E.FUSE_ACT
        E.FUSE_ACT = fuse
        try:
            with torch.no_grad():
                outs.append(s.G(x, z=z).cpu())
        finally:
            E.FUSE_ACT = prev
    assert max_abs(outs[0], outs[1]) <= 3e-4


@pytest.mark.parametrize("B,L,kind", [(3, 16384, "speech"), (2, 4096, "white"), (5, 16384, "weak_hf")])
def test_spectral_loss_gemm_vs_torch_stft(B, L, kind):
    """WSEGAN's log-power STFT L1 (model.py:638-653) as one tap-GEMM over the frames (engine.SpectralLoss) against
    torch.stft + autograd in fp64: loss to 1e-4 relative (two-halves fp16 operands), gradient to 1 % rel-L2 (bf16
    dL/dX).  'weak_hf' = a 70 dB spectral tilt: the bins an un-split fp16 transform would bury in rounding noise."""
    g = _gen(51)
    x = torch.randn(B, 1, L, generator=g)
    if kind != "white":
        # low-pass tilt: running mean filters make the high bins 40-70 dB weaker than the low ones
        k = 9 if kind == "speech" else 33
        for _ in range(2):
            x = F.avg_pool1d(F.pad(x, (k // 2, k // 2), mode="reflect"), k, stride=1)
        x = x / x.abs().max()
    y = (x + 0.05 * torch.randn(B, 1, L, generator=g) * (1.0 if kind == "white" else 0.01)).clamp(-1, 1)

    def logpow(t):
        st = torch.stft(t.squeeze(1), n_fft=2048, hop_length=160, win_length=320, normalized=True, return_complex=True)
        return 10 * torch.log10(st.real ** 2 + st.imag ** 2 + 10e-20)
    yd = y.double().requires_grad_(True)
    ref = 0.37 * (logpow(yd) - logpow(x.double())).abs().mean()
    gref, = torch.autograd.grad(ref, yd)
    sp = E.SpectralLoss(torch.device(DEV))
    loss = torch.zeros(1, device=DEV)
    gw = torch.zeros(B, 1, L, device=DEV)
    sp(y.to(DEV), x.to(DEV), 0.37, C.c_void_p(loss.data_ptr()), g_wave=gw, g_scale=8.0)
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) <= 1e-4 * abs(float(ref)), (float(loss), float(ref))
    assert rel_err(gw.cpu() / 8.0, gref.float()) <= 1e-2
    # loss only (no gradient buffers touched)
    loss2 = torch.zeros(1, device=DEV)
    sp(y.to(DEV), x.to(DEV), 0.37, C.c_void_p(loss2.data_ptr()))
    assert float(loss2) == pytest.approx(float(loss), rel=2e-5)          # atomics: summation order differs run to run


@pytest.mark.parametrize("C_,L,roll,halo,B", [(64, 1024, 3, 16, 160), (128, 256, -5, 16, 300), (512, 64, 1, 16, 300),
                                               (1024, 16, 0, 0, 300), (64, 4096, -2, 16, 24)])
def test_tma_staged_glue_kernels_match_register_staged(C_, L, roll, halo, B):
    """stream_ew.cu (variant vec 16: cp.async.bulk row tiles through an mbarrier ring, two row ranges per batch element
    at the phase-shift wrap) against the register-staged kernels at sizes where every CTA walks more tiles than its
    ring has stages: forward and BN-backward outputs bit-identical (same fp32 arithmetic per element), reductions equal
    up to the summation order."""
    lib = _lib.load()
    g = _gen(31)
    a = torch.randn(B, L, C_, generator=g).to(torch.float16).to(DEV)
    gh = torch.randn(B, L + 2 * halo, C_, generator=g).to(E.GT).to(DEV)
    gadd = torch.randn(B, L, C_, generator=g).to(E.GT).to(DEV)
    ss = torch.randn(2, C_, generator=g).to(DEV)
    mi = (torch.randn(2, C_, generator=g).abs() + 0.5).to(DEV)
    slope = (0.2 * torch.rand(C_, generator=g)).to(DEV)
    roll_dev = torch.tensor([roll], dtype=torch.int32, device=DEV)
    outs = {}
    for tag, variants in (("reg", EW_DEFAULT_REG), ("tma", {k: (16, 2, 2) for k in (1, 2, 3, 4)})):
        for kind, v in variants.items():
            assert lib.sg_set_ew_variant(kind, *v) == 0
        stats = torch.zeros(8, 2, C_, dtype=torch.float64, device=DEV)
        _lib.call("sg_bn_stats", _p(a), SG_F16, B * L, C_, _p(stats), _stream())
        h = torch.zeros(B, L + 2 * halo, C_, dtype=torch.float16, device=DEV)
        _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(slope), 1, 0, _p(roll_dev), halo, _p(h), None, None,
                  _stream())
        red = torch.zeros(8, 3, C_, dtype=torch.float64, device=DEV)
        _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, roll, None, None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
                  _p(slope), 1, _p(red), None, _stream())
        ga = torch.zeros(B, L, C_, dtype=E.GT, device=DEV)
        _lib.call("sg_act_bwd_apply", _p(gh), C_, halo, 0, _p(roll_dev), None, 0, _p(a), SG_F16, B, L, C_, _p(ss), _p(mi),
                  _p(slope), 1, _p(red), 1, _p(ga), _stream())
        # Generator-encoder form: no BN, skip gradient joins after the activation derivative, g_pre written by pass 1
        red2 = torch.zeros(8, 3, C_, dtype=torch.float64, device=DEV)
        ga2 = torch.zeros(B, L, C_, dtype=E.GT, device=DEV)
        _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, 0, None, _p(gadd), C_, _p(a), SG_F16, B, L, C_, None, None,
                  _p(slope), 1, _p(red2), _p(ga2), _stream())
        torch.cuda.synchronize()
        outs[tag] = (stats.sum(0), h, red.sum(0), ga, red2.sum(0), ga2)
    r, t = outs["reg"], outs["tma"]
    assert rel_err(t[0], r[0]) <= 1e-6
    assert torch.equal(t[1], r[1])
    assert rel_err(t[2], r[2]) <= 1e-5
    assert rel_err(t[3].float(), r[3].float()) <= 2e-3          # pass 2 consumes each run's own (re-ordered) sums
    assert rel_err(t[4], r[4]) <= 1e-5
    assert torch.equal(t[5], r[5])


@pytest.mark.parametrize("cin,L,roll", [(2, 2048, 3), (1, 16384, 0), (2, 1280, -5)])
def test_wave_im2col_matches_unfold(cin, L, roll):
    """sg_wave_im2col (shared-memory staged tiles): col[b][t][ci * 32 + k] = pad(shift(v_ci))[4 t + k - 14], reflect
    padding (14, 15) of the stride-4 k = 31 conv (modules.py:91-98), columns 31 / 63 and absent channels zero."""
    g = _gen(41)
    B = 3
    x = [torch.randn(B, L, generator=g) for _ in range(cin)]
    col = torch.full((B, L // 4, 64), 7.0, dtype=torch.float16, device=DEV)
    xd = [t.to(DEV) for t in x]
    _lib.call("sg_wave_im2col", _p(xd[0]), _p(xd[1]) if cin == 2 else None, cin, B, L, roll, None, 1, 14, _p(col), None,
              _stream())
    rdev = torch.tensor([roll], dtype=torch.int32, device=DEV)
    col_d = torch.zeros_like(col)
    _lib.call("sg_wave_im2col", _p(xd[0]), _p(xd[1]) if cin == 2 else None, cin, B, L, 0, _p(rdev), 1, 14, _p(col_d), None,
              _stream())
    torch.cuda.synchronize()
    ref = torch.zeros(B, L // 4, 64)
    for ci in range(cin):
        xp = F.pad(O.phase_roll(x[ci].unsqueeze(1), roll), (14, 15), mode="reflect").squeeze(1)
        ref[:, :, ci * 32:ci * 32 + 31] = xp.unfold(1, 31, 4)
    assert torch.equal(col.float().cpu(), ref.to(torch.float16).float())
    assert torch.equal(col_d, col)
