"""The forward-form tap-GEMM (form F: tapgemm_tc.cu tapgemm_f_tc<TN, format>, tapgemm_ref.cu tapgemm_f_ffma) launched
through sg_tapgemm_f_run against an fp64 evaluation of
    out[b][m][n] = bias[n % bias_mod] + sum_d sum_kc A[b][m + d][kc] * W[d + 4 - w_tap0][n][kc]
(tests/tapgemm_model.py ref_f), optionally followed by PReLU (slope[n % slope_mod]) into `out` itself or into a
second output out2 with a reflect halo.

Every case places out (and out2) inside guard bands of 4096 elements; 16-bit buffers start as a sentinel bit pattern,
fp32 ones as random values with -0.0f in half of the dead elements.  Inside the launch's region
  16-bit:  c_f = (|out - ref| - half an ulp of ref) / (2^-24 * sum |a w| * (1 + stages / 32))  <=  16
  fp32:    c_w = |out - out0 - ref| / (2^-24 * (sum |a w| + |out0|) * (1 + stages / 32))     <=  16
(out0 = the initial value where the launch accumulates, ksplit > 1; 0 where it overwrites, ksplit = 1; `stages` =
the 64-channel k-steps one tensor-core accumulator walks, tapgemm_model.f_stages, 0 on the FFMA kernel); every other
element, guard bands included, keeps its initial bits.  out2 is compared with PReLU of the fp64 value where no
summation order can flip its sign.  Both back-ends run wherever the FFMA kernel serves the launch (no out2 / slope /
BatchNorm statistics) and agree within 2 * 16 (c_pair); 16-bit tensor-core results are bitwise repeatable; after every
tensor-core launch the stream-K counters (the first 8 KB of the stream's workspace) are zero again.  A operands
without a halo have +-64 as the first and last row of every batch element: a row read from the neighbouring packed
batch element instead of the zero fill moves the result by hundreds of products.

Which instantiation a case launches: TN = 256 / 128 / 64 from ncols = n_hi - n_lo (or the tile_n hint); M tile =
TB batch elements x TR rows, TR = min(rows_m, 128), TB = min(128 / TR, batch).  Every id runs as `<id>-f16` and,
where marked *, also as `<id>-bf16`:

  id                      TN   TR x TB    sources       taps / d              split / epilogue
  tn64_conv *             64   64 x 2     256           conv_fwd              bias nc
  tn128_deconv *          128  64 x 2     256           deconv_fwd, n 0..384  bias 128 (repeating)
  tn256_conv *            256  64 x 2     256           conv_fwd              bias nc
  tile_n64_hint *         64   64 x 2     256           conv_fwd, nc 256      tile_n = 64
  tile_n128_hint          128  64 x 2     256           conv_fwd, nc 256      tile_n = 128
  rows1_b70               256  1 x 70     256           full, d 0, tap0 4     (TB clamped to the batch)
  rows12_b23              256  12 x 10    128           conv_dgrad, m -4..8   (out_halo 4)
  rows16_b11 *            128  16 x 8     256           conv_fwd              bias nc
  rows24_b13              256  24 x 5     128           conv_dgrad            -
  rows40_b7               256  40 x 3     128           conv_dgrad            -
  rows64_b5               256  64 x 2     256           conv_fwd              bias nc
  rows72_b3 / rows104_b3  256  72, 104 x 1 128          conv_dgrad            (one partial M tile)
  rows128_b3              256  128 x 1    256           conv_fwd              bias nc
  rows264_b2 *            256  128 x 1    128           conv_dgrad            (partial third M tile)
  deconv_dgrad_tn64       64   64 x 2     256           deconv_dgrad, n 0..192
  full_tap0_4             128  64 x 2     192           full, d 0, tap0 4     bias nc
  skipconv_k11 *          256  64 x 2     256           skip conv k 11, d -2..2, tap0 2
  skipconv_k33            256  64 x 2     256           skip conv k 33, d -4..4
  dsub_conv_fwd ...       256  64 x 2     256 / 128     each table, d -2..3 / -4..-1 / 1..4 / -3..2
  no_live_tap_tile        64   64 x 2     256           full, n 0..64 only    bias nc: tiles 64..191 = bias
  src_128_128             256  64 x 2     128 + 128     deconv_fwd            bias 64
  src_64_192 / 192_64     128  64 x 2     64 + 192 ...  full                  -
  src_64_1024 *           256  16 x 8     64 + 1024     deconv_fwd, nc 2048   (--z_dim 64 decoder block 0)
  n_sub_range *           128  64 x 2     256           deconv_dgrad, n 64..192
  concat_dst              128  64 x 2     256           conv_fwd              out_ld 384, out_col0 192
  wave_half_lo / _hi      64   128 x 1    64            full, n 0..64 / 64..128  out_ld 64, out_col0 0
  bias_mod192 / 320       128  64 x 2     256           full, nc 384 / 640    bias_mod 192 / 320
  out2_h0 / h4 / h16 ...  all  ...        ...           conv_fwd, deconv_fwd  out2 + PReLU, slope_mod nc / 192 / 320
  prelu_in_place *        128  64 x 2     256           conv_fwd              PReLU into out
  f16_saturates           256  64 x 2     256           conv_fwd              |values| >> 65504
  f32_* ...               ...             ...           full / conv_fwd       ksplit 1 (overwrite), 2, 3, 7, 9
                                                                              (empty splits), fc.0 K 16384 / 16
Forced stream-K (sg_set_stream_k(16, 1e-6)): test_stream_k_vs_fp64 (conv / deconv / dgrad x TN x format, out2 +
concat + two sources), two streams, and a tile with fewer k-steps than the split (empty pieces).
Batch 300 under the default cost model: test_production_scale.  Argument errors: test_tapgemm_f_refuses.
Run on an H100:  python -m pytest tests/test_gpu_tapgemm_f.py -m gpu -s"""
import ctypes as C
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                                           # noqa: E402
from segan_pytorch_b200._lib import (SG_BF16, SG_F16, SG_F32, BACKEND_FFMA, BACKEND_TCGEN05,   # noqa: E402
                                     TapGemmF)
from tests import tapgemm_model as M                                                        # noqa: E402

DEV = "cuda"
GUARD = 4096                  # elements before and after out / out2
SENTINEL = 0x7E5A
FMT = {"f16": (SG_F16, torch.float16), "bf16": (SG_BF16, torch.bfloat16)}
BACKENDS = {"ffma": BACKEND_FFMA, "tc": BACKEND_TCGEN05}
EDGE = 64.0


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _kc(c):
    return c["a0_c"] + c.get("a1_c", 0)


def _taps(c):
    """(taps, d_lo, d_hi, w_tap0)"""
    kind, kc, nc = c["taps"], _kc(c), c["nc"]
    if kind == "skipconv":
        d_lo, d_hi, tap0, fwd, _ = E.skipconv_geometry(kc // 4, c["skip_k"])
        return fwd, d_lo, d_hi, tap0
    if kind == "custom":
        return [list(t) for t in c["table"]], c["d"][0], c["d"][1], c.get("tap0", 0)
    ch = {"conv_fwd": kc // 4, "deconv_dgrad": kc // 4, "conv_dgrad": nc // 4, "deconv_fwd": nc // 4, "full": 0}[kind]
    d = c.get("d", (-4, 4))
    return E.tap_ranges(kind, ch, kc, nc, c.get("k", 31)), d[0], d[1], c.get("tap0", 0)


def _geom(c):
    """Rows and columns of the launch: (rows, halo, out_halo, m_lo, m_hi, n_lo, n_hi, ld, col0)."""
    R = c["rows"]
    dgrad = c["taps"] == "conv_dgrad"
    out_halo = 4 if dgrad else 0
    m_lo, m_hi = (-4, R + 4) if dgrad else (0, R)
    n_lo, n_hi = c.get("n", (0, c["nc"]))
    ld = c.get("out_ld", 0)
    col0 = c.get("out_col0", 0) if ld > 0 else n_lo
    return R, c.get("halo", 0), out_halo, m_lo, m_hi, n_lo, n_hi, (ld if ld > 0 else c["nc"]), col0


def tc_tile_n(c):
    _, _, _, _, _, n_lo, n_hi, _, _ = _geom(c)
    ncols = n_hi - n_lo
    tn = 256 if ncols % 256 == 0 else (128 if ncols % 128 == 0 else 64)
    t = c.get("tile_n", 0)
    return t if t in (64, 128, 256) and ncols % t == 0 and t < tn else tn


def _operands(c, fmt, seed, batch=None):
    """A0 / A1 [B][R + 2 halo][.] ~ N(0,1) (+-EDGE first and last rows without a halo), W [slots][nc][kc] ~ w_std
    N(0,1), zero outside every tap's live box (the layout's structural zeros), bias / slope [mod]."""
    g = _gen(seed)
    tdt = FMT[fmt][1]
    B = c["batch"] if batch is None else batch
    R, halo = c["rows"], c.get("halo", 0)
    taps, d_lo, d_hi, tap0 = _taps(c)
    srcs = []
    for ch in (c["a0_c"], c.get("a1_c", 0)):
        if ch == 0:
            srcs.append(None)
            continue
        a = torch.randn(B, R + 2 * halo, ch, generator=g, device=DEV)
        if halo == 0 and not c.get("no_edge"):
            sign = torch.where(torch.rand(B, 2, ch, generator=g, device=DEV) < 0.5, -EDGE, EDGE)
            a[:, 0], a[:, -1] = sign[:, 0], sign[:, 1]
        srcs.append(a.to(tdt))
    slots = d_hi + 4 - tap0 + 1
    w = c.get("w_std", 0.05) * torch.randn(slots, c["nc"], _kc(c), generator=g, device=DEV)
    live = torch.zeros_like(w, dtype=torch.bool)
    for d in range(d_lo, d_hi + 1):
        i = d + 4
        live[i - tap0, taps[2][i]:taps[3][i], taps[0][i]:taps[1][i]] = True
    w = torch.where(live, w, torch.zeros_like(w)).to(tdt)
    bias = slope = None
    bmod = c.get("bias")
    if bmod is not None:
        bias = torch.randn(c["nc"] if bmod == "nc" else bmod, generator=g, device=DEV)
    smod = c.get("slope")
    if smod is not None:
        slope = 0.3 * torch.rand(c["nc"] if smod == "nc" else smod, generator=g, device=DEV)
    return srcs[0], srcs[1], w, bias, slope


class _Out(object):
    """A [B][rows][ld] destination inside guard bands; `live` marks what the launch may write."""

    def __init__(self, B, rows, ld, tdt, seed, live_fn):
        n = B * rows * ld
        live = torch.zeros(B, rows, ld, dtype=torch.bool, device=DEV)
        live_fn(live)
        self.live = torch.zeros(n + 2 * GUARD, dtype=torch.bool, device=DEV)
        self.live[GUARD:GUARD + n] = live.reshape(-1)
        if tdt == torch.float32:
            self.buf = torch.randn(n + 2 * GUARD, generator=_gen(seed), device=DEV)
            neg = ~self.live
            neg[1::2] = False
            self.buf[neg] = -0.0
            self.bits = lambda t: t.view(torch.int32)
        else:
            self.buf = torch.empty(n + 2 * GUARD, dtype=tdt, device=DEV)
            self.buf.view(torch.int16).fill_(SENTINEL)
            self.bits = lambda t: t.view(torch.int16)
        self.buf0 = self.buf.clone()
        self.t = self.buf[GUARD:GUARD + n].view(B, rows, ld)
        self.t0 = self.buf0[GUARD:GUARD + n].view(B, rows, ld)

    def untouched_outside(self):
        dead = ~self.live
        return torch.equal(self.bits(self.buf)[dead], self.bits(self.buf0)[dead])

    def unchanged(self):
        return torch.equal(self.bits(self.buf), self.bits(self.buf0))


def _mirror(m, out_rows, h):
    if 1 <= m <= h:
        return -m
    if out_rows - 1 - h <= m <= out_rows - 2:
        return 2 * (out_rows - 1) - m
    return None


def _make_q(c, fmt, backend, a0, a1, w, bias, slope, out, out2, ksplit, batch=None, sk_ws=None):
    taps, d_lo, d_hi, tap0 = _taps(c)
    R, halo, out_halo, m_lo, m_hi, n_lo, n_hi, ld, col0 = _geom(c)
    sdt = FMT[fmt][0]
    q = TapGemmF()
    q.a0, q.a1 = C.c_void_p(a0.data_ptr()), (None if a1 is None else C.c_void_p(a1.data_ptr()))
    q.a0_c, q.a1_c = c["a0_c"], c.get("a1_c", 0)
    q.a_rows, q.a_halo, q.a_dtype = R, halo, sdt
    q.w, q.w_dtype, q.w_tap0 = C.c_void_p(w.data_ptr()), sdt, tap0
    q.kc, q.nc, q.d_lo, q.d_hi = _kc(c), c["nc"], d_lo, d_hi
    for i in range(9):
        q.tap_k_lo[i], q.tap_k_hi[i], q.tap_n_lo[i], q.tap_n_hi[i] = taps[0][i], taps[1][i], taps[2][i], taps[3][i]
    q.out = C.c_void_p(out.data_ptr())
    q.out_ld, q.out_col0 = c.get("out_ld", 0), c.get("out_col0", 0)
    q.out_dtype = SG_F32 if c.get("f32") else sdt
    q.out_rows, q.out_halo = R, out_halo
    q.m_lo, q.m_hi, q.n_lo, q.n_hi = m_lo, m_hi, n_lo, n_hi
    q.bias = None if bias is None else C.c_void_p(bias.data_ptr())
    q.bias_mod = 0 if bias is None else bias.numel()
    q.batch = c["batch"] if batch is None else batch
    q.ksplit = ksplit
    q.backend, q.tile_n = backend, c.get("tile_n", 0)
    q.bn_stats = None
    q.out2 = None if out2 is None else C.c_void_p(out2.data_ptr())
    q.out2_halo = c.get("out2", 0) if out2 is not None else 0
    q.slope = None if slope is None else C.c_void_p(slope.data_ptr())
    q.slope_mod = 0 if slope is None else slope.numel()
    ws = (E.sk_workspace(DEV) if sk_ws is None else sk_ws) if backend == BACKEND_TCGEN05 else None
    q.sk_ws = None if ws is None else C.c_void_p(ws.data_ptr())
    return q


def _launch(q):
    _lib.call("sg_tapgemm_f_run", C.byref(q), E._stream())


def _ref(c, a0, a1, w, bias):
    taps, d_lo, d_hi, tap0 = _taps(c)
    R, halo, _, m_lo, m_hi, n_lo, n_hi, _, _ = _geom(c)
    return M.ref_f(a0, a1, halo, w, taps, m_lo, m_hi, d_lo, d_hi, tap0, bias)


def _stages(c, backend, ksplit=1):
    """Per column of [n_lo, n_hi): the k-steps the tensor-core accumulator of that column's tiles walks (0 on FFMA).
    A stream-K split shortens only the leftover tiles; the tiles above them in the same columns walk all steps."""
    _, _, _, _, _, n_lo, n_hi, _, _ = _geom(c)
    st = torch.zeros(n_hi - n_lo, dtype=torch.float64, device=DEV)
    if backend != "tc":
        return st
    taps, d_lo, d_hi, _ = _taps(c)
    tn = tc_tile_n(c)
    for n0 in range(n_lo, n_hi, tn):
        st[n0 - n_lo:n0 - n_lo + tn] = M.f_stages(taps, d_lo, d_hi, n0, n0 + tn, ksplit)
    return st


def _counters_zero(ws=None):
    ws = E.sk_workspace(DEV) if ws is None else ws
    return ws is None or int(ws[:8192].count_nonzero()) == 0


def _outputs(c, fmt, seed, B=None):
    R, halo, out_halo, m_lo, m_hi, n_lo, n_hi, ld, col0 = _geom(c)
    B = c["batch"] if B is None else B
    f32 = c.get("f32")
    tdt = torch.float32 if f32 else FMT[fmt][1]
    ncols = n_hi - n_lo

    def live_out(lv):
        lv[:, out_halo + m_lo:out_halo + m_hi, col0:col0 + ncols] = True
    out = _Out(B, R + 2 * out_halo, ld, tdt, seed, live_out)
    out2 = None
    if "out2" in c:
        h = c["out2"]

        def live_out2(lv):
            lv[:, h + m_lo:h + m_hi, col0:col0 + ncols] = True
            for m in range(m_lo, m_hi):
                mm = _mirror(m, R, h) if h > 0 else None
                if mm is not None:
                    lv[:, h + mm, col0:col0 + ncols] = True
        out2 = _Out(B, R + 2 * h, ld, tdt, seed + 1, live_out2)
    return out, out2


def _check(label, c, fmt, bk, out, out2, ref, mag, slope, stages, ksplit):
    """Gate the region(s), the bits outside them; returns (values, den) for the back-end comparison."""
    R, halo, out_halo, m_lo, m_hi, n_lo, n_hi, ld, col0 = _geom(c)
    ncols = n_hi - n_lo
    ref, mag = ref[..., n_lo:n_hi], mag[..., n_lo:n_hi]
    assert out.untouched_outside(), (label, "out written outside the launch's region")
    region = out.t[:, out_halo + m_lo:out_halo + m_hi, col0:col0 + ncols]
    if c.get("f32"):
        d0 = out.t0[:, out_halo + m_lo:out_halo + m_hi, col0:col0 + ncols].double()
        if ksplit == 1:
            d0 = torch.zeros_like(d0)                        # ksplit 1 overwrites
        got, den = region.double() - d0, mag + d0.abs()
        cc = M.c_w(got, ref, den, trunc_stages=stages)
        print("tapgemm_f %s %s: c = %.2f (tol %g)" % (label, bk, cc, M.C_TOL))
        assert cc <= M.C_TOL, (label, bk, cc)
        return got, den
    if slope is not None and "out2" not in c:                # PReLU in place
        act, mag_act = M.prelu_ref(ref, mag, slope[torch.arange(n_lo, n_hi, device=DEV) % slope.numel()])
        safe = M.sign_safe(ref, mag)
        assert float(safe.double().mean()) > 0.99
        cc = M.c_f(region[safe], act[safe], mag_act[safe], fmt, stages.expand_as(ref)[safe])
        print("tapgemm_f %s %s (in place): c = %.2f (tol %g)" % (label, bk, cc, M.C_TOL))
        assert cc <= M.C_TOL, (label, bk, cc)
        return region, mag_act
    cc = M.c_f(region, ref, mag, fmt, stages)
    print("tapgemm_f %s %s: c = %.2f (tol %g)" % (label, bk, cc, M.C_TOL))
    assert cc <= M.C_TOL, (label, bk, cc)
    if out2 is not None:
        h = c["out2"]
        assert out2.untouched_outside(), (label, "out2 written outside its rows and columns")
        sl = slope[torch.arange(n_lo, n_hi, device=DEV) % slope.numel()]
        act, mag_act = M.prelu_ref(ref, mag, sl)
        safe = M.sign_safe(ref, mag)
        inner = out2.t[:, h + m_lo:h + m_hi, col0:col0 + ncols]
        c2 = M.c_f(inner[safe], act[safe], mag_act[safe], fmt, stages.expand_as(ref)[safe])
        print("tapgemm_f %s %s out2: c = %.2f" % (label, bk, c2))
        assert c2 <= M.C_TOL, (label, bk, "out2", c2)
        b2 = out2.bits(out2.t)
        for m in range(m_lo, m_hi):                        # reflect-halo rows: bit copies
            mm = _mirror(m, R, h) if h > 0 else None
            if mm is not None:
                assert torch.equal(b2[:, h + mm, col0:col0 + ncols], b2[:, h + m, col0:col0 + ncols]), (label, m)
    return region, mag


def _run_case(name, c, fmt, seed):
    taps, d_lo, d_hi, tap0 = _taps(c)
    a0, a1, w, bias, slope = _operands(c, fmt, seed)
    ref, mag = _ref(c, a0, a1, w, bias)
    ksplit = c.get("ksplit", 1)
    ffma_ok = slope is None and "out2" not in c
    res = {}
    for bk in (("ffma", "tc") if ffma_ok else ("tc",)):
        out, out2 = _outputs(c, fmt, seed + 1)
        q = _make_q(c, fmt, BACKENDS[bk], a0, a1, w, bias, slope, out.t, None if out2 is None else out2.t, ksplit)
        _launch(q)
        torch.cuda.synchronize()
        if bk == "tc":
            assert _counters_zero(), (name, "stream-K counters left non-zero")
        st = _stages(c, bk, ksplit)
        res[bk] = _check("%s-%s" % (name, fmt), c, fmt, bk, out, out2, ref, mag, slope, st, ksplit)
        if bk == "tc" and not c.get("f32"):                 # bitwise repeatable
            again, again2 = _outputs(c, fmt, seed + 1)
            _launch(_make_q(c, fmt, BACKEND_TCGEN05, a0, a1, w, bias, slope, again.t,
                            None if again2 is None else again2.t, ksplit))
            torch.cuda.synchronize()
            assert torch.equal(out.bits(out.buf), again.bits(again.buf)), (name, fmt, "not repeatable")
            if out2 is not None:
                assert torch.equal(out2.bits(out2.buf), again2.bits(again2.buf)), (name, fmt, "out2 not repeatable")
    if len(res) == 2:
        st = _stages(c, "tc", ksplit)
        den = torch.maximum(res["tc"][1], res["ffma"][1])
        cb = M.c_pair(res["tc"][0], res["ffma"][0], den, None if c.get("f32") else fmt, st)
        print("tapgemm_f %s-%s back-ends: c = %.2f (tol %g)" % (name, fmt, cb, 2 * M.C_TOL))
        assert cb <= 2 * M.C_TOL, (name, fmt, "back-ends disagree", cb)


_CONV = dict(a0_c=256, taps="conv_fwd", halo=4)
_DG = dict(a0_c=128, nc=256, taps="conv_dgrad")
CASES = {
    # instantiations: TN x format
    "tn64_conv": dict(_CONV, nc=192, rows=64, batch=5, bias="nc", bf16=True),
    "tn128_deconv": dict(a0_c=256, nc=512, n=(0, 384), taps="deconv_fwd", rows=64, batch=5, bias=128, bf16=True),
    "tn256_conv": dict(_CONV, nc=256, rows=64, batch=5, bias="nc", bf16=True),
    "tile_n64_hint": dict(_CONV, nc=256, rows=64, batch=5, bias="nc", tile_n=64, bf16=True),
    "tile_n128_hint": dict(_CONV, nc=256, rows=64, batch=5, bias="nc", tile_n=128),
    # row packing (rows_m = m_hi - m_lo; conv_dgrad computes rows -4 .. R + 4 into out_halo = 4)
    "rows1_b70": dict(a0_c=256, nc=256, taps="full", d=(0, 0), tap0=4, rows=1, batch=70, bias="nc"),
    "rows12_b23": dict(_DG, rows=4, batch=23),
    "rows16_b11": dict(_CONV, nc=128, rows=16, batch=11, bias="nc", bf16=True),
    "rows24_b13": dict(_DG, rows=16, batch=13),
    "rows40_b7": dict(_DG, rows=32, batch=7),
    "rows64_b5": dict(_CONV, nc=256, rows=64, batch=5, bias="nc"),
    "rows72_b3": dict(_DG, rows=64, batch=3),
    "rows104_b3": dict(_DG, rows=96, batch=3),
    "rows128_b3": dict(_CONV, nc=256, rows=128, batch=3, bias="nc"),
    "rows264_b2": dict(_DG, rows=256, batch=2, bf16=True),
    # tap tables
    "deconv_dgrad_tn64": dict(a0_c=256, nc=256, n=(0, 192), taps="deconv_dgrad", rows=64, batch=5),
    "full_tap0_4": dict(a0_c=192, nc=128, taps="full", d=(0, 0), tap0=4, rows=64, batch=5, bias="nc"),
    "skipconv_k11": dict(a0_c=256, nc=256, taps="skipconv", skip_k=11, rows=64, batch=5, bias=64, bf16=True),
    "skipconv_k33": dict(a0_c=256, nc=256, taps="skipconv", skip_k=33, rows=64, batch=5),
    "dsub_conv_fwd": dict(_CONV, nc=256, d=(-2, 3), rows=64, batch=5, bias="nc"),
    "dsub_conv_dgrad": dict(_DG, d=(-4, -1), rows=64, batch=3),
    "dsub_deconv_fwd": dict(a0_c=128, nc=256, taps="deconv_fwd", d=(1, 4), rows=64, batch=5),
    "dsub_deconv_dgrad": dict(a0_c=256, nc=128, taps="deconv_dgrad", d=(-3, 2), rows=64, batch=5),
    "no_live_tap_tile": dict(a0_c=256, nc=192, taps="custom", d=(-1, 1), rows=64, batch=5, bias="nc",
                             table=([0] * 9, [256] * 9, [0] * 9, [64] * 9)),
    # sources
    "src_128_128": dict(a0_c=128, a1_c=128, nc=256, taps="deconv_fwd", rows=64, batch=5, bias=64),
    "src_64_192": dict(a0_c=64, a1_c=192, nc=128, taps="full", rows=64, batch=5),
    "src_192_64": dict(a0_c=192, a1_c=64, nc=128, taps="full", rows=64, batch=5),
    "src_64_1024": dict(a0_c=64, a1_c=1024, nc=2048, taps="deconv_fwd", rows=16, batch=9, bias=512, bf16=True),
    # columns
    "n_sub_range": dict(a0_c=256, nc=256, n=(64, 192), taps="deconv_dgrad", rows=64, batch=5, bf16=True),
    "concat_dst": dict(_CONV, nc=128, rows=64, batch=5, bias="nc", out_ld=384, out_col0=192),
    "wave_half_lo": dict(a0_c=64, nc=128, n=(0, 64), taps="full", d=(0, 0), tap0=4, rows=512, batch=3, out_ld=64,
                         out_col0=0),
    "wave_half_hi": dict(a0_c=64, nc=128, n=(64, 128), taps="full", d=(0, 0), tap0=4, rows=512, batch=3, out_ld=64,
                         out_col0=0),
    # bias moduli that are not powers of two
    "bias_mod192": dict(a0_c=256, nc=384, taps="full", d=(-1, 1), rows=64, batch=5, bias=192),
    "bias_mod320": dict(a0_c=256, nc=640, taps="full", d=(-1, 1), rows=64, batch=5, bias=320),
    # fused epilogue
    "out2_h0_tn64": dict(_CONV, nc=192, rows=64, batch=5, bias="nc", slope="nc", out2=0, bf16=True),
    "out2_h4_rows16": dict(_CONV, nc=128, rows=16, batch=11, bias="nc", slope="nc", out2=4),
    "out2_h16_tn64": dict(a0_c=64, nc=64, taps="full", d=(0, 0), tap0=4, rows=256, batch=3, bias=64, slope=64, out2=16,
                          bf16=True),
    "out2_h16_tn256": dict(_CONV, nc=256, rows=160, batch=3, bias="nc", slope="nc", out2=16, bf16=True),
    "out2_deconv_slope192": dict(a0_c=128, nc=768, taps="full", d=(-1, 1), rows=64, batch=3, bias=192, slope=192,
                                 out2=0),
    "out2_slope320": dict(a0_c=128, nc=640, taps="full", d=(-1, 1), rows=64, batch=3, bias=320, slope=320, out2=4),
    "prelu_in_place": dict(_CONV, nc=128, rows=160, batch=3, bias="nc", slope="nc", bf16=True),
    "f16_saturates": dict(_CONV, nc=256, rows=64, batch=3, bias="nc", w_std=3000.0),
    # fp32 outputs: ksplit 1 overwrites, ksplit > 1 accumulates (full, kc 256: 4 k-steps per tile)
    "f32_ksplit1": dict(_CONV, nc=128, rows=64, batch=3, bias="nc", f32=True),
    "f32_ksplit2": dict(a0_c=256, nc=128, taps="full", d=(0, 0), tap0=4, rows=64, batch=3, bias="nc", f32=True,
                        ksplit=2),
    "f32_ksplit3": dict(a0_c=256, nc=128, taps="full", d=(-1, 0), rows=64, batch=3, f32=True, ksplit=3),
    "f32_ksplit7": dict(_CONV, nc=128, rows=64, batch=3, bias="nc", f32=True, ksplit=7),
    "f32_ksplit9_empty": dict(a0_c=256, nc=128, taps="full", d=(0, 0), tap0=4, rows=64, batch=3, bias="nc",
                              f32=True, ksplit=9),
    "f32_fc0_k16": dict(a0_c=16384, nc=256, taps="full", d=(0, 0), tap0=4, rows=1, batch=7, bias="nc", f32=True,
                        ksplit=16),
}
PARAMS = [(n, f) for n, c in CASES.items() for f in (("f16", "bf16") if c.get("bf16") else ("f16",))]


@pytest.mark.parametrize("name,fmt", PARAMS, ids=["%s-%s" % p for p in PARAMS])
def test_tapgemm_f_vs_fp64(name, fmt):
    _run_case(name, CASES[name], fmt, 5000 + 11 * list(CASES).index(name))


def test_every_tensor_core_instantiation_is_launched():
    launched = {(tc_tile_n(CASES[n]), f) for n, f in PARAMS}
    assert launched == {(tn, f) for tn in (64, 128, 256) for f in ("f16", "bf16")}


def test_ffma_and_tensor_cores_overwrite_an_fp32_destination():
    """ksplit = 1 into an fp32 destination twice: the second launch leaves what the first one did (the engine's
    Generator output P and SpectralLoss buffers are reused without zeroing)."""
    c = CASES["f32_ksplit1"]
    a0, a1, w, bias, _ = _operands(c, "f16", 5900)
    for bk in ("ffma", "tc"):
        out, _ = _outputs(c, "f16", 5901)
        for _ in range(2):
            _launch(_make_q(c, "f16", BACKENDS[bk], a0, a1, w, bias, None, out.t, None, 1))
        torch.cuda.synchronize()
        once, _ = _outputs(c, "f16", 5902)
        _launch(_make_q(c, "f16", BACKENDS[bk], a0, a1, w, bias, None, once.t, None, 1))
        torch.cuda.synchronize()
        region = once.live[GUARD:GUARD + once.t.numel()].view_as(once.t)
        assert torch.equal(out.t[region], once.t[region]), (bk, "a second launch accumulated")


def test_generator_forward_twice_under_ffma_is_repeatable():
    """Two identical Generator forwards with the FFMA back-end give the same waveform."""
    from tests.util import build_segan
    s = build_segan().to(DEV)
    s.G.eval()
    s.G.engine.backend = BACKEND_FFMA
    g = _gen(5903)
    x = (0.3 * torch.randn(1, 1, 16384, generator=g, device=DEV)).clamp(-1, 1)
    z = torch.randn(1, 1024, 16, generator=g, device=DEV)
    with torch.no_grad():
        y1 = s.G(x, z=z).clone()
        y2 = s.G(x, z=z).clone()
    torch.cuda.synchronize()
    assert torch.equal(y1, y2), float((y1 - y2).abs().max())


# ---------------------------------------------------------------------------------------------------------------
# stream-K: the leftover tiles of the last wave split along K (forced), finished by the warp that counts last
# ---------------------------------------------------------------------------------------------------------------
class _ForcedStreamK(object):
    def __enter__(self):
        self.lib = _lib.load()
        self.prev = E.STREAM_K
        E.STREAM_K = True
        self.lib.sg_set_stream_k(16, 1e-6)
        return self

    def __exit__(self, *a):
        E.STREAM_K = self.prev
        self.lib.sg_set_stream_k(16, 4.5)                     # the default cost model
        return False


def _sk_case(kind, tn):
    """Shapes with more tiles than SMs and a ragged last wave (M tiles of 128 rows, TB 1)."""
    if kind == "conv":
        c = dict(_CONV, nc={64: 192, 128: 384, 256: 256}[tn], rows=128, bias="nc")
    elif kind == "deconv":
        c = dict(a0_c=128, taps="deconv_fwd", nc={64: 256, 128: 512, 256: 256}[tn], rows=128, bias=64,
                 n={64: (0, 192), 128: (0, 384), 256: (0, 256)}[tn])
    else:
        c = dict(a0_c=128, taps="conv_dgrad", nc={64: 256, 128: 512, 256: 256}[tn], rows=120,
                 n={64: (64, 256), 128: (128, 512), 256: (0, 256)}[tn])
    n_tiles = (c.get("n", (0, c["nc"]))[1] - c.get("n", (0, c["nc"]))[0]) // tn
    b = -(-140 // n_tiles)
    while (b * n_tiles) % E.NUM_SMS == 0:
        b += 1
    c["batch"] = b
    return c


SK_PARAMS = [(k, tn, f) for k in ("conv", "deconv", "dgrad") for tn in (64, 128, 256) for f in ("f16", "bf16")]
SK_EXTRA = {
    # out2 with a reflect halo of 16, a concat destination and two sources
    "out2_concat_two_src": dict(a0_c=128, a1_c=128, nc=256, taps="deconv_fwd", rows=128, batch=135, bias=64,
                                slope=64, out2=16, out_ld=512, out_col0=128),
}


def _run_sk(label, c, fmt, seed):
    a0, a1, w, bias, slope = _operands(c, fmt, seed)
    ref, mag = _ref(c, a0, a1, w, bias)
    ws = E.sk_workspace(DEV)
    ws[8192:].fill_(0xFF)                      # NaN in every partial slot: a piece overwrites its own before use
    out, out2 = _outputs(c, fmt, seed + 1)
    with _ForcedStreamK():
        _launch(_make_q(c, fmt, BACKEND_TCGEN05, a0, a1, w, bias, slope, out.t, None if out2 is None else out2.t, 1))
        torch.cuda.synchronize()
    split, zero = bool((ws[8192:] != 0xFF).any()), _counters_zero()
    ws[8192:].zero_()
    print("tapgemm_f %s: split-K ran %s, counters zero afterwards %s" % (label, split, zero))
    _check(label, c, fmt, "tc stream-K", out, out2, ref, mag, slope, _stages(c, "tc"), 1)
    assert split, (label, "the split-K path did not run")
    assert zero, (label, "stream-K counters left non-zero")


@pytest.mark.parametrize("kind,tn,fmt", SK_PARAMS, ids=["%s-tn%d-%s" % p for p in SK_PARAMS])
def test_stream_k_vs_fp64(kind, tn, fmt):
    c = _sk_case(kind, tn)
    assert tc_tile_n(c) == tn
    _run_sk("stream_k %s tn%d-%s" % (kind, tn, fmt), c, fmt, 6000 + SK_PARAMS.index((kind, tn, fmt)))


@pytest.mark.parametrize("name", list(SK_EXTRA))
def test_stream_k_fused_epilogue_vs_fp64(name):
    _run_sk("stream_k %s" % name, SK_EXTRA[name], "f16", 6100)


def test_stream_k_on_two_streams():
    """Two forced-split launches enqueued on two side streams at once, each with its own workspace."""
    c = _sk_case("conv", 128)
    sides = [torch.cuda.Stream(), torch.cuda.Stream()]
    probs = [_operands(c, "f16", 6200 + i) for i in range(2)]
    outs = [_outputs(c, "f16", 6210 + i)[0] for i in range(2)]
    wss = []
    for side in sides:
        with E.on_side(side):
            wss.append(E.sk_workspace(DEV))
    torch.cuda.synchronize()
    with _ForcedStreamK():
        for side, (a0, a1, w, bias, _), out, ws in zip(sides, probs, outs, wss):
            with E.on_side(side):
                _launch(_make_q(c, "f16", BACKEND_TCGEN05, a0, a1, w, bias, None, out.t, None, 1, sk_ws=ws))
        for side in sides:
            E.join_side(side)
        torch.cuda.synchronize()
    for i, ((a0, a1, w, bias, _), out, ws) in enumerate(zip(probs, outs, wss)):
        assert _counters_zero(ws), (i, "stream-K counters left non-zero")
        ref, mag = _ref(c, a0, a1, w, bias)
        _check("stream_k two streams %d" % i, c, "f16", "tc", out, None, ref, mag, None, _stages(c, "tc"), 1)


FEWER_STEPS = {
    # conv_dgrad, taps -4 only (N 0..128): 67 x 2 = 134 tiles on 132 CTAs, the two leftover tiles are the second N
    # tile, which no tap reaches (0 k-steps), split 2 ways: every piece is empty, the finisher writes the bias
    "zero_steps": dict(a0_c=256, nc=512, taps="conv_dgrad", d=(-4, -4), rows=120, batch=67, bias="nc"),
    # tap -4: N 0..256, 4 k-steps; tap -3: N 0..512, 2 k-steps.  The leftover second N tile has 2 k-steps, split 3
    # ways: one piece is empty and must still count, or the tile is never finished and its counter stays at 2
    "two_steps_three_pieces": dict(a0_c=256, nc=512, taps="custom", d=(-4, -3), rows=128, batch=67, bias="nc",
                                   table=([0] * 9, [256, 128] + [256] * 7, [0] * 9, [256, 512] + [512] * 7)),
}


@pytest.mark.parametrize("name", list(FEWER_STEPS))
def test_stream_k_tile_with_fewer_steps_than_the_split(name):
    ws = E.sk_workspace(DEV)
    try:
        _run_sk("stream_k %s" % name, FEWER_STEPS[name], "f16", 6300)
    finally:
        ws[:8192].zero_()                      # whatever happened, later launches on this stream start from zero


# ---------------------------------------------------------------------------------------------------------------
# batch 300, tensor cores, default cost model
# ---------------------------------------------------------------------------------------------------------------
def _conv(cin, cout, R, out2=None, fmt="f16"):
    c = dict(a0_c=4 * cin, nc=cout, taps="conv_fwd", rows=R, halo=4, batch=300, bias="nc", no_edge=True)
    if out2 is not None:
        c.update(slope="nc", out2=out2)
    return c


def _deconv(cin, cout, R, mode=None):
    c = dict(a0_c=cin // 2, a1_c=cin // 2, nc=4 * cout, taps="deconv_fwd", rows=R, batch=300, bias=cout, no_edge=True)
    if mode == "out2":
        c.update(slope=cout, out2=0)
    elif mode == "inplace":
        c.update(slope=cout)
    return c


def _dgrad(cin, cout, R):
    return dict(a0_c=cout, nc=4 * cin, taps="conv_dgrad", rows=R, batch=300, no_edge=True)


_WAVE = dict(a0_c=64, nc=64, taps="full", d=(0, 0), tap0=4, rows=4096, batch=300, bias=64, no_edge=True)
PRODUCTION = {
    # tools/dump_tapgemm_f.py SHAPES
    "genc0_out2_h16": (dict(_WAVE, slope=64, out2=16), "f16"),
    "denc0": (dict(_WAVE), "f16"),
    "genc1_out2_h16": (_conv(64, 128, 1024, 16), "f16"),
    "enc1": (_conv(64, 128, 1024), "f16"),
    "enc2": (_conv(128, 256, 256), "f16"),
    "genc3_out2_h16": (_conv(256, 512, 64, 16), "f16"),
    "enc4": (_conv(512, 1024, 16), "f16"),
    "gdec0_out2": (_deconv(2048, 512, 16, "out2"), "f16"),
    "gdec1_out2": (_deconv(1024, 256, 64, "out2"), "f16"),
    "gdec2_inplace": (_deconv(512, 128, 256, "inplace"), "f16"),
    "dec3": (_deconv(256, 64, 1024), "f16"),
    "dgrad1": (_dgrad(64, 128, 1024), "f16"),
    "dgrad3_bf16": (_dgrad(256, 512, 64), "bf16"),
    "dgrad4": (_dgrad(512, 1024, 16), "f16"),
    "wave_dgrad": (dict(a0_c=64, nc=128, n=(64, 128), taps="full", d=(0, 0), tap0=4, rows=4096, batch=300, out_ld=64,
                        out_col0=0, no_edge=True), "f16"),
    # D's fc.0 (interleaved k-split into a zeroed fp32 accumulator), a skip conv, WSEGAN's spectral loss GEMMs
    "fc0": (dict(a0_c=16384, nc=256, taps="full", d=(0, 0), tap0=4, rows=1, batch=300, f32=True, ksplit=16,
                 no_edge=True), "f16"),
    "skipconv_k11": (dict(a0_c=256, nc=256, taps="skipconv", skip_k=11, rows=1024, batch=300, bias=64, no_edge=True),
                     "f16"),
    "spectral_fwd": (dict(a0_c=960, nc=2176, taps="full", d=(0, 0), tap0=4, rows=2 * 300 * 103, batch=1, f32=True,
                          no_edge=True, w_std=0.02), "f16"),
    "spectral_bwd": (dict(a0_c=2176, nc=320, taps="full", d=(0, 0), tap0=4, rows=300 * 103, batch=1, f32=True,
                          no_edge=True, w_std=0.02), "bf16"),
}


def test_production_covers_the_dump_tool():
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "dump_tapgemm_f.py")
    spec = importlib.util.spec_from_file_location("dump_tapgemm_f", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert {n for n, _ in mod.SHAPES} <= set(PRODUCTION)


def _ref_chunked(c, a0, a1, w, bias, region, stages, fmt, budget=1 << 25):
    """max c over the region, the fp64 reference evaluated a few batch elements (or rows) at a time."""
    taps, d_lo, d_hi, tap0 = _taps(c)
    R, halo, out_halo, m_lo, m_hi, n_lo, n_hi, ld, col0 = _geom(c)
    width = max(_kc(c), c["nc"])
    B = a0.shape[0]
    per_b = (m_hi - m_lo) * width
    worst = [0.0, 0.0]
    bstep = max(1, budget // per_b)
    mstep = (m_hi - m_lo) if bstep > 1 or per_b <= budget else max(128, budget // width)
    for b0 in range(0, B, bstep):
        b1 = min(B, b0 + bstep)
        for r0 in range(m_lo, m_hi, mstep):
            r1 = min(m_hi, r0 + mstep)
            x1 = None if a1 is None else a1[b0:b1]
            ref, mag = M.ref_f(a0[b0:b1], x1, halo, w, taps, r0, r1, d_lo, d_hi, tap0, bias)
            ref, mag = ref[..., n_lo:n_hi], mag[..., n_lo:n_hi]
            got = region[b0:b1, r0 - m_lo:r1 - m_lo]
            for i, s in enumerate((stages, 0)):
                if c.get("f32"):
                    cc = M.c_w(got, ref, mag, trunc_stages=s)
                else:
                    cc = M.c_f(got, ref, mag, fmt, s)
                worst[i] = max(worst[i], cc)
            del ref, mag
    return worst


@pytest.mark.parametrize("name", list(PRODUCTION))
def test_production_scale(name):
    """The step's launch at batch 300 under the default stream-K cost model.  Prints c with and without the
    per-stage truncation allowance and whether the launch split its last wave."""
    c, fmt = PRODUCTION[name]
    R, halo, out_halo, m_lo, m_hi, n_lo, n_hi, ld, col0 = _geom(c)
    a0, a1, w, bias, slope = _operands(c, fmt, 7000 + list(PRODUCTION).index(name))
    out, out2 = _outputs(c, fmt, 7100)
    if c.get("f32"):
        out.t.zero_()                                       # the engine's fc.0 accumulator is zeroed first
        out.buf0.copy_(out.buf)
    ws = E.sk_workspace(DEV)
    ws[8192:].zero_()
    _lib.load().sg_set_stream_k(16, 4.5)
    _launch(_make_q(c, fmt, BACKEND_TCGEN05, a0, a1, w, bias, slope, out.t, None if out2 is None else out2.t,
                    c.get("ksplit", 1)))
    torch.cuda.synchronize()
    split = int(ws[8192:].count_nonzero()) > 0
    assert _counters_zero(), (name, "stream-K counters left non-zero")
    assert out.untouched_outside(), (name, "out written outside the launch's region")
    ncols = n_hi - n_lo
    region = out.t[:, out_halo + m_lo:out_halo + m_hi, col0:col0 + ncols]
    stages = _stages(c, "tc", c.get("ksplit", 1))
    worst = [0.0, 0.0]
    if slope is None or out2 is not None:
        worst = _ref_chunked(c, a0, a1, w, bias, region, stages, fmt)
    else:
        # PReLU in place: against PReLU of the fp64 value where its sign is certain
        taps, d_lo, d_hi, tap0 = _taps(c)
        for b0 in range(0, 300, 25):
            ref, mag = M.ref_f(a0[b0:b0 + 25], a1[b0:b0 + 25], halo, w, taps, m_lo, m_hi, d_lo, d_hi, tap0, bias)
            act, mag_act = M.prelu_ref(ref, mag, slope)
            safe = M.sign_safe(ref, mag)
            got = out.t[b0:b0 + 25, out_halo + m_lo:out_halo + m_hi, col0:col0 + ncols]
            st = stages.expand_as(ref)[safe]
            worst[0] = max(worst[0], M.c_f(got[safe], act[safe], mag_act[safe], fmt, st))
            worst[1] = max(worst[1], M.c_f(got[safe], act[safe], mag_act[safe], fmt))
    if out2 is not None:
        assert out2.untouched_outside(), (name, "out2 written outside its rows and columns")
        h = c["out2"]
        taps, d_lo, d_hi, tap0 = _taps(c)
        bstep = 25
        for b0 in range(0, 300, bstep):
            x1 = None if a1 is None else a1[b0:b0 + bstep]
            ref, mag = M.ref_f(a0[b0:b0 + bstep], x1, halo, w, taps, m_lo, m_hi, d_lo, d_hi, tap0, bias)
            act, mag_act = M.prelu_ref(ref, mag, slope)
            safe = M.sign_safe(ref, mag)
            got = out2.t[b0:b0 + bstep, h + m_lo:h + m_hi, col0:col0 + ncols]
            worst[0] = max(worst[0], M.c_f(got[safe], act[safe], mag_act[safe], fmt, stages.expand_as(ref)[safe]))
            del ref, mag, act, mag_act
    print("tapgemm_f production %s (%s, TN %d, k-steps <= %d, stream-K %s): c = %.2f, without the stage allowance "
          "%.2f (tol %g)" % (name, fmt, tc_tile_n(c), int(stages.max()), "split" if split else "whole", worst[0],
                             worst[1], M.C_TOL))
    assert worst[0] <= M.C_TOL, (name, worst)


# ---------------------------------------------------------------------------------------------------------------
# argument errors: refused on the host, nothing launched, the destination keeps its bits
# ---------------------------------------------------------------------------------------------------------------
_RC = dict(a0_c=128, nc=128, taps="full", d=(-1, 1), rows=64, batch=2, bias="nc")


def _set_tap(i, k_lo=None, k_hi=None, n_lo=None, n_hi=None):
    def f(q):
        for arr, v in ((q.tap_k_lo, k_lo), (q.tap_k_hi, k_hi), (q.tap_n_lo, n_lo), (q.tap_n_hi, n_hi)):
            if v is not None:
                arr[i] = v
    return f


def _set(**kw):
    def f(q):
        for k, v in kw.items():
            setattr(q, k, v)
    return f


REFUSED = {
    "null_a0": _set(a0=None),
    "null_w": _set(w=None),
    "null_out": _set(out=None),
    "a0_c_not_64": _set(a0_c=96, kc=96),
    "a1_c_not_64": _set(a1_c=32, kc=160),
    "kc_not_the_sum": _set(kc=192),
    "a1_without_channels": "a1",
    "a1_channels_without_a1": _set(a1_c=64, kc=192),
    "nc_not_64": _set(nc=96),
    "n_lo_not_64": _set(n_lo=32),
    "n_hi_past_nc": _set(n_hi=192),
    "n_empty": _set(n_lo=64, n_hi=64),
    "n_lo_negative": _set(n_lo=-64),
    "d_lo_below_-4": _set(d_lo=-5),
    "d_hi_above_4": _set(d_hi=5),
    "d_lo_above_d_hi": _set(d_lo=1, d_hi=0),
    "tap_k_past_kc": _set_tap(4, k_hi=192),
    "tap_k_unaligned": _set_tap(4, k_lo=32),
    "tap_k_empty": _set_tap(4, k_lo=64, k_hi=64),
    "tap_n_past_nc": _set_tap(3, n_hi=192),
    "tap_n_unaligned": _set_tap(5, n_hi=96),
    "a_dtype": _set(a_dtype=SG_F32),
    "w_dtype": _set(w_dtype=7),
    "out_dtype": _set(out_dtype=9),
    "ksplit_16bit_out": _set(ksplit=2),
    "m_lo_below_halo": _set(m_lo=-1),
    "m_hi_past_rows": _set(m_hi=65),
    "m_empty": _set(m_lo=10, m_hi=10),
    "batch_0": _set(batch=0),
    "a_rows_0": _set(a_rows=0),
    "a_halo_negative": _set(a_halo=-1),
    "out2_without_slope": "out2",
    "slope_mod_0": "slope_mod_0",
    "slope_mod_not_64": "slope_mod_96",
    "slope_with_f32_out": "slope_f32",
    "out2_halo_negative": "out2_halo_-1",
    "out2_halo_with_m_range": "out2_halo_m",
    "out2_halo_too_few_rows": "out2_halo_rows",
    "mixed_formats_on_tensor_cores": _set(w_dtype=SG_BF16),
    "bn_stats_n_sub_range": "bn_stats",
    "tma_store_ld_not_8": _set(out_ld=130, out_col0=0),
    "unknown_backend": _set(backend=7),
    # the column range stays inside one row; pairs are stored together
    "columns_past_out_ld": _set(out_ld=128, out_col0=64),
    "out_col0_negative": _set(out_ld=256, out_col0=-64),
    "bias_mod_not_64": _set(bias_mod=96),
    "f32_out_ld_odd": ("f32", _set(out_ld=129, out_col0=0)),
    "f32_out_col0_odd": ("f32", _set(out_ld=256, out_col0=1)),
    "f32_out_misaligned": ("f32", "misalign"),
    "f16_out_misaligned": "misalign",
    # the FFMA kernel has no fused epilogues
    "ffma_out2": ("ffma", "out2_ok"),
    "ffma_slope": ("ffma", "slope_ok"),
    "ffma_bn_stats": ("ffma", "bn_stats_ok"),
}


def _refusal(name):
    r = REFUSED[name]
    backend, f32 = BACKEND_TCGEN05, False
    if isinstance(r, tuple):
        if r[0] == "ffma":
            backend = BACKEND_FFMA
        else:
            f32 = True
        r = r[1]
    c = dict(_RC, f32=True) if f32 else dict(_RC)
    a0, a1, w, bias, _ = _operands(c, "f16", 8000)
    big = _Out(2, 64 + 8, 256, torch.float32 if f32 else torch.float16, 8001, lambda lv: None)
    dst = big.t
    extra = {}
    q = _make_q(c, "f16", backend, a0, a1, w, bias, None, dst, None, 1)
    q.out_ld, q.out_col0 = 256, 0
    slope = torch.rand(128, device=DEV)
    out2 = _Out(2, 64 + 8, 256, torch.float16, 8002, lambda lv: None)
    if callable(r):
        r(q)
    elif r == "a1":
        extra["a1"] = torch.zeros(2, 64, 64, dtype=torch.float16, device=DEV)
        q.a1 = C.c_void_p(extra["a1"].data_ptr())
    elif r in ("out2", "out2_ok"):
        q.out2, q.out2_halo = C.c_void_p(out2.t.data_ptr()), 0
        if r == "out2_ok":
            q.slope, q.slope_mod = C.c_void_p(slope.data_ptr()), 128
    elif r in ("slope_ok", "slope_mod_0", "slope_mod_96", "slope_f32"):
        q.slope, q.slope_mod = C.c_void_p(slope.data_ptr()), {"slope_mod_0": 0, "slope_mod_96": 96}.get(r, 128)
        if r == "slope_f32":
            q.out_dtype = SG_F32
    elif r.startswith("out2_halo"):
        q.out2, q.slope, q.slope_mod = C.c_void_p(out2.t.data_ptr()), C.c_void_p(slope.data_ptr()), 128
        q.out2_halo = {"out2_halo_-1": -1, "out2_halo_m": 4, "out2_halo_rows": 31}[r]
        if r == "out2_halo_m":
            q.m_lo = 1
    elif r in ("bn_stats", "bn_stats_ok"):
        extra["st"] = torch.zeros(8, 2, 128, dtype=torch.float64, device=DEV)
        q.bn_stats = C.c_void_p(extra["st"].data_ptr())
        if r == "bn_stats":
            q.n_lo = 64
    elif r == "misalign":
        q.out = C.c_void_p(dst.data_ptr() + (4 if f32 else 2))
    return q, big, out2, extra


@pytest.mark.parametrize("name", list(REFUSED))
def test_tapgemm_f_refuses(name):
    q, big, out2, extra = _refusal(name)
    torch.cuda.synchronize()
    with pytest.raises(_lib.SeganB200Error):
        _launch(q)
    torch.cuda.synchronize()
    assert big.unchanged() and out2.unchanged(), (name, "a refused launch wrote")


def test_refusal_baseline_launches():
    """The valid problem every refusal starts from runs on both back-ends (so each refusal is its own change)."""
    for backend in (BACKEND_TCGEN05, BACKEND_FFMA):
        for f32 in (False, True):
            c = dict(_RC, f32=True) if f32 else dict(_RC)
            a0, a1, w, bias, _ = _operands(c, "f16", 8000)
            big = _Out(2, 64 + 8, 256, torch.float32 if f32 else torch.float16, 8001, lambda lv: None)
            q = _make_q(c, "f16", backend, a0, a1, w, bias, None, big.t, None, 1)
            q.out_ld, q.out_col0 = 256, 0
            _launch(q)
            torch.cuda.synchronize()
            assert not big.unchanged()
