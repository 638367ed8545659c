"""The hidden layers' tap-GEMM launches at every kernel width 4..32 against fp64 evaluations of the reference modules
(tests/kwidth_layer_model.py): encoder conv forward / data gradient / weight gradient, the Discriminator's conv data
gradient, and decoder deconv forward / data gradient / weight gradient with two sources.

Every layer goes through the engine's own path: a reference-layout fp32 weight -> sg_pack_weights_kw (fp32 master) ->
sg_emit_operands (f16 forward operand, f16 / bf16 data-gradient operand, alpha on the skip half of the decoder's
"skip" sources) -> engine.run_f / run_w with the engine's tap tables, spans, row ranges, halos, bias_mod and
wgrad_ksplit -> sg_unpack_wgrad_kw (weight gradients back to reference layout).  The fp64 references never see the
engine's tables or packing: they take the same 16-bit-rounded operands in reference layout.

Gates (tests/tapgemm_model.py, harness of test_gpu_tapgemm_f.py / _w.py):
  forward-form outputs   c_f <= 16 per back-end, c_pair <= 32 between FFMA and tensor cores, 16-bit tensor-core
                         results bitwise repeatable, every element outside the launch's rows and columns (guard bands
                         included) keeps its sentinel bits, stream-K counters zero afterwards
  weight gradients       accumulated into a pre-filled packed slot: c_w <= 16 in reference layout, back-ends within
                         32, and every element that holds no weight of the width-k layer (kwidth_layer_model
                         .packed_live: structural zeros, unused taps, guard bands) keeps its initial bits

Cases: every width at c = 64 (the phase blocks start at odd multiples of 64 inside the 256-wide K / N tiles) and at
c = 256 (ranges that cross tile boundaries); rows per batch element 16 / 64 / 128 by width (row packing, partial M
tiles: the data gradient's 24 / 72 / 136 rows); decoder sources by width: "skip" (c + c, alpha on the second),
"block0" (64 + c, the data gradient from column 64 only), "convskip" (c + c, the data gradient split over two
destinations).  Batch 300 under the default cost model at widths 4, 5, 11, 20, 32 and one forced stream-K launch.
Run on an H100:  python -m pytest tests/test_gpu_kwidth_layers.py -m gpu -s"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                              # noqa: E402
from segan_pytorch_b200._lib import SG_F16, SG_F32, BACKEND_TCGEN05            # noqa: E402
from tests import kwidth_layer_model as K, tapgemm_model as M                 # noqa: E402
from tests import test_gpu_tapgemm_f as TF, test_gpu_tapgemm_w as TW          # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream
ZC = 64                       # z channels of the "block0" decoder sources (--z_dim 64)
KINDS = ("enc_fwd", "enc_dgrad", "d_dgrad", "enc_wgrad", "dec_fwd", "dec_dgrad", "dec_wgrad")
# (form, tap table) each kind launches: the coverage test in tests/test_kwidth_layer_model.py reads it
TABLES = {"enc_fwd": ("F", "conv_fwd"), "enc_dgrad": ("F", "conv_dgrad"), "d_dgrad": ("F", "conv_dgrad"),
          "enc_wgrad": ("W", "conv_fwd"), "dec_fwd": ("F", "deconv_fwd"), "dec_dgrad": ("F", "deconv_dgrad"),
          "dec_wgrad": ("W", "deconv_fwd")}
CHANNELS = (64, 256)
ROWS = (16, 64, 128)
SOURCES = ("skip", "block0", "convskip")
CASES = [(kind, k, c) for kind in KINDS for c in CHANNELS for k in K.WIDTHS]
PRODUCTION_WIDTHS = (4, 5, 11, 20, 32)
PRODUCTION = [(kind, k) for kind in KINDS for k in PRODUCTION_WIDTHS]


def rows_of(k):
    return ROWS[k % 3]


def sources_of(k):
    return SOURCES[(k // 3) % 3]


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


class _Layer(object):
    """A width-k conv (kind 0: W[cout][cin][k]) or deconv (kind 1: W[cin][cout][k]) through the engine's packing:
    reference-layout fp32 -> sg_pack_weights_kw -> fp32 master [9][nc][kc] -> sg_emit_operands."""

    def __init__(self, kind, c_out, c_in, k, g, alpha_from=0):
        self.kind, self.c_out, self.c_in, self.k = kind, c_out, c_in, k
        self.w = 0.05 * torch.randn((c_out, c_in, k) if kind == 0 else (c_in, c_out, k), generator=g, device=DEV)
        self.alpha_from = alpha_from
        self.alpha = 0.5 + torch.rand(c_in - alpha_from, generator=g, device=DEV) if alpha_from else None
        self.nc, self.kc = (c_out, 4 * c_in) if kind == 0 else (4 * c_out, c_in)
        self.master = torch.full((9, self.nc, self.kc), float("nan"), device=DEV)
        _lib.call("sg_pack_weights_kw", kind, _p(self.w), c_out, c_in, 0, k, None, 0, _p(self.master), None, SG_F32,
                  SG_F32, _stream())

    def emit(self, fmt):
        """(forward operand f16 [9][nc][kc], data-gradient operand in fmt [9][kc][nc])"""
        wf = torch.empty(9, self.nc, self.kc, dtype=torch.float16, device=DEV)
        wd = torch.empty(9, self.kc, self.nc, dtype=TF.FMT[fmt][1], device=DEV)
        _lib.call("sg_emit_operands", _p(self.master), 9, self.nc, self.kc, _p(self.alpha), self.alpha_from, _p(wf),
                  _p(wd), SG_F16, TF.FMT[fmt][0], None, _stream())
        return wf, wd

    def weff(self, fmt):
        """The weight the emitted operand holds, in reference layout: W (alpha on the input channels >= alpha_from),
        rounded once to fmt."""
        w = self.w.clone()
        if self.alpha is not None:
            w[self.alpha_from:] *= self.alpha.view(-1, 1, 1)
        return w.to(TF.FMT[fmt][1])

    def unpack(self, packed):
        """Packed slots [>= d_hi + 5][nc][kc] (fp32) -> reference layout through sg_unpack_wgrad_kw (a copy)."""
        m = torch.zeros(9, self.nc, self.kc, device=DEV)
        n = min(9, packed.shape[0])
        m[:n] = packed[:n]
        out = torch.empty_like(self.w)
        _lib.call("sg_unpack_wgrad_kw", self.kind, _p(m), self.c_out, self.c_in, 0, self.k, None, None, 0, _p(out),
                  None, 0, _stream())
        return out


def _rows(x):
    """[B][C][R] -> [B][R][C] (one position per row: the decoder's input and the conv's output rows)"""
    return x.permute(0, 2, 1).contiguous()


def _f_launch(c, fmt, launch, ref, mag, seed, backends=("ffma", "tc")):
    """One form-F launch per back-end into a guarded destination: gated against fp64, the back-ends against each other
    and, where both run (batch 3: a single wave, no stream-K split), the tensor cores repeated bitwise."""
    label = "%s k%d c%d %s%s" % (c["name"], c["k"], c["ch"], fmt, c.get("part", ""))
    res = {}
    for bk in backends:
        out, _ = TF._outputs(c, fmt, seed)
        launch(out.t, TF.BACKENDS[bk])
        torch.cuda.synchronize()
        if bk == "tc":
            assert TF._counters_zero(), (label, "stream-K counters left non-zero")
        res[bk] = TF._check(label, c, fmt, bk, out, None, ref, mag, None, TF._stages(c, bk), 1)
        if bk == "tc" and len(backends) == 2:
            again, _ = TF._outputs(c, fmt, seed)
            launch(again.t, BACKEND_TCGEN05)
            torch.cuda.synchronize()
            assert torch.equal(out.bits(out.buf), again.bits(again.buf)), (label, "not repeatable")
    if len(res) == 2:
        den = torch.maximum(res["tc"][1], res["ffma"][1])
        cb = M.c_pair(res["tc"][0], res["ffma"][0], den, fmt, TF._stages(c, "tc"))
        print("kwidth layer %s back-ends: c = %.2f (tol %g)" % (label, cb, 2 * M.C_TOL))
        assert cb <= 2 * M.C_TOL, (label, "back-ends disagree", cb)


def _w_launch(c, fmt, layer, launch, ref, mag, ksplit, seed, backends=("ffma", "tc")):
    """One form-W launch per back-end into a packed gradient slot pre-filled with random values (-0.0f in half of its
    structural zeros), checked in reference layout after sg_unpack_wgrad_kw."""
    label = "%s k%d c%d %s" % (c["name"], c["k"], c["ch"], fmt)
    taps, d_lo, d_hi = c["table"], c["d"][0], c["d"][1]
    live = K.packed_live(layer.kind, layer.k, layer.c_out, layer.c_in, DEV)
    res = {}
    for bk in backends:
        dw = TW._Dw(c, taps, d_lo, d_hi, 0, seed)
        n = dw.dw.numel()
        assert not live[dw.slots:].any()
        dw.live.zero_()
        dw.live[TW.GUARD:TW.GUARD + n].view_as(dw.dw)[:9] = live[:dw.slots]
        launch(dw.dw, TF.BACKENDS[bk])
        torch.cuda.synchronize()
        assert dw.untouched_outside(), (label, bk, "wrote an element that holds no weight")
        dw0 = dw.buf0[TW.GUARD:TW.GUARD + n].view_as(dw.dw)
        got0 = layer.unpack(dw0).double()
        got = layer.unpack(dw.dw).double() - got0
        den = mag + got0.abs()
        cc = M.c_w(got, ref, den, trunc_stages=TW._stages(c, ksplit, bk))
        print("kwidth layer %s %s: ksplit %d c = %.2f (tol %g)" % (label, bk, ksplit, cc, M.C_TOL))
        assert cc <= M.C_TOL, (label, bk, cc)
        assert float(got.abs().max()) > 0
        res[bk] = (got, den)
    if len(res) == 2:
        cb = M.c_w(res["tc"][0] - res["ffma"][0], torch.zeros_like(ref), torch.maximum(res["tc"][1], res["ffma"][1]))
        print("kwidth layer %s back-ends: c = %.2f (tol %g)" % (label, cb, 2 * M.C_TOL))
        assert cb <= 2 * M.C_TOL, (label, "back-ends disagree", cb)


def _encoder(kind, k, c, B, R, fmt, g):
    """Conv cin = c -> cout = 2c over L = 4R positions between 16-position reflect halos (rows: R + 8 of 4c)."""
    cin, cout = c, 2 * c
    tdt = TF.FMT[fmt][1]
    lay = _Layer(0, cout, cin, k, g)
    taps = E.tap_ranges("conv_fwd", cin, 4 * cin, cout, k)
    x = torch.randn(B, cin, 4 * R, generator=g, device=DEV)
    xp = F.pad(x, (K.HALO, K.HALO), mode="reflect").to(tdt)
    a = K.ncl_to_rows(xp).contiguous()
    base = dict(name=kind, k=k, ch=c, rows=R, batch=B)
    if kind == "enc_fwd":
        d_lo, d_hi = E.tap_span(taps)
        bias = torch.randn(cout, generator=g, device=DEV)
        wf, _ = lay.emit(fmt)
        ref, mag = K.conv_fwd(xp, lay.weff(fmt), k, bias)
        cc = dict(base, taps="conv_fwd", d=(d_lo, d_hi), a0_c=4 * cin, nc=cout, halo=4)

        def launch(out, bk):
            E.run_f(a, None, R, 4, SG_F16, wf, SG_F16, 4 * cin, cout, taps, out, SG_F16, R, 0, 0, R, B, d_lo=d_lo,
                    d_hi=d_hi, bias=bias, bias_mod=cout, backend=bk)
        return "F", [(cc, launch, _rows(ref), _rows(mag))]
    gy = (0.1 * torch.randn(B, cout, R, generator=g, device=DEV)).to(tdt)
    gr = _rows(gy)
    if kind == "enc_wgrad":
        d_lo, d_hi = E.tap_span(taps)
        ref, mag = K.conv_wgrad(xp, gy, k)
        n_tiles = 9 * (cout // 128) * max(1, 4 * cin // 256)
        ksplit = E.wgrad_ksplit(B * R, n_tiles, taps, 4 * cin, cout, d_lo, d_hi)
        cc = dict(base, table=taps, d=(d_lo, d_hi), a0_c=4 * cin, nc=cout)

        def launch(dw, bk):
            E.run_w(gr, R, TF.FMT[fmt][0], a, None, R, 4, TF.FMT[fmt][0], 4 * cin, cout, taps, dw, B, d_lo=d_lo,
                    d_hi=d_hi, ksplit=ksplit, backend=bk)
        return "W", [(cc, launch, ref, mag, lay, ksplit)]
    # data gradient: the Generator mirrors the forward span, the Discriminator takes the span of the dgrad table
    taps_dg = E.tap_ranges("conv_dgrad", cin, cout, 4 * cin, k)
    d_lo, d_hi = E.dgrad_span(taps) if kind == "enc_dgrad" else E.tap_span(taps_dg)
    _, wd = lay.emit(fmt)
    ref, mag = K.conv_dgrad(gy, lay.weff(fmt), k)
    cc = dict(base, taps="conv_dgrad", d=(d_lo, d_hi), a0_c=cout, nc=4 * cin)
    S = TF.FMT[fmt][0]

    def launch(out, bk):
        E.run_f(gr, None, R, 0, S, wd, S, cout, 4 * cin, taps_dg, out, S, R, 4, -4, R + 4, B, d_lo=d_lo, d_hi=d_hi,
                backend=bk)
    return "F", [(cc, launch, K.ncl_to_rows(ref), K.ncl_to_rows(mag))]


def _decoder(kind, k, c, B, R, fmt, g, srcs):
    """Deconv cout = c over two sources of R rows each: skip (c + c, alpha on the second), block0 (ZC + c: the data
    gradient from column ZC, as for decoder block 0 whose z gets none), convskip (c + c, the data gradient written to
    two destinations of cin / 2 columns)."""
    c0 = ZC if srcs == "block0" else c
    c1, cout = c, c
    cin = c0 + c1
    tdt = TF.FMT[fmt][1]
    lay = _Layer(1, cout, cin, k, g, alpha_from=c0 if srcs == "skip" else 0)
    taps = E.tap_ranges("deconv_fwd", cout, cin, 4 * cout, k)
    d_lo, d_hi = E.tap_span(taps)
    x = torch.randn(B, cin, R, generator=g, device=DEV).to(tdt)
    s0, s1 = _rows(x[:, :c0]), _rows(x[:, c0:])
    base = dict(name="%s_%s" % (kind, srcs), k=k, ch=c, rows=R, batch=B)
    S = TF.FMT[fmt][0]
    if kind == "dec_fwd":
        bias = torch.randn(cout, generator=g, device=DEV)
        wf, _ = lay.emit(fmt)
        ref, mag = K.deconv_fwd(x, lay.weff(fmt), k, bias)
        cc = dict(base, taps="deconv_fwd", d=(d_lo, d_hi), a0_c=c0, a1_c=c1, nc=4 * cout)

        def launch(out, bk):
            E.run_f(s0, s1, R, 0, SG_F16, wf, SG_F16, cin, 4 * cout, taps, out, SG_F16, R, 0, 0, R, B, d_lo=d_lo,
                    d_hi=d_hi, bias=bias, bias_mod=cout, a0_c=c0, a1_c=c1, backend=bk)
        return "F", [(cc, launch, K.ncl_to_rows(ref), K.ncl_to_rows(mag))]
    gy = (0.1 * torch.randn(B, cout, 4 * R, generator=g, device=DEV)).to(tdt)
    gr = K.ncl_to_rows(gy).contiguous()
    if kind == "dec_wgrad":
        ref, mag = K.deconv_wgrad(x, gy, k)
        n_tiles = 9 * (4 * cout // 128) * max(1, cin // 256)
        ksplit = E.wgrad_ksplit(B * R, n_tiles, taps, cin, 4 * cout, d_lo, d_hi)
        cc = dict(base, table=taps, d=(d_lo, d_hi), a0_c=c0, a1_c=c1, nc=4 * cout)

        def launch(dw, bk):
            E.run_w(gr, R, S, s0, s1, R, 0, S, cin, 4 * cout, taps, dw, B, d_lo=d_lo, d_hi=d_hi, ksplit=ksplit,
                    a0_c=c0, a1_c=c1, backend=bk)
        return "W", [(cc, launch, ref, mag, lay, ksplit)]
    taps_dg = E.tap_ranges("deconv_dgrad", cout, 4 * cout, cin, k)
    dg_lo, dg_hi = E.dgrad_span(taps)
    _, wd = lay.emit(fmt)
    ref, mag = K.deconv_dgrad(gy, lay.weff(fmt), k)
    ref, mag = _rows(ref), _rows(mag)
    cc = dict(base, taps="deconv_dgrad", d=(dg_lo, dg_hi), a0_c=4 * cout, nc=cin)
    if srcs != "convskip":
        n_lo = ZC if srcs == "block0" else 0
        cc["n"] = (n_lo, cin)

        def launch(out, bk):
            E.run_f(gr, None, R, 0, S, wd, S, 4 * cout, cin, taps_dg, out, S, R, 0, 0, R, B, d_lo=dg_lo, d_hi=dg_hi,
                    n_lo=n_lo, n_hi=cin, backend=bk)
        return "F", [(cc, launch, ref, mag)]
    parts = []
    half = cin // 2
    for i, n0 in enumerate((0, half)):
        def launch(out, bk, n0=n0):
            E.run_f(gr, None, R, 0, S, wd, S, 4 * cout, cin, taps_dg, out, S, R, 0, 0, R, B, d_lo=dg_lo, d_hi=dg_hi,
                    n_lo=n0, n_hi=n0 + half, out_ld=half, out_col0=0, backend=bk)
        parts.append((dict(cc, n=(n0, n0 + half), out_ld=half, out_col0=0, part=" dst%d" % i), launch, ref, mag))
    return "F", parts


def _run(kind, k, c, B, R, fmt, seed, backends=("ffma", "tc")):
    g = _gen(seed)
    if kind.startswith("dec"):
        form, parts = _decoder(kind, k, c, B, R, fmt, g, sources_of(k))
    else:
        form, parts = _encoder(kind, k, c, B, R, fmt, g)
    for i, part in enumerate(parts):
        if form == "F":
            cc, launch, ref, mag = part
            _f_launch(cc, fmt, launch, ref, mag, seed + 1 + i, backends)
        else:
            cc, launch, ref, mag, lay, ksplit = part
            _w_launch(cc, fmt, lay, launch, ref, mag, ksplit, seed + 1 + i, backends)


def _fmts(kind):
    return ("f16",) if kind.endswith("fwd") else ("f16", "bf16")


@pytest.mark.parametrize("kind,k,c", CASES, ids=["%s-k%d-c%d" % p for p in CASES])
def test_layer_vs_fp64(kind, k, c):
    for j, fmt in enumerate(_fmts(kind)):
        _run(kind, k, c, 3, rows_of(k), fmt, 20000 + 1000 * KINDS.index(kind) + 40 * k + c + 17 * j)


@pytest.mark.parametrize("kind,k", PRODUCTION, ids=["%s-k%d" % p for p in PRODUCTION])
def test_production_scale(kind, k):
    """Batch 300, 64 rows, c = 64, f16, tensor cores, the default stream-K cost model and wgrad_ksplit."""
    _lib.load().sg_set_stream_k(16, 4.5)
    _run(kind, k, 64, 300, 64, "f16", 30000 + 100 * KINDS.index(kind) + k, backends=("tc",))


@pytest.fixture
def forced_stream_k():
    with TF._ForcedStreamK():
        yield


def test_forced_stream_k(forced_stream_k):
    """Deconv at k = 5, c = 256, batch 300, 16 rows: 38 M tiles x 4 N tiles of 256 columns = 152 tiles on 132 SMs; the
    N tiles see different taps (their phase blocks), so the 20 leftover tiles split along K walk unequal step counts.
    Every partial slot starts as NaN: a piece that adds a slot it did not write first poisons the output."""
    ws = E.sk_workspace(DEV)
    ws[8192:].fill_(0xFF)
    _run("dec_fwd", 5, 256, 300, 16, "f16", 31000, backends=("tc",))
    split = bool((ws[8192:] != 0xFF).any())
    ws[8192:].zero_()
    assert split, "the split-K path did not run"
