"""The weight-gradient tap-GEMM (form W: tapgemm_tc.cu tapgemm_w_tc<TK, format>, tapgemm_ref.cu tapgemm_w_ffma)
launched through engine.run_w against an fp64 evaluation of  dW[d][n][kc] += sum_{b,m} G[b][m][n] A[b][m + d][kc].

Every case accumulates into a dw pre-filled with random fp32 values dw0 (-0.0f in half of the dead elements: a
stray accumulation of 0.0f flips that sign bit).  Afterwards, inside the taps' live (n, kc) boxes
  c = max |dw - dw0 - scale * ref| / (2^-24 * scale * (sum |g a| + |dw0|) * (1 + stages / 32))  <=  16
(tests/tapgemm_model.py; the last term is the tensor-core accumulator's truncation over the 64-position stages of one
split: decoder block 1 at batch 300 runs unsplit, 300 stages, and comes out 2e-5 smaller than the fp64 sum)
and every other element -- structural-zero blocks, tap slots outside [d_lo, d_hi], the guard bands before and
after dw -- is bit-identical to dw0.  Where both back-ends run they agree at c <= 32.

Which tensor-core instantiation a case launches (TK = 256 / 128 / 64 from kc % 256, kc % 128; one 64-position stage
= PB batch elements x PR rows; pos_steps = ceil(rows / PR) * ceil(batch / PB)); every id runs as `<id>-f16` and,
where marked *, also as `<id>-bf16`:

  id                  TK   PR x PB   sources      taps                 ksplit / pos_steps
  kc64_full *         64   64 x 1    64           full, 9 taps         2 / 3
  kc192_deconv *      64   64 x 1    192          deconv_fwd (n)       2 / 3
  z64_dec0 *          64   16 x 4    64 + 1024    deconv_fwd (n)       2 / 2      (--z_dim 64 decoder block 0)
  kc128_full *        128  64 x 1    128          full, 9 taps         2 / 3
  kc384_deconv *      128  64 x 1    384          deconv_fwd (n)       2 / 3
  kc256_conv *        256  64 x 1    256          conv_fwd (k)         2 / 3
  kc512_conv_n512 *   256  64 x 1    512          conv_fwd (k)         2 / 3
  skipconv_k11 *      256  64 x 1    256          skip conv, d -2..2   2 / 3      (dw_tap0 = 2)
  taps3_conv          256  64 x 1    256          conv_fwd, d -1..1    2 / 3      (dw_tap0 = 0: slots 0-2, 6 unused)
  src_128_128         256  64 x 1    128 + 128    deconv_fwd (n)       2 / 3
  src_64_192          256  64 x 1    64 + 192     full                 2 / 3
  src_192_64 *        256  64 x 1    192 + 64     full                 2 / 3
  src_64_64           128  64 x 1    64 + 64      full                 2 / 3
  src_256_128         128  64 x 1    256 + 128    full                 2 / 3      (split on a TK boundary)
  src_256_256         256  64 x 1    256 + 256    conv_fwd (k)         2 / 3      (split on a TK boundary)
  rows1_b70_h0        256  1 x 64    256          full, d = 0          1 / 2      (last box: 6 of 64 batch elements)
  rows1_b1_h0         256  1 x 64    256          full, d = 0          1 / 1
  rows2_b33_h4        256  2 x 32    256          conv_fwd             2 / 2
  rows4_b17_h0        256  4 x 16    256          conv_fwd             2 / 2
  rows8_b9_h4         256  8 x 8     256          conv_fwd             2 / 2
  rows16_b5_h0 *      256  16 x 4    256          conv_fwd             2 / 2
  rows32_b3_h0        256  32 x 2    256          conv_fwd             2 / 2
  rows32_b1_h4        256  32 x 2    256          conv_fwd             1 / 1
  rows64_b3_h0        256  64 x 1    256          conv_fwd             2 / 3
  rows128_b2_h4       256  64 x 1    256          conv_fwd             3 / 4
  mlp_rows4800_b1     256  64 x 1    1024         full, d = 0          wgrad_ksplit / 75
  split_1 / 3 / 7 / 40     64 x 1    256          conv_fwd             1, 3, 7 (2 empty splits), 40 (clamped) / 10
  split_engine        256  64 x 1    256          conv_fwd             wgrad_ksplit / 24
  wave_b4_k74  ...    128  64 x 1    128          full, d = 0          74 / 128 (10 empty), 148 / 128 (clamped),
  wave_b16_k148                                                        74 / 512, 148 / 512 (20 empty)
  out_scale_k1 / k3   256  64 x 1    256          conv_fwd             1, 3 / 3   (device scalar, pointer offset)
Production scale (batch 300, fp16, tensor cores, ksplit from engine.wgrad_ksplit): test_production_scale.
Run on an H100:  python -m pytest tests -m gpu"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                                     # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, BACKEND_FFMA, BACKEND_TCGEN05   # noqa: E402
from tests import tapgemm_model as M                                                  # noqa: E402

DEV = "cuda"
GUARD = 4096                  # floats before and after the dw view
FMT = {"f16": (SG_F16, torch.float16), "bf16": (SG_BF16, torch.bfloat16)}
BACKENDS = {"ffma": BACKEND_FFMA, "tc": BACKEND_TCGEN05}
EDGE = 64.0                   # |first and last row| of every batch element when a_halo = 0


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _taps(c):
    kind, kc, nc = c["taps"], c["a0_c"] + c.get("a1_c", 0), c["nc"]
    if kind == "skipconv":
        d_lo, d_hi, tap0, fwd, _ = E.skipconv_geometry(kc // 4, c["skip_k"])
        return fwd, d_lo, d_hi, tap0
    ch = {"conv_fwd": kc // 4, "deconv_fwd": nc // 4, "full": 0}[kind]
    d = c.get("d", (-4, 4))
    return E.tap_ranges(kind, ch, kc, nc), d[0], d[1], c.get("tap0", 0)


def tc_tile_k(kc):
    return 256 if kc % 256 == 0 else (128 if kc % 128 == 0 else 64)


def _operands(c, fmt, seed):
    """G [B][R][nc] ~ 0.1 N(0,1); A0 / A1 [B][R + 2 halo][.] ~ N(0,1) in separate allocations.  Without a halo the
    first and last row of every batch element are +-EDGE, so a read that strays into the neighbouring batch
    element (instead of the zero fill) moves the result by hundreds of products."""
    g = _gen(seed)
    tdt = FMT[fmt][1]
    B, R, halo = c["batch"], c["rows"], c.get("halo", 0)
    gg = (0.1 * torch.randn(B, R, c["nc"], generator=g)).to(tdt).to(DEV)
    srcs = []
    for ch in (c["a0_c"], c.get("a1_c", 0)):
        if ch == 0:
            srcs.append(None)
            continue
        a = torch.randn(B, R + 2 * halo, ch, generator=g)
        if halo == 0:
            sign = torch.where(torch.rand(B, 2, ch, generator=g) < 0.5, -EDGE, EDGE)
            a[:, 0], a[:, -1] = sign[:, 0], sign[:, 1]
        srcs.append(a.to(tdt).to(DEV))
    return gg, srcs[0], srcs[1]


class _Dw(object):
    """dw [slots][nc][kc] inside guard bands, pre-filled; `live` marks what the launch may touch."""

    def __init__(self, c, taps, d_lo, d_hi, tap0, seed):
        kc, nc = c["a0_c"] + c.get("a1_c", 0), c["nc"]
        self.slots = d_hi + 4 - tap0 + 2                     # one unused slot after the last tap
        n = self.slots * nc * kc
        live = torch.zeros(self.slots, nc, kc, dtype=torch.bool, device=DEV)
        for d in range(d_lo, d_hi + 1):
            i = d + 4
            live[i - tap0, taps[2][i]:taps[3][i], taps[0][i]:taps[1][i]] = True
        self.live = torch.zeros(n + 2 * GUARD, dtype=torch.bool, device=DEV)
        self.live[GUARD:GUARD + n] = live.reshape(-1)
        self.buf = torch.randn(n + 2 * GUARD, generator=_gen(seed)).to(DEV)
        neg = ~self.live
        neg[1::2] = False
        self.buf[neg] = -0.0
        self.buf0 = self.buf.clone()
        self.dw = self.buf[GUARD:GUARD + n].view(self.slots, nc, kc)
        self.d_lo, self.d_hi, self.tap0 = d_lo, d_hi, tap0

    def untouched_outside(self):
        dead = ~self.live
        return torch.equal(self.buf.view(torch.int32)[dead], self.buf0.view(torch.int32)[dead])

    def unchanged(self):
        return torch.equal(self.buf.view(torch.int32), self.buf0.view(torch.int32))

    def delta(self):
        """(dw - dw0, |dw0|) over the taps d_lo..d_hi, float64."""
        s = slice(self.d_lo + 4 - self.tap0, self.d_hi + 4 - self.tap0 + 1)
        dw0 = self.buf0[GUARD:GUARD + self.dw.numel()].view_as(self.dw)[s].double()
        return self.dw[s].double() - dw0, dw0.abs()


def _launch(c, fmt, backend, gg, a0, a1, taps, d_lo, d_hi, tap0, dw, ksplit, out_scale=None):
    E.run_w(gg, c["rows"], FMT[fmt][0], a0, a1, c["rows"], c.get("halo", 0), FMT[fmt][0], c["a0_c"] + c.get("a1_c", 0),
            c["nc"], taps, dw, c["batch"], d_lo=d_lo, d_hi=d_hi, dw_tap0=tap0, ksplit=ksplit, backend=backend,
            a0_c=c["a0_c"], a1_c=c.get("a1_c", 0), out_scale=out_scale)


def _stages(c, ksplit, backend):
    """64-position stages one tensor-core accumulator walks (mirror of tapgemm_w_tc_launch); 0 for the FFMA kernel,
    whose fmaf rounds to nearest."""
    if backend != "tc":
        return 0
    pr = min(c["rows"], 64)
    pos_steps = -(-c["rows"] // pr) * -(-c["batch"] // (64 // pr))
    return -(-pos_steps // max(1, min(ksplit, pos_steps)))


def _ksplit(c, taps, d_lo, d_hi):
    if c.get("ksplit") == "engine":
        kc = c["a0_c"] + c.get("a1_c", 0)
        return E.wgrad_ksplit(c["batch"] * c["rows"], 0, taps, kc, c["nc"], d_lo, d_hi)
    return c.get("ksplit", 2)


def _run_case(name, c, fmt, backends, seed):
    taps, d_lo, d_hi, tap0 = _taps(c)
    gg, a0, a1 = _operands(c, fmt, seed)
    ksplit = _ksplit(c, taps, d_lo, d_hi)
    scale, osc = 1.0, None
    if c.get("out_scale"):
        sdev = torch.tensor([3.0, c["out_scale"]], device=DEV)       # the scalar sits behind a pointer offset
        scale, osc = float(sdev[1]), sdev[1:]
    ref, mag = M.ref_w(gg, a0, a1, c.get("halo", 0), taps, d_lo, d_hi)
    deltas = {}
    for bk in backends:
        dw = _Dw(c, taps, d_lo, d_hi, tap0, seed + 1)
        _launch(c, fmt, BACKENDS[bk], gg, a0, a1, taps, d_lo, d_hi, tap0, dw.dw, ksplit, osc)
        torch.cuda.synchronize()
        got, dw0 = dw.delta()
        cc = M.c_w(got, ref, mag + dw0 / abs(scale), scale, _stages(c, ksplit, bk))
        print("tapgemm_w %s-%s %s: TK %d ksplit %s c = %.2f (tol %g)" % (name, fmt, bk, tc_tile_k(ref.shape[-1]),
                                                                          ksplit, cc, M.C_TOL))
        assert dw.untouched_outside(), (name, fmt, bk, "written outside the taps' live ranges")
        assert cc <= M.C_TOL, (name, fmt, bk, cc)
        assert float(got.abs().max()) > 0
        deltas[bk] = (got, mag + dw0 / abs(scale))
    if len(deltas) == 2:
        cb = M.c_w(deltas["tc"][0] - deltas["ffma"][0], torch.zeros_like(ref), deltas["tc"][1], scale)
        assert cb <= 2 * M.C_TOL, (name, fmt, "back-ends disagree", cb)


_CONV = dict(a0_c=256, nc=128, taps="conv_fwd")
CASES = {
    # instantiations: TK x format
    "kc64_full": dict(a0_c=64, nc=128, taps="full", rows=64, batch=3, halo=4, bf16=True),
    "kc192_deconv": dict(a0_c=192, nc=256, taps="deconv_fwd", rows=64, batch=3, bf16=True),
    "z64_dec0": dict(a0_c=64, a1_c=1024, nc=512, taps="deconv_fwd", rows=16, batch=5, bf16=True),
    "kc128_full": dict(a0_c=128, nc=128, taps="full", rows=64, batch=3, bf16=True),
    "kc384_deconv": dict(a0_c=384, nc=256, taps="deconv_fwd", rows=64, batch=3, halo=4, bf16=True),
    "kc256_conv": dict(_CONV, rows=64, batch=3, halo=4, bf16=True),
    "kc512_conv_n512": dict(a0_c=512, nc=512, taps="conv_fwd", rows=64, batch=3, halo=4, bf16=True),
    "skipconv_k11": dict(a0_c=256, nc=256, taps="skipconv", skip_k=11, rows=64, batch=3, bf16=True),
    "taps3_conv": dict(_CONV, d=(-1, 1), rows=64, batch=3, halo=4),
    # two sources
    "src_128_128": dict(a0_c=128, a1_c=128, nc=256, taps="deconv_fwd", rows=64, batch=3),
    "src_64_192": dict(a0_c=64, a1_c=192, nc=128, taps="full", rows=64, batch=3),
    "src_192_64": dict(a0_c=192, a1_c=64, nc=128, taps="full", rows=64, batch=3, bf16=True),
    "src_64_64": dict(a0_c=64, a1_c=64, nc=128, taps="full", rows=64, batch=3),
    "src_256_128": dict(a0_c=256, a1_c=128, nc=128, taps="full", rows=64, batch=3),
    "src_256_256": dict(a0_c=256, a1_c=256, nc=128, taps="conv_fwd", rows=64, batch=3, halo=4),
    # rows per batch element and batch tails
    "rows1_b70_h0": dict(a0_c=256, nc=128, taps="full", d=(0, 0), tap0=4, rows=1, batch=70, ksplit=1),
    "rows1_b1_h0": dict(a0_c=256, nc=128, taps="full", d=(0, 0), tap0=4, rows=1, batch=1, ksplit=1),
    "rows2_b33_h4": dict(_CONV, rows=2, batch=33, halo=4),
    "rows4_b17_h0": dict(_CONV, rows=4, batch=17),
    "rows8_b9_h4": dict(_CONV, rows=8, batch=9, halo=4),
    "rows16_b5_h0": dict(_CONV, rows=16, batch=5, bf16=True),
    "rows32_b3_h0": dict(_CONV, rows=32, batch=3),
    "rows32_b1_h4": dict(_CONV, rows=32, batch=1, halo=4, ksplit=1),
    "rows64_b3_h0": dict(_CONV, rows=64, batch=3),
    "rows128_b2_h4": dict(_CONV, rows=128, batch=2, halo=4, ksplit=3),
    "mlp_rows4800_b1": dict(a0_c=1024, nc=1024, taps="full", d=(0, 0), tap0=4, rows=4800, batch=1, ksplit="engine"),
    # position splits: pos_steps = 10
    "split_1": dict(_CONV, rows=64, batch=10, halo=4, ksplit=1),
    "split_3": dict(_CONV, rows=64, batch=10, halo=4, ksplit=3),
    "split_7_two_empty": dict(_CONV, rows=64, batch=10, halo=4, ksplit=7),
    "split_40_clamped": dict(_CONV, rows=64, batch=10, halo=4, ksplit=40),
    "split_engine": dict(_CONV, rows=64, batch=24, halo=4, ksplit="engine"),
    # the waveform-end position-pair GEMMs with the engine's fixed split counts at batches other than 300
    "wave_b4_k74": dict(a0_c=128, nc=128, taps="full", d=(0, 0), tap0=4, rows=2048, batch=4, ksplit=74),
    "wave_b4_k148": dict(a0_c=128, nc=128, taps="full", d=(0, 0), tap0=4, rows=2048, batch=4, ksplit=148),
    "wave_b16_k74": dict(a0_c=128, nc=128, taps="full", d=(0, 0), tap0=4, rows=2048, batch=16, ksplit=74),
    "wave_b16_k148": dict(a0_c=128, nc=128, taps="full", d=(0, 0), tap0=4, rows=2048, batch=16, ksplit=148),
    # 1 / sigma of a spectrally normalised layer
    "out_scale_k1": dict(_CONV, rows=64, batch=3, halo=4, ksplit=1, out_scale=0.37),
    "out_scale_k3": dict(_CONV, rows=64, batch=3, halo=4, ksplit=3, out_scale=0.37),
}
PARAMS = [(n, f) for n, c in CASES.items() for f in (("f16", "bf16") if c.get("bf16") else ("f16",))]


@pytest.mark.parametrize("name,fmt", PARAMS, ids=["%s-%s" % p for p in PARAMS])
def test_tapgemm_w_vs_fp64(name, fmt):
    _run_case(name, CASES[name], fmt, ("ffma", "tc"), 1000 + 7 * list(CASES).index(name))


def test_every_tensor_core_instantiation_is_launched():
    launched = {(tc_tile_k(CASES[n]["a0_c"] + CASES[n].get("a1_c", 0)), f) for n, f in PARAMS}
    assert launched == {(tk, f) for tk in (64, 128, 256) for f in ("f16", "bf16")}


@pytest.mark.parametrize("backend", ["ffma", "tc"])
def test_tapgemm_w_accumulates_from_two_streams(backend):
    """Two launches with different operands enqueued on two side streams into one dw (the gradient bucket of a layer
    both Discriminator lanes reach), joined before the check: dw0 + ref_1 + ref_2."""
    c = dict(_CONV, rows=64, batch=6, halo=4)
    taps, d_lo, d_hi, tap0 = _taps(c)
    ops = [_operands(c, "f16", 2000 + i) for i in range(2)]
    dw = _Dw(c, taps, d_lo, d_hi, tap0, 2002)
    torch.cuda.synchronize()
    sides = [torch.cuda.Stream(), torch.cuda.Stream()]
    for side, (gg, a0, a1) in zip(sides, ops):
        with E.on_side(side):
            _launch(c, "f16", BACKENDS[backend], gg, a0, a1, taps, d_lo, d_hi, tap0, dw.dw, 3)
    for side in sides:
        E.join_side(side)
    refs = [M.ref_w(gg, a0, a1, 4, taps) for gg, a0, a1 in ops]
    torch.cuda.synchronize()
    got, dw0 = dw.delta()
    cc = M.c_w(got, refs[0][0] + refs[1][0], refs[0][1] + refs[1][1] + dw0)
    print("tapgemm_w two streams %s: c = %.2f (tol %g)" % (backend, cc, M.C_TOL))
    assert dw.untouched_outside() and cc <= M.C_TOL


# Batch 300 as GeneratorEngine / DiscriminatorEngine launch it (split count from engine.wgrad_ksplit; fc.0 runs
# unsplit): a CTA walks several tiles and the stage ring wraps many times.
PRODUCTION = {
    "enc1": dict(a0_c=256, nc=128, taps="conv_fwd", rows=1024, batch=300, halo=4, ksplit="engine"),
    "enc3": dict(a0_c=1024, nc=512, taps="conv_fwd", rows=64, batch=300, halo=4, ksplit="engine"),
    "enc4_pb4": dict(a0_c=2048, nc=1024, taps="conv_fwd", rows=16, batch=300, halo=4, ksplit="engine"),
    "dec1_two_src": dict(a0_c=512, a1_c=512, nc=1024, taps="deconv_fwd", rows=64, batch=300, ksplit="engine"),
    "fc0": dict(a0_c=16384, nc=256, taps="full", d=(0, 0), tap0=4, rows=1, batch=300, ksplit=1),
    "skipconv_l0": dict(a0_c=256, nc=256, taps="skipconv", skip_k=11, rows=1024, batch=300, ksplit="engine"),
}


@pytest.mark.parametrize("name", list(PRODUCTION))
def test_production_scale(name):
    """fp16, tensor cores.  Launched twice from the same dw0: fp32 atomics make the two results differ, by no more
    than the model allows either of them."""
    c = PRODUCTION[name]
    taps, d_lo, d_hi, tap0 = _taps(c)
    gg, a0, a1 = _operands(c, "f16", 3000 + list(PRODUCTION).index(name))
    ksplit = _ksplit(c, taps, d_lo, d_hi)
    got = []
    for _ in range(2):
        dw = _Dw(c, taps, d_lo, d_hi, tap0, 3100)
        _launch(c, "f16", BACKEND_TCGEN05, gg, a0, a1, taps, d_lo, d_hi, tap0, dw.dw, ksplit)
        torch.cuda.synchronize()
        assert dw.untouched_outside(), (name, "written outside the taps' live ranges")
        got.append(dw.delta())
    ref, mag = M.ref_w(gg, a0, a1, c.get("halo", 0), taps, d_lo, d_hi)
    scale = mag + got[0][1]
    cc = [M.c_w(g_, ref, scale, trunc_stages=_stages(c, ksplit, "tc")) for g_, _ in got]
    rr = M.c_w(got[0][0] - got[1][0], torch.zeros_like(ref), scale)
    print("tapgemm_w production %s: ksplit %d c = %.2f, %.2f run-to-run %.2f (tol %g)"
          % (name, ksplit, cc[0], cc[1], rr, M.C_TOL))
    assert max(cc) <= M.C_TOL and rr <= 2 * M.C_TOL


REFUSED = {
    "rows_24": dict(rows=24),
    "rows_160": dict(rows=160),
    "nc_64": dict(nc=64),
    "kc_not_the_sum_of_sources": dict(kc=320),
    "a1_without_channels": dict(a1=True),
    "mixed_formats_on_tensor_cores": dict(a_fmt="bf16"),
    "tap_range_outside_kc": dict(k_hi=320),
    "tap_range_unaligned": dict(k_lo=32),
}


@pytest.mark.parametrize("name", list(REFUSED))
def test_tapgemm_w_refuses(name):
    """Argument errors are reported on the host: nothing is launched, dw and its guard bands keep their bits."""
    r = REFUSED[name]
    rows, nc, kc = r.get("rows", 64), r.get("nc", 128), 256
    c = dict(a0_c=kc, nc=nc, taps="full", rows=rows, batch=3)
    taps, d_lo, d_hi, tap0 = _taps(c)
    gg, a0, _ = _operands(c, "f16", 4000)
    a1 = torch.zeros(3, rows, 64, dtype=torch.float16, device=DEV) if r.get("a1") else None
    if r.get("a_fmt"):
        a0 = a0.to(FMT[r["a_fmt"]][1])
    taps[1][2] = r.get("k_hi", taps[1][2])
    taps[0][2] = r.get("k_lo", taps[0][2])
    dw = _Dw(c, E.tap_ranges("full", 0, kc, nc), d_lo, d_hi, tap0, 4001)
    with pytest.raises(_lib.SeganB200Error):
        E.run_w(gg, rows, SG_F16, a0, a1, rows, 0, FMT[r.get("a_fmt", "f16")][0], r.get("kc", kc), nc, taps, dw.dw, 3,
                ksplit=2, backend=BACKEND_TCGEN05, a0_c=kc, a1_c=0)
    torch.cuda.synchronize()
    assert dw.unchanged()
