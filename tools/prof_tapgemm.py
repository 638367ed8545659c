"""Launches representative SEGAN+ layer shapes of the two tensor-core tap-GEMMs at batch 300 (for timing): conv
forward and data gradient of every encoder level, the decoder deconvs (two K sources), the weight gradients, the
Generator's fused PReLU + reflect-halo outputs (out2) and the waveform-end single-tap GEMMs.  Prints CUDA-event times
and TFLOP/s.  `one <names>` runs single shapes; with SEGAN_B200_DEBUG=1048576 it also prints each one's per-CTA
phase timeline."""
import os
import sys

import torch

from segan_pytorch_b200 import engine as E
from segan_pytorch_b200._lib import SG_BF16, SG_F16

B = int(sys.argv[1]) if len(sys.argv) > 1 else 300
REP = int(sys.argv[2]) if len(sys.argv) > 2 else 5
COMPARE = sys.argv[3] if len(sys.argv) > 3 else ""
MODEL_ATOMIC = float(sys.argv[4]) if len(sys.argv) > 4 and sys.argv[3] == "streamk" else 4.5
dev = "cuda"
h = lambda *s: (torch.randn(*s, device=dev) * 0.5).half()
b = lambda *s: (torch.randn(*s, device=dev) * 0.5).bfloat16()


def timeit(name, fn, flops):
    """COMPARE = "compare": wave split on / off;  "splitk": split-K tail on / off;  "streamk": stream-K split factors."""
    from segan_pytorch_b200 import _lib
    lib = _lib.load()
    if COMPARE == "splitk":
        settings = [("splitk", lambda: setattr(E, "SPLITK_TAIL", True)), ("plain", lambda: setattr(E, "SPLITK_TAIL", False))]
    elif COMPARE == "streamk":
        # split factor of the leftover tiles of the last wave: off, forced 2..37 (cost constant ~0), then the model
        settings = [("off", lambda: lib.sg_set_stream_k(0, -1.0))] + \
                   [("S<=%d" % S, (lambda S=S: lib.sg_set_stream_k(S, 1e-6))) for S in (2, 4, 8, 16, 37)] + \
                   [("model", lambda: lib.sg_set_stream_k(16, MODEL_ATOMIC))]
    elif COMPARE == "compare":
        settings = [("split", lambda: setattr(E, "SPLIT_WAVES", True)), ("unsplit", lambda: setattr(E, "SPLIT_WAVES", False))]
    else:
        settings = [("", lambda: None)]
    res = []
    for _, setup in settings:
        setup()
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(REP):
            fn()
        e.record()
        torch.cuda.synchronize()
        res.append(s.elapsed_time(e) / REP)
    if COMPARE == "streamk":
        print("%-28s %s" % (name, " | ".join("%s %.3f" % (settings[i][0], ms) for i, ms in enumerate(res))))
        return
    print("%-28s %s" % (name, "   | ".join("%-7s %8.3f ms  %7.1f TFLOP/s" % (settings[i][0], ms, flops / ms / 1e9)
                                          for i, ms in enumerate(res))))


def _out2(rows, cols, halo):
    """The Generator blocks' fused second output: PReLU(out) with a reflect halo (sg_tapgemm_f.out2)."""
    if halo is None:
        return {}
    return dict(out2=torch.empty(B, rows + 2 * halo, cols, device=dev, dtype=torch.float16), out2_halo=halo,
                slope=torch.rand(cols, device=dev) * 0.3, slope_mod=cols)


def conv_fwd(cin, cout, R, out2_halo=None):
    """out2_halo: None = the Discriminator's conv (one output), else the Generator's encoder block with its out2."""
    a = h(B, R + 8, 4 * cin)
    w = h(9, cout, 4 * cin)
    out = torch.empty(B, R, cout, device=dev, dtype=torch.float16)
    bias = torch.randn(cout, device=dev)
    taps = E.tap_ranges("conv_fwd", cin, 4 * cin, cout)
    fl = E._tap_flops(taps, -4, 4, 0, cout, R * B)
    kw = _out2(R, cout, out2_halo)
    timeit("conv_fwd %d->%d R=%d%s" % (cin, cout, R, "" if out2_halo is None else " out2 halo %d" % out2_halo),
           lambda: E.run_f(a, None, R, 4, SG_F16, w, SG_F16, 4 * cin, cout, taps, out, SG_F16, R, 0, 0, R, B,
                           bias=bias, bias_mod=cout, backend=1, **kw), fl)


def deconv_fwd(cin, cout, R, out2=False):
    """out2: the Generator's decoder block as the train step runs it (raw output + PReLU output, no halo)."""
    a0, a1 = h(B, R, cin // 2), h(B, R, cin // 2)
    w = h(9, 4 * cout, cin)
    out = torch.empty(B, R, 4 * cout, device=dev, dtype=torch.float16)
    bias = torch.randn(cout, device=dev)
    taps = E.tap_ranges("deconv_fwd", cout, cin, 4 * cout)
    fl = E._tap_flops(taps, -4, 4, 0, 4 * cout, R * B)
    kw = _out2(R, 4 * cout, 0 if out2 else None)
    if out2:
        kw["slope_mod"] = cout
    timeit("deconv_fwd %d->%d R=%d%s" % (cin, cout, R, " out2" if out2 else ""),
           lambda: E.run_f(a0, a1, R, 0, SG_F16, w, SG_F16, cin, 4 * cout, taps, out, SG_F16, R, 0, 0, R, B,
                           bias=bias, bias_mod=cout, a0_c=cin // 2, a1_c=cin // 2, backend=1, **kw), fl)


def conv_dgrad(cin, cout, R):
    g = b(B, R, cout)
    w = b(9, 4 * cin, cout)
    out = torch.empty(B, R + 8, 4 * cin, device=dev, dtype=torch.bfloat16)
    taps = E.tap_ranges("conv_dgrad", cin, cout, 4 * cin)
    fl = E._tap_flops(taps, -4, 4, 0, 4 * cin, (R + 8) * B)
    timeit("conv_dgrad %d<-%d R=%d" % (cin, cout, R),
           lambda: E.run_f(g, None, R, 0, SG_BF16, w, SG_BF16, cout, 4 * cin, taps, out, SG_BF16, R, 4, -4, R + 4, B,
                           backend=1), fl)


def conv_wgrad(cin, cout, R):
    g = b(B, R, cout)
    a = b(B, R + 8, 4 * cin)
    dw = torch.zeros(9, cout, 4 * cin, device=dev)
    taps = E.tap_ranges("conv_fwd", cin, 4 * cin, cout)
    fl = E._tap_flops(taps, -4, 4, 0, cout, R * B)
    nt = 9 * (cout // 128) * max(1, 4 * cin // 256)
    ks = E.wgrad_ksplit(B * R, nt)
    timeit("conv_wgrad %d->%d R=%d ks=%d" % (cin, cout, R, ks),
           lambda: E.run_w(g, R, SG_BF16, a, None, R, 4, SG_BF16, 4 * cin, cout, taps, dw, B, ksplit=ks, backend=1), fl)


def wave0(out2_halo=None):
    """The waveform-end layer as it runs in the step: single-tap GEMM over the 64-column im2col (K = 64, N = 64).
    out2_halo None: the Discriminator's enc0 (one output); 16: the Generator's enc0 with its fused out2."""
    col = h(B, 4096, 64)
    w = h(1, 64, 64)
    bias = torch.randn(64, device=dev)
    out = torch.empty(B, 4096, 64, device=dev, dtype=torch.float16)
    taps = E.tap_ranges("full", 0, 64, 64)
    fl = 2.0 * B * 4096 * 64 * 64
    kw = _out2(4096, 64, out2_halo)
    timeit("wave0 im2col-GEMM 64x64 R=4096%s" % ("" if out2_halo is None else " out2 halo %d" % out2_halo),
           lambda: E.run_f(col, None, 4096, 0, SG_F16, w, SG_F16, 64, 64, taps, out, SG_F16, 4096, 0, 0, 4096, B,
                           bias=bias, bias_mod=64, d_lo=0, d_hi=0, w_tap0=4, backend=1, **kw), fl)


def dump_timeline(name):
    """SEGAN_B200_DEBUG bit 20: per-CTA phase stamps of the LAST tapgemm_f_tc launch (sg_debug_timeline)."""
    import ctypes as C
    from segan_pytorch_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    buf = (C.c_uint64 * (160 * 32))()
    lib.sg_debug_timeline.argtypes = [C.c_void_p, C.c_int]
    n = lib.sg_debug_timeline(buf, 160 * 32)
    rows = []
    for cta in range(160):
        w = [buf[cta * 32 + i] for i in range(32)]
        w = [x for x in w if x]
        if w:
            rows.append((cta, w))
    if not rows:
        print("no timeline recorded")
        return
    t0 = min(w[0] & ~(1 << 63) for _, w in rows)
    print("# %s timeline (us since the earliest CTA start): cta: start | per piece (acc ready, epilogue done, *finisher done) | exit" % name)
    ends = []
    for cta, w in rows:
        vals = ["%s%.1f" % ("*" if x >> 63 else "", ((x & ~(1 << 63)) - t0) / 1e3) for x in w]
        ends.append(((w[-1] & ~(1 << 63)) - t0) / 1e3)
        if cta < 32 or cta % 16 == 0:
            print("cta %3d: %s" % (cta, " ".join(vals)))
    ends.sort()
    print("exit times us: min %.1f median %.1f max %.1f" % (ends[0], ends[len(ends) // 2], ends[-1]))


ONE = {"wave0": wave0, "denc0": wave0, "genc0": lambda: wave0(16),
       "enc1": lambda: conv_fwd(64, 128, 1024), "genc1": lambda: conv_fwd(64, 128, 1024, 16),
       "enc3": lambda: conv_fwd(256, 512, 64), "gdec1": lambda: deconv_fwd(1024, 256, 64, out2=True),
       "enc4": lambda: conv_fwd(512, 1024, 16), "dec1": lambda: deconv_fwd(1024, 256, 64),
       "dgrad3": lambda: conv_dgrad(256, 512, 64), "wgrad3": lambda: conv_wgrad(256, 512, 64),
       "wgrad4": lambda: conv_wgrad(512, 1024, 16)}

if __name__ == "__main__":
    if COMPARE == "one":                # a single shape (ncu captures): python tools/prof_tapgemm.py 300 2 one enc3
        COMPARE = ""
        for name in sys.argv[4:]:
            ONE[name]()
            if int(os.environ.get("SEGAN_B200_DEBUG", "0")) & (1 << 20):
                dump_timeline(name)
        sys.exit(0)
    if COMPARE == "streamk":
        for fn, args in ((conv_fwd, (64, 128, 1024)), (conv_fwd, (128, 256, 256)), (conv_fwd, (256, 512, 64)),
                         (conv_fwd, (512, 1024, 16)), (deconv_fwd, (2048, 512, 16)), (deconv_fwd, (1024, 256, 64)),
                         (deconv_fwd, (512, 128, 256)), (deconv_fwd, (256, 64, 1024)), (conv_dgrad, (512, 1024, 16)),
                         (conv_dgrad, (256, 512, 64)), (conv_dgrad, (128, 256, 256)), (conv_dgrad, (64, 128, 1024))):
            fn(*args)
        sys.exit(0)
    wave0()
    wave0(16)
    conv_fwd(64, 128, 1024)
    conv_fwd(64, 128, 1024, 16)
    conv_fwd(128, 256, 256)
    conv_fwd(256, 512, 64)
    conv_fwd(512, 1024, 16)
    deconv_fwd(2048, 512, 16)
    deconv_fwd(1024, 256, 64, out2=True)
    deconv_fwd(1024, 256, 64)
    deconv_fwd(512, 128, 256)
    deconv_fwd(256, 64, 1024)
    conv_dgrad(512, 1024, 16)
    conv_dgrad(256, 512, 64)
    conv_dgrad(128, 256, 256)
    conv_dgrad(64, 128, 1024)
    conv_wgrad(64, 128, 1024)
    conv_wgrad(128, 256, 256)
    conv_wgrad(256, 512, 64)
    conv_wgrad(512, 1024, 16)
