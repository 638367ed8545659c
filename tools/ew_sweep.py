"""Sweeps the streaming-kernel variants (sg_set_ew_variant) of the HBM-bound glue kernels on the
SEGAN+ layer shapes at batch 300 and prints CUDA-event times and effective GB/s (algorithmic bytes:
every tensor read or written once).  Optionally co-runs a tap-GEMM on a second stream to measure
the overlapped rate (`--with-gemm`).

    python tools/ew_sweep.py [--batch 300] [--rep 10] [--with-gemm] > profiles/ew_sweep.txt
"""
import argparse
import sys

import torch

sys.path.insert(0, ".")
from segan_pytorch_b200 import _lib, engine as E          # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16       # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=300)
ap.add_argument("--rep", type=int, default=10)
ap.add_argument("--with-gemm", action="store_true")
ap.add_argument("--default-only", action="store_true", help="only the built-in variant of each kernel (ncu captures)")
ap.add_argument("--shapes", type=int, default=5, help="first N layer shapes")
args = ap.parse_args()
B, REP = args.batch, args.rep
dev = "cuda"
_p, _stream = E._p, E._stream
lib = _lib.load()

SHAPES = [(64, 4096), (128, 1024), (256, 256), (512, 64), (1024, 16)]      # (C, L) of enc0..enc4
# (vec, unroll, cap) per kernel family (kind 1 act_fwd, 2 bn_stats, 3 bwd_reduce, 4 bwd_apply; for the backward
# kinds vec 8 = tiled kernel, vec 4 = generic kernel; vec 16 = the TMA-staged kernels of stream_ew.cu)
VARIANTS = {
    1: [(8, 4, 4), (8, 4, 2), (16, 2, 2)],
    2: [(4, 4, 3), (4, 8, 3), (8, 4, 2), (16, 2, 2)],
    3: [(8, 2, 2), (8, 4, 2), (16, 2, 2)],
    4: [(8, 2, 2), (8, 2, 4), (8, 4, 2), (16, 2, 2)],
}
if args.default_only:
    VARIANTS = {1: [(8, 4, 2)], 2: [(4, 4, 3)], 3: [(8, 2, 2)], 4: [(8, 2, 4)]}      # elementwise.cu g_ew
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, side_fn=None):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    side = torch.cuda.Stream() if side_fn is not None else None
    for _ in range(REP):
        flush.zero_()                                   # > L2: every repetition streams from HBM
        if side is not None:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                side_fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        tot += s.elapsed_time(e)
    return tot / REP


def gemm_side():
    """A dense conv-dgrad tap-GEMM (enc3, 0.2 ms) to co-run with the streaming kernel."""
    cin, cout, R = 256, 512, 64
    g = (torch.randn(B, R, cout, device=dev) * 0.5).bfloat16()
    w = (torch.randn(9, 4 * cin, cout, device=dev) * 0.05).bfloat16()
    out = torch.empty(B, R + 8, 4 * cin, device=dev, dtype=torch.bfloat16)
    taps = E.tap_ranges("conv_dgrad", cin, cout, 4 * cin)

    def run():
        for _ in range(2):
            E.run_f(g, None, R, 0, SG_BF16, w, SG_BF16, cout, 4 * cin, taps, out, SG_BF16, R, 4, -4, R + 4, B, backend=1)
    return run


side_fn = gemm_side() if args.with_gemm else None
print("# batch %d, rep %d, with_gemm %s" % (B, REP, args.with_gemm))
# calibration: plain device copy of the largest activation
x = torch.empty(B, 4096, 64, dtype=torch.float16, device=dev).normal_()
y = torch.empty_like(x)
ms = timeit(lambda: y.copy_(x))
print("copy 157MB->157MB: %.1f us  %.0f GB/s" % (ms * 1e3, 2 * x.numel() * 2 / ms / 1e6))

for C_, L in SHAPES[:args.shapes]:
    halo = 16 if L >= 64 else 0
    roll = 3 if halo else 0
    a = torch.empty(B, L, C_, dtype=torch.float16, device=dev).normal_()
    gh = torch.empty(B, L + 2 * halo, C_, dtype=torch.bfloat16, device=dev).normal_()
    gadd = torch.empty(B, L, 2 * C_, dtype=torch.bfloat16, device=dev).normal_()
    h = torch.empty(B, L + 2 * halo, C_, dtype=torch.float16, device=dev)
    hb = torch.empty(B, L + 2 * halo, C_, dtype=torch.bfloat16, device=dev)
    ga = torch.empty(B, L, C_, dtype=torch.bfloat16, device=dev)
    ss = torch.randn(2, C_, device=dev)
    mi = torch.randn(2, C_, device=dev).abs() + 0.5
    slope = torch.rand(C_, device=dev) * 0.2
    stats = torch.zeros(8, 2, C_, dtype=torch.float64, device=dev)
    red = torch.zeros(8, 3, C_, dtype=torch.float64, device=dev)
    gadd_ptr = E.C.c_void_p(gadd.data_ptr() + 2 * C_)
    n = B * L * C_ * 2          # bytes of one exact-geometry 16-bit tensor
    nh = B * (L + 2 * halo) * C_ * 2
    kernels = {
        "bn_stats": (2, lambda: _lib.call("sg_bn_stats", _p(a), SG_F16, B * L, C_, _p(stats), _stream()), n),
        "act_fwd(D: h+twin)": (1, lambda: _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(slope), 1, roll, None, halo,
                                                 _p(h), _p(hb), None, _stream()), n + 2 * nh),
        "act_fwd(D3: h)": (1, lambda: _lib.call("sg_act_fwd", _p(a), SG_F16, B, L, C_, _p(ss), _p(slope), 1, roll, None, halo,
                                             _p(h), None, None, _stream()), n + nh),
        "bwd_reduce(D)": (3, lambda: _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, roll, None, None, 0, _p(a), SG_F16, B, L, C_,
                                            _p(ss), _p(mi), _p(slope), 1, _p(red), None, _stream()), n + nh),
        "bwd_apply(D)": (4, lambda: _lib.call("sg_act_bwd_apply", _p(gh), C_, halo, roll, None, None, 0, _p(a), SG_F16, B, L, C_,
                                           _p(ss), _p(mi), _p(slope), 1, _p(red), 1, _p(ga), _stream()), 2 * n + nh),
        "bwd_reduce(G enc: +skip,+out)": (3, lambda: _lib.call("sg_act_bwd_reduce", _p(gh), C_, halo, 0, None, gadd_ptr, 2 * C_, _p(a),
                                                            SG_F16, B, L, C_, None, None, _p(slope), 1, _p(red), _p(ga),
                                                            _stream()), 3 * n + nh),
    }
    for kname, (kind, fn, nbytes) in kernels.items():
        row = []
        for v in VARIANTS[kind]:
            assert lib.sg_set_ew_variant(kind, *v) == 0
            ms = timeit(fn, side_fn)
            row.append((ms, v))
        best = min(row)
        print("C=%4d L=%4d %-30s %s" % (C_, L, kname, "  ".join(
            "%d,%d,%d:%.0fus/%.0fGB/s" % (v + (ms * 1e3, nbytes / ms / 1e6)) for ms, v in row)))
        print("    best %s  %.1f us  %.0f GB/s" % (best[1], best[0] * 1e3, nbytes / best[0] / 1e6))
    sys.stdout.flush()
