"""Host-side orchestration of the H100 kernels for the SEGAN+ Generator and Discriminator.

PyTorch is used for device memory (caching allocator), streams and parameter storage only; every
FLOP of the hot path runs in libsegan_b200.so through the C ABI (segan_pytorch_b200._lib).

Layer geometry follows the reference (file:line into santi-pdp/segan_pytorch):
  encoder block  = reflect-pad(k//2-1,k//2) -> Conv1d(k,s4) -> [BatchNorm1d] -> PReLU   segan/models/modules.py:91-105
  decoder block  = ConvTranspose1d(k,s4,p=(k-4)//2)[:-1 if k odd] -> PReLU | Tanh     segan/models/modules.py:135-141
                   (k = 31 in SEGAN+; every width 4 <= k <= 32 is served, see kwidth_served)
  G wiring       = 5 enc -> cat(z, h) -> 5 x (cat(h, alpha*skip), dec)              segan/models/generator.py:180-230
                   (no_z: h alone into dec 0; skip=False: every dec block reads h alone)
  D wiring       = 5 x (phase shift, enc with BN) -> FC 16384-256-128-1             segan/models/discriminator.py:150-194

HBM layouts are described in include/segan_b200.h and DESIGN.md.
"""
import ctypes as C
import math
import os

import torch

from . import _lib
from ._lib import (ACT_NONE, ACT_PRELU, BACKEND_FFMA, BACKEND_TCGEN05, SG_BF16, SG_DHEAD_CONV, SG_DHEAD_GAVG,
                   SG_DHEAD_GMAX, SG_DHEAD_MLP, SG_F16, SG_F32, TapGemmF, TapGemmW)

# Kernel widths of the stride-4 convs and transposed convs: activations are rows of 4 positions with a 16-position
# halo, so a width-k layer is a 9-tap (d = -4..4) GEMM over those rows for every k <= 35.  The bound 32 is the
# waveform-end layers' im2col (32 columns per input channel); below 4 the reference's transposed conv does not give
# 4 * Lin samples, so its skip concat fails.
KW_MIN, KW_MAX = 4, 32


def kwidth_served(k):
    return isinstance(k, int) and not isinstance(k, bool) and KW_MIN <= k <= KW_MAX


def conv_offset(k):
    """Left reflect pad of a width-k encoder conv (modules.py:94-97): tap index = 4d + p + conv_offset(k)."""
    return k // 2 - 1


def deconv_padding(k):
    """Padding of a width-k stride-4 ConvTranspose1d (modules.py:116): tap index = -4d + r + deconv_padding(k)."""
    return max(0, (4 - k) // -2)


# Discriminator pool_type -> head kernel selector of sg_dhead_fwd / _bwd ('none' runs fc.0 + sg_fc_tail instead)
DHEAD_KINDS = {"conv": SG_DHEAD_CONV, "gmax": SG_DHEAD_GMAX, "gavg": SG_DHEAD_GAVG, "mlp": SG_DHEAD_MLP}


def wave_on_tensor_cores():
    """Waveform-end layers through im2col + tensor-core tap-GEMMs (default) or the CUDA-core kernels."""
    return os.environ.get("SEGAN_B200_WAVE", "tc").lower() not in ("cuda", "ffma", "0")


def wave_col_weights(w, dev):
    """Conv1d weight [64][cin][k] -> single-tap operand Wcol[co][ci*32 + j] = W[co][ci][j] for j < k (fp32, [64][64])."""
    wc = torch.zeros(w.shape[0], 2, 32, dtype=torch.float32, device=dev)
    wc[:, :w.shape[1], :w.shape[2]] = w
    return wc.view(w.shape[0], 64)


_DEC_LAST_KIDX = {}


def dec_last_tap_index(dev, k=31):
    """jj = (d+4)*4 + r  ->  j = -4d + r + deconv_padding(k) (or -1 outside [0, k)): column order of the last decoder
    block's GEMM for a width-k transposed conv."""
    key = (dev, k)
    if key not in _DEC_LAST_KIDX:
        idx = []
        for jj in range(64):
            d, r = jj // 4 - 4, jj % 4
            j = -4 * d + r + deconv_padding(k)
            idx.append(j if (jj < 36 and 0 <= j < k) else -1)
        _DEC_LAST_KIDX[key] = torch.tensor(idx, device=dev)
    return _DEC_LAST_KIDX[key]


def default_backend():
    v = os.environ.get("SEGAN_B200_BACKEND", "tcgen05").lower()
    return BACKEND_FFMA if v in ("ffma", "ref", "0") else BACKEND_TCGEN05


def _p(t):
    if t is None or isinstance(t, C.c_void_p):
        return t
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# --------------------------------------------------------------------------------------------
# side streams: the HBM-bound glue kernels run concurrently with the tensor-bound tap-GEMMs
# --------------------------------------------------------------------------------------------
# A persistent tap-GEMM CTA leaves ~45 K registers and ~29 KB of shared memory per SM unused, and
# the tensor pipe does not compete with HBM streaming: the weight-gradient chain (wgrad GEMM +
# unpack) of a backward pass therefore runs on side stream 0 while the data-gradient chain (dgrad
# GEMM -> activation backward) continues on the caller's stream, and the Generator forward of a
# train step runs on side stream 1 next to the Discriminator's real pass.  SEGAN_B200_OVERLAP=0
# (or engine.OVERLAP = False) serialises everything on the caller's stream (bench.py does that for
# its per-call profile so that per-kernel times are exclusive).
OVERLAP = os.environ.get("SEGAN_B200_OVERLAP", "1").lower() not in ("0", "off", "no", "false")
# CUDA graphs: SEGAN.train_step captures the whole step after GRAPH_WARMUP eager steps of the same shape
# and replays it (SEGAN_B200_GRAPH=0 keeps the eager schedule).
GRAPHS = os.environ.get("SEGAN_B200_GRAPH", "1").lower() not in ("0", "off", "no", "false")
GRAPH_WARMUP = 2
_SIDE = {}


def side_stream(dev, which):
    """Side stream `which` of device `dev`, or None when overlap is disabled."""
    if not OVERLAP:
        return None
    key = (torch.device(dev).index if torch.device(dev).index is not None else torch.cuda.current_device(), which)
    st = _SIDE.get(key)
    if st is None:
        st = torch.cuda.Stream(device=key[0])
        _SIDE[key] = st
    return st


class on_side(object):
    """`with on_side(side):` enqueues the enclosed launches on `side`, ordered after everything
    enqueued so far on the current stream (fork).  side=None: plain in-line execution."""

    def __init__(self, side):
        self.side = side
        self.ctx = None

    def __enter__(self):
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream())
            self.ctx = torch.cuda.stream(self.side)
            self.ctx.__enter__()
        return self

    def __exit__(self, *a):
        if self.ctx is not None:
            self.ctx.__exit__(*a)
        return False


def join_side(side):
    """The current stream waits for everything enqueued on `side` (join)."""
    if side is not None:
        torch.cuda.current_stream().wait_stream(side)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.SeganB200Error(
                "segan_pytorch_b200 runs on H100 GPUs only: got a CPU tensor (there is no CPU path; "
                "the CPU restatement under oracle/ is test infrastructure)")


# --------------------------------------------------------------------------------------------
# structural-zero tap ranges of the four packed weight layouts
# --------------------------------------------------------------------------------------------
def _phase_span(kind, d, k):
    """Stride phases (lo, hi inclusive) that forward tap d of a width-k layer reads, or None: conv phase p holds tap
    index 4d + p + conv_offset(k), deconv phase r holds -4d + r + deconv_padding(k); valid indices are [0, k)."""
    if kind == "conv":
        ph = [p for p in range(4) if 0 <= 4 * d + p + conv_offset(k) < k]
    else:
        ph = [r for r in range(4) if 0 <= -4 * d + r + deconv_padding(k) < k]
    return (ph[0], ph[-1]) if ph else None


def tap_ranges(kind, c, kc, nc, k=31):
    """kind: conv_fwd | conv_dgrad | deconv_fwd | deconv_dgrad | full ; c = the channel count whose
    four stride phases are interleaved (Cin for conv, Cout for deconv); k = the kernel width.  Blocks of phases a tap
    does not read are structurally zero in the packed weight and are skipped; a tap that reads none gets an empty
    range (tap_span gives the d_lo, d_hi of the others).  k = 31: d=-4 reads conv phases {2,3} / deconv phases
    {0,1}, d=+4 conv phase 0 / deconv phase 3."""
    k_lo, k_hi, n_lo, n_hi = [0] * 9, [kc] * 9, [0] * 9, [nc] * 9
    if kind == "full":
        return k_lo, k_hi, n_lo, n_hi
    if kind not in ("conv_fwd", "conv_dgrad", "deconv_fwd", "deconv_dgrad"):
        raise ValueError(kind)
    base, form = kind.split("_")
    # the data-gradient operand's tap d is the transpose of the forward tap -d: its phases move to the other side
    on_k = (base == "conv") == (form == "fwd")          # conv_fwd / deconv_dgrad: phases are K; else N
    lo, hi = (k_lo, k_hi) if on_k else (n_lo, n_hi)
    for i in range(9):
        d = i - 4 if form == "fwd" else 4 - i
        span = _phase_span(base, d, k)
        if span is None:
            lo[i], hi[i] = 0, 0
        elif span != (0, 3):
            lo[i], hi[i] = span[0] * c, (span[1] + 1) * c
    return k_lo, k_hi, n_lo, n_hi


def tap_span(taps):
    """(d_lo, d_hi) of the non-empty taps of a tap table (they are contiguous for every width >= 4)."""
    live = [i - 4 for i in range(9) if taps[1][i] > taps[0][i] and taps[3][i] > taps[2][i]]
    return live[0], live[-1]


def dgrad_span(fwd_taps):
    """(d_lo, d_hi) of a layer's data-gradient tap-GEMM from its forward tap table: data-gradient tap d is the
    transpose of forward tap -d, so the span is the forward span mirrored (= tap_span of the data-gradient table)."""
    d_lo, d_hi = tap_span(fwd_taps)
    return -d_hi, -d_lo


# optional live profiling (bench.py): list of (kind, start_event, end_event, algorithmic_flops)
PROFILE = None


def _tap_flops(taps, d_lo, d_hi, n_lo, n_hi, rows):
    f = 0
    for d in range(d_lo, d_hi + 1):
        i = d + 4
        nn = max(0, min(n_hi, taps[3][i]) - max(n_lo, taps[2][i]))
        f += 2 * rows * nn * (taps[1][i] - taps[0][i])
    return f


class _Prof(object):
    def __init__(self, kind, flops):
        self.kind, self.flops = kind, flops

    def __enter__(self):
        if PROFILE is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *a):
        if PROFILE is not None:
            self.e.record()
            PROFILE.append((self.kind, self.s, self.e, self.flops))
        return False


NUM_SMS = 132      # H100 SXM
# BatchNorm statistics in the conv epilogue (sg_tapgemm_f.bn_stats).  Off by default: the D conv GEMMs with short K
# are epilogue-bound, so the extra epilogue work can cost what the separate bn_stats launches cost; the fused path is
# kept tested but not used (not measured to pay off on H100).
FUSE_BN_STATS = os.environ.get("SEGAN_B200_FUSE_BN_STATS", "0").lower() not in ("0", "off", "no", "false")
# Off by default: a tile's A-operand fill does not shrink with its width, so a narrow-tile tail costs about as much
# as the wave it replaces (not measured to pay off on H100).
SPLIT_WAVES = os.environ.get("SEGAN_B200_WAVE_SPLIT", "0").lower() not in ("0", "off", "no", "false")


def _f_tiling(rows_m, batch, ncols, tile_n=0):
    """Tiling model of the optional wave-split planners below, in units of two 128-row M tiles ("pairs", NUM_SMS // 2
    of them per wave): (TB, m_tiles_per_b, TN, pair tiles, batch granularity of a pair-aligned group)."""
    if rows_m >= 128:
        tb, mpb = 1, (rows_m + 127) // 128
    else:
        tb, mpb = max(1, min(128 // rows_m, batch, 256)), 1
    tn = 256 if ncols % 256 == 0 else (128 if ncols % 128 == 0 else 64)
    if tile_n in (64, 128, 256) and ncols % tile_n == 0 and tile_n < tn:
        tn = tile_n
    m_tiles = mpb * ((batch + tb - 1) // tb)
    tiles = ((m_tiles + 1) // 2) * (ncols // tn)
    gran = 2 * tb if mpb % 2 else tb          # batch elements per group of whole CTA pairs
    return tb, mpb, tn, tiles, gran


def _plan_f_split(rows_m, batch, ncols):
    """Wave quantisation: batch 300 puts many layers just over a whole number of waves (e.g. 4.05 waves -> 5).  Returns (B1, tail_tile_n): the launch is split into the first B1 batch
    elements as whole waves of full-width tiles and the rest as one short wave of narrow tiles; (batch, 0)
    when splitting does not pay."""
    pairs_hw = NUM_SMS // 2
    tb, mpb, tn, tiles, gran = _f_tiling(rows_m, batch, ncols)
    waves = -(-tiles // pairs_hw)
    if tiles <= pairs_hw or tiles % pairs_hw == 0 or waves > 12:
        return batch, 0
    per_gran = _f_tiling(rows_m, gran, ncols)[3]              # tiles of one pair-aligned batch group
    full_tiles = (tiles // pairs_hw) * pairs_hw
    b1 = min(batch, (full_tiles // per_gran) * gran)
    if b1 <= 0 or b1 >= batch:
        return batch, 0
    best = None
    for t, penalty in ((64, 1.3), (128, 1.15), (256, 1.0)):
        if ncols % t or t > tn:
            continue
        tt = _f_tiling(rows_m, batch - b1, ncols, t)[3]
        cost = -(-tt // pairs_hw) * (t / float(tn)) * penalty
        if best is None or cost < best[0]:
            best = (cost, t)
    head_waves = -(-_f_tiling(rows_m, b1, ncols)[3] // pairs_hw)
    if head_waves + best[0] + 0.05 >= waves * 0.97:
        return batch, 0
    return b1, (best[1] if best[1] < tn else 0)


# Off by default: bit-correct, but the two extra launches (tail GEMM + convert) and the tail kernel's own prologue
# can cost more than the partial wave they remove (not measured to pay off on H100).
SPLITK_TAIL = os.environ.get("SEGAN_B200_SPLITK_TAIL", "0").lower() not in ("0", "off", "no", "false")
# PReLU (+ reflect halo) of the Generator's blocks in the tap-GEMM epilogue (sg_tapgemm_f.out2 / .slope)
FUSE_ACT = os.environ.get("SEGAN_B200_FUSE_ACT", "1").lower() not in ("0", "off", "no", "false")


def _plan_f_tail_splitk(rows_m, batch, ncols, ksteps):
    """Split-K tail against wave quantisation: (B1, s).  The first B1 batch elements run as whole waves; the
    leftover tiles (fewer than half a wave) run as a second launch whose k-steps are split s ways over the idle
    CTA pairs, accumulating fp32 partial sums that a small kernel converts.  Unlike narrow tiles, a split's
    operand fill shrinks with its work.  (batch, 0) when it does not apply."""
    pairs_hw = NUM_SMS // 2
    tb, mpb, tn, tiles, gran = _f_tiling(rows_m, batch, ncols)
    waves = -(-tiles // pairs_hw)
    rem = tiles % pairs_hw
    if tiles <= pairs_hw or rem == 0 or waves > 10:
        return batch, 0
    per_gran = _f_tiling(rows_m, gran, ncols)[3]
    full_tiles = (tiles // pairs_hw) * pairs_hw
    b1 = min(batch, (full_tiles // per_gran) * gran)
    if b1 <= 0 or b1 >= batch:
        return batch, 0
    tail_tiles = _f_tiling(rows_m, batch - b1, ncols)[3]
    s = min(pairs_hw // max(1, tail_tiles), ksteps // 4, 32)
    if s < 2:
        return batch, 0
    return b1, s


_SK_WS = {}
STREAM_K = os.environ.get("SEGAN_B200_STREAMK", "1").lower() not in ("0", "off", "no", "false")


def sk_workspace(dev):
    """Stream-K workspace of the CURRENT stream (sg_tapgemm_f.sk_ws): zero-filled once, left zeroed by every launch;
    one per stream because launches on different streams may run concurrently."""
    if not STREAM_K:
        return None
    idx = torch.device(dev).index
    key = (torch.cuda.current_device() if idx is None else idx, torch.cuda.current_stream().cuda_stream)
    ws = _SK_WS.get(key)
    if ws is None:
        ws = _SK_WS[key] = torch.zeros(int(_lib.load().sg_tapgemm_f_workspace_bytes()), dtype=torch.uint8, device=dev)
    return ws


def f_pair_tiles(rows_m, batch):
    """M tiles of a form-F launch (mirror of tapgemm_f_tc_launch); the fused-activation path is used from two on."""
    tb, mpb = _f_tiling(rows_m, batch, 64)[:2]
    return mpb * ((batch + tb - 1) // tb)


def run_f(a0, a1, a_rows, a_halo, a_dtype, w, w_dtype, kc, nc, taps, out, out_dtype, out_rows, out_halo,
          m_lo, m_hi, batch, bias=None, bias_mod=0, n_lo=0, n_hi=None, d_lo=-4, d_hi=4, w_tap0=0,
          out_ld=0, out_col0=0, ksplit=1, backend=None, a0_c=None, a1_c=0, stats=None,
          out2=None, out2_halo=0, slope=None, slope_mod=0):
    """stats: optional [SL][2][nc] float64 tensor: BatchNorm batch statistics of the output, fused into the
    epilogue of the tensor-core kernel (see sg_tapgemm_f.bn_stats).
    slope (+ out2): PReLU fused into the epilogue -- into `out2` (with reflect halo) next to the raw `out`, or,
    without out2, into `out` itself (see sg_tapgemm_f.out2)."""
    n_hi = nc if n_hi is None else n_hi
    a0_c = kc if a0_c is None else a0_c
    backend = default_backend() if backend is None else backend
    b1, tail_tn, tail_ks = batch, 0, 0
    if backend == BACKEND_TCGEN05 and ksplit == 1 and batch > 1 and stats is None:
        if SPLITK_TAIL and out_dtype != SG_F32 and m_lo == -out_halo and m_hi == out_rows + out_halo:
            ksteps = sum((taps[1][d + 4] - taps[0][d + 4]) // 64 for d in range(d_lo, d_hi + 1))
            b1, tail_ks = _plan_f_tail_splitk(m_hi - m_lo, batch, n_hi - n_lo, ksteps)
        elif SPLIT_WAVES:
            b1, tail_tn = _plan_f_split(m_hi - m_lo, batch, n_hi - n_lo)
    esz = 4 if out_dtype == SG_F32 else 2
    old = (out_ld if out_ld > 0 else nc)
    out_brows = out_rows + 2 * out_halo
    ws = None
    if tail_ks:
        # fp32 workspace with the geometry of the tail's slice of `out` (from the caching allocator: per stream,
        # static inside a captured graph)
        ws = torch.zeros((batch - b1) * out_brows * old, dtype=torch.float32, device=out.device)
    for b_off, nb, tn in ((0, b1, 0), (b1, batch - b1, tail_tn)):
        if nb <= 0:
            continue
        tail = b_off > 0 and tail_ks > 0
        q = TapGemmF()
        a_stride = (a_rows + 2 * a_halo) * 2
        q.a0 = _p(a0) if b_off == 0 else C.c_void_p(a0.data_ptr() + b_off * a_stride * a0_c)
        q.a1 = _p(a1) if (a1 is None or b_off == 0) else C.c_void_p(a1.data_ptr() + b_off * a_stride * a1_c)
        q.a0_c, q.a1_c = a0_c, a1_c
        q.a_rows, q.a_halo, q.a_dtype = a_rows, a_halo, a_dtype
        q.w, q.w_dtype, q.w_tap0 = _p(w), w_dtype, w_tap0
        q.kc, q.nc, q.d_lo, q.d_hi = kc, nc, d_lo, d_hi
        for i in range(9):
            q.tap_k_lo[i], q.tap_k_hi[i], q.tap_n_lo[i], q.tap_n_hi[i] = taps[0][i], taps[1][i], taps[2][i], taps[3][i]
        if tail:
            q.out = _p(ws)
        else:
            q.out = _p(out) if b_off == 0 else C.c_void_p(out.data_ptr() + b_off * out_brows * old * esz)
        q.out_ld, q.out_col0 = out_ld, out_col0
        q.out_dtype, q.out_rows, q.out_halo = (SG_F32 if tail else out_dtype), out_rows, out_halo
        q.m_lo, q.m_hi, q.n_lo, q.n_hi = m_lo, m_hi, n_lo, n_hi
        q.bias, q.bias_mod = _p(bias), bias_mod
        q.batch, q.ksplit = nb, (tail_ks if tail else ksplit)
        q.backend, q.tile_n = backend, tn
        q.bn_stats = _p(stats)
        assert (out2 is None and slope is None) or b1 == batch, "fused activation outputs are not split"
        q.out2, q.out2_halo, q.slope, q.slope_mod = _p(out2), out2_halo, _p(slope), slope_mod
        q.sk_ws = _p(sk_workspace(out.device)) if backend == BACKEND_TCGEN05 else None
        with _Prof("tapgemm_f", _tap_flops(taps, d_lo, d_hi, q.n_lo, q.n_hi, (m_hi - m_lo) * nb)):
            _lib.call("sg_tapgemm_f_run", C.byref(q), _stream())
        if tail:
            # columns the launch wrote: [col_lo, col_lo + n_hi - n_lo) of every row of the slice
            col_lo = out_col0 if out_ld > 0 else n_lo
            _lib.call("sg_convert_f32_rows", _p(ws), C.c_void_p(out.data_ptr() + b_off * out_brows * old * esz),
                      out_dtype, nb * out_brows, old, col_lo, n_hi - n_lo, _stream())


def run_w(g, g_rows, g_dtype, a0, a1, a_rows, a_halo, a_dtype, kc, nc, taps, dw, batch, d_lo=-4, d_hi=4,
          dw_tap0=0, ksplit=1, backend=None, a0_c=None, a1_c=0, out_scale=None):
    q = TapGemmW()
    q.out_scale = _p(out_scale)
    q.g, q.g_rows, q.g_dtype = _p(g), g_rows, g_dtype
    q.a0, q.a1 = _p(a0), _p(a1)
    q.a0_c = kc if a0_c is None else a0_c
    q.a1_c = a1_c
    q.a_rows, q.a_halo, q.a_dtype = a_rows, a_halo, a_dtype
    q.kc, q.nc, q.d_lo, q.d_hi = kc, nc, d_lo, d_hi
    for i in range(9):
        q.tap_k_lo[i], q.tap_k_hi[i], q.tap_n_lo[i], q.tap_n_hi[i] = taps[0][i], taps[1][i], taps[2][i], taps[3][i]
    q.dw, q.dw_tap0 = _p(dw), dw_tap0
    q.batch, q.ksplit = batch, ksplit
    q.backend = default_backend() if backend is None else backend
    with _Prof("tapgemm_w", _tap_flops(taps, d_lo, d_hi, 0, nc, g_rows * batch)):
        _lib.call("sg_tapgemm_w_run", C.byref(q), _stream())


def wgrad_ksplit(total_positions, n_tiles, taps=None, kc=None, nc=None, d_lo=-4, d_hi=4):
    """Position-range splits of a weight-gradient tap-GEMM.  With the tap table the number of non-empty
    (tap, n, kc) tiles is counted exactly (mirror of tapgemm_w_tc's decode()) and the split count is the
    one that minimises waves / splits over the NUM_SMS SMs (265 tiles = 2.008 waves would run as 3); without
    it: about two waves."""
    steps = max(1, total_positions // 64)
    if taps is None:
        want = max(1, (2 * NUM_SMS + n_tiles - 1) // max(1, n_tiles))
        return int(max(1, min(want, steps)))
    tk = 256 if kc >= 256 else kc
    valid = 0
    for d in range(d_lo, d_hi + 1):
        i = d + 4
        for n0 in range(0, nc, 128):
            if n0 + 128 <= taps[2][i] or n0 >= taps[3][i]:
                continue
            for k0 in range(0, kc, tk):
                if k0 + tk <= taps[0][i] or k0 >= taps[1][i]:
                    continue
                valid += 1
    valid = max(1, valid)
    # time ~ waves / ks (a tile's work shrinks with the split count); small preferences: at least ~1.5 waves
    # (so a CTA's epilogue overlaps its next tile) and fewer splits (every split adds a pass of fp32 atomics)
    best = None
    for ks in range(1, min(steps, max(1, -(-8 * NUM_SMS // valid))) + 1):
        tiles = valid * ks
        cost = (-(-tiles // NUM_SMS)) / float(ks)
        if tiles < 1.5 * NUM_SMS:
            cost *= 1.15
        cost *= 1.0 + 0.004 * ks
        if best is None or cost < best[0] - 1e-12:
            best = (cost, ks)
    return best[1]


class _Buffers:
    """Named device buffers, reused across steps (keyed by name; re-allocated on shape change)."""

    def __init__(self):
        self.t = {}

    def get(self, name, shape, dtype, device, zero=False):
        cur = self.t.get(name)
        shape = tuple(int(s) for s in shape)
        if cur is None or tuple(cur.shape) != shape or cur.dtype != dtype or cur.device != device:
            cur = torch.empty(shape, dtype=dtype, device=device)
            self.t[name] = cur
            if not zero:
                cur.zero_()       # never expose uninitialised halos
        if zero:
            cur.zero_()
        return cur


def stat_arena(buf, name, shapes, device):
    """One zero-fill for all per-channel statistic buffers of a pass: views of shapes[i] (float64) into a
    single tensor that is zeroed once (each buffer used to get its own tiny fill launch on the critical chain)."""
    sizes = [int(torch.Size(sh).numel()) for sh in shapes]
    flat = buf.get(name, (sum(sizes),), torch.float64, device, zero=True)
    out, off = [], 0
    for sh, n in zip(shapes, sizes):
        out.append(flat[off:off + n].view(sh))
        off += n
    return out


F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
SL = 8   # SG_STAT_SLICES: statistic buffers are [SL][n_stats][C]; the statistic is the sum over slices

# ---- gradient precision -------------------------------------------------------------------------
# Gradient tensors are fp16 (11 significant bits) with a static loss scale: the loss gradients are multiplied by
# LOSS_SCALE at their source (sg_fc_tail_bwd / sg_l1_loss_bwd), every gradient tensor and the flat parameter-
# gradient buckets carry the factor, and the optimiser kernels divide it out (their grad_scale argument).  16-bit
# stores saturate at +-65504.  With fp16 gradients the weight-gradient tap-GEMMs read the forward activations
# directly (same 16-bit format on both wgmma operands), so no bf16 twins are written.
# SEGAN_B200_GRAD_DTYPE=bf16 (or set_grad_dtype('bf16')) restores round 1's bf16 gradient tensors + twins
# (loss scale 1): the measured control for the parity gates (DESIGN.md section 4).
if os.environ.get("SEGAN_B200_GRAD_DTYPE", "f16").lower() == "bf16":     # _lib.load() applies the same variable
    GT, GS, LOSS_SCALE = BF16, SG_BF16, 1.0
else:
    GT, GS, LOSS_SCALE = F16, SG_F16, float(os.environ.get("SEGAN_B200_LOSS_SCALE", "1024"))


def set_grad_dtype(kind, loss_scale=None):
    """kind: 'f16' | 'bf16'.  Affects engines built afterwards (packed dgrad operands are re-made on the next pack)."""
    global GT, GS, LOSS_SCALE
    if kind in ("bf16", BF16):
        GT, GS = BF16, SG_BF16
        LOSS_SCALE = 1.0 if loss_scale is None else float(loss_scale)
    else:
        GT, GS = F16, SG_F16
        LOSS_SCALE = float(os.environ.get("SEGAN_B200_LOSS_SCALE", "1024")) if loss_scale is None else float(loss_scale)
    _lib.load().sg_set_grad_dtype(GS)


def twins_or_alias(alias, twins):
    """A forward pass that a weight-gradient computation will follow (its saved activations feed tapgemm_w)."""
    return bool(alias or twins)


def grad_twins():
    """bf16 gradient tensors need bf16 copies of the forward activations for the weight-gradient GEMMs."""
    return GS == SG_BF16


class PackedLayer(object):
    """One tap-GEMM layer whose fp32 master, optimiser state and gradient live in the layout of its forward
    operand, M[T][nc][kc] (include/segan_b200.h "Packed-master path").
      kind 0: Conv1d W[cout][cin][kw]          -> M[9][cout][4cin]
      kind 1: ConvTranspose1d W[cin][cout][kw] -> M[9][4cout][cin]   (alpha: GSkip scale of the columns >= alpha_from)
      kind 2: Linear W[nout][C*T]              -> M[1][nout][T*C]"""

    def __init__(self, name, kind, c_out, c_in, t_len, f_key, dg_key, alpha_name=None, tied=False, kw=31):
        """tied (skip_merge='sum', generator.py:72-74): W (hi + alpha*skip) = [W | alpha W] cat(hi, skip) -- the
        layer runs as the two-source concat GEMM over 2*Cin' input channels whose two halves hold the SAME weights:
        `c_in` is the doubled count, import duplicates the parameter, export returns the first half, and the
        gradients of the two halves are summed into both (finish_grads) so the copies never drift apart."""
        self.name, self.kind, self.c_out, self.c_in, self.t_len = name, kind, c_out, c_in, t_len
        self.f_key, self.dg_key, self.alpha_name, self.tied = f_key, dg_key, alpha_name, tied
        self.kw = kw
        if kind == 0:
            self.T, self.nc, self.kc = 9, c_out, 4 * c_in
        elif kind == 1:
            self.T, self.nc, self.kc = 9, 4 * c_out, c_in
        else:
            self.T, self.nc, self.kc = 1, c_out, c_in * t_len
        self.alpha_from = c_in // 2 if alpha_name is not None else 0
        self.numel = self.T * self.nc * self.kc
        self.off = 0


def _tap_pad(kind, k):
    """Left zero pad that places the k taps of a width-k weight in the 36 = 9 x 4 (tap, phase) slots."""
    return 16 - (conv_offset(k) if kind == 0 else deconv_padding(k))


def pack_reference(kind, w, c_out, c_in, t_len, k=31):
    """Reference layout -> packed master layout M[T][nc][kc], as tensor algebra (host-side twin of sg_pack_weights_kw:
    used for CPU-resident modules -- optimiser state dicts, checkpoints -- and as the kernels' cross-check).
    k = kernel width of kinds 0 and 1."""
    if kind == 0:        # M[d+4][co][p*Cin+ci] = W[co][ci][4d+p+conv_offset(k)]
        lp = _tap_pad(0, k)
        wp = torch.nn.functional.pad(w.reshape(c_out, c_in, k), (lp, 36 - k - lp))
        return wp.view(c_out, c_in, 9, 4).permute(2, 0, 3, 1).reshape(9, c_out, 4 * c_in).contiguous()
    if kind == 1:        # M[d+4][r*Cout+co][ci] = W[ci][co][-4d+r+deconv_padding(k)]
        lp = _tap_pad(1, k)
        wp = torch.nn.functional.pad(w.reshape(c_in, c_out, k), (lp, 36 - k - lp))
        return wp.view(c_in, c_out, 9, 4).flip(2).permute(2, 3, 1, 0).reshape(9, 4 * c_out, c_in).contiguous()
    return w.reshape(c_out, c_in, t_len).permute(0, 2, 1).reshape(1, c_out, t_len * c_in).contiguous()


def unpack_reference(kind, m, c_out, c_in, t_len, k=31):
    """Inverse of pack_reference (host-side twin of sg_unpack_wgrad_kw without alpha)."""
    if kind == 0:
        lp = _tap_pad(0, k)
        return m.reshape(9, c_out, 4, c_in).permute(1, 3, 0, 2).reshape(c_out, c_in, 36)[..., lp:lp + k].contiguous()
    if kind == 1:
        lp = _tap_pad(1, k)
        return m.reshape(9, 4, c_out, c_in).permute(3, 2, 0, 1).flip(2).reshape(c_in, c_out, 36)[..., lp:lp + k].contiguous()
    return m.reshape(c_out, t_len, c_in).permute(0, 2, 1).reshape(c_out, c_in * t_len).contiguous()


# --------------------------------------------------------------------------------------------
# convolutional skip connection (GSkip skip_type='conv', generator.py:43-49): Conv1d(C, C, K, padding K//2) on the
# grouped rows [B][L/4][4C] is a forward-form tap-GEMM over the taps d = -D..D (include/segan_b200.h)
# --------------------------------------------------------------------------------------------
def skipconv_served(k):
    """Odd kernel widths up to 33 fit the tap-GEMMs' 9-entry tap table (D <= 4); an even width makes the
    reference's own output one sample too long (padding K//2 on both ends), so it cannot be merged either."""
    return isinstance(k, int) and k >= 1 and k % 2 == 1 and k <= 33


def skipconv_geometry(c, k):
    """(d_lo, d_hi, w_tap0, forward tap table, data-gradient tap table) of the skip conv of C = c channels.  A tap's
    valid ranges are the bounding box of its non-zero C x C blocks (skip_conv.cu's fold kernel clears the same boxes)."""
    p, D = k // 2, (k // 2 + 3) // 4
    fwd = [[0] * 9, [4 * c] * 9, [0] * 9, [4 * c] * 9]
    for d in range(-D, D + 1):
        blocks = [(po, pi) for po in range(4) for pi in range(4) if 0 <= 4 * d + pi - po + p < k]
        pos, pis = [b[0] for b in blocks], [b[1] for b in blocks]
        fwd[0][d + 4], fwd[1][d + 4] = min(pis) * c, (max(pis) + 1) * c
        fwd[2][d + 4], fwd[3][d + 4] = min(pos) * c, (max(pos) + 1) * c
    # data gradient: tap d reads the transpose of the forward tap -d (K and N ranges swap)
    dg = [[fwd[2][8 - i] for i in range(9)], [fwd[3][8 - i] for i in range(9)],
          [fwd[0][8 - i] for i in range(9)], [fwd[1][8 - i] for i in range(9)]]
    return -D, D, 4 - D, fwd, dg


def skipconv_pack_reference(w):
    """Conv1d weight W[C][C][K] -> forward operand W'[2D+1][4C][4C] as tensor algebra (host-side twin of
    sg_skipconv_emit): W'[d + D][(po, co)][(pi, ci)] = W[co][ci][4d + pi - po + K//2], zero outside [0, K)."""
    c, _, k = w.shape
    p, D = k // 2, (k // 2 + 3) // 4
    out = torch.zeros(2 * D + 1, 4, c, 4, c, dtype=w.dtype, device=w.device)
    for d in range(-D, D + 1):
        for po in range(4):
            for pi in range(4):
                t = 4 * d + pi - po + p
                if 0 <= t < k:
                    out[d + D, po, :, pi, :] = w[:, :, t]
    return out.reshape(2 * D + 1, 4 * c, 4 * c)


def skipconv_grouped_reference(a, wp, bias=None):
    """The tap-GEMM the engine runs, on the host: a [B][L][C] (read as [B][L/4][4C]), wp from
    skipconv_pack_reference; rows outside the sequence read as zero.  Returns [B][L][C]."""
    B, L, c = a.shape
    D = (wp.shape[0] - 1) // 2
    ag = torch.nn.functional.pad(a.reshape(B, L // 4, 4 * c), (0, 0, D, D))
    out = torch.zeros(B, L // 4, 4 * c, dtype=a.dtype, device=a.device)
    for d in range(-D, D + 1):
        out += ag[:, D + d:D + d + L // 4] @ wp[d + D].t()
    out = out.reshape(B, L, c)
    return out if bias is None else out + bias


# Gradient buckets are cleared by the optimiser kernels as they read them (sg_rmsprop_step clear_grad): a step
# needs no fill launches.  KEEP_GRADS = True (tests, inspection) leaves the gradients in place after a step; the
# next backward then zeroes the bucket itself.
KEEP_GRADS = os.environ.get("SEGAN_B200_KEEP_GRADS", "0").lower() not in ("0", "off", "no", "false")


class _NetEngine:
    """Shared machinery: ONE fp32 bucket per network holding the packed masters of the tap-GEMM layers followed by
    every other ("small") parameter in reference layout, a gradient bucket of the same layout (the NCCL buffer),
    and the lazily re-emitted 16-bit operands.

    The nn.Parameters of the module keep the reference's names and shapes: small parameters ARE views into the
    bucket; the big weights are reference-layout MIRRORS that are refreshed from the packed master only when
    somebody looks (state_dict(), checkpoints, .to(), grad_of()) and imported into the master when somebody wrote
    them (load_state_dict, init functions: detected through the tensors' version counters)."""

    def __init__(self, module):
        self.module = module
        self.flat = None            # packed masters | small parameters
        self.grad = None
        self.index = {}             # small parameter name -> (offset, numel, shape) in the bucket
        self.layers = []            # PackedLayer descriptors (offsets into the bucket)
        self.by_name = {}
        self.buf = _Buffers()
        self.backend = None
        self._mirror_stale = False  # the packed masters are newer than the reference-layout mirrors
        self._ops_stale = True      # the 16-bit operands are older than the masters / small parameters
        self._seen = None           # version counters of the module's parameters at the last look
        self._grad_dirty = False    # the gradient bucket holds something
        self._alpha_fixed = False   # sg_alpha_grad has been applied to the current gradients

    def packed_layers(self):
        raise NotImplementedError

    # -- parameters -------------------------------------------------------------------------
    def bind(self):
        ps = list(self.module.named_parameters())
        dev = ps[0][1].device
        ok = self.flat is not None and self.flat.device == dev
        if ok:
            for name, p in ps:
                ent = self.index.get(name)
                if ent is not None and p.data_ptr() != self.flat.data_ptr() + 4 * ent[0]:
                    ok = False
                    break
                if ent is None and (p.device != dev or self._mirror_ptr.get(name) != p.data_ptr()):
                    ok = False
                    break
        if not ok:
            self._build(ps, dev)
        return self

    def _build(self, ps, dev):
        """(Re)creates the buckets from the module's parameters (first use, or after .to(device))."""
        self.layers = self.packed_layers()
        self.by_name = {l.name: l for l in self.layers}
        off = 0
        for l in self.layers:
            l.off = off
            off += l.numel
        self.index = {}
        for name, p in ps:
            if name not in self.by_name:
                self.index[name] = (off, p.numel(), tuple(p.shape))
                off += (p.numel() + 3) // 4 * 4                  # 16-byte aligned views
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev)
        # the gradient bucket may carry a gradient-only tail past the parameters (_grad_tail): all-reduced with
        # the gradients, never stepped by the optimiser (it steps flat.numel() elements)
        self.grad = torch.zeros(off + self._grad_tail(), dtype=torch.float32, device=dev)
        self._mirror_ptr = {}
        for name, p in ps:
            p.grad = None
            if name in self.by_name:
                p.data = p.data.contiguous().float()
                self._mirror_ptr[name] = p.data_ptr()
            else:
                o, n, shape = self.index[name]
                self.flat[o:o + n].copy_(p.data.reshape(-1))
                p.data = self.flat[o:o + n].view(shape)
        for l in self.layers:
            self._import(l)
        self._mirror_stale, self._ops_stale = False, True
        self._grad_dirty, self._alpha_fixed = False, False
        self._seen = self._versions()
        if hasattr(self, "sn"):
            self.sn = {}                     # spectral-norm state is rebuilt from the module's buffers

    def _grad_tail(self):
        return 0

    def _versions(self):
        return tuple(p._version for _, p in self.module.named_parameters())

    def mview(self, l):
        """Packed master of layer `l` (fp32 [T][nc][kc])."""
        return self.flat[l.off:l.off + l.numel]

    def mgrad(self, l):
        return self.grad[l.off:l.off + l.numel]

    def _param(self, name):
        return dict(self.module.named_parameters())[name]

    def _import(self, l, src=None, dst=None):
        """reference layout -> packed (master by default)."""
        src = self._param(l.name).data if src is None else src
        dst = self.mview(l) if dst is None else dst
        if l.tied:
            src = torch.cat((src, src), 0).contiguous()          # both halves of the doubled input = the parameter
        if not dst.is_cuda:
            dst.copy_(pack_reference(l.kind, src.float(), l.c_out, l.c_in, l.t_len, l.kw).reshape(-1))
            return
        _lib.call("sg_pack_weights_kw", l.kind, _p(src), l.c_out, l.c_in, l.t_len, l.kw, None, 0, _p(dst), None, SG_F32,
                  SG_F32, _stream())

    def _export(self, l, src, dst):
        """packed -> reference layout (pure layout transform)."""
        if l.tied:
            full = torch.empty((2 * dst.shape[0],) + tuple(dst.shape[1:]), dtype=dst.dtype, device=dst.device)
            self._export_plain(l, src, full)
            dst.copy_(full[:dst.shape[0]])
            return
        self._export_plain(l, src, dst)

    def _export_plain(self, l, src, dst):
        if not src.is_cuda:
            dst.copy_(unpack_reference(l.kind, src, l.c_out, l.c_in, l.t_len, l.kw).reshape(dst.shape))
            return
        _lib.call("sg_unpack_wgrad_kw", l.kind, _p(src), l.c_out, l.c_in, l.t_len, l.kw, None, None, 0, _p(dst), None, 0,
                  _stream())

    def notice_external_writes(self):
        """Parameters written through torch since the last look (load_state_dict, init functions, p.data.copy_):
        big weights are imported into their packed master, everything marks the operands stale."""
        v = self._versions()
        if v == self._seen:
            return
        for (name, p), new, old in zip(self.module.named_parameters(), v, self._seen):
            if new != old:
                self._ops_stale = True
                if name in self.by_name:
                    self._import(self.by_name[name])
        self._seen = v

    def sync_to_reference(self):
        """Refreshes the reference-layout mirrors of the big weights from the packed masters (no-op when nothing
        changed).  Called by state_dict() / save / .to() / grad_of()."""
        if self.flat is None:
            return
        self.notice_external_writes()
        if self._mirror_stale:
            for l in self.layers:
                self._export(l, self.mview(l), self._param(l.name).data)
            self._mirror_stale = False

    def pview(self, name):
        """Current value of a parameter: bucket view (small parameters) or the reference-layout mirror."""
        ent = self.index.get(name)
        if ent is not None:
            off, n, shape = ent
            return self.flat[off:off + n].view(shape)
        return self._param(name).data

    def gview(self, name):
        """Gradient slot of a SMALL parameter (bucket view, carries LOSS_SCALE)."""
        off, n, shape = self.index[name]
        return self.grad[off:off + n].view(shape)

    def master_updated(self):
        """An optimiser step changed the bucket in place."""
        self._mirror_stale = True
        self._ops_stale = True

    def mark_dirty(self):
        self._ops_stale = True

    # -- gradients --------------------------------------------------------------------------
    def zero_grad(self):
        if self._grad_dirty:
            self.grad.zero_()
        self._grad_dirty, self._alpha_fixed = False, False

    def finish_grads(self):
        """Hook between the (all-reduced) raw gradients and the optimiser: the decoder's alpha-scaled layers turn
        their dWeff into dW and produce the alpha gradients (linear in the gradients: safe after the all-reduce)."""
        self._alpha_fixed = True

    def grads_consumed(self, cleared):
        if cleared:
            self._grad_dirty, self._alpha_fixed = False, False

    def grad_of(self, name):
        """Gradient of parameter `name` in true units and reference layout (tests, autograd API)."""
        if not self._alpha_fixed:
            self.finish_grads()
        l = self.by_name.get(name)
        if l is None:
            return self.gview(name) * (1.0 / LOSS_SCALE)
        out = torch.empty_like(self._param(name).data)
        self._export(l, self.mgrad(l), out)
        return out.mul_(1.0 / LOSS_SCALE)

    def export_grads(self):
        """Copies the gradients into per-parameter .grad tensors (API compatibility)."""
        for name, p in self.module.named_parameters():
            if p.requires_grad:
                g = self.grad_of(name)
                if p.grad is None:
                    p.grad = g
                else:
                    p.grad.copy_(g)

    # -- 16-bit operands ----------------------------------------------------------------------
    def ensure_packed(self):
        """Re-emits the 16-bit operands when the masters changed.  With overlap on, the kernels go to side
        stream 4 and record one event per operand: the forward that triggered them waits for each layer's event
        right before that layer's tap-GEMM (`wait_packed`), so the emission hides behind the first layers
        instead of preceding them on the critical chain."""
        self.bind()
        self.notice_external_writes()
        if self._ops_stale:
            self.pack_ev = {}
            self._pack_side = side_stream(self.flat.device, 4)
            with on_side(self._pack_side):
                self.pack()
            self._ops_stale = False

    def emit(self, l, alpha=None, scale=None):
        """Forward + data-gradient operand of packed layer `l` out of its master (scale: device scalar, 1/sigma)."""
        dev = self.flat.device
        wf = self.buf.get(l.f_key, (l.T, l.nc, l.kc), F16, dev)
        wd = self.buf.get(l.dg_key, (l.T, l.kc, l.nc), GT, dev)
        _lib.call("sg_emit_operands", _p(self.mview(l)), l.T, l.nc, l.kc, _p(alpha), l.alpha_from, _p(wf), _p(wd),
                  SG_F16, GS, _p(scale), _stream())
        self.packed[l.f_key], self.packed[l.dg_key] = wf, wd
        self._mark_packed(l.f_key)

    def _mark_packed(self, *keys):
        if getattr(self, "_pack_side", None) is not None:
            ev = torch.cuda.Event()
            ev.record()
            for k in keys:
                self.pack_ev[k] = ev

    def wait_packed(self, key):
        ev = getattr(self, "pack_ev", {}).get(key)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def packs_consumed(self):
        """End of the forward that triggered a pack: later users are ordered after it by their streams."""
        if getattr(self, "_pack_side", None) is not None:
            join_side(self._pack_side)
            self._pack_side = None
        self.pack_ev = {}


# --------------------------------------------------------------------------------------------
# spectral normalisation (norm_type='snorm', torch.nn.utils.spectral_norm) -- shared by both networks
# --------------------------------------------------------------------------------------------
def sn_v_layout(pl):
    """(reference shape of weight_v as a weight with one output channel, c_in of that weight) of packed layer `pl`.
    Conv1d (dim 0): v runs over (ci, k) -> [1][Cin][kw]; ConvTranspose1d (dim 1): v runs over (ci, k) of
    W[Cin][Cout][kw] -> [Cin][1][kw]; a tied master holds [W | W], whose v covers one half."""
    vin = pl.c_in // 2 if pl.tied else pl.c_in
    if pl.kind == 0:
        return (1, vin, pl.kw), vin
    if pl.kind == 1:
        return (vin, 1, pl.kw), vin
    return (1, -1), vin


def sn_pack_v(pl, vref):
    """weight_v (reference layout, flat) -> the packed slots the power iteration of `pl` runs on."""
    shape, vin = sn_v_layout(pl)
    return pack_reference(pl.kind, vref.reshape(shape), 1, vin, pl.t_len, pl.kw).reshape(-1).contiguous()


def sn_unpack_v(pl, v):
    return unpack_reference(pl.kind, v, 1, sn_v_layout(pl)[1], pl.t_len, pl.kw).reshape(-1)


def sn_geometry(pl):
    """(n_taps, nc, kc, ld) of the power iteration on the packed master of `pl` (include/segan_b200.h): kind 0 / 2
    as packed (dim 0); kind 1 as [36][Cout][Cin] (dim 1: u per output channel); a tied master's first half."""
    _, vin = sn_v_layout(pl)
    if pl.kind == 1:
        return 36, pl.c_out, vin, pl.kc
    return pl.T, pl.nc, pl.kc, pl.kc


class _SpectralNorm(object):
    """Per-pass spectral-norm state of the normalised weights of a network (names ending in weight_orig): the
    power-iteration vectors (u: the module's buffer itself; v: packed slots for the tap-GEMM layers, the module's
    buffer for the small ones), per-pass copies of both, the per-pass [unused, unused, sigma, 1/sigma] scalars and
    the per-pass sigma-term coefficients."""
    SN_SLOTS = 5                    # up to 4 accumulating passes per optimiser step (WSEGAN) + 1 gradient-free pass

    def _sn_coef(self, name):
        """Storage of the per-pass sigma-term coefficients of packed layer `name` (SN_SLOTS floats)."""
        return torch.zeros(self.SN_SLOTS, device=self.flat.device)

    def _sn_state(self, name):
        st = self.sn.get(name)
        if st is not None:
            return st
        dev = self.flat.device
        mod = dict(self.module.named_buffers())
        base = name[:-len("weight_orig")]
        u, vref = mod[base + "weight_u"], mod[base + "weight_v"]
        pl = self.by_name.get(name)
        if pl is not None:
            T, nc, kc, ld = sn_geometry(pl)
            v = sn_pack_v(pl, vref)
        else:
            # reference layout [height][rest]: dim 0, or dim 1 of a transposed conv with one output channel
            nc = u.numel()
            T, kc = 1, self.index[name][1] // nc
            ld = kc
            v = vref
        P = self.SN_SLOTS
        st = self.sn[name] = dict(T=T, nc=nc, kc=kc, ld=ld, u=u, v=v, vref=vref, pl=pl,
                                  scal=torch.zeros(P, 4, device=dev), u_p=torch.zeros(P, nc, device=dev),
                                  v_p=torch.zeros(P, T * kc, device=dev),
                                  coef=self._sn_coef(name) if pl is not None else None,
                                  work=torch.zeros(nc + T * ((kc + 255) // 256) + 4, device=dev),
                                  seen=(u._version, vref._version))
        return st

    def _sn_master(self, name):
        pl = self.by_name.get(name)
        return self.mview(pl) if pl is not None else self.pview(name)

    def sn_inv_sigma(self, name, slot=None):
        """Device scalar 1 / sigma of `name` for pass slot `slot` (default: the current one)."""
        return self._sn_state(name)["scal"][self._sn_slot if slot is None else slot][3:4]

    def sync_to_reference(self):
        super().sync_to_reference()
        for name, st in self.sn.items():          # packed v -> the module's reference-layout buffer
            pl = st["pl"]
            if pl is not None:
                st["vref"].copy_(sn_unpack_v(pl, st["v"]))
                st["seen"] = (st["u"]._version, st["vref"]._version)

    def _sn_fix_small(self, nm, scratch, slot):
        """scratch gradient w.r.t. the normalised small tensor `nm` -> gradient w.r.t. weight_orig, into the bucket."""
        stt = self._sn_state(nm)
        _lib.call("sg_snorm_grad", _p(scratch), _p(self.pview(nm)), 1, stt["nc"], stt["kc"], _p(stt["u_p"][slot]),
                  _p(stt["v_p"][slot]), _p(stt["scal"][slot]), _p(stt["work"][stt["nc"]:]), _stream())
        self.gview(nm).add_(scratch)


# ============================================================================================
# Generator
# ============================================================================================
class GeneratorEngine(_SpectralNorm, _NetEngine):
    def __init__(self, module):
        super().__init__(module)
        m = module
        self.fmaps = list(m.enc_fmaps)
        self.nl = len(self.fmaps)
        self.enc_bias = m.bias
        # topology: z channels ahead of the code in decoder block 0 (0 with no_z) and whether the decoder merges
        # skips at all (skip=False: every decoder block and the waveform end read the previous block alone)
        self.zc = 0 if getattr(m, "no_z", False) else m.z_dim
        self.has_skip = getattr(m, "skip", True)
        self.sum_merge = self.has_skip and getattr(m, "skip_merge", "concat") == "sum"
        # skip_type='conv': the skip of encoder level l is Conv1d(C, C, K)(a[l]) (weights alpha_l.skip_k.weight /
        # .bias, small region of the bucket) and has no alpha -- every alpha use below reads 1
        self.conv_skip = self.has_skip and getattr(m, "skip_type", "alpha") == "conv"
        self.skip_kw = getattr(m, "skip_kwidth", 11)
        # kernel width of every encoder conv and decoder deconv (31 in SEGAN+; Generator._served admits 4..32)
        self.kw_enc = [b.kwidth for b in m.enc_blocks]
        self.kw_dec = [b.kwidth for b in m.dec_blocks]
        self.packed = {}
        # norm_type='snorm' (modules.py:12-14): every encoder conv (dim 0) and decoder deconv (dim 1) is divided by its
        # spectral norm, re-estimated by one power iteration per training forward; the parameters are then called
        # weight_orig.  Skip convs and alphas are not normalised.
        self.snorm = getattr(m, "norm_type", None) == "snorm"
        self.wsfx = "_orig" if self.snorm else ""
        self.sn = {}
        self._sn_reset()

    def _require_wave_route(self):
        if not wave_on_tensor_cores() and any(k != 31 for k in self.kw_enc + self.kw_dec):
            raise NotImplementedError("Generator kernel widths other than 31 need the tensor-core waveform route "
                                      "(SEGAN_B200_WAVE=tc)")

    def _sn_reset(self):
        # Pass slots: a forward that a backward will follow takes a slot that is neither outstanding (forward run,
        # backward not yet) nor done (gradients in the bucket).  A step's G forward runs BEFORE Gopt.zero_grad()
        # (SEGAN / WSEGAN), so zero_grad() drops only the done slots.  The done slots' sigma terms are applied in
        # finish_grads().
        self._sn_live = {}          # slot -> ticket of the outstanding forward that holds it
        self._sn_done = []          # slots whose gradients are in the bucket
        self._sn_ticket = 0
        self._sn_slot = self.SN_SLOTS - 1
        self._sn_eval_ok = False    # the operands hold the eval-mode sigma of the current masters and vectors
        self._ops_slot = None       # the pass slot whose 1 / sigma the current 16-bit operands carry

    def wname(self, block, l):
        """Name of the weight of encoder ('enc') or decoder ('dec') block l (weight_orig with snorm)."""
        return ("enc_blocks.%d.conv.weight%s" if block == "enc" else "dec_blocks.%d.deconv.weight%s") % (l, self.wsfx)

    # -- weights ----------------------------------------------------------------------------
    def packed_layers(self):
        """Bucket order = the order in which a backward pass completes the gradients, so that the data-parallel
        all-reduce can leave in contiguous chunks while the rest of the backward still runs (grad_chunks):
        decoder (dec3 .. dec0 finish first), then enc4, then enc3 .. enc1 and the small parameters."""
        fm, nl = self.fmaps, self.nl
        ls = []
        for l in range(nl - 1):
            ls.append(PackedLayer(self.wname("dec", l), 1, self.dec_cout(l), self.dec_cin(l), 0,
                                  "Wt%d" % l, "Wtd%d" % l,
                                  alpha_name=(("alpha_%d.skip_k" % (nl - 1 - l))
                                              if l > 0 and self.has_skip and not self.conv_skip else None),
                                  tied=(self.sum_merge and l > 0), kw=self.kw_dec[l]))
        ls += [PackedLayer(self.wname("enc", l), 0, fm[l], fm[l - 1], 0, "Wf%d" % l, "Wdg%d" % l, kw=self.kw_enc[l])
               for l in range(nl - 1, 0, -1)]
        return ls

    # -- spectral norm (state: _SpectralNorm) ------------------------------------------------------
    def _sn_names(self):
        return [self.wname("enc", l) for l in range(self.nl)] + [self.wname("dec", l) for l in range(self.nl)]

    def _grad_tail(self):
        """snorm: the per-pass sigma-term coefficients of the packed layers ride at the end of the gradient bucket, so
        that the data-parallel all-reduce sums them with the gradients: the sigma terms applied after it
        (finish_grads) then use the coefficients of the whole batch."""
        return len(self.layers) * self.SN_SLOTS if self.snorm else 0

    def _sn_coef(self, name):
        i = self.layers.index(self.by_name[name])
        o = self.flat.numel() + i * self.SN_SLOTS
        return self.grad[o:o + self.SN_SLOTS]

    def _build(self, ps, dev):
        super()._build(ps, dev)
        self._sn_reset()

    def _sn_iterate(self, training, slot):
        """sigma of every normalised weight for the coming pass (one power iteration when training) into pass slot
        `slot`, with copies of the vectors for that pass's backward.  sg_snorm_sigma_ld sums in a fixed order: ranks
        holding the same masters and vectors compute the same bits, so u, v and sigma never drift apart."""
        st_ = _stream()
        for name in self._sn_names():
            st = self._sn_state(name)
            _lib.call("sg_snorm_sigma_ld", _p(self._sn_master(name)), st["T"], st["nc"], st["kc"], st["ld"], _p(st["u"]),
                      _p(st["v"]), _p(st["scal"][slot]), _p(st["work"]), 1 if training else 0, st_)
            st["u_p"][slot].copy_(st["u"])
            st["v_p"][slot].copy_(st["v"].reshape(-1))
        self._sn_slot = slot

    def _sn_take_slot(self):
        """Pass slot of a forward that a backward will follow (see _sn_reset).  With every slot taken, the oldest
        outstanding forward's slot is reused: its backward then raises."""
        busy = set(self._sn_live) | set(self._sn_done)
        free = [s for s in range(self.SN_SLOTS - 1) if s not in busy]
        if free:
            slot = free[0]
        elif self._sn_live:
            slot = min(self._sn_live, key=self._sn_live.get)
        else:
            raise RuntimeError("more than %d accumulating Generator passes per optimiser step" % (self.SN_SLOTS - 1))
        self._sn_ticket += 1
        self._sn_live[slot] = self._sn_ticket
        return slot, self._sn_ticket

    def _sn_notice_buffers(self):
        """weight_u / weight_v written through torch (load_state_dict, copy_): the packed v is re-imported in place
        and the operands are re-emitted with the new sigma."""
        for st in self.sn.values():
            seen = (st["u"]._version, st["vref"]._version)
            if seen != st["seen"]:
                if st["pl"] is not None:
                    st["v"].copy_(sn_pack_v(st["pl"], st["vref"]))
                st["seen"] = seen
                self._ops_stale, self._sn_eval_ok = True, False

    def notice_external_writes(self):
        super().notice_external_writes()
        if self.snorm:
            self._sn_notice_buffers()

    def master_updated(self):
        super().master_updated()
        self._sn_eval_ok = False

    def zero_grad(self):
        super().zero_grad()
        self._sn_done = []

    def grads_consumed(self, cleared):
        super().grads_consumed(cleared)
        if cleared:
            self._sn_done = []
            if self.snorm:
                # the optimiser clears the parameters' gradients only: clear the coefficient tail too, so that no stale
                # value is all-reduced (and multiplied by the world size) step after step
                self.grad[self.flat.numel():].zero_()

    def grad_chunks(self):
        """[(offset, numel)]: decoder weights (complete after dec0's weight gradient) | enc_{nl-1} | the rest."""
        a = sum(l.numel for l in self.layers[:self.nl - 1])
        b = a + self.layers[self.nl - 1].numel
        return [(0, a), (a, b - a), (b, self.grad.numel() - b)]

    def pack(self):
        dev = self.flat.device
        # last decoder layer (Cout = 1): fp32 [cin][31] with alpha folded (tiny: torch ops); snorm: every operand below
        # and the waveform-end conv's are made of W / sigma
        l = self.nl - 1
        w = self.pview(self.wname("dec", l))[:, 0, :]
        w0 = self.pview(self.wname("enc", 0))
        if self.snorm:
            self._ops_slot = self._sn_slot
            w = w * self.sn_inv_sigma(self.wname("dec", l))
            w0 = w0 * self.sn_inv_sigma(self.wname("enc", 0))
        if self.sum_merge:                      # tied halves: W (hi + alpha skip) = [W | alpha W] cat(hi, skip)
            w = torch.cat((w, w), 0)
        self.packed["w_last_dup"] = w.reshape(w.shape[0], 1, self.kw_dec[l]).contiguous()
        weff = w.clone()
        if self.has_skip:
            half = w.shape[0] // 2
            weff[half:] = weff[half:] * self.alpha_for_dec(l).view(-1, 1)
        self.packed["w_last_eff"] = weff.contiguous()
        # tensor-core route of the waveform-end layers: single-tap operands (tiny tensors, torch ops)
        wcol = wave_col_weights(w0, dev)
        self.packed["Wcol0"] = wcol.half().contiguous()
        kidx = dec_last_tap_index(dev, self.kw_dec[l])
        w2 = weff.t()[kidx.clamp(min=0)] * (kidx >= 0).float().unsqueeze(1)       # [64][cin]
        self.packed["W2_last"] = w2.half().contiguous()
        wg = torch.zeros(weff.shape[0], 64, dtype=torch.float32, device=dev)
        wg[:, :self.kw_dec[l]] = weff
        self.packed["Wg_last"] = wg.to(GT).contiguous()
        self._mark_packed("small")
        if self.conv_skip:
            # skip convs: grouped 16-bit operands [2D+1][4C][4C] out of the reference-layout fp32 master
            D = (self.skip_kw // 2 + 3) // 4
            for l in range(self.nl - 1):
                c = self.fmaps[l]
                wf = self.buf.get("Wsk%d" % l, (2 * D + 1, 4 * c, 4 * c), F16, dev)
                wd = self.buf.get("Wskd%d" % l, (2 * D + 1, 4 * c, 4 * c), GT, dev)
                _lib.call("sg_skipconv_emit", _p(self.pview("alpha_%d.skip_k.weight" % l)), c, self.skip_kw,
                          _p(wf), _p(wd), SG_F16, GS, _stream())
                self.packed["Wsk%d" % l], self.packed["Wskd%d" % l] = wf, wd
                self._mark_packed("Wsk%d" % l)
        for pl in self.layers:
            self.emit(pl, self.pview(pl.alpha_name).reshape(-1) if pl.alpha_name else None,
                      scale=self.sn_inv_sigma(pl.name) if self.snorm else None)

    def finish_grads(self):
        """Per packed layer, in this order: the alpha fix (dWeff -> dW and dalpha), the sum of the tied halves, and with
        snorm the sigma terms of the step's passes.  Each pass's weight-gradient GEMM scaled by 1/sigma_p, so the
        alpha fix against the master W gives sum_p <dWeff_p, W / sigma_p> = dalpha, and afterwards the bucket holds
        sum_p (dL/dW~_p) / sigma_p, from which sg_snorm_rank1_ld subtracts sum_p coef_p u_p v_p^T (on both tied
        copies).  The sigma term must come after the alpha fix: the fix multiplies the skip columns by alpha."""
        if self._alpha_fixed:
            return
        runs = []
        for s in sorted(self._sn_done) if self.snorm else ():
            if runs and runs[-1][0] + runs[-1][1] == s:
                runs[-1][1] += 1
            else:
                runs.append([s, 1])
        for pl in self.layers:
            if pl.alpha_name is not None:
                trainable = self._param(pl.alpha_name).requires_grad
                _lib.call("sg_alpha_grad", _p(self.mgrad(pl)), _p(self.mview(pl)), pl.T, pl.nc, pl.kc,
                          _p(self.pview(pl.alpha_name).reshape(-1)), pl.alpha_from,
                          _p(self.gview(pl.alpha_name).view(-1)) if trainable else None, _stream())
            if pl.tied:                          # dW = dW_a + alpha dW_b, written to both copies
                g2 = self.mgrad(pl).view(pl.T, pl.nc, 2, pl.kc // 2)
                tot = g2[:, :, 0] + g2[:, :, 1]
                g2[:, :, 0] = tot
                g2[:, :, 1] = tot
            if runs:
                st = self._sn_state(pl.name)
                for s0, n in runs:
                    _lib.call("sg_snorm_rank1_ld", _p(self.mgrad(pl)), st["T"], st["nc"], st["kc"], st["ld"],
                              2 if pl.tied else 1, n, _p(st["u_p"][s0]), _p(st["v_p"][s0]), _p(st["coef"][s0:]),
                              _stream())
        self._alpha_fixed = True

    def dec_cin(self, l):
        """Input channels of decoder block l AS THE GEMM SEES THEM: cat(z, code) (the code alone with no_z) for
        block 0, cat(decoder, skip) afterwards -- also with skip_merge='sum', which runs as the concat GEMM with
        tied weight halves -- or the decoder output alone without skips."""
        if l == 0:
            return self.zc + self.fmaps[-1]
        return (2 if self.has_skip else 1) * self.fmaps[self.nl - 1 - l]

    def dec_cout(self, l):
        return self.fmaps[self.nl - 2 - l] if l < self.nl - 1 else 1

    def alpha_for_dec(self, l):
        """alpha of the skip merged before decoder block l (None for block 0: cat(z, h), and without skips)."""
        if l == 0 or not self.has_skip:
            return None
        if self.conv_skip:                       # the skip conv's output is merged unscaled
            c, key = self.fmaps[self.nl - 1 - l], "g.ones%d" % self.fmaps[self.nl - 1 - l]
            ones = self.buf.t.get(key)
            if ones is None or ones.device != self.flat.device:
                ones = self.buf.t[key] = torch.ones(c, dtype=F32, device=self.flat.device)
            return ones
        return self.pview("alpha_%d.skip_k" % (self.nl - 1 - l)).reshape(-1)

    # -- forward ----------------------------------------------------------------------------
    def forward(self, x, z, want_ctx=True, fresh=False, twins=None, training=True):
        """x: (B,1,L) fp32 cuda, z: (B, C4, L/1024) fp32 cuda.  Returns y (B,1,L) fp32.
        twins (default = want_ctx): also write the bf16 copies of the activations that only the weight-gradient
        tap-GEMMs read; inference passes False (one store per activation instead of two or three).
        fresh=True gives the saved activations their own storage (generic autograd use, where several
        forwards may precede a backward); the fused train step reuses one persistent workspace.
        training (snorm only, the module's mode): one power iteration that updates weight_u / weight_v; eval mode
        uses the stored vectors and leaves them unchanged."""
        _require_cuda(x, z)
        self._require_wave_route()
        twins = want_ctx if twins is None else (twins and want_ctx)
        bwd = twins                               # a backward pass will read this forward's saved tensors
        alias = twins and not grad_twins()        # fp16 gradients: the weight-gradient GEMMs read the forward tensors
        twins = twins and grad_twins()
        sn_slot = None
        if self.snorm:
            if not wave_on_tensor_cores():
                raise NotImplementedError("norm_type='snorm' needs the tensor-core waveform route (SEGAN_B200_WAVE=tc)")
            self.bind()
            self.notice_external_writes()
            if bwd:
                sn_slot = self._sn_take_slot()
                self._sn_iterate(training, sn_slot[0])
                self._ops_stale, self._sn_eval_ok = True, False
            elif training or not self._sn_eval_ok or self._ops_stale:
                # gradient-free pass: slot SN_SLOTS - 1; an eval-mode sigma stays valid until the masters or the
                # vectors change
                self._sn_iterate(training, self.SN_SLOTS - 1)
                self._ops_stale, self._sn_eval_ok = True, not training
        self.ensure_packed()
        self.wait_packed("small")
        B, _, L = x.shape
        fm, nl, dev, st = self.fmaps, self.nl, x.device, _stream()
        buf = _Buffers() if fresh else self.buf
        assert L % (4 ** nl) == 0 and L // (4 ** nl) >= 1 and L >= 4096, "window length must be a multiple of 1024, >= 4096"
        x = x.contiguous().float()
        Lq = [L // 4 ** (l + 1) for l in range(nl)]
        a, hp = [None] * nl, [None] * nl
        # bf16 twins (only when a backward will follow): operands of the weight-gradient tap-GEMMs
        hpb, ab, ddb, z16b = [None] * nl, [None] * nl, [None] * nl, None
        # skip_type='conv': the skip convs' outputs (what the decoder merges instead of a[l]) and their 16-bit
        # weight-gradient operands (bf16 twin, or the output itself with fp16 gradients)
        sk, skb = [None] * nl, [None] * nl
        # The Generator has no norm layer between a contraction and its PReLU, so the activation (and the reflect
        # halo of the next conv) is written by the tap-GEMM epilogue next to the raw pre-activation: no separate
        # pass over the tensor.  Needs the tensor-core backend, no bf16 twins, and tensors long
        # enough for the mirror logic; otherwise sg_act_fwd does it as before.
        eff_backend = default_backend() if self.backend is None else self.backend
        fuse_ok = FUSE_ACT and eff_backend == BACKEND_TCGEN05 and not twins

        def fused(rows_m, halo):
            return fuse_ok and f_pair_tiles(rows_m, B) >= 2 and (halo == 0 or rows_m >= 2 * halo + 3)
        # ---- encoder
        for l in range(nl):
            cout = fm[l]
            a[l] = buf.get("g.a%d" % l, (B, Lq[l], cout), F16, dev)
            bias = self.pview("enc_blocks.%d.conv.bias" % l) if self.enc_bias else None
            halo = 16 if l < nl - 1 else 0
            hp[l] = buf.get("g.hp%d" % l, (B, Lq[l] + 2 * halo, cout), F16, dev)
            slope = self.pview("enc_blocks.%d.act.weight" % l)
            fz = fused(Lq[l], halo) and (l > 0 or wave_on_tensor_cores())
            fkw = dict(out2=hp[l], out2_halo=halo, slope=slope, slope_mod=cout) if fz else {}
            if l == 0 and wave_on_tensor_cores():
                col16 = buf.get("g.col16", (B, Lq[0], 64), F16, dev)
                colb = buf.get("g.colb", (B, Lq[0], 64), GT, dev) if twins else None
                _lib.call("sg_wave_im2col_kw", _p(x), None, 1, B, L, 0, None, 1, conv_offset(self.kw_enc[0]),
                          self.kw_enc[0], _p(col16), _p(colb), st)
                if alias:
                    colb = col16
                self.wait_packed("small")
                run_f(col16, None, Lq[0], 0, SG_F16, self.packed["Wcol0"], SG_F16, 64, 64,
                      tap_ranges("full", 0, 64, 64), a[0], SG_F16, Lq[0], 0, 0, Lq[0], B, bias=bias, bias_mod=64,
                      d_lo=0, d_hi=0, w_tap0=4, backend=self.backend, **fkw)
            elif l == 0:
                colb = None
                _lib.call("sg_wave_conv_fwd", _p(x), None, 1, B, L, 0, _p(self.pview("enc_blocks.0.conv.weight")),
                          _p(bias), cout, _p(a[0]), None, None, st)
            else:
                cin = fm[l - 1]
                self.wait_packed("Wf%d" % l)
                taps = tap_ranges("conv_fwd", cin, 4 * cin, cout, self.kw_enc[l])
                d_lo, d_hi = tap_span(taps)
                run_f(hp[l - 1], None, Lq[l], 4, SG_F16, self.packed["Wf%d" % l], SG_F16, 4 * cin, cout,
                      taps, a[l], SG_F16, Lq[l], 0, 0, Lq[l], B, d_lo=d_lo, d_hi=d_hi,
                      bias=bias, bias_mod=cout, backend=self.backend, **fkw)
            if twins:
                hpb[l] = buf.get("g.hpb%d" % l, (B, Lq[l] + 2 * halo, cout), GT, dev)
                if l < nl - 1:
                    ab[l] = buf.get("g.ab%d" % l, (B, Lq[l], cout), GT, dev)
            if not fz:
                _lib.call("sg_act_fwd", _p(a[l]), SG_F16, B, Lq[l], cout, None, _p(slope), ACT_PRELU, 0, None, halo,
                          _p(hp[l]), _p(hpb[l]), _p(ab[l]), st)
            if alias:
                hpb[l], ab[l] = hp[l], a[l]
            if self.conv_skip and l < nl - 1:
                sk[l], skb[l] = self._skip_conv_fwd(l, a[l], B, Lq[l], buf, twins, alias)
        # ---- z (none with no_z: decoder block 0 reads the code alone)
        z16 = None
        if self.zc:
            zc = z.shape[1]
            assert zc == self.zc, "z has %d channels, the Generator was built with z_dim %d" % (zc, self.zc)
            z16 = buf.get("g.z16", (B, Lq[-1], zc), F16, dev)
            zf = z.contiguous().float()
            _lib.call("sg_ncl_to_nlc", _p(zf), B, zc, Lq[-1], _p(z16), SG_F16, st)
            if twins:
                z16b = buf.get("g.z16b", (B, Lq[-1], zc), GT, dev)
                _lib.call("sg_ncl_to_nlc", _p(zf), B, zc, Lq[-1], _p(z16b), GS, st)
            elif alias:
                z16b = z16
        # ---- decoder
        ad, dd = [None] * nl, [None] * nl
        src0, src1 = (z16, hp[nl - 1]) if self.zc else (hp[nl - 1], None)
        lin = Lq[-1]
        for l in range(nl - 1):
            cin, cout = self.dec_cin(l), self.dec_cout(l)
            c1 = 0 if src1 is None else src1.shape[-1]
            assert src0.shape[-1] + c1 == cin
            dd[l] = buf.get("g.dd%d" % l, (B, 4 * lin, cout), F16, dev)
            slope = self.pview("dec_blocks.%d.act.weight" % l)
            fz = fused(lin, 0)
            if fz and not bwd:
                # inference: nobody reads the decoder's pre-activation -- PReLU applied to the only output
                ad[l] = None
                fkw = dict(slope=slope, slope_mod=cout)
                dst = dd[l]
            else:
                ad[l] = buf.get("g.ad%d" % l, (B, lin, 4 * cout), F16, dev)
                fkw = dict(out2=dd[l], slope=slope, slope_mod=cout) if fz else {}
                dst = ad[l]
            self.wait_packed("Wt%d" % l)
            taps = tap_ranges("deconv_fwd", cout, cin, 4 * cout, self.kw_dec[l])
            d_lo, d_hi = tap_span(taps)
            run_f(src0, src1, lin, 0, SG_F16, self.packed["Wt%d" % l], SG_F16, cin, 4 * cout,
                  taps, dst, SG_F16, lin, 0, 0, lin, B, d_lo=d_lo, d_hi=d_hi,
                  bias=self.pview("dec_blocks.%d.deconv.bias" % l), bias_mod=cout,
                  a0_c=src0.shape[-1], a1_c=c1, backend=self.backend, **fkw)
            if twins:
                ddb[l] = buf.get("g.ddb%d" % l, (B, 4 * lin, cout), GT, dev)
            if not fz:
                _lib.call("sg_act_fwd", _p(ad[l]), SG_F16, B, 4 * lin, cout, None, _p(slope), ACT_PRELU, 0, None, 0,
                          _p(dd[l]), _p(ddb[l]), None, st)
            if alias:
                ddb[l] = dd[l]
            lin *= 4
            src0 = dd[l]
            src1 = (sk if self.conv_skip else a)[nl - 2 - l] if self.has_skip else None
        y = torch.empty(B, 1, L, dtype=F32, device=dev)
        blast = self.pview("dec_blocks.%d.deconv.bias" % (nl - 1))
        if wave_on_tensor_cores():
            c1 = 0 if src1 is None else src1.shape[-1]
            cl = src0.shape[-1] + c1
            P = buf.get("g.P", (B, lin, 64), F32, dev)
            run_f(src0, src1, lin, 0, SG_F16, self.packed["W2_last"], SG_F16, cl, 64, tap_ranges("full", 0, cl, 64),
                  P, SG_F32, lin, 0, 0, lin, B, d_lo=0, d_hi=0, w_tap0=4, a0_c=src0.shape[-1], a1_c=c1,
                  backend=self.backend)
            _lib.call("sg_wave_shiftadd_tanh", _p(P), B, lin, _p(blast), _p(y), st)
        else:
            if not self.has_skip:
                raise NotImplementedError("a Generator without skips (skip=False) needs the tensor-core waveform "
                                          "route (SEGAN_B200_WAVE=tc)")
            _lib.call("sg_wave_deconv_fwd", _p(src0), src0.shape[-1], _p(src1), src1.shape[-1], B, lin,
                      _p(self.packed["w_last_eff"]), _p(blast), _p(y), st)
        self.packs_consumed()
        ctx = dict(x=x, B=B, L=L, Lq=Lq, a=a, hp=hp, z16=z16, ad=ad, dd=dd, y=y, hpb=hpb, ab=ab, ddb=ddb,
                   z16b=z16b, colb=colb, skb=skb if self.conv_skip else ab, sn_slot=sn_slot) if want_ctx else None
        return y, ctx

    def _skip_conv_fwd(self, l, a_l, B, lq, buf, twins, alias):
        """Skip conv of encoder level l on its pre-activation a_l [B][lq][C]: one tap-GEMM over the grouped rows
        (zero padding = rows outside the sequence).  Returns (output, weight-gradient operand of the decoder)."""
        c, dev = self.fmaps[l], a_l.device
        d_lo, d_hi, tap0, taps, _ = skipconv_geometry(c, self.skip_kw)
        bias_name = "alpha_%d.skip_k.bias" % l
        bias = self.pview(bias_name) if bias_name in self.index else None
        outs = [(buf.get("g.sk%d" % l, (B, lq, c), F16, dev), SG_F16)]
        if twins:                                 # bf16 gradients: a bf16 twin for the decoder's weight gradient
            outs.append((buf.get("g.skb%d" % l, (B, lq, c), GT, dev), GS))
        self.wait_packed("Wsk%d" % l)
        for out, dt in outs:
            run_f(a_l, None, lq // 4, 0, SG_F16, self.packed["Wsk%d" % l], SG_F16, 4 * c, 4 * c, taps, out, dt,
                  lq // 4, 0, 0, lq // 4, B, bias=bias, bias_mod=c, d_lo=d_lo, d_hi=d_hi, w_tap0=tap0,
                  backend=self.backend)
        s = outs[0][0]
        return s, (outs[1][0] if twins else (s if alias else None))

    def hidden_ncl(self, ctx, only=None):
        """`hall` of generator.py:186-227 as fp32 NCL tensors (inspection path).  only: optional set of keys."""
        nl, st = self.nl, _stream()
        B, Lq = ctx["B"], ctx["Lq"]
        hall = {}

        def to_ncl(t16, C_, L_):
            out = torch.empty(B, C_, L_, dtype=F32, device=t16.device)
            _lib.call("sg_nlc_to_ncl", _p(t16), SG_F16, B, C_, L_, _p(out), st)
            return out
        want = (lambda k: True) if only is None else (lambda k: k in only)
        want_zc = self.zc > 0 and want("enc_zc")          # no_z: the reference's hall has no enc_zc
        for l in range(nl):
            if want("enc_%d" % l) or (l == nl - 1 and want_zc):
                a = to_ncl(ctx["a"][l], self.fmaps[l], Lq[l])
                hall["enc_%d" % l] = torch.nn.functional.prelu(a, self.pview("enc_blocks.%d.act.weight" % l))
        if want_zc:
            zc = ctx["z16"].shape[-1]
            hall["enc_zc"] = torch.cat((to_ncl(ctx["z16"], zc, Lq[-1]), hall["enc_%d" % (nl - 1)]), 1)
        lin = Lq[-1]
        for l in range(nl - 1):
            if want("dec_%d" % l):
                hall["dec_%d" % l] = to_ncl(ctx["dd"][l], self.dec_cout(l), 4 * lin)
            lin *= 4
        if want("dec_%d" % (nl - 1)):
            hall["dec_%d" % (nl - 1)] = ctx["y"]
        return hall

    # -- backward ---------------------------------------------------------------------------
    def backward(self, ctx, gy, accumulate=False, reducer=None):
        """gy: (B,1,L) fp32 gradient w.r.t. the output.  Fills self.grad (the packed bucket).
        reducer: optional model.GradReducer -- chunk i of grad_chunks() is all-reduced on the communication stream
        as soon as its last weight-gradient GEMM has been enqueued, while the rest of the backward runs."""
        fm, nl, st, buf = self.fmaps, self.nl, _stream(), self.buf
        B, L, Lq = ctx["B"], ctx["L"], ctx["Lq"]
        a, hp, ad, dd = ctx["a"], ctx["hp"], ctx["ad"], ctx["dd"]
        dev = gy.device
        gy = gy.contiguous().float()
        slot, sn_small = None, {}
        if self.snorm:
            slot, ticket = ctx["sn_slot"]
            if self._sn_live.get(slot) != ticket:
                raise RuntimeError("this Generator forward's spectral-norm state was reused by %d later forward passes "
                                   "that kept their graphs: run at most %d forward passes ahead of their backward "
                                   "passes" % (self.SN_SLOTS - 1, self.SN_SLOTS - 1))
        if self.snorm and self._ops_slot != slot:
            # another forward (a second outstanding pass, or a gradient-free training pass) re-emitted the operands with
            # its own sigma since this pass's forward: the data-gradient GEMMs and the last block's fold read W / sigma
            # of THIS pass, so the operands are emitted again for its slot, in line on this stream
            self.packs_consumed()
            self._sn_slot = slot
            self.pack()
            self._sn_eval_ok = False
        if not accumulate:
            self.zero_grad()
        self._grad_dirty = True
        if self.snorm:
            del self._sn_live[slot]
            self._sn_done.append(slot)
            # the waveform ends are small tensors: this pass's gradient w.r.t. W / sigma goes to a scratch buffer and
            # sg_snorm_grad turns it into the weight_orig gradient (_sn_fix_small)
            for nm in (self.wname("enc", 0), self.wname("dec", nl - 1)):
                sn_small[nm] = buf.get("g.sng." + nm, self.index[nm][2], F32, dev, zero=True)

        def wgrad_dst(nm):
            """Where this pass's gradient of the small weight `nm` is accumulated."""
            return sn_small[nm] if nm in sn_small else self.gview(nm)

        def sn_coef(red, bias, c, pl_name):
            """snorm: sigma-term coefficient <dL/dW~, W~> / sigma of this pass from the layer's output statistics."""
            if self.snorm:
                stt = self._sn_state(pl_name)
                _lib.call("sg_snorm_coef", _p(red), _p(bias), c, _p(stt["scal"][slot]), _p(stt["coef"][slot:slot + 1]),
                          st)
        osc = (lambda nm: self.sn_inv_sigma(nm, slot)) if self.snorm else (lambda nm: None)
        side = side_stream(dev, 0)       # weight-gradient tap-GEMM of every layer (writes the packed gradient bucket)
        red_dec = stat_arena(buf, "g.red_dec", [(SL, 3, self.dec_cout(l)) for l in range(nl - 1)], dev)
        red_enc = stat_arena(buf, "g.red_enc", [(SL, 3, fm[l]) for l in range(nl)], dev)
        # ---- last decoder block (tanh, Cout = 1)
        l = nl - 1
        lin = Lq[0]
        cin = self.dec_cin(l)
        half = cin // 2
        # skip_type='conv': the data gradients of the blocks with a skip are written as two tensors -- decoder half
        # and skip half -- because the skip conv's data gradient reads its half through the contiguous grouped view
        g_in = buf.get("g.gin%d" % l, (B, lin, half if self.conv_skip else cin), GT, dev)
        gpre = buf.get("g.gpre", (B, L), F32, dev)
        gb = self.gview("dec_blocks.%d.deconv.bias" % l)
        src0 = dd[l - 1]
        src1 = a[0]
        if wave_on_tensor_cores():
            _lib.call("sg_tanh_bwd", _p(gy), _p(ctx["y"]), B * L, _p(gpre), _p(gb), st)
            colg = buf.get("g.colg", (B, lin, 64), GT, dev)
            kl = self.kw_dec[l]
            _lib.call("sg_wave_im2col_kw", _p(gpre), None, 1, B, L, 0, None, 0, deconv_padding(kl), kl,
                      _p(colg) if GS == SG_F16 else None, _p(colg) if GS != SG_F16 else None, st)
            if self.conv_skip:
                for dst, n0 in ((g_in, 0), (buf.get("g.gsk0", (B, lin, half), GT, dev), half)):
                    run_f(colg, None, lin, 0, GS, self.packed["Wg_last"], GS, 64, cin, tap_ranges("full", 0, 64, cin),
                          dst, GS, lin, 0, 0, lin, B, n_lo=n0, n_hi=n0 + half, out_ld=half, out_col0=0, d_lo=0,
                          d_hi=0, w_tap0=4, backend=self.backend)
            else:
                run_f(colg, None, lin, 0, GS, self.packed["Wg_last"], GS, 64, cin, tap_ranges("full", 0, 64, cin),
                      g_in, GS, lin, 0, 0, lin, B, d_lo=0, d_hi=0, w_tap0=4, backend=self.backend)
            # dW'[n=(s,k)][kc=(src,s',c)] over position pairs; the s == s' blocks are the gradient: folded (and
            # cleared for the next step) by sg_last_deconv_wgrad_fold into dW (alpha on the skip half) and dalpha
            dwq = buf.get("g.dwq_last", (128 * 2 * cin,), F32, dev)
            if not self.has_skip:
                # one source: kc = (s', c) over the decoder output alone, folded without alpha
                with on_side(side):
                    run_w(colg, lin // 2, GS, ctx["ddb"][l - 1], None, lin // 2, 0, GS, 2 * cin, 128,
                          tap_ranges("full", 0, 2 * cin, 128), dwq, B, d_lo=0, d_hi=0, dw_tap0=4, ksplit=74,
                          a0_c=2 * cin, backend=self.backend)
                    _lib.call("sg_last_deconv_wgrad_fold_1src_kw", _p(dwq), cin, kl,
                              _p(wgrad_dst(self.wname("dec", l))), _stream())
                    if sn_small:
                        self._sn_fix_small(self.wname("dec", l), sn_small[self.wname("dec", l)], slot)
            else:
                a_train = not self.conv_skip and self._param("alpha_0.skip_k").requires_grad
                with on_side(side):
                    run_w(colg, lin // 2, GS, ctx["ddb"][l - 1], ctx["skb"][0], lin // 2, 0, GS, 2 * cin, 128,
                          tap_ranges("full", 0, 2 * cin, 128), dwq, B, d_lo=0, d_hi=0, dw_tap0=4, ksplit=74,
                          a0_c=cin, a1_c=cin, backend=self.backend)
                    gw_dst = wgrad_dst(self.wname("dec", l))
                    if self.sum_merge:
                        gw_dst = buf.get("g.gw_last2", (cin, 1, kl), F32, dev, zero=True)
                    # snorm: w_last_dup is W / sigma, so the fold's dalpha is <dWeff, W~> as the reference's
                    _lib.call("sg_last_deconv_wgrad_fold_kw", _p(dwq), half, kl, _p(self.packed["w_last_dup"]),
                              _p(self.alpha_for_dec(l)), _p(gw_dst),
                              _p(self.gview("alpha_0.skip_k").view(-1)) if a_train else None, _stream())
                    if self.sum_merge:
                        wgrad_dst(self.wname("dec", l)).add_(gw_dst[:half] + gw_dst[half:])
                    if sn_small:
                        self._sn_fix_small(self.wname("dec", l), sn_small[self.wname("dec", l)], slot)
        else:
            if not self.has_skip:
                raise NotImplementedError("a Generator without skips (skip=False) needs the tensor-core waveform "
                                          "route (SEGAN_B200_WAVE=tc)")
            if self.conv_skip:
                raise NotImplementedError("skip_type='conv' needs the tensor-core waveform route (SEGAN_B200_WAVE=tc)")
            dweff = buf.get("g.dweff", (cin, self.kw_dec[l]), F32, dev, zero=True)
            _lib.call("sg_wave_deconv_bwd", _p(src0), half, _p(src1), half, B, lin, _p(self.packed["w_last_eff"]),
                      _p(gy), _p(ctx["y"]), _p(gpre), _p(g_in), _p(dweff), _p(gb), st)
            if self.sum_merge:
                raise NotImplementedError("skip_merge='sum' needs the tensor-core waveform route (SEGAN_B200_WAVE=tc)")
            w_last = self.pview("dec_blocks.%d.deconv.weight" % l)[:, 0, :]
            alpha = self.alpha_for_dec(l)
            gw = self.gview("dec_blocks.%d.deconv.weight" % l)[:, 0, :]
            gw[:half] += dweff[:half]
            gw[half:] += dweff[half:] * alpha.view(-1, 1)
            self.gview("alpha_0.skip_k").view(-1).add_((dweff[half:] * w_last[half:]).sum(1))
        # ---- decoder blocks nl-2 .. 0
        g_next = g_in            # gradient w.r.t. cat(dd[l-1], alpha*a_skip) of block l
        for l in range(nl - 2, -1, -1):
            cin, cout = self.dec_cin(l), self.dec_cout(l)
            lin = Lq[nl - 1 - l]
            cnext = g_next.shape[-1]
            # PReLU backward on [B, 4*lin, cout]
            g_ad = buf.get("g.gad%d" % l, (B, lin, 4 * cout), GT, dev)
            red = red_dec[l]
            _lib.call("sg_act_bwd_reduce", _p(g_next), cnext, 0, 0, None, None, 0, _p(ad[l]), SG_F16, B, 4 * lin, cout,
                      None, None, _p(self.pview("dec_blocks.%d.act.weight" % l)), ACT_PRELU, _p(red), _p(g_ad), st)
            _lib.call("sg_stat_grads", _p(red), cout, 3, _p(self.gview("dec_blocks.%d.act.weight" % l)),
                      _p(self.gview("dec_blocks.%d.deconv.bias" % l)), None, st)
            sn_coef(red, self.pview("dec_blocks.%d.deconv.bias" % l), cout, self.wname("dec", l))
            if l == 0:
                s0, s1 = (ctx["z16b"], ctx["hpb"][nl - 1]) if self.zc else (ctx["hpb"][nl - 1], None)
            else:
                s0, s1 = ctx["ddb"][l - 1], (ctx["skb"][nl - 1 - l] if self.has_skip else None)
            c0, c1 = s0.shape[-1], (0 if s1 is None else s1.shape[-1])
            taps = tap_ranges("deconv_fwd", cout, cin, 4 * cout, self.kw_dec[l])
            d_lo, d_hi = tap_span(taps)
            taps_dg = tap_ranges("deconv_dgrad", cout, 4 * cout, cin, self.kw_dec[l])
            dg_lo, dg_hi = dgrad_span(taps)
            dwp = self.mgrad(self.by_name[self.wname("dec", l)])     # packed gradient slot (dWeff; snorm: / sigma)
            with on_side(side):
                n_tiles = 9 * (4 * cout // 128) * max(1, cin // 256)
                run_w(g_ad, lin, GS, s0, s1, lin, 0, GS, cin, 4 * cout, taps, dwp, B, d_lo=d_lo, d_hi=d_hi,
                      ksplit=wgrad_ksplit(B * lin, n_tiles, taps, cin, 4 * cout, d_lo, d_hi), a0_c=c0, a1_c=c1,
                      backend=self.backend, out_scale=osc(self.wname("dec", l)))
                if l == 0 and reducer is not None:
                    reducer.ready(0, launch=True)              # every decoder weight gradient has been enqueued
            # data gradient w.r.t. cat(s0, s1); block 0 only needs the code's columns [zc, zc + C) (z gets no
            # gradient)
            if self.conv_skip and l > 0:
                g_in = buf.get("g.gin%d" % l, (B, lin, cin // 2), GT, dev)
                for dst, n0 in ((g_in, 0), (buf.get("g.gsk%d" % (nl - 1 - l), (B, lin, cin // 2), GT, dev), cin // 2)):
                    run_f(g_ad, None, lin, 0, GS, self.packed["Wtd%d" % l], GS, 4 * cout, cin,
                          taps_dg, dst, GS, lin, 0, 0, lin, B, d_lo=dg_lo, d_hi=dg_hi,
                          n_lo=n0, n_hi=n0 + cin // 2, out_ld=cin // 2, out_col0=0, backend=self.backend)
            else:
                g_in = buf.get("g.gin%d" % l, (B, lin, cin), GT, dev)
                run_f(g_ad, None, lin, 0, GS, self.packed["Wtd%d" % l], GS, 4 * cout, cin,
                      taps_dg, g_in, GS, lin, 0, 0, lin, B, d_lo=dg_lo, d_hi=dg_hi,
                      n_lo=(self.zc if l == 0 else 0), n_hi=cin, backend=self.backend)
            g_next = g_in
        # ---- encoder blocks nl-1 .. 0
        g_hp = None
        for l in range(nl - 1, -1, -1):
            cout = fm[l]
            g_a = buf.get("g.ga%d" % l, (B, Lq[l], cout), GT, dev)
            red = red_enc[l]
            slope = self.pview("enc_blocks.%d.act.weight" % l)
            if l == nl - 1:
                gin0 = buf.t["g.gin0"]                  # [B][Lq][zc + C]: the code's gradient from column zc
                gh_ptr = C.c_void_p(gin0.data_ptr() + 2 * self.zc)
                _lib.call("sg_act_bwd_reduce", gh_ptr, gin0.shape[-1], 0, 0, None, None, 0, _p(a[l]), SG_F16, B, Lq[l],
                          cout, None, None, _p(slope), ACT_PRELU, _p(red), _p(g_a), st)
            else:
                if not self.has_skip:
                    gadd_ptr, gadd_ld = None, 0
                elif self.conv_skip:
                    gadd_ptr, gadd_ld = _p(self._skip_conv_bwd(l, ctx, side)), cout
                else:
                    gsk = buf.t["g.gin%d" % (nl - 1 - l)]
                    gadd_ptr, gadd_ld = C.c_void_p(gsk.data_ptr() + 2 * (gsk.shape[-1] // 2)), gsk.shape[-1]
                _lib.call("sg_act_bwd_reduce", _p(g_hp), cout, 16, 0, None, gadd_ptr, gadd_ld, _p(a[l]), SG_F16,
                          B, Lq[l], cout, None, None, _p(slope), ACT_PRELU, _p(red), _p(g_a), st)
            _lib.call("sg_stat_grads", _p(red), cout, 3, _p(self.gview("enc_blocks.%d.act.weight" % l)),
                      _p(self.gview("enc_blocks.%d.conv.bias" % l)) if self.enc_bias else None, None, st)
            if l == 0:
                dwq = buf.get("g.dwq0", (128 * 128,), F32, dev)
                with on_side(side):
                    if ctx.get("colb") is not None:
                        run_w(g_a, Lq[0] // 2, GS, ctx["colb"], None, Lq[0] // 2, 0, GS, 128, 128,
                              tap_ranges("full", 0, 128, 128), dwq, B, d_lo=0, d_hi=0, dw_tap0=4, ksplit=148,
                              backend=self.backend)
                        _lib.call("sg_wave_wgrad_fold_kw", _p(dwq), 1, self.kw_enc[0],
                                  _p(wgrad_dst(self.wname("enc", 0))), _stream())
                    else:
                        _lib.call("sg_wave_conv_wgrad", _p(ctx["x"]), None, 1, B, L, 0, _p(g_a), cout,
                                  _p(self.gview("enc_blocks.0.conv.weight")), None, _stream())
                    if sn_small:
                        self._sn_fix_small(self.wname("enc", 0), sn_small[self.wname("enc", 0)], slot)
                break
            sn_coef(red, self.pview("enc_blocks.%d.conv.bias" % l) if self.enc_bias else None, cout,
                    self.wname("enc", l))
            cin = fm[l - 1]
            taps = tap_ranges("conv_fwd", cin, 4 * cin, cout, self.kw_enc[l])
            d_lo, d_hi = tap_span(taps)
            dwp_l = self.mgrad(self.by_name[self.wname("enc", l)])
            with on_side(side):
                n_tiles = 9 * (cout // 128) * max(1, 4 * cin // 256)
                run_w(g_a, Lq[l], GS, ctx["hpb"][l - 1], None, Lq[l], 4, GS, 4 * cin, cout, taps, dwp_l, B,
                      d_lo=d_lo, d_hi=d_hi, ksplit=wgrad_ksplit(B * Lq[l], n_tiles, taps, 4 * cin, cout, d_lo, d_hi),
                      backend=self.backend, out_scale=osc(self.wname("enc", l)))
                if l == nl - 1 and reducer is not None:
                    reducer.ready(1, launch=True)
            g_hp = buf.get("g.ghp%d" % (l - 1), (B, Lq[l] + 8, 4 * cin), GT, dev)
            dg_lo, dg_hi = dgrad_span(taps)
            run_f(g_a, None, Lq[l], 0, GS, self.packed["Wdg%d" % l], GS, cout, 4 * cin,
                  tap_ranges("conv_dgrad", cin, cout, 4 * cin, self.kw_enc[l]), g_hp, GS, Lq[l], 4, -4, Lq[l] + 4, B,
                  d_lo=dg_lo, d_hi=dg_hi, backend=self.backend)
        join_side(side)
        if reducer is not None:
            reducer.ready(2, launch=True)
        return self.grad

    def _skip_conv_bwd(self, l, ctx, side):
        """Backward of the skip conv of encoder level l given the gradient of its output (g.gsk<l>, [B][Lq][C]):
        the data gradient w.r.t. a[l] is returned ([B][Lq][C], the encoder's extra pre-activation gradient); the
        weight gradient (tap-GEMM into a workspace of the grouped layout, folded into reference layout) and the
        bias gradient run on `side`, which serialises the levels' use of the one workspace."""
        buf, B, lq = self.buf, ctx["B"], ctx["Lq"][l]
        c, dev = self.fmaps[l], self.flat.device
        D = (self.skip_kw // 2 + 3) // 4
        d_lo, d_hi, tap0, taps, taps_dg = skipconv_geometry(c, self.skip_kw)
        g_s = buf.t["g.gsk%d" % l]
        g_a = buf.get("g.gask%d" % l, (B, lq, c), GT, dev)
        run_f(g_s, None, lq // 4, 0, GS, self.packed["Wskd%d" % l], GS, 4 * c, 4 * c, taps_dg, g_a, GS, lq // 4, 0, 0,
              lq // 4, B, d_lo=d_lo, d_hi=d_hi, w_tap0=tap0, backend=self.backend)
        cmax = self.fmaps[self.nl - 2]
        ws = buf.get("g.dwq_sk", ((2 * D + 1) * 16 * cmax * cmax,), F32, dev)     # left zeroed by every fold
        dwq = ws[:(2 * D + 1) * 16 * c * c]
        with on_side(side):
            run_w(g_s, lq // 4, GS, ctx["ab"][l], None, lq // 4, 0, GS, 4 * c, 4 * c, taps, dwq, B, d_lo=d_lo,
                  d_hi=d_hi, dw_tap0=tap0, ksplit=wgrad_ksplit(B * lq // 4, 0, taps, 4 * c, 4 * c, d_lo, d_hi),
                  backend=self.backend)
            _lib.call("sg_skipconv_wgrad_fold", _p(dwq), c, self.skip_kw,
                      _p(self.gview("alpha_%d.skip_k.weight" % l)), _stream())
            bias_name = "alpha_%d.skip_k.bias" % l
            if bias_name in self.index:
                tmp = buf.get("g.sk_tmp", (SL * cmax,), F64, dev)
                _lib.call("sg_colsum", _p(g_s), GS, B * lq, c, c, _p(self.gview(bias_name)), 1, _p(tmp), _stream())
        return g_a


# ============================================================================================
# Discriminator
# ============================================================================================
class DiscriminatorEngine(_SpectralNorm, _NetEngine):
    def __init__(self, module):
        super().__init__(module)
        self.fmaps = list(module.fmaps)
        self.nl = len(self.fmaps)
        self.kw = module.enc_blocks[0].kwidth          # one width for every tower conv (Discriminator._served: 4..32)
        self.packed = {}
        self.eps = 1e-5
        self.momentum = 0.1
        # norm_type='snorm' (modules.py:12-14, discriminator.py:118-121): no BatchNorm; every conv, fc.0, fc.2 and the
        # fc.3 PReLU slope vector are divided by their spectral norm, re-estimated by one power iteration per
        # training forward (sg_snorm_sigma).  The parameters are then called weight_orig.
        self.snorm = getattr(module, "norm_type", "bnorm") == "snorm"
        self.wsfx = "_orig" if self.snorm else ""
        self.sn = {}                # name -> spectral-norm state (see _sn_state)
        self._sn_pass = 0           # forward passes with parameter gradients since the last zero_grad
        self._sn_slot = 0           # slot of the pass whose operands are current
        # lane 1: a second workspace so that one pass (the real pair of a train step) can run on its own stream
        # concurrently with another pass of the same network.  Both lanes accumulate into the SAME gradient
        # bucket: every parameter-gradient writer is atomic (red.add in the wgrad epilogue, atomicAdd elsewhere).
        self.buf1 = _Buffers()
        # pool_type 'none': fc.0 (a tap-GEMM) + sg_fc_tail; 'conv' / 'gmax' / 'gavg': the small pooled heads of
        # discriminator.py:122-137, one sg_dhead_fwd / _bwd launch each; 'mlp' (discriminator.py:138-143): its
        # C x C 1x1 conv mlp.0 is a single-tap tap-GEMM over the B * Lq positions, the PReLU(C) mlp.1 runs on the
        # tower's activation kernels and the per-position C -> 1 conv mlp.2 + loss on sg_dhead_fwd / _bwd
        self.pool_type = getattr(module, "pool_type", "none")

    def packed_layers(self):
        """Bucket order = gradient completion order of a backward pass: [fc.0 | mlp.0,] enc4 | enc3 .. enc1, small."""
        fm = self.fmaps
        ls = []
        if self.pool_type == "none":
            nout, kin = self._param("fc.0.weight" + self.wsfx).shape
            ls.append(PackedLayer("fc.0.weight" + self.wsfx, 2, nout, fm[-1], kin // fm[-1], "W1p", "W1dg"))
        elif self.pool_type == "mlp":        # Conv1d(C, C, 1) weight [C][C][1] = a Linear with t_len 1
            ls.append(PackedLayer("mlp.0.weight" + self.wsfx, 2, fm[-1], fm[-1], 1, "Wm0", "Wm0dg"))
        ls += [PackedLayer("enc_blocks.%d.conv.weight%s" % (l, self.wsfx), 0, fm[l], fm[l - 1], 0, "Wf%d" % l, "Wdg%d" % l,
                           kw=self.kw)
               for l in range(self.nl - 1, 0, -1)]
        return ls

    # -- spectral norm (state: _SpectralNorm) ------------------------------------------------------
    # the head's spectrally normalised tensors (discriminator.py:118-121,125-137)
    HEAD_SN = {"none": ("fc.0.weight_orig", "fc.2.weight_orig", "fc.3.weight_orig"),
               "conv": ("pool_conv.weight_orig", "fc.weight_orig"), "gmax": ("fc.weight_orig",),
               "gavg": ("fc.weight_orig",), "mlp": ("mlp.0.weight_orig", "mlp.1.weight_orig")}

    def _sn_names(self):
        return ["enc_blocks.%d.conv.weight_orig" % l for l in range(self.nl)] + list(self.HEAD_SN[self.pool_type])

    def _sn_iterate(self, training, slot):
        """sigma of every normalised weight for the coming pass (one power iteration when training), kept in pass
        slot `slot` together with copies of the vectors: the backward of that pass and the sigma terms need them."""
        st_ = _stream()
        for name in self._sn_names():
            st = self._sn_state(name)
            _lib.call("sg_snorm_sigma", _p(self._sn_master(name)), st["T"], st["nc"], st["kc"], _p(st["u"]), _p(st["v"]),
                      _p(st["scal"][slot]), _p(st["work"]), 1 if training else 0, st_)
            st["u_p"][slot].copy_(st["u"])
            st["v_p"][slot].copy_(st["v"].reshape(-1))
        self._sn_slot = slot

    def zero_grad(self):
        super().zero_grad()
        self._sn_pass = 0

    def finish_grads(self):
        """snorm: the sigma terms of every accumulating pass of this step, one sweep per tap-GEMM layer
        (dW -= sum_p coef_p u_p v_p^T; the G / sigma_p part was applied by the weight-gradient GEMMs)."""
        if self._alpha_fixed:
            return
        if self.snorm and self._sn_pass > 0:
            for pl in self.layers:
                stt = self._sn_state(pl.name)
                _lib.call("sg_snorm_rank1", _p(self.mgrad(pl)), pl.T, pl.nc, pl.kc, self._sn_pass, _p(stt["u_p"]),
                          _p(stt["v_p"]), _p(stt["coef"]), _stream())
        self._alpha_fixed = True

    def grad_chunks(self):
        """[fc.0 | mlp.0 +] enc4 (complete once the last tower layer's weight gradient is enqueued) | the rest."""
        a = sum(l.numel for l in self.layers[:2 if self.pool_type in ("none", "mlp") else 1])
        return [(0, a), (a, self.grad.numel() - a)]

    def pack(self):
        dev = self.flat.device
        w0 = self.pview("enc_blocks.0.conv.weight" + self.wsfx)
        if self.snorm:
            w0 = w0 * self.sn_inv_sigma("enc_blocks.0.conv.weight_orig")
            # the head's small normalised tensors, consumed by sg_fc_tail_fwd / _bwd or sg_dhead_fwd / _bwd
            for nm in self.HEAD_SN[self.pool_type]:
                if nm not in self.by_name:          # fc.0 / mlp.0: packed layers, emitted with their 1/sigma below
                    self.packed[nm + "/n"] = (self.pview(nm) * self.sn_inv_sigma(nm)).contiguous()
        wcol = wave_col_weights(w0, dev)
        self.packed["Wcol0"] = wcol.half().contiguous()
        self.packed["WcolT0"] = wcol.t().to(GT).contiguous()
        self._mark_packed("small")
        for pl in self.layers:
            self.emit(pl, scale=self.sn_inv_sigma(pl.name) if self.snorm else None)
            if pl.f_key == "W1p":  # fc.0's operands are used as 2-D [nout][kin] / [kin][nout]
                self.packed["W1p"] = self.packed["W1p"].view(pl.nc, pl.kc)
                self.packed["W1dg"] = self.packed["W1dg"].view(pl.kc, pl.nc)

    def forward(self, x0, x1, shifts, training=True, fresh=False, twins=True, lane=0, shifts_dev=None):
        """x0: candidate (B,1,L), x1: reference/noisy (B,1,L) -- the reference's cat((x_, ref), 1)
        (model.py:173-175) is never materialised.  shifts: nl signed phase shifts.  shifts_dev: optional
        device int32 tensor holding the same nl shifts; the kernels then read them from memory (no
        per-step scalar in the launches, so the step can be replayed from a CUDA graph)."""
        _require_cuda(x0, x1)
        if self.kw != 31 and not wave_on_tensor_cores():
            raise NotImplementedError("Discriminator kernel widths other than 31 need the tensor-core waveform route "
                                      "(SEGAN_B200_WAVE=tc)")
        alias = twins and not grad_twins()
        twins = twins and grad_twins()
        sn_slot = None
        if self.snorm:
            # a new sigma (training: after one more power iteration) for this pass -> the operands are re-emitted
            self.bind()
            self.notice_external_writes()
            if training and twins_or_alias(alias, twins):
                sn_slot = self._sn_pass
                assert sn_slot < self.SN_SLOTS - 1, "more accumulating D passes per optimiser step than SN_SLOTS"
                self._sn_pass += 1
            else:
                sn_slot = self.SN_SLOTS - 1               # gradient-free pass (G step, inference)
            self._sn_iterate(training, sn_slot)
            self._ops_stale = True
        self.ensure_packed()
        self.wait_packed("small")
        m = self.module
        B, _, L = x0.shape
        fm, nl, dev, st = self.fmaps, self.nl, x0.device, _stream()
        buf = _Buffers() if fresh else (self.buf1 if lane == 1 else self.buf)
        x0 = x0.contiguous().float()
        x1 = x1.contiguous().float()
        Lq = [L // 4 ** (l + 1) for l in range(nl)]
        if self.pool_type == "none":
            assert Lq[-1] * fm[-1] == self._param("fc.0.weight" + self.wsfx).shape[1], "D expects L = 16384"
        elif self.pool_type == "conv":
            assert Lq[-1] == self._param("fc.weight" + self.wsfx).shape[1], "D expects L = 4^n_layers * pool_slen"
        if shifts_dev is not None and not wave_on_tensor_cores():
            raise _lib.SeganB200Error("device-resident phase shifts need the tensor-core waveform route")

        def rptr(i):
            return None if shifts_dev is None else C.c_void_p(shifts_dev.data_ptr() + 4 * i)
        a, hp, ss, mi, hpb = [None] * nl, [None] * nl, [None] * nl, [None] * nl, [None] * nl
        bnorm = not self.snorm
        stats = stat_arena(buf, "d.stats", [(SL, 2, fm[l]) for l in range(nl)], dev) if (training and bnorm) else None
        # BatchNorm statistics in the conv epilogue (tensor-core kernel; used with B * L/4 >= 256)
        eff_backend = default_backend() if self.backend is None else self.backend
        fuse_stats = (training and bnorm and FUSE_BN_STATS and eff_backend == BACKEND_TCGEN05 and B * Lq[-1] >= 256)
        for l in range(nl):
            cout = fm[l]
            a[l] = buf.get("d.a%d" % l, (B, Lq[l], cout), F16, dev)
            bias = self.pview("enc_blocks.%d.conv.bias" % l) if m.bias else None
            colb = None
            if l == 0 and wave_on_tensor_cores():
                col16 = buf.get("d.col16", (B, Lq[0], 64), F16, dev)
                colb0 = buf.get("d.colb", (B, Lq[0], 64), GT, dev) if twins else None
                _lib.call("sg_wave_im2col_kw", _p(x0), _p(x1), 2, B, L, int(shifts[0]), rptr(0), 1, conv_offset(self.kw),
                          self.kw, _p(col16), _p(colb0), st)
                if alias:
                    colb0 = col16
                self.wait_packed("small")
                run_f(col16, None, Lq[0], 0, SG_F16, self.packed["Wcol0"], SG_F16, 64, 64,
                      tap_ranges("full", 0, 64, 64), a[0], SG_F16, Lq[0], 0, 0, Lq[0], B, bias=bias, bias_mod=64,
                      d_lo=0, d_hi=0, w_tap0=4, backend=self.backend, stats=stats[0] if fuse_stats else None)
            elif l == 0:
                colb0 = None
                w0 = self.pview("enc_blocks.0.conv.weight" + self.wsfx)
                if self.snorm:
                    w0 = (w0 * self.sn_inv_sigma("enc_blocks.0.conv.weight_orig")).contiguous()
                _lib.call("sg_wave_conv_fwd", _p(x0), _p(x1), 2, B, L, int(shifts[0]),
                          _p(w0), _p(bias), cout, _p(a[0]), None, None, st)
            else:
                cin = fm[l - 1]
                self.wait_packed("Wf%d" % l)
                taps = tap_ranges("conv_fwd", cin, 4 * cin, cout, self.kw)
                d_lo, d_hi = tap_span(taps)
                run_f(hp[l - 1], None, Lq[l], 4, SG_F16, self.packed["Wf%d" % l], SG_F16, 4 * cin, cout,
                      taps, a[l], SG_F16, Lq[l], 0, 0, Lq[l], B, d_lo=d_lo, d_hi=d_hi,
                      bias=bias, bias_mod=cout, backend=self.backend, stats=stats[l] if fuse_stats else None)
            bn = m.enc_blocks[l].norm
            if bnorm:
                ss[l] = buf.get("d.ss%d" % l, (2, cout), F32, dev)
                mi[l] = buf.get("d.mi%d" % l, (2, cout), F32, dev)
            if not bnorm:
                pass                                   # snorm: conv -> PReLU, no statistics
            elif training:
                st2 = stats[l]
                if not (fuse_stats and (l > 0 or wave_on_tensor_cores())):
                    _lib.call("sg_bn_stats", _p(a[l]), SG_F16, B * Lq[l], cout, _p(st2), st)
                _lib.call("sg_bn_finalize", _p(st2), B * Lq[l], cout,
                          _p(self.pview("enc_blocks.%d.norm.weight" % l)),
                          _p(self.pview("enc_blocks.%d.norm.bias" % l)), self.eps, self.momentum,
                          _p(bn.running_mean), _p(bn.running_var), _p(ss[l]), _p(mi[l]), st)
                bn.num_batches_tracked += 1
            else:
                invstd = torch.rsqrt(bn.running_var + self.eps)
                sc = self.pview("enc_blocks.%d.norm.weight" % l) * invstd
                ss[l][0].copy_(sc)
                ss[l][1].copy_(self.pview("enc_blocks.%d.norm.bias" % l) - bn.running_mean * sc)
                mi[l][0].copy_(bn.running_mean)
                mi[l][1].copy_(invstd)
            halo = 16 if l < nl - 1 else 0
            roll = int(shifts[l + 1]) if l < nl - 1 else 0
            hp[l] = buf.get("d.hp%d" % l, (B, Lq[l] + 2 * halo, cout), F16, dev)
            hpb[l] = buf.get("d.hpb%d" % l, (B, Lq[l] + 2 * halo, cout), GT, dev) if twins else None
            _lib.call("sg_act_fwd", _p(a[l]), SG_F16, B, Lq[l], cout, _p(ss[l]),
                      _p(self.pview("enc_blocks.%d.act.weight" % l)), ACT_PRELU, roll, rptr(l + 1) if l < nl - 1 else None,
                      halo, _p(hp[l]), _p(hpb[l]), None, st)
            if alias:
                hpb[l] = hp[l]
        if self.pool_type == "mlp":
            logit, head = self._mlp_head_fwd(hp[-1], B, Lq[-1], buf)
        elif self.pool_type != "none":
            logit = torch.empty(B, 1, dtype=F32, device=dev)
            head = self._pool_head_fwd(hp[-1], B, Lq[-1], buf, logit)
        else:
            # ---- FC head
            kin = Lq[-1] * fm[-1]
            acc = buf.get("d.fc0", (B, 256), F32, dev, zero=True)
            self.wait_packed("W1p")
            run_f(hp[-1], None, 1, 0, SG_F16, self.packed["W1p"], SG_F16, kin, 256,
                  tap_ranges("full", 0, kin, 256), acc, SG_F32, 1, 0, 0, 1, B, d_lo=0, d_hi=0, w_tap0=4,
                  ksplit=16, backend=self.backend)
            z1 = buf.get("d.z1", (B, 256), F32, dev)
            z2 = buf.get("d.z2", (B, 128), F32, dev)
            logit = torch.empty(B, 1, dtype=F32, device=dev)
            w2 = self.packed["fc.2.weight_orig/n"] if self.snorm else self.pview("fc.2.weight")
            s3 = self.packed["fc.3.weight_orig/n"] if self.snorm else self.pview("fc.3.weight")
            _lib.call("sg_fc_tail_fwd", _p(acc), _p(self.pview("fc.0.bias")), _p(self.pview("fc.1.weight")),
                      _p(w2), _p(self.pview("fc.2.bias")), _p(s3),
                      _p(self.pview("fc.4.weight")), _p(self.pview("fc.4.bias")), B, _p(z1), _p(z2), _p(logit), st)
            head = dict(z1=z1, z2=z2, acc=acc, w2=w2, s3=s3)
        self.packs_consumed()
        ctx = dict(x0=x0, x1=x1, B=B, L=L, Lq=Lq, a=a, hp=hp, hpb=hpb, colb=colb0, ss=ss, mi=mi,
                   logit=logit, lane=lane, shifts_dev=shifts_dev, sn_slot=sn_slot,
                   shifts=[int(s) for s in shifts], **head)
        return logit, ctx

    # -- pooled heads (pool_type 'conv' / 'gmax' / 'gavg') --------------------------------------------
    def _head_weights(self):
        """(pool_conv weight, pool_conv bias, fc weight, fc bias) as the head kernels read them: the spectrally
        normalised copies made by pack() where norm_type='snorm'; the pool_conv entries are None without one."""
        w = lambda nm: self.packed[nm + "_orig/n"] if self.snorm else self.pview(nm)
        pw = w("pool_conv.weight") if self.pool_type == "conv" else None
        pb = self.pview("pool_conv.bias") if self.pool_type == "conv" else None
        return pw, pb, w("fc.weight"), self.pview("fc.bias")

    def _pool_head_fwd(self, h, B, lq, buf, logit):
        """h: the last tower activation [B][lq][C] fp16.  Fills logit (B, 1); returns the head's saved tensors."""
        dev, c = h.device, self.fmaps[-1]
        kind = DHEAD_KINDS[self.pool_type]
        pw, pb, fw, fb = self._head_weights()
        pooled = buf.get("d.pooled", (B, lq if kind == SG_DHEAD_CONV else c), F32, dev)
        argmax = buf.get("d.argmax", (B, c), torch.int32, dev) if kind == SG_DHEAD_GMAX else None
        _lib.call("sg_dhead_fwd", kind, _p(h), B, lq, c, _p(pw), _p(pb), _p(fw), _p(fb), _p(pooled), _p(argmax),
                  _p(logit), _stream())
        return dict(pooled=pooled, argmax=argmax, pw=pw, fw=fw)

    def _mlp_head_fwd(self, h, B, lq, buf):
        """pool_type 'mlp' on the last tower activation h [B][lq][C] fp16: logits (B, 1, lq) and the saved tensors."""
        dev, c, rows, st = h.device, self.fmaps[-1], B * lq, _stream()
        pl = self.by_name["mlp.0.weight" + self.wsfx]
        z = buf.get("d.mlp.z", (B, lq, c), F16, dev)
        self.wait_packed(pl.f_key)
        run_f(h, None, rows, 0, SG_F16, self.packed[pl.f_key], SG_F16, c, c, tap_ranges("full", 0, c, c), z, SG_F16,
              rows, 0, 0, rows, 1, bias=self.pview("mlp.0.bias"), bias_mod=c, d_lo=0, d_hi=0, w_tap0=4,
              backend=self.backend)
        slope = self.packed["mlp.1.weight_orig/n"] if self.snorm else self.pview("mlp.1.weight")
        hm = buf.get("d.mlp.h", (B, lq, c), F16, dev)
        _lib.call("sg_act_fwd", _p(z), SG_F16, B, lq, c, None, _p(slope), ACT_PRELU, 0, None, 0, _p(hm), None, None, st)
        logit = torch.empty(B, 1, lq, dtype=F32, device=dev)
        _lib.call("sg_dhead_fwd", SG_DHEAD_MLP, _p(hm), B, lq, c, _p(self.pview("mlp.2.weight")),
                  _p(self.pview("mlp.2.bias")), None, None, None, None, _p(logit), st)
        return logit, dict(mlp_z=z, mlp_h=hm, mlp_slope=slope)

    def _mlp_head_bwd(self, ctx, target, weight, param_grads, loss_out, g_logit, g_h, buf, slot, side):
        """Loss + backward of the mlp head: mlp.2 and the loss in sg_dhead_bwd, the PReLU through the tower's
        activation backward (its slope and mlp.0's bias from the reduction), mlp.0's weight gradient on the side
        stream and its data gradient into g_h."""
        B, lq, c, st = ctx["B"], ctx["Lq"][-1], self.fmaps[-1], _stream()
        dev, rows, sn = g_h.device, B * lq, self.snorm
        pl = self.by_name["mlp.0.weight" + self.wsfx]
        g_hm = buf.get("d.mlp.gh", (B, lq, c), GT, dev)
        gv = (lambda n: _p(self.gview(n))) if param_grads else (lambda n: None)
        _lib.call("sg_dhead_bwd", SG_DHEAD_MLP, _p(ctx["mlp_h"]), B, lq, c, _p(self.pview("mlp.2.weight")), None, None,
                  None, _p(ctx["logit"]), _p(g_logit), float(target), float(weight), _p(loss_out), _p(g_hm),
                  gv("mlp.2.weight"), gv("mlp.2.bias"), None, None, float(LOSS_SCALE), st)
        red = buf.get("d.mlp.red", (SL, 3, c), F64, dev, zero=True)
        g_z = buf.get("d.mlp.gz", (B, lq, c), GT, dev)
        _lib.call("sg_act_bwd_reduce", _p(g_hm), c, 0, 0, None, None, 0, _p(ctx["mlp_z"]), SG_F16, B, lq, c, None, None,
                  _p(ctx["mlp_slope"]), ACT_PRELU, _p(red), _p(g_z), st)
        taps = tap_ranges("full", 0, c, c)
        if param_grads:
            g_slope = buf.get("d.sng.mlp.1", (c,), F32, dev, zero=True) if sn else self.gview("mlp.1.weight")
            # red is [SL][3][C] (sg_stat_grads strides its slices by n_stats): 3 statistics, the third unused
            _lib.call("sg_stat_grads", _p(red), c, 3, _p(g_slope), _p(self.gview("mlp.0.bias")), None, st)
            osc = None
            if sn:
                self._sn_fix_small("mlp.1.weight_orig", g_slope, slot)
                stt = self._sn_state(pl.name)
                _lib.call("sg_snorm_coef", _p(red), _p(self.pview("mlp.0.bias")), c, _p(stt["scal"][slot]),
                          _p(stt["coef"][slot:slot + 1]), st)
                osc = stt["scal"][slot][3:4]
            with on_side(side):
                run_w(g_z, rows, GS, ctx["hpb"][-1], None, rows, 0, GS, c, c, taps, self.mgrad(pl), 1, d_lo=0, d_hi=0,
                      dw_tap0=4, ksplit=wgrad_ksplit(rows, 0, taps, c, c, 0, 0), backend=self.backend, out_scale=osc)
        run_f(g_z, None, rows, 0, GS, self.packed[pl.dg_key], GS, c, c, taps, g_h, GS, rows, 0, 0, rows, 1, d_lo=0,
              d_hi=0, w_tap0=4, backend=self.backend)

    def _pool_head_bwd(self, ctx, target, weight, param_grads, loss_out, g_logit, g_h, buf, slot):
        """Loss + backward of a pooled head into g_h (every element written) and, with param_grads, the head's
        parameter gradients into the bucket (snorm: through per-pass scratch gradients and sg_snorm_grad)."""
        B, lq, c = ctx["B"], ctx["Lq"][-1], self.fmaps[-1]
        kind = DHEAD_KINDS[self.pool_type]
        conv = kind == SG_DHEAD_CONV
        g = {}
        if param_grads:
            for nm in ("pool_conv.weight", "pool_conv.bias", "fc.weight", "fc.bias"):
                if not conv and nm.startswith("pool_conv"):
                    continue
                if self.snorm and nm.endswith("weight"):
                    g[nm] = buf.get("d.sng." + nm, self.index[nm + "_orig"][2], F32, ctx["x0"].device, zero=True)
                else:
                    g[nm] = self.gview(nm)
        _lib.call("sg_dhead_bwd", kind, _p(ctx["hp"][-1]), B, lq, c, _p(ctx["pw"]), _p(ctx["fw"]), _p(ctx["pooled"]),
                  _p(ctx["argmax"]), _p(ctx["logit"]), _p(g_logit), float(target), float(weight), _p(loss_out),
                  _p(g_h), _p(g.get("pool_conv.weight")), _p(g.get("pool_conv.bias")), _p(g.get("fc.weight")),
                  _p(g.get("fc.bias")), float(LOSS_SCALE), _stream())
        if param_grads and self.snorm:
            for nm in self.HEAD_SN[self.pool_type]:
                self._sn_fix_small(nm, g[nm[:-len("_orig")]], slot)

    def backward(self, ctx, target, weight=1.0, param_grads=True, input_grad=None, loss_out=None, g_logit=None,
                 input_grad1=None, reducer=None, reduce_now=True):
        """Backward of  weight * mean((logit - target)^2)  (nn.MSELoss, model.py:298,305,316).
        param_grads: accumulate parameter gradients into self.grad (D steps) or skip them (G step).
        input_grad: optional fp32 (B,1,L) buffer that receives (+=) the gradient w.r.t. x0."""
        m = self.module
        lane = ctx.get("lane", 0)
        shifts_dev = ctx.get("shifts_dev")

        def rptr(i):
            return None if shifts_dev is None else C.c_void_p(shifts_dev.data_ptr() + 4 * i)
        fm, nl, st, buf = self.fmaps, self.nl, _stream(), (self.buf1 if lane == 1 else self.buf)
        grad_flat = self.grad if param_grads else None
        if param_grads:
            self._grad_dirty = True
        gview = self.gview
        B, L, Lq = ctx["B"], ctx["L"], ctx["Lq"]
        a, hp, ss, mi, shifts = ctx["a"], ctx["hp"], ctx["ss"], ctx["mi"], ctx["shifts"]
        dev = ctx["x0"].device
        fc_head = self.pool_type == "none"
        if fc_head:
            kin = Lq[-1] * fm[-1]
            g_z1 = buf.get("d.gz1", (B, 256), GT, dev)
            ws = buf.get("d.fcws", (B * (1 + 128 + 256 + 256),), F32, dev)
        gv = (lambda n: _p(gview(n))) if param_grads else (lambda n: None)
        sn, slot, wsfx = self.snorm, ctx.get("sn_slot"), self.wsfx
        sn_small = {}             # snorm: per-pass scratch gradients of the small normalised tensors
        if sn and param_grads:
            head_sn = ("fc.2.weight_orig", "fc.3.weight_orig") if fc_head else ()
            for nm in head_sn + ("enc_blocks.0.conv.weight_orig",):
                sn_small[nm] = buf.get("d.sng." + nm, self.index[nm][2], F32, dev, zero=True)
        # weight-gradient chain (wgrad GEMM + unpack) of every layer: side stream 0, next to the
        # data-gradient chain (dgrad GEMM -> BatchNorm/PReLU backward) on the caller's stream
        side = side_stream(dev, 3 if lane == 1 else 0) if param_grads else None
        if not fc_head:
            g_h = buf.get("d.gh%d" % (nl - 1), (B, Lq[-1], fm[-1]), GT, dev)
            if self.pool_type == "mlp":
                self._mlp_head_bwd(ctx, target, weight, param_grads, loss_out, g_logit, g_h, buf, slot, side)
            else:
                self._pool_head_bwd(ctx, target, weight, param_grads, loss_out, g_logit, g_h, buf, slot)
        else:
            g_w2 = _p(sn_small["fc.2.weight_orig"]) if sn_small else gv("fc.2.weight")
            g_s3 = _p(sn_small["fc.3.weight_orig"]) if sn_small else gv("fc.3.weight")
            _lib.call("sg_fc_tail_bwd", _p(ctx["z1"]), _p(ctx["z2"]), _p(ctx["logit"]), _p(g_logit), float(target),
                      float(weight),
                      _p(self.pview("fc.1.weight")), _p(ctx["w2"]), _p(ctx["s3"]),
                      _p(self.pview("fc.4.weight")), B, _p(loss_out), _p(g_z1), _p(ws),
                      gv("fc.0.bias"), gv("fc.1.weight"), g_w2, gv("fc.2.bias"), g_s3,
                      gv("fc.4.weight"), gv("fc.4.bias"), float(LOSS_SCALE), st)
            if sn_small:
                self._sn_fix_small("fc.2.weight_orig", sn_small["fc.2.weight_orig"], slot)
                self._sn_fix_small("fc.3.weight_orig", sn_small["fc.3.weight_orig"], slot)
            if param_grads:
                fc0 = self.by_name["fc.0.weight" + wsfx]
                dw1 = self.mgrad(fc0)
                osc = None
                if sn:
                    # <dL/dW~, W~> of fc.0 = <g_z1, fc0 output without bias>; coefficient of this pass's sigma term
                    stt = self._sn_state(fc0.name)
                    gz1f = ws[B * 129:B * 129 + B * 256]
                    stt["coef"][slot] = (gz1f * ctx["acc"].reshape(-1)).sum() * stt["scal"][slot][3]
                    osc = stt["scal"][slot][3:4]
                with on_side(side):
                    run_w(g_z1, 1, GS, ctx["hpb"][-1], None, 1, 0, GS, kin, 256, tap_ranges("full", 0, kin, 256),
                          dw1, B, d_lo=0, d_hi=0, dw_tap0=4, ksplit=1, backend=self.backend, out_scale=osc)
            g_h = buf.get("d.gh%d" % (nl - 1), (B, Lq[-1], fm[-1]), GT, dev)
            run_f(g_z1, None, 1, 0, GS, self.packed["W1dg"], GS, 256, kin, tap_ranges("full", 0, 256, kin),
                  g_h, GS, 1, 0, 0, 1, B, d_lo=0, d_hi=0, w_tap0=4, backend=self.backend)
        tmp = buf.get("d.cstmp", (SL * 2048,), F64, dev)
        reds = stat_arena(buf, "d.red", [(SL, 3, fm[l]) for l in range(nl)], dev)
        for l in range(nl - 1, -1, -1):
            cout = fm[l]
            halo = 16 if l < nl - 1 else 0
            roll = shifts[l + 1] if l < nl - 1 else 0
            rp = rptr(l + 1) if l < nl - 1 else None
            g_a = buf.get("d.ga%d" % l, (B, Lq[l], cout), GT, dev)
            redl = reds[l]
            slope = self.pview("enc_blocks.%d.act.weight" % l)
            if sn:
                # no norm layer: one pass gives the final gradient of the pre-activation (as in the Generator)
                _lib.call("sg_act_bwd_reduce", _p(g_h), cout, halo, roll, rp, None, 0, _p(a[l]), SG_F16, B, Lq[l], cout,
                          None, None, _p(slope), ACT_PRELU, _p(redl), _p(g_a), st)
                if param_grads:
                    bias_l = self.pview("enc_blocks.%d.conv.bias" % l) if m.bias else None
                    _lib.call("sg_stat_grads", _p(redl), cout, 3, _p(gview("enc_blocks.%d.act.weight" % l)),
                              _p(gview("enc_blocks.%d.conv.bias" % l)) if m.bias else None, None, st)
                    if l > 0:        # sigma-term coefficient of this pass (layer 0 is a small tensor, fixed below)
                        stt = self._sn_state("enc_blocks.%d.conv.weight_orig" % l)
                        _lib.call("sg_snorm_coef", _p(redl), _p(bias_l), cout, _p(stt["scal"][slot]),
                                  _p(stt["coef"][slot:slot + 1]), st)
            else:
                _lib.call("sg_act_bwd_reduce", _p(g_h), cout, halo, roll, rp, None, 0, _p(a[l]), SG_F16, B, Lq[l], cout,
                          _p(ss[l]), _p(mi[l]), _p(slope), ACT_PRELU, _p(redl), None, st)
                _lib.call("sg_act_bwd_apply", _p(g_h), cout, halo, roll, rp, None, 0, _p(a[l]), SG_F16, B, Lq[l], cout,
                          _p(ss[l]), _p(mi[l]), _p(slope), ACT_PRELU, _p(redl), 1, _p(g_a), st)
            if param_grads and not sn:
                _lib.call("sg_stat_grads", _p(redl), cout, 3, _p(gview("enc_blocks.%d.act.weight" % l)),
                          _p(gview("enc_blocks.%d.norm.bias" % l)),
                          _p(gview("enc_blocks.%d.norm.weight" % l)), st)
                # conv biases feed BatchNorm: their gradient is exactly zero (the BN backward output has
                # zero mean per channel); the reference only sees rounding noise there.  Left at zero
                # (SEGAN_B200_EXACT_BIAS_GRAD=1 computes the column sums anyway).
                if m.bias and not sn and os.environ.get("SEGAN_B200_EXACT_BIAS_GRAD") == "1":
                    _lib.call("sg_colsum", _p(g_a), GS, B * Lq[l], cout, cout,
                              _p(gview("enc_blocks.%d.conv.bias" % l)), 1, _p(tmp), st)
            if l == 0:
                w0 = self.pview("enc_blocks.0.conv.weight" + wsfx)
                if sn:
                    w0 = (w0 * self.sn_inv_sigma("enc_blocks.0.conv.weight_orig", slot)).contiguous()
                g_w0 = (sn_small["enc_blocks.0.conv.weight_orig"] if sn_small else gview("enc_blocks.0.conv.weight")) \
                    if param_grads else None
                if param_grads and ctx.get("colb") is not None:
                    dwq = buf.get("d.dwq0", (128 * 128,), F32, dev)
                    with on_side(side):
                        run_w(g_a, Lq[0] // 2, GS, ctx["colb"], None, Lq[0] // 2, 0, GS, 128, 128,
                              tap_ranges("full", 0, 128, 128), dwq, B, d_lo=0, d_hi=0, dw_tap0=4, ksplit=148,
                              backend=self.backend)
                        _lib.call("sg_wave_wgrad_fold_kw", _p(dwq), 2, self.kw, _p(g_w0), _stream())
                        if sn_small:
                            self._sn_fix_small("enc_blocks.0.conv.weight_orig",
                                               sn_small["enc_blocks.0.conv.weight_orig"], slot)
                elif param_grads:
                    with on_side(side):
                        _lib.call("sg_wave_conv_wgrad", _p(ctx["x0"]), _p(ctx["x1"]), 2, B, L, shifts[0], _p(g_a),
                                  cout, _p(g_w0), None, _stream())
                        if sn_small:
                            self._sn_fix_small("enc_blocks.0.conv.weight_orig",
                                               sn_small["enc_blocks.0.conv.weight_orig"], slot)
                if (input_grad is not None or input_grad1 is not None) and wave_on_tensor_cores():
                    P2 = buf.get("d.P2", (B, Lq[0], 64), GT, dev)
                    run_f(g_a, None, Lq[0], 0, GS, self.packed["WcolT0"], GS, 64, 64,
                          tap_ranges("full", 0, 64, 64), P2, GS, Lq[0], 0, 0, Lq[0], B, d_lo=0, d_hi=0, w_tap0=4,
                          backend=self.backend)
                    if input_grad is not None:
                        _lib.call("sg_wave_col2im_fold_kw", _p(P2), 0, B, L, shifts[0], rptr(0), self.kw,
                                  _p(input_grad), st)
                    if input_grad1 is not None:
                        _lib.call("sg_wave_col2im_fold_kw", _p(P2), 32, B, L, shifts[0], rptr(0), self.kw,
                                  _p(input_grad1), st)
                else:
                    if input_grad is not None:
                        _lib.call("sg_wave_conv_dgrad", _p(g_a), B, L, shifts[0], _p(w0), 2, cout, _p(input_grad), 1, st)
                    if input_grad1 is not None:     # gradient w.r.t. the second input channel
                        w1 = C.c_void_p(w0.data_ptr() + 4 * self.kw)
                        _lib.call("sg_wave_conv_dgrad", _p(g_a), B, L, shifts[0], w1, 2, cout, _p(input_grad1), 1, st)
                break
            cin = fm[l - 1]
            if param_grads:
                pl_l = self.by_name["enc_blocks.%d.conv.weight%s" % (l, wsfx)]
                dwp_l = self.mgrad(pl_l)
                osc = self.sn_inv_sigma(pl_l.name, slot) if sn else None
                with on_side(side):
                    n_tiles = 9 * (cout // 128) * max(1, 4 * cin // 256)
                    taps_w = tap_ranges("conv_fwd", cin, 4 * cin, cout, self.kw)
                    d_lo, d_hi = tap_span(taps_w)
                    run_w(g_a, Lq[l], GS, ctx["hpb"][l - 1], None, Lq[l], 4, GS, 4 * cin, cout, taps_w, dwp_l, B,
                          d_lo=d_lo, d_hi=d_hi, ksplit=wgrad_ksplit(B * Lq[l], n_tiles, taps_w, 4 * cin, cout, d_lo,
                                                                    d_hi), backend=self.backend, out_scale=osc)
                    if l == nl - 1 and reducer is not None:
                        # fc.0 and enc4 of THIS pass are enqueued; the chunk leaves once every accumulating pass
                        # (real / fake / misaligned ...) has said so: reduce_now marks the last one
                        reducer.ready(0, launch=reduce_now)
            g_h = buf.get("d.gh%d" % (l - 1), (B, Lq[l] + 8, 4 * cin), GT, dev)
            taps_dg = tap_ranges("conv_dgrad", cin, cout, 4 * cin, self.kw)
            d_lo, d_hi = tap_span(taps_dg)
            run_f(g_a, None, Lq[l], 0, GS, self.packed["Wdg%d" % l], GS, cout, 4 * cin,
                  taps_dg, g_h, GS, Lq[l], 4, -4, Lq[l] + 4, B, d_lo=d_lo, d_hi=d_hi, backend=self.backend)
        join_side(side)
        if reducer is not None and param_grads:
            reducer.ready(1, launch=reduce_now)
        return grad_flat


class SpectralLoss(object):
    """WSEGAN's spectral regression term (model.py:638-653): pow_weight * L1 between the log-power spectrograms of the
    enhanced and the clean batch -- torch.stft(n_fft 2048, hop 160, win_length 320 rectangular, centred, normalised),
    10 log10(|X|^2 + 1e-19).  Only the window's 320 samples of every 2048-sample frame are non-zero, so the transform
    of all B x (1 + L/160) frames of BOTH signals is one dense GEMM on the tensor cores (the tap-GEMM with one tap):
        [2 B frames][960 = hi | lo | hi] x [960 = Dhi ; Dhi ; Dlo][2176 = re(1025) pad | im(1025) pad]  (fp16, fp32 out)
    the two-halves split of both operands (x = hi + lo) keeps the weak bins of a 60 dB spectrum out of the fp16
    rounding floor.  |X| does not depend on where the window sits in the frame: the DFT runs over n = 0..319.
    Backward: dL/dX (bf16: 1/|X|^2 has a wide range) x D^T (bf16) -> dL/dframes, overlap-added into dL/dwave."""

    WIN, HOP, NFFT, BINS, HALF = 320, 160, 2048, 1025, 1088

    def __init__(self, device):
        self.dev = device
        self.buf = _Buffers()
        n = torch.arange(self.WIN, dtype=torch.float64)
        f = torch.arange(self.BINS, dtype=torch.float64)
        ang = 2.0 * math.pi * torch.outer(f, n) / self.NFFT                  # [bins][win]
        d = torch.zeros(2 * self.HALF, self.WIN, dtype=torch.float64)
        d[:self.BINS] = torch.cos(ang) / math.sqrt(self.NFFT)                # normalized=True: frame_length ** -0.5
        d[self.HALF:self.HALF + self.BINS] = -torch.sin(ang) / math.sqrt(self.NFFT)
        hi = d.to(torch.float16)
        lo = (d - hi.double()).to(torch.float16)
        self.w_fwd = torch.cat((hi, hi, lo), dim=1).contiguous().to(device)               # F[n = column][k = 960]
        self.w_bwd = d.t().contiguous().to(torch.bfloat16).to(device)                     # F[n = sample][k = column]
        self.taps_f = tap_ranges("full", 0, 3 * self.WIN, 2 * self.HALF)
        self.taps_b = tap_ranges("full", 0, 2 * self.HALF, self.WIN)

    def __call__(self, gen, clean, weight, loss_out, g_wave=None, g_scale=1.0):
        """loss_out (device float*) += weight * mean|logpow(gen) - logpow(clean)|; g_wave (fp32 (B,1,L), optional)
        += g_scale * d loss / d gen."""
        B, _, L = gen.shape
        assert L > self.NFFT // 2 and gen.dtype == torch.float32 and clean.dtype == torch.float32
        fr = 1 + L // self.HOP
        rows = B * fr
        dev = gen.device
        K, N = 3 * self.WIN, 2 * self.HALF
        frames = self.buf.get("frames", (2 * rows, K), F16, dev)
        _lib.call("sg_stft_frames", _p(gen.contiguous()), B, L, _p(frames), SG_F16, 1, _stream())
        _lib.call("sg_stft_frames", _p(clean.contiguous()), B, L, C.c_void_p(frames.data_ptr() + rows * K * 2),
                  SG_F16, 1, _stream())
        X = self.buf.get("X", (2 * rows, N), F32, dev)
        run_f(frames, None, 2 * rows, 0, SG_F16, self.w_fwd, SG_F16, K, N, self.taps_f, X, SG_F32, 2 * rows, 0,
              0, 2 * rows, 1, d_lo=0, d_hi=0, w_tap0=4)
        gX = None
        if g_wave is not None:
            gX = self.buf.get("gX", (rows, N), BF16, dev)          # pad columns stay zero (never written)
        _lib.call("sg_logpow_l1", _p(X), C.c_void_p(X.data_ptr() + rows * N * 4), rows, self.BINS, self.HALF, N,
                  float(weight), loss_out, _p(gX), SG_BF16, 1.0, _stream())
        if g_wave is not None:
            gf = self.buf.get("gf", (rows, self.WIN), F32, dev)
            run_f(gX, None, rows, 0, SG_BF16, self.w_bwd, SG_BF16, N, self.WIN, self.taps_b, gf, SG_F32, rows, 0,
                  0, rows, 1, d_lo=0, d_hi=0, w_tap0=4)
            _lib.call("sg_stft_frames_fold", _p(gf), B, L, float(g_scale), _p(g_wave), _stream())
