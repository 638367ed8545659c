"""The forward-form tap-GEMM's two row segments (tapgemm_tc.cu tapgemm_f_tc_launch, f_tile): a launch whose rows
[m_lo, m_hi) pack badly into 128-row M tiles (a conv data gradient computes R + 8 rows per batch element) is covered
by a leading segment of R0 rows (a multiple of 128, or the largest power of two <= the row count) and the remaining
R1 < 128 rows, each packed on its own, when that strictly lowers the M tile count and leaves at least one tile per SM
(132 on an H100).  Launched through sg_tapgemm_f_run and held to fp64 by the checks of test_gpu_tapgemm_f.py: the
c <= 16 gate, guard bands and dead elements keeping their bits, bitwise repeatability, and agreement with the FFMA
back-end.

  id                  rows_m  batch  segments (R x TB -> M tiles)            TN x N tiles   sources
  rows72_b251 *       72      251    64 x 2 -> 126, 8 x 16 -> 16              256 x 1        128
  rows72_b57_tn64 *   72      57     64 x 2 -> 29,  8 x 16 -> 4               64 x 4         128
  rows72_b115_tn128 * 72      115    64 x 2 -> 58,  8 x 16 -> 8               128 x 2        128
  rows72_b300         72      300    64 x 2 -> 150, 8 x 16 -> 19              256 x 1        128
  rows264_b65 *       264     65     256 -> 2 x 65, 8 x 16 -> 5               256 x 1        128
  rows1032_b17        1032    17     1024 -> 8 x 17, 8 x 16 -> 2              256 x 1        128
  rows24_b705         24      705    16 x 8 -> 89, 8 x 16 -> 45               256 x 1        128
  rows40_b423 *       40      423    32 x 4 -> 106, 8 x 16 -> 27              256 x 1        128
  rows72_b251_src2    72      251    as rows72_b251                           256 x 1        64 + 64
  rows72_b251_f32     72      251    as rows72_b251, fp32 out (fragment epilogue)  256 x 1   128
  rows72_b3           72      3      one segment: 72 x 1 -> 3 (two would be 2 + 1)
  rows72_b17          72      17     one segment: 72 x 1 -> 17 (two would be 9 + 2, fewer tiles than SMs)

(* also in bf16.)  Forced stream-K: 72 rows at batch 239 is 120 + 15 = 135 M tiles on 132 CTAs, so the three
leftover tiles, split along K, are all segment-1 tiles, the last one a partial batch tile.  At batch 300, the four
data gradients of the train step (conv levels 1-4, rows 1032 / 264 / 72 / 24) run under the default cost model.
Run on an H100:  python -m pytest tests/test_gpu_tapgemm_f_rowsplit.py -m gpu -s"""
import pytest

from tests import test_gpu_tapgemm_f as tf


def m_tiling(rows_m, batch, n_tiles=1):
    """The launch's M tiling: [(rows, TR, TB, M tiles)] per segment (mirrors tapgemm_f_tc_launch)."""
    def seg(r):
        tr = min(r, 128)
        tb = 1 if r >= 128 else min(128 // r, batch)
        return (r, tr, tb, -(-r // tr) * -(-batch // tb))
    whole = seg(rows_m)
    r0 = 128 * (rows_m // 128) if rows_m > 128 else 1 << (rows_m.bit_length() - 1)
    if r0 < rows_m:
        two = [seg(r0), seg(rows_m - r0)]
        if two[0][3] + two[1][3] < whole[3] and (two[0][3] + two[1][3]) * n_tiles >= tf.E.NUM_SMS:
            return two
    return [whole]


_DG = dict(a0_c=128, nc=256, taps="conv_dgrad")
CASES = {
    "rows72_b251": dict(_DG, rows=64, batch=251, bf16=True),
    "rows72_b57_tn64": dict(_DG, rows=64, batch=57, tile_n=64, bf16=True),
    "rows72_b115_tn128": dict(_DG, rows=64, batch=115, tile_n=128, bf16=True),
    "rows72_b300": dict(_DG, rows=64, batch=300),
    "rows264_b65": dict(_DG, rows=256, batch=65, bf16=True),
    "rows1032_b17": dict(_DG, rows=1024, batch=17),
    "rows24_b705": dict(_DG, rows=16, batch=705),
    "rows40_b423": dict(_DG, rows=32, batch=423, bf16=True),
    "rows72_b251_src2": dict(_DG, a0_c=64, a1_c=64, rows=64, batch=251),
    "rows72_b251_f32": dict(_DG, rows=64, batch=251, f32=True),
    "rows72_b3": dict(_DG, rows=64, batch=3),
    "rows72_b17": dict(_DG, rows=64, batch=17),
}
NO_SPLIT = {"rows72_b3", "rows72_b17"}
PARAMS = [(n, f) for n, c in CASES.items() for f in (("f16", "bf16") if c.get("bf16") else ("f16",))]

SK_CASE = dict(_DG, rows=64, batch=239)

STEP = {                                         # conv level: (cin, cout, R); rows_m = R + 8
    "dgrad1": (64, 128, 1024),
    "dgrad2": (128, 256, 256),
    "dgrad3": (256, 512, 64),
    "dgrad4": (512, 1024, 16),
}


def test_cases_cover_both_segments():
    """Every split case ends both segments in a partial batch tile where its table says so, and the tile count the
    step's data gradients drop to."""
    for name, c in CASES.items():
        segs = m_tiling(c["rows"] + 8, c["batch"], c["nc"] // tf.tc_tile_n(c))
        assert (len(segs) == 2) == (name not in NO_SPLIT), (name, segs)
    for name in ("rows72_b251", "rows72_b57_tn64", "rows72_b115_tn128", "rows24_b705", "rows40_b423"):
        c = CASES[name]
        for r, tr, tb, _ in m_tiling(c["rows"] + 8, c["batch"], c["nc"] // tf.tc_tile_n(c)):
            assert tb > 1 and c["batch"] % tb != 0, (name, r, tb)
    step_tiles = [sum(s[3] for s in m_tiling(R + 8, 300, 4 * cin // 256)) for cin, _, R in STEP.values()]
    assert step_tiles == [2419, 619, 169, 57], step_tiles
    # the forced stream-K case: every leftover tile of the last wave is a segment-1 tile
    s0, s1 = m_tiling(SK_CASE["rows"] + 8, SK_CASE["batch"])
    tiles = s0[3] + s1[3]
    left = tiles % tf.E.NUM_SMS
    assert tiles > tf.E.NUM_SMS and 0 < left <= s1[3] and SK_CASE["batch"] % s1[2] != 0, (s0, s1)


@pytest.mark.gpu
@pytest.mark.parametrize("name,fmt", PARAMS, ids=["%s-%s" % p for p in PARAMS])
def test_rowsplit_vs_fp64(name, fmt):
    tf._run_case(name, CASES[name], fmt, 8000 + 11 * list(CASES).index(name))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f16", "bf16"])
def test_rowsplit_stream_k_leftovers_in_segment_1(fmt):
    tf._run_sk("stream_k rows72_b239-%s" % fmt, SK_CASE, fmt, 8200 + (fmt == "bf16"))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f16", "bf16"])
@pytest.mark.parametrize("name", list(STEP))
def test_rowsplit_step_data_gradients(name, fmt, monkeypatch):
    key = "%s_%s" % (name, fmt)
    monkeypatch.setitem(tf.PRODUCTION, key, (tf._dgrad(*STEP[name]), fmt))
    tf.test_production_scale(key)
