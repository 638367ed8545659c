"""The forward-form tap-GEMM's whole-tile output staging (tapgemm_tc.cu f_epilogue_tma, FSmem) over many tiles per
CTA: the sentinel-filled cases of test_gpu_f_epilogue.py at sizes where every one of the 132 CTAs stages at least
three tiles in a row, so that the two alternating staging buffers of 64-wide tiles wrap, the single buffer of 128-
and 256-wide tiles is rewritten behind its own stores, and 256-wide tiles with a second output leave in four rounds.
Run on an H100:  python -m pytest tests -m gpu"""
import pytest

from tests import test_gpu_f_epilogue as fe

pytestmark = pytest.mark.gpu

# 160 rows = a full and a partial 128-row M tile per batch element; 198 batch elements = 396 tiles = 3 per CTA, so
# every CTA's last tile (CTA 131's: a partial M tile) is followed by the kernel's exit
CASES = {
    "tn64_three_tiles_partial_m_exit": dict(kind="conv_fwd", cin=64, cout=64, R=160, B=198),
    "tn64_out2_three_tiles_bf16": dict(kind="conv_fwd", cin=64, cout=64, R=160, B=198, out2_halo=16, bf16=True),
    "tn256_out2_three_tiles": dict(kind="conv_fwd", cin=64, cout=256, R=160, B=198, out2_halo=16),
    # 400 tiles on 132 CTAs: three staged tiles per CTA, then the 4 leftover tiles split along K and finished from
    # the fragment into the same out / out2
    "stream_k_after_three_staged_tiles": dict(kind="conv_fwd", cin=64, cout=128, R=1024, B=50, out2_halo=16,
                                              stream_k=True),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_f_staging_region_and_sentinel(case, monkeypatch):
    monkeypatch.setitem(fe.CASES, case, CASES[case])
    fe.test_f_epilogue_region_and_sentinel(case)
