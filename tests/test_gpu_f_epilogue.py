"""The forward-form tap-GEMM's TMA-store epilogue (tapgemm_tc.cu f_epilogue_tma): whole tiles of a 16-bit output are
staged in shared memory and leave through TMA tensor stores clipped at the launch's rows, batch elements and columns.
Every output buffer starts as a sentinel bit pattern; after the launch the computed region matches the fp32 reference
and every other element still holds the sentinel.  Run on an H100:  python -m pytest tests -m gpu"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                            # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, BACKEND_TCGEN05      # noqa: E402
from tests.test_gpu_kernels import _gen, _packed_random, _ref_f          # noqa: E402
from tests.util import max_abs                                             # noqa: E402

DEV = "cuda"
SENTINEL = 0x7E5A          # an int16 bit pattern no launch writes by accident

# kind: conv_fwd (rows [0, R), a halo of 4), conv_dgrad (rows [-4, R+4) into an output halo of 4), deconv_dgrad
CASES = {
    "partial_m_tile": dict(kind="conv_fwd", cin=64, cout=128, R=160, B=3),                  # 128 + 32 rows
    "small_rows_batch_tail": dict(kind="conv_fwd", cin=128, cout=256, R=16, B=11),          # TR 16, TB 8
    "dgrad_16_rows": dict(kind="conv_dgrad", cin=64, cout=128, R=8, B=11),                   # TR 16, TB 8
    "dgrad_24_rows_bf16": dict(kind="conv_dgrad", cin=64, cout=256, R=16, B=7, bf16=True),   # TR 24, TB 5
    "dgrad_halo_two_m_tiles": dict(kind="conv_dgrad", cin=64, cout=128, R=128, B=3),         # rows -4..132
    "n_sub_range_bf16": dict(kind="deconv_dgrad", cin=256, cout=64, R=64, B=3, n_lo=128, n_hi=256, bf16=True),
    "concat_destination": dict(kind="conv_fwd", cin=64, cout=128, R=64, B=3, out_ld=384, out_col0=192),
    "concat_n_sub_range": dict(kind="deconv_dgrad", cin=256, cout=64, R=64, B=3, n_lo=64, n_hi=192, out_ld=320,
                               out_col0=64),
    "out2_halo0": dict(kind="conv_fwd", cin=64, cout=128, R=256, B=5, out2_halo=0),
    "out2_halo4_small_rows": dict(kind="conv_fwd", cin=64, cout=128, R=16, B=11, out2_halo=4),   # mirrors, TB 8
    "out2_halo16": dict(kind="conv_fwd", cin=64, cout=128, R=256, B=5, out2_halo=16),
    "out2_halo16_bf16": dict(kind="conv_fwd", cin=64, cout=256, R=160, B=3, out2_halo=16, bf16=True),
    "prelu_in_place": dict(kind="conv_fwd", cin=64, cout=256, R=160, B=3, inplace=True),
    # 192 tiles on 132 CTAs: the 60 leftover tiles are split along K and finished by single warps with direct
    # stores, next to the TMA-stored tiles of the same out / out2
    "stream_k_shared_output": dict(kind="conv_fwd", cin=64, cout=512, R=1024, B=12, out2_halo=16, stream_k=True),
}


def _sentinel(shape, tdt):
    t = torch.empty(shape, dtype=tdt, device=DEV)
    t.view(torch.int16).fill_(SENTINEL)
    return t


def _problem(c):
    g = _gen(31)
    tdt = torch.bfloat16 if c.get("bf16") else torch.float16
    sdt = SG_BF16 if c.get("bf16") else SG_F16
    kind, cin, cout, R, B = c["kind"], c["cin"], c["cout"], c["R"], c["B"]
    if kind == "conv_fwd":
        kc, nc, halo, m_lo, m_hi, out_halo, cpack = 4 * cin, cout, 4, 0, R, 0, cin
    elif kind == "conv_dgrad":
        kc, nc, halo, m_lo, m_hi, out_halo, cpack = cout, 4 * cin, 0, -4, R + 4, 4, cin
    else:
        kc, nc, halo, m_lo, m_hi, out_halo, cpack = 4 * cout, cin, 0, 0, R, 0, cout
    w, taps = _packed_random(kind, cpack, kc, nc, g, tdt)
    a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(tdt).to(DEV)
    bias = torch.randn(nc, generator=g).to(DEV) if kind == "conv_fwd" else None
    slope = (0.3 * torch.rand(nc, generator=g)).to(DEV) if ("out2_halo" in c or c.get("inplace")) else None
    return dict(tdt=tdt, sdt=sdt, kc=kc, nc=nc, halo=halo, m_lo=m_lo, m_hi=m_hi, out_halo=out_halo, w=w, taps=taps,
                a0=a0, bias=bias, slope=slope)


def _run(c, pr):
    B, R, nc = c["B"], c["R"], pr["nc"]
    n_lo, n_hi = c.get("n_lo", 0), c.get("n_hi", nc)
    ld = c.get("out_ld", nc)
    out = _sentinel((B, R + 2 * pr["out_halo"], ld), pr["tdt"])
    out2 = None
    kw = {}
    if "out2_halo" in c:
        out2 = _sentinel((B, R + 2 * c["out2_halo"], ld), pr["tdt"])
        kw = dict(out2=out2, out2_halo=c["out2_halo"], slope=pr["slope"], slope_mod=nc)
    elif c.get("inplace"):
        kw = dict(slope=pr["slope"], slope_mod=nc)
    if "out_ld" in c:
        kw.update(out_ld=c["out_ld"], out_col0=c["out_col0"])
    lib = _lib.load()
    if c.get("stream_k"):
        ws = E.sk_workspace(DEV)
        ws[8192:].zero_()
        lib.sg_set_stream_k(16, 1e-6)          # force the split of the leftover tiles
    try:
        E.run_f(pr["a0"], None, R, pr["halo"], pr["sdt"], pr["w"], pr["sdt"], pr["kc"], nc, pr["taps"], out, pr["sdt"],
                R, pr["out_halo"], pr["m_lo"], pr["m_hi"], B, bias=pr["bias"],
                bias_mod=nc if pr["bias"] is not None else 0, n_lo=n_lo, n_hi=n_hi, backend=BACKEND_TCGEN05, **kw)
        torch.cuda.synchronize()
    finally:
        if c.get("stream_k"):
            lib.sg_set_stream_k(16, 4.5)
    if c.get("stream_k"):
        assert int(E.sk_workspace(DEV)[8192:].count_nonzero()) > 0, "the split-K path did not run"
    return out, out2


@pytest.mark.parametrize("case", sorted(CASES))
def test_f_epilogue_region_and_sentinel(case):
    c = CASES[case]
    pr = _problem(c)
    B, R, nc = c["B"], c["R"], pr["nc"]
    n_lo, n_hi = c.get("n_lo", 0), c.get("n_hi", nc)
    col0 = c.get("out_col0", n_lo)
    ncols = n_hi - n_lo
    out, out2 = _run(c, pr)

    ref = _ref_f(pr["a0"].float().cpu(), pr["halo"], pr["w"].cpu(), pr["m_lo"], pr["m_hi"])[:, :, n_lo:n_hi]
    if pr["bias"] is not None:
        ref = ref + pr["bias"].cpu()[n_lo:n_hi]
    sl = pr["slope"].cpu()[n_lo:n_hi] if pr["slope"] is not None else None
    act = torch.where(ref > 0, ref, ref * sl) if sl is not None else None
    tol = 3e-2 * max(1.0, float(ref.abs().max()))

    # out: the region holds the result, everything else the sentinel
    r0 = pr["out_halo"] + pr["m_lo"]
    o = out.cpu()
    region = o[:, r0:r0 + (pr["m_hi"] - pr["m_lo"]), col0:col0 + ncols]
    assert max_abs(region.float(), act if c.get("inplace") else ref) <= tol, case
    mask = torch.ones(o.shape, dtype=torch.bool)
    mask[:, r0:r0 + (pr["m_hi"] - pr["m_lo"]), col0:col0 + ncols] = False
    assert bool((o.view(torch.int16)[mask] == SENTINEL).all()), "%s: out written outside the launch's region" % case

    if out2 is not None:
        h = c["out2_halo"]
        o2 = out2.cpu()
        inner = o2[:, h:h + R, col0:col0 + ncols]
        assert max_abs(inner.float(), act) <= tol, case
        mask2 = torch.ones(o2.shape, dtype=torch.bool)
        mask2[:, :, col0:col0 + ncols] = False
        assert bool((o2.view(torch.int16)[mask2] == SENTINEL).all()), "%s: out2 written outside its columns" % case
        o2i, oi = o2.view(torch.int16), o.view(torch.int16)
        # the reflect-halo rows are bit-copies of their mirror rows
        for k in range(1, h + 1):
            assert torch.equal(o2i[:, h - k], o2i[:, h + k]), (case, k)
            assert torch.equal(o2i[:, h + R - 1 + k], o2i[:, h + R - 1 - k]), (case, k)
        # PReLU leaves positive values alone: same bits as out there
        pos = region.float() > 0
        assert torch.equal(oi[:, r0:r0 + R, col0:col0 + ncols][pos], o2i[:, h:h + R, col0:col0 + ncols][pos]), case

    # bitwise repeatable
    out_b, out2_b = _run(c, pr)
    assert torch.equal(out.view(torch.int16), out_b.view(torch.int16)), case
    if out2 is not None:
        assert torch.equal(out2.view(torch.int16), out2_b.view(torch.int16)), case


def test_f_epilogue_refuses_unaligned_destination():
    """TMA stores need 16-byte aligned rows and column offsets: such a launch is an argument error, not a fallback."""
    c = dict(kind="conv_fwd", cin=64, cout=128, R=64, B=2)
    pr = _problem(c)
    out = _sentinel((2, 64, 136), torch.float16)
    with pytest.raises(_lib.SeganB200Error):
        E.run_f(pr["a0"], None, 64, 4, SG_F16, pr["w"], SG_F16, pr["kc"], 128, pr["taps"], out, SG_F16, 64, 0, 0, 64, 2,
                out_ld=136, out_col0=4, backend=BACKEND_TCGEN05)
    torch.cuda.synchronize()
    assert bool((out.view(torch.int16) == SENTINEL).all())
