"""The forward-form tap-GEMM (form F: tapgemm_tc.cu tapgemm_f_tc, tapgemm_ref.cu tapgemm_f_ffma) held to its
arithmetic: 16-bit operands multiplied exactly, fp32 accumulation, one rounding of the output.  The shapes are the
ones the max-abs tests already launch (test_gpu_kernels.py: test_tapgemm_f, test_tapgemm_f_a_reuse, the stream-K
shapes; test_gpu_f_epilogue.py: CASES), imported from there; the reference is fp64 and the gate is
tests/tapgemm_model.py's: the error beyond half an ulp of the stored 16-bit value is at most 16 * 2^-24 * sum |a w|
(+ |bias|) per element.  out2 is compared with PReLU of the fp64 value where the sign of that value is beyond the
reach of the summation order.  fp32 outputs (fc.0's interleaved k-split, accumulated into a pre-filled
destination) have no output rounding to take off.  Sentinels, bit-copies of halo rows and the stream-K counters
stay with the tests that own those shapes.  Run on an H100:  python -m pytest tests -m gpu"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                                          # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, SG_F32, BACKEND_FFMA, BACKEND_TCGEN05   # noqa: E402
from tests import tapgemm_model as M                                                       # noqa: E402
from tests import test_gpu_f_epilogue as EP                                                # noqa: E402
from tests.test_gpu_kernels import (F_CASES, F_REUSE_CASES, _f_case, _f_reuse_case, _gen, _sk_case)   # noqa: E402

DEV = "cuda"


@pytest.fixture(autouse=True)
def _restore_schedule_switches():
    yield
    _lib.load().sg_set_cta_pair(1)


def _fmt(sg_dtype):
    return "bf16" if sg_dtype == SG_BF16 else "f16"


def _gate(label, got, ref, mag, fmt):
    c = M.c_f(got, ref, mag, fmt)
    print("tapgemm_f %s (%s): c = %.2f (tol %g)" % (label, fmt, c, M.C_TOL))
    assert c <= M.C_TOL, (label, c)
    assert float(got.double().abs().max()) > 0


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05, 2])
@pytest.mark.parametrize("case", F_CASES)
def test_tapgemm_f_cases_vs_fp64(backend, case):
    """backend 1 = tensor cores with sg_set_cta_pair(0), 2 = tensor cores with sg_set_cta_pair(1)."""
    _lib.load().sg_set_cta_pair(1 if backend == 2 else 0)
    label = "%s backend %d" % (case, backend)
    if backend == 2:
        backend = BACKEND_TCGEN05
    c = _f_case(case)
    B, nc, m_lo, m_hi, out_halo = c["B"], c["nc"], c["m_lo"], c["m_hi"], c["out_halo"]
    n_lo, n_hi = c["n_lo"], nc if c["n_hi"] is None else c["n_hi"]
    f32 = c["out_dtype"] == SG_F32
    out0 = torch.randn(B, c["out_rows"] + 2 * out_halo, nc, generator=_gen(77)).to(c["tdt"]).to(DEV)
    if not (f32 and c["ksplit"] > 1):
        out0.zero_()                                   # every other launch overwrites its region
    out = out0.clone()
    bias = c["bias"]
    E.run_f(c["a0"], c["a1"], c["R"], c["halo"], c["adt"], c["w"], c["wdt"], c["kc"], nc, c["taps"], out, c["out_dtype"],
            c["out_rows"], out_halo, m_lo, m_hi, B, bias=bias, bias_mod=(bias.numel() if bias is not None else 0),
            n_lo=c["n_lo"], n_hi=c["n_hi"], d_lo=c["d_lo"], d_hi=c["d_hi"], w_tap0=c["w_tap0"], ksplit=c["ksplit"],
            backend=backend, a0_c=c["a0"].shape[-1], a1_c=c["a1_c"])
    ref, mag = M.ref_f(c["a0"], c["a1"], c["halo"], c["w"], c["taps"], m_lo, m_hi, c["d_lo"], c["d_hi"], c["w_tap0"], bias)
    torch.cuda.synchronize()
    region = (slice(None), slice(out_halo + m_lo, out_halo + m_hi), slice(n_lo, n_hi))
    ref, mag = ref[..., n_lo:n_hi], mag[..., n_lo:n_hi]
    if f32:
        d0 = out0[region].double()
        cc = M.c_w(out[region].double() - d0, ref, mag + d0.abs())
        print("tapgemm_f %s (f32, ksplit %d): c = %.2f (tol %g)" % (label, c["ksplit"], cc, M.C_TOL))
        assert cc <= M.C_TOL, (label, cc)
    else:
        _gate(label, out[region], ref, mag, _fmt(c["out_dtype"]))


@pytest.mark.parametrize("case", F_REUSE_CASES)
def test_tapgemm_f_a_reuse_cases_vs_fp64(case):
    _lib.load().sg_set_cta_pair(2)
    c = _f_reuse_case(case)
    B, nc, m_lo, m_hi, out_halo = c["B"], c["nc"], c["m_lo"], c["m_hi"], c["out_halo"]
    n_lo, n_hi = c["n_lo"], nc if c["n_hi"] is None else c["n_hi"]
    bias = c["bias"]
    out = torch.zeros(B, c["out_rows"] + 2 * out_halo, nc, dtype=c["tdt"], device=DEV)
    E.run_f(c["a0"], c["a1"], c["R"], c["halo"], c["adt"], c["w"], c["adt"], c["kc"], nc, c["taps"], out, c["odt"],
            c["out_rows"], out_halo, m_lo, m_hi, B, bias=bias, bias_mod=(bias.numel() if bias is not None else 0),
            n_lo=c["n_lo"], n_hi=c["n_hi"], d_lo=c["d_lo"], d_hi=c["d_hi"], backend=BACKEND_TCGEN05,
            a0_c=c["a0"].shape[-1], a1_c=c["a1_c"])
    ref, mag = M.ref_f(c["a0"], c["a1"], c["halo"], c["w"], c["taps"], m_lo, m_hi, c["d_lo"], c["d_hi"], 0, bias)
    torch.cuda.synchronize()
    _gate("a_reuse %s" % case, out[:, out_halo + m_lo:out_halo + m_hi, n_lo:n_hi], ref[..., n_lo:n_hi],
          mag[..., n_lo:n_hi], _fmt(c["odt"]))


@pytest.mark.parametrize("case", sorted(EP.CASES))
def test_f_epilogue_cases_vs_fp64(case):
    """out, and out2 / the in-place activation against PReLU of the fp64 value."""
    c = EP.CASES[case]
    pr = EP._problem(c)
    R, nc = c["R"], pr["nc"]
    n_lo, n_hi = c.get("n_lo", 0), c.get("n_hi", nc)
    col0 = c.get("out_col0", n_lo)
    out, out2 = EP._run(c, pr)
    ref, mag = M.ref_f(pr["a0"], None, pr["halo"], pr["w"], pr["taps"], pr["m_lo"], pr["m_hi"], bias=pr["bias"])
    ref, mag = ref[..., n_lo:n_hi], mag[..., n_lo:n_hi]
    fmt = "bf16" if c.get("bf16") else "f16"
    r0 = pr["out_halo"] + pr["m_lo"]
    region = out[:, r0:r0 + (pr["m_hi"] - pr["m_lo"]), col0:col0 + (n_hi - n_lo)]
    if pr["slope"] is not None:
        act, mag_act = M.prelu_ref(ref, mag, pr["slope"][n_lo:n_hi])
        safe = M.sign_safe(ref, mag)
        assert float(safe.double().mean()) > 0.99
    if c.get("inplace"):
        _gate("epilogue %s in place" % case, region[safe], act[safe], mag_act[safe], fmt)
        return
    _gate("epilogue %s out" % case, region, ref, mag, fmt)
    if out2 is not None:
        h = c["out2_halo"]
        inner = out2[:, h:h + R, col0:col0 + (n_hi - n_lo)]
        _gate("epilogue %s out2" % case, inner[safe], act[safe], mag_act[safe], fmt)


@pytest.mark.parametrize("case", ["conv_fwd", "deconv_fwd", "conv_dgrad"])
@pytest.mark.parametrize("stream_k", [False, True])
def test_tapgemm_f_stream_k_cases_vs_fp64(case, stream_k):
    """More tiles than SMs with a ragged last wave: unsplit, and with the leftover tiles split along K."""
    g = _gen(21)
    B, kc, nc, R, halo, m_lo, m_hi, out_halo, w, taps, a0 = _sk_case(case, g)
    bias = torch.randn(nc, generator=g).to(DEV)
    ws = E.sk_workspace(DEV)
    ws[8192:].zero_()
    lib = _lib.load()
    prev = E.STREAM_K
    E.STREAM_K = stream_k
    lib.sg_set_stream_k(16, 1e-6)              # force the split whatever the cost model says about this shape
    try:
        out = torch.zeros(B, R + 2 * out_halo, nc, dtype=torch.float16, device=DEV)
        E.run_f(a0, None, R, halo, SG_F16, w, SG_F16, kc, nc, taps, out, SG_F16, R, out_halo, m_lo, m_hi, B, bias=bias,
                bias_mod=nc, backend=BACKEND_TCGEN05)
        torch.cuda.synchronize()
    finally:
        E.STREAM_K = prev
        lib.sg_set_stream_k(16, 4.5)             # the default cost model
    assert (int(ws[8192:].count_nonzero()) > 0) == stream_k
    ref, mag = M.ref_f(a0, None, halo, w, taps, m_lo, m_hi, bias=bias)
    _gate("stream_k=%s %s" % (stream_k, case), out[:, out_halo + m_lo:out_halo + m_hi], ref, mag, "f16")
