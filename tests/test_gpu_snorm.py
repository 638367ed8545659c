"""Spectral normalisation kernels (norm_type='snorm', torch.nn.utils.spectral_norm) against fp64 references of the
same operation: sg_snorm_sigma (one power iteration / eval sigma), sg_snorm_grad, sg_snorm_coef, sg_snorm_rank1, the
activation-backward statistic red[2] = sum g_pre * x that feeds sg_snorm_coef, the 1/sigma scale options of the
weight-gradient tap-GEMM and of sg_emit_operands; and one engine-level invariant that needs no oracle: with u and v
held constant, W / sigma(W) does not change when W is scaled, so every weight_orig gradient is orthogonal to W.
An fp32 sum must satisfy |err| <= c * 2^-24 * sum|terms| for every output (U below).
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C
import random

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E          # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, BACKEND_FFMA, BACKEND_TCGEN05  # noqa: E402
from oracle import segan_oracle as O                       # noqa: E402
from tests.util import load_opts, seed_all                 # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream
U = 2.0 ** -24
KW = 31
FM = [64, 128, 256, 512, 1024]


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _ratio(err, scale):
    return float((err.abs() / (U * scale.clamp_min(1e-300))).max())


@pytest.fixture(autouse=True)
def _restore_ew_variant():
    yield
    _lib.load().sg_set_ew_variant(3, 16, 4, 2)        # elementwise.cu's default for sg_act_bwd_reduce


# Every spectrally normalised tensor of the Discriminator (discriminator.py:110-146): name -> (kind, reference
# shape, c_in, t_len).  kind 0 / 2 are packed tap-GEMM masters (engine.PackedLayer), None the small tensors that
# sg_snorm_grad handles in reference layout (T = 1, nc = dim 0, kc = the rest).
SN_TENSORS = {
    "enc1": (0, (128, 64, KW), 64, 0), "enc2": (0, (256, 128, KW), 128, 0), "enc3": (0, (512, 256, KW), 256, 0),
    "enc4": (0, (1024, 512, KW), 512, 0),
    "fc.0": (2, (256, 16 * 1024), 1024, 16),
    "mlp.0": (2, (1024, 1024, 1), 1024, 1),
    "enc0": (None, (64, 2, KW), 0, 0), "fc.2": (None, (128, 256), 0, 0), "pool_conv": (None, (1, 1024, 1), 0, 0),
    "fc.conv_head": (None, (1, 16), 0, 0), "fc.gavg_head": (None, (1, 1024), 0, 0),
    "fc.3": (None, (128,), 0, 0), "mlp.1": (None, (1024,), 0, 0),
}


def _sn_case(name, seed):
    """(packed master M [T][nc][kc] on the device, W [nc][K] fp64 reference layout, u0 [nc], v0 reference layout,
    v0 in the kernel's slots, pack(v) -> reference layout)."""
    kind, shape, c_in, t_len = SN_TENSORS[name]
    g = _gen(seed)
    w = 0.05 * torch.randn(*shape, generator=g)
    nc = shape[0]
    wm = w.reshape(nc, -1)
    u0 = F.normalize(torch.randn(nc, generator=g), dim=0, eps=1e-12)
    v0 = F.normalize(torch.randn(wm.shape[1], generator=g), dim=0, eps=1e-12)
    if kind is None:
        m = wm.reshape(1, nc, -1)
        return m.to(DEV).contiguous(), wm.double().to(DEV), u0, v0, v0.clone(), (lambda v: v)
    m = E.pack_reference(kind, w, nc, c_in, t_len)
    vshape = (1, c_in, KW) if kind == 0 else (1, -1)
    vp = E.pack_reference(kind, v0.reshape(vshape), 1, c_in, t_len).reshape(-1)
    unpack = lambda v: E.unpack_reference(kind, v, 1, c_in, t_len).reshape(-1)     # noqa: E731
    assert torch.equal(unpack(vp), v0)
    return m.to(DEV).contiguous(), wm.double().to(DEV), u0, v0, vp, unpack


class _Holder(torch.nn.Module):
    def __init__(self, w):
        super().__init__()
        self.weight = torch.nn.Parameter(w)


def _torch_power_iteration(wm, u0, v0):
    """torch.nn.utils.spectral_norm in fp64: one training-mode power iteration from (u0, v0); returns u, v, sigma."""
    h = _Holder(wm.detach().cpu().clone())
    torch.nn.utils.spectral_norm(h)
    h.weight_u.copy_(u0.double())
    h.weight_v.copy_(v0.double())
    hook = next(iter(h._forward_pre_hooks.values()))
    with torch.no_grad():
        w_sn = hook.compute_weight(h, do_power_iteration=True)
    u, v = h.weight_u.clone(), h.weight_v.clone()
    sigma = float(torch.dot(u, h.weight_orig.detach() @ v))
    assert torch.allclose(w_sn, h.weight_orig.detach() / sigma, rtol=1e-12, atol=0)
    return u.to(DEV), v.to(DEV), sigma


@pytest.mark.parametrize("name", list(SN_TENSORS))
def test_snorm_sigma_training_vs_torch_spectral_norm(name):
    """One power iteration v = normalize(W^T u), u = normalize(W v), sigma = u^T W v on the packed master against
    torch's spectral_norm in fp64 (u, the unpacked v, sigma, 1/sigma).  Per element, c = 32 of
    2^-24 * (the sum of |terms| of that element's dot product / the norm it is divided by + |value|)."""
    m, wm, u0, v0, vp, unpack = _sn_case(name, 200 + list(SN_TENSORS).index(name))
    T, nc, kc = m.shape
    u = u0.to(DEV).contiguous()
    v = vp.to(DEV).contiguous()
    scal = torch.full((4,), 5.0, device=DEV)
    work = torch.zeros(nc + 4, device=DEV)
    _lib.call("sg_snorm_sigma", _p(m), T, nc, kc, _p(u), _p(v), _p(scal), _p(work), 1, _stream())
    u_t, v_t, sig_t = _torch_power_iteration(wm, u0, v0)
    torch.cuda.synchronize()
    vg = unpack(v.cpu()).double().to(DEV)
    ug = u.double()
    # v = normalize(W^T u0): torch's v is exactly this fp64 reference
    vr = wm.t() @ u0.double().to(DEV)
    sv = wm.abs().t() @ u0.double().abs().to(DEV)
    cv = _ratio(vg - v_t, sv / vr.norm() + v_t.abs())
    # u = normalize(W v) given the v the kernel produced, and sigma = ||W v||
    ur = wm @ vg
    su = wm.abs() @ vg.abs()
    sig_r = float(ur.norm())
    cu = _ratio(ug - ur / sig_r, su / sig_r + (ur / sig_r).abs())
    sig, inv = float(scal[2]), float(scal[3])
    cs = abs(sig - sig_r) / (U * (float(((ur / sig_r).abs() * su).sum()) + sig_r))
    print("snorm_sigma %s (T %d, nc %d, kc %d): c v %.2f u %.2f sigma %.2f (tol 32); vs torch: |du| %.2e |dsigma|/sigma %.2e"
          % (name, T, nc, kc, cv, cu, cs, float((ug - u_t).abs().max()), abs(sig - sig_t) / sig_t))
    assert cv <= 32 and cu <= 32 and cs <= 32
    assert abs(inv - 1.0 / sig) <= 2 * U * abs(1.0 / sig)                 # 1/sigma: one fp32 rounding
    # the same numbers against torch's own iteration (u differs only through the kernel's v, within its bound)
    assert float((ug - u_t).norm()) <= 1e-5 and abs(sig - sig_t) <= 1e-5 * sig_t


@pytest.mark.parametrize("name", ["enc2", "fc.0", "enc0", "fc.3", "pool_conv"])
def test_snorm_sigma_eval_uses_stored_vectors(name):
    """training = 0: sigma = u^T W v from the stored vectors (c = 32 of 2^-24 * sum_n |u_n| (|W| |v|)_n), u and v
    left bit-for-bit untouched."""
    m, wm, u0, v0, vp, unpack = _sn_case(name, 300)
    T, nc, kc = m.shape
    u = u0.to(DEV).contiguous()
    v = vp.to(DEV).contiguous()
    u_before, v_before = u.clone(), v.clone()
    scal = torch.full((4,), 5.0, device=DEV)
    work = torch.zeros(nc + 4, device=DEV)
    _lib.call("sg_snorm_sigma", _p(m), T, nc, kc, _p(u), _p(v), _p(scal), _p(work), 0, _stream())
    torch.cuda.synchronize()
    u64, v64 = u0.double().to(DEV), v0.double().to(DEV)
    ref = float(u64 @ (wm @ v64))
    scale = float(u64.abs() @ (wm.abs() @ v64.abs()))
    c = abs(float(scal[2]) - ref) / (U * scale)
    print("snorm_sigma eval %s: c = %.2f (tol 32)" % (name, c))
    assert c <= 32
    assert abs(float(scal[3]) - 1.0 / float(scal[2])) <= 2 * U / abs(float(scal[2]))
    assert torch.equal(u, u_before) and torch.equal(v, v_before)


@pytest.mark.parametrize("shape", [(1, 64, 62), (1, 128, 256), (1, 128, 1), (1, 1, 1024), (1, 1, 16), (1, 1024, 1),
                                   (9, 128, 256)])
def test_snorm_grad_vs_fp64_autograd(shape):
    """dL/dW of L = <G, W / sigma(W)>, sigma = u^T W v with u, v constants, by fp64 autograd: per element c = 8 of
    2^-24 * (|G| / sigma + sum|G * W| / sigma^2 * |u_n v_k| + |dW|)."""
    T, nc, kc = shape
    g = _gen(400 + T + nc + kc)
    M = (0.05 * torch.randn(T, nc, kc, generator=g)).to(DEV)
    G = torch.randn(T, nc, kc, generator=g).to(DEV)
    u = F.normalize(torch.randn(nc, generator=g), dim=0).to(DEV)
    v = F.normalize(torch.randn(T * kc, generator=g), dim=0).to(DEV)
    M64 = M.double().requires_grad_(True)
    sigma = (u.double().view(1, nc, 1) * M64 * v.double().view(T, 1, kc)).sum()
    (G.double() * M64 / sigma).sum().backward()
    ref = M64.grad
    sig = float(sigma)
    scal = torch.tensor([7.0, 7.0, sig, 1.0 / sig], device=DEV)
    dw = G.clone()
    dot_ws = torch.full((1,), 9.0, device=DEV)
    _lib.call("sg_snorm_grad", _p(dw), _p(M), T, nc, kc, _p(u), _p(v), _p(scal), _p(dot_ws), _stream())
    torch.cuda.synchronize()
    uv = (u.double().view(1, nc, 1) * v.double().view(T, 1, kc)).abs()
    scale = G.double().abs() / abs(sig) + float((G.double() * M.double()).abs().sum()) / sig ** 2 * uv + ref.abs()
    c = _ratio(dw.double() - ref, scale)
    print("snorm_grad %s: c = %.2f (tol 8)" % (str(shape), c))
    assert c <= 8


@pytest.mark.parametrize("Cc,with_bias", [(64, True), (64, False), (300, True), (1024, True), (1024, False)])
def test_snorm_coef_hand_built(Cc, with_bias):
    """coef = scal[3] * sum_c (sum_slices red[.,2,c] - b_c * sum_slices red[.,1,c]): summed in double, one fp32
    rounding.  scal[0..2] hold garbage that must not be read."""
    g = _gen(500 + Cc)
    red = torch.randn(8, 3, Cc, generator=g, dtype=torch.float64) * 10
    bias = 0.3 * torch.randn(Cc, generator=g) if with_bias else None
    scal = torch.tensor([1e30, -1e30, 1e30, 0.37])
    coef = torch.full((1,), 7.0, device=DEV)
    red_d, scal_d = red.to(DEV), scal.to(DEV)          # kept alive until the launch has run
    bias_d = bias.to(DEV) if with_bias else None
    _lib.call("sg_snorm_coef", _p(red_d), _p(bias_d), Cc, _p(scal_d), _p(coef), _stream())
    b = bias.double() if with_bias else torch.zeros(Cc, dtype=torch.float64)
    s = red[:, 2].sum(0) - b * red[:, 1].sum(0)
    exp = float(scal[3]) * float(s.sum())
    torch.cuda.synchronize()
    assert abs(float(coef) - exp) <= U * abs(exp) + 1e-12 * float(s.abs().sum()), (float(coef), exp)


@pytest.mark.parametrize("n_pass", [1, 2, 4, 5])
@pytest.mark.parametrize("shape", [(9, 128, 256), (1, 256, 16384)])
def test_snorm_rank1_vs_fp64(shape, n_pass):
    """dWp -= sum_{p < P} coef_p u_p v_p^T over P pass slots out of 5 stored ones: c = 12 of
    2^-24 * (|dWp| + sum_p |coef_p u_p v_p|) per element."""
    T, nc, kc = shape
    g = _gen(600 + n_pass)
    dwp = torch.randn(T, nc, kc, generator=g).to(DEV)
    u = F.normalize(torch.randn(5, nc, generator=g), dim=1).to(DEV)
    v = F.normalize(torch.randn(5, T * kc, generator=g), dim=1).to(DEV)
    coef = (100 * torch.randn(5, generator=g)).to(DEV)
    d0 = dwp.double()
    ref, scale = d0.clone(), d0.abs()
    for p in range(n_pass):
        t = coef[p].double() * u[p].double().view(1, nc, 1) * v[p].double().view(T, 1, kc)
        ref -= t
        scale = scale + t.abs()
    _lib.call("sg_snorm_rank1", _p(dwp), T, nc, kc, n_pass, _p(u), _p(v), _p(coef), _stream())
    torch.cuda.synchronize()
    c = _ratio(dwp.double() - ref, scale)
    print("snorm_rank1 %s P=%d: c = %.2f (tol 12)" % (str(shape), n_pass, c))
    assert c <= 12


@pytest.mark.parametrize("variant", [(4, 2, 3), (8, 2, 2), (16, 2, 2)], ids=["reg_vec4", "tiled_vec8", "tma_vec16"])
@pytest.mark.parametrize("Cc,L,roll", [(64, 256, 3), (256, 64, -5), (128, 96, 4)])
@pytest.mark.parametrize("roll_on_device", [False, True])
def test_act_bwd_reduce_without_bn_feeds_snorm_coef(variant, Cc, L, roll, roll_on_device):
    """The snorm D tower's activation backward (no BatchNorm, reflect halo 16, phase roll, no g_add): red[2] =
    sum g_pre * x and red[1] = sum g_pre per channel against fp64 autograd of PReLU -> roll -> reflect pad (c = 32
    of 2^-24 * sum|terms|), for the register-staged, tiled and TMA-staged kernels; then sg_snorm_coef on that red
    against scal[3] * sum g_pre * (x - bias) in fp64."""
    assert _lib.load().sg_set_ew_variant(3, *variant) == 0
    g = _gen(700 + Cc)
    B, halo = 6, 16
    a = torch.randn(B, L, Cc, generator=g).to(torch.float16).to(DEV)
    gh = torch.randn(B, L + 2 * halo, Cc, generator=g).to(E.GT).to(DEV)
    slope = (0.2 * torch.rand(Cc, generator=g)).to(DEV)
    bias = (0.1 * torch.randn(Cc, generator=g)).to(DEV)
    red = torch.zeros(8, 3, Cc, dtype=torch.float64, device=DEV)
    ga = torch.zeros(B, L, Cc, dtype=E.GT, device=DEV)
    rdev = torch.tensor([11, roll], dtype=torch.int32, device=DEV)
    rptr = C.c_void_p(rdev.data_ptr() + 4) if roll_on_device else None
    _lib.call("sg_act_bwd_reduce", _p(gh), Cc, halo, 0 if roll_on_device else roll, rptr, None, 0, _p(a), SG_F16, B, L,
              Cc, None, None, _p(slope), 1, _p(red), _p(ga), _stream())
    scal = torch.tensor([0.0, 0.0, 1.0 / 0.37, 0.37], device=DEV)
    coef = torch.zeros(1, device=DEV)
    _lib.call("sg_snorm_coef", _p(red), _p(bias), Cc, _p(scal), _p(coef), _stream())
    an = a.double().permute(0, 2, 1).requires_grad_(True)
    y = F.prelu(an, slope.double())
    yr = F.pad(O.phase_roll(y, roll), (halo, halo), mode="reflect")
    (yr * gh.double().permute(0, 2, 1)).sum().backward()
    gpre = an.grad                                                   # [B][C][L]
    x = an.detach()
    r2, s2 = (gpre * x).sum((0, 2)), (gpre * x).abs().sum((0, 2))
    r1, s1 = gpre.sum((0, 2)), gpre.abs().sum((0, 2))
    torch.cuda.synchronize()
    rs = red.sum(0)
    c2, c1 = _ratio(rs[2] - r2, s2), _ratio(rs[1] - r1, s1)
    b64 = bias.double().view(1, Cc, 1)
    exp = 0.37 * float((gpre * (x - b64)).sum())
    cc = abs(float(coef) - exp) / (U * 0.37 * float((gpre * (x - b64)).abs().sum()))
    print("act_bwd_reduce %s C=%d L=%d roll=%d dev=%s: c red2 %.2f red1 %.2f coef %.2f (tol 32)"
          % (variant, Cc, L, roll, roll_on_device, c2, c1, cc))
    assert c2 <= 32 and c1 <= 32 and cc <= 32


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05])
@pytest.mark.parametrize("ksplit", [1, 3])
def test_tapgemm_w_out_scale(backend, ksplit):
    """sg_tapgemm_w.out_scale (1/sigma of a snorm layer) multiplies the accumulated products: against the unscaled
    launch times the device scalar, c = 16 of 2^-24 * s * sum|g a| per element (the split-K partial sums are scaled
    before they are added)."""
    g = _gen(800)
    B, cin, cout, R, halo = 3, 64, 128, 128, 4
    kc, nc = 4 * cin, cout
    taps = E.tap_ranges("conv_fwd", cin, kc, nc)
    a0 = torch.randn(B, R + 2 * halo, kc, generator=g).to(torch.bfloat16).to(DEV)
    gg = (torch.randn(B, R, nc, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    s = torch.tensor([0.0, 0.37], device=DEV)
    dws = []
    for osc in (None, s[1:]):
        dw = torch.zeros(9, nc, kc, device=DEV)
        E.run_w(gg, R, SG_BF16, a0, None, R, halo, SG_BF16, kc, nc, taps, dw, B, ksplit=ksplit, backend=backend,
                out_scale=osc)
        dws.append(dw)
    ap = F.pad(a0.double(), (0, 0, 16, 16))
    gabs = gg.double().abs()
    asum = torch.stack([torch.einsum("bmn,bmk->nk", gabs, ap[:, 16 + halo + d: 16 + halo + d + R].abs())
                        for d in range(-4, 5)])
    torch.cuda.synchronize()
    c = _ratio(dws[1].double() - 0.37 * dws[0].double(), 0.37 * asum)
    print("tapgemm_w out_scale backend %d ksplit %d: c = %.2f (tol 16)" % (backend, ksplit, c))
    assert c <= 16
    assert float(dws[1].abs().max()) > 0


@pytest.mark.parametrize("dt", [SG_F16, SG_BF16])
def test_emit_operands_scale_dev(dt):
    """sg_emit_operands(scale_dev = 1/sigma) packs W / sigma: the forward and data-gradient operands are the
    unscaled emission of the fp32 product M * s bit for bit, and within one 16-bit rounding of M * s in fp64."""
    g = _gen(900)
    T, nc, kc = 9, 128, 256
    tdt = torch.float16 if dt == SG_F16 else torch.bfloat16
    m = torch.randn(T, nc, kc, generator=g).to(DEV)
    s = torch.tensor([0.0, 0.37], device=DEV)
    f1 = torch.zeros(T, nc, kc, dtype=tdt, device=DEV)
    d1 = torch.zeros(T, kc, nc, dtype=tdt, device=DEV)
    _lib.call("sg_emit_operands", _p(m), T, nc, kc, None, 0, _p(f1), _p(d1), dt, dt, C.c_void_p(s.data_ptr() + 4),
              _stream())
    ms = (m * s[1]).contiguous()
    f0, d0 = torch.zeros_like(f1), torch.zeros_like(d1)
    _lib.call("sg_emit_operands", _p(ms), T, nc, kc, None, 0, _p(f0), _p(d0), dt, dt, None, _stream())
    torch.cuda.synchronize()
    assert torch.equal(f1, f0) and torch.equal(d1, d0)
    exact = m.double() * 0.37
    p = 11 if dt == SG_F16 else 8
    bound = (2.0 ** -p + 2.0 ** -23) * exact.abs() + 2.0 ** -25
    assert bool(((f1.double() - exact).abs() <= bound).all())
    assert torch.equal(d1, f1.flip(0).transpose(1, 2))         # Dg[t][k][n] = F[T-1-t][n][k]


# ------------------------------------------------------------------------------------------------------
# engine-level invariant: <dL/dW_orig, W_orig> = 0 for every spectrally normalised weight
# ------------------------------------------------------------------------------------------------------
# |<g, W>| / sum_p |coef_p sigma_p| measured on one H100 80GB HBM3 (700 W): at most 5e-4 for the two-pass D backward
# and 5e-3 for the WSEGAN step (the fp16 pre-activations and gradients behind coef); dropping one pass's rank-1 term
# gives 0.59 - 0.99.
ORTHO_TOL = 2e-2


def _record_small_sigma_terms(de):
    """Wraps the engine's small-tensor snorm fix so that each pass's sigma-term coefficient <G, W> / sigma^2 (the dot
    product sg_snorm_grad leaves in its scratch float) is kept with that pass's u and v, stream-ordered."""
    recs = {}
    orig = de._sn_fix_small

    def fix(nm, scratch, slot):
        orig(nm, scratch, slot)
        stt = de._sn_state(nm)
        inv = stt["scal"][slot][3]
        recs.setdefault(nm, []).append(((stt["work"][stt["nc"]] * inv * inv).clone(), stt["u_p"][slot].clone(),
                                        stt["v_p"][slot].clone()))
    de._sn_fix_small = fix
    return recs


def _orthogonality(de, w0, recs, label):
    """For every weight_orig: |<g, W>| / sum_p |coef_p u_p^T W v_p| (the size of the sigma correction), and the same
    ratio with the rank-1 term of the largest pass added back in fp64 (what a missing correction would leave)."""
    de.finish_grads()
    torch.cuda.synchronize()
    items = []
    for pl in de.layers:
        stt = de._sn_state(pl.name)
        terms = [(stt["coef"][p], stt["u_p"][p], stt["v_p"][p]) for p in range(de._sn_pass)]
        items.append((pl.name, de.mgrad(pl), w0[pl.off:pl.off + pl.numel], pl.T, pl.nc, pl.kc, terms))
    for nm, terms in recs.items():
        off, n, _ = de.index[nm]
        stt = de._sn_state(nm)
        items.append((nm, de.gview(nm).reshape(-1), w0[off:off + n], 1, stt["nc"], stt["kc"], terms))
    out = {}
    for nm, gr, w, T, nc, kc, terms in items:
        assert len(terms) == de._sn_pass, (nm, len(terms))
        g64, w64 = gr.double(), w.double()
        dot = float(g64 @ w64)
        wt = w64.view(T, nc, kc)
        sig_terms = [float(cf) * float((u.double().view(1, nc, 1) * wt * v.double().view(T, 1, kc)).sum())
                     for cf, u, v in terms]
        scale = sum(abs(t) for t in sig_terms)
        ratio = abs(dot) / scale
        missing = max(abs(dot + t) for t in sig_terms) / scale
        rel_corr = sum(abs(float(cf)) for cf, _, _ in terms) / float(g64.norm())
        out[nm] = (ratio, missing)
        print("%s %-32s |<g,W>|/sum|coef sigma| %.2e | one pass's term dropped %.3f | sum|coef| / |g| %.3e | "
              "sum|coef sigma| / (|g| |W|) %.3e" % (label, nm, ratio, missing, rel_corr,
                                                    scale / float(g64.norm() * w64.norm())))
    return out


def _build_d(head):
    from segan_pytorch_b200.segan.models import Discriminator
    seed_all(111)
    return Discriminator(2, FM, 31, [4, 4, 4, 4, 4], pool_type=head, pool_slen=16, norm_type="snorm",
                         phase_shift=5).to(DEV)


def _waves(B, seed):
    g = _gen(seed)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    return clean, noisy


@pytest.mark.parametrize("head", ["none", "mlp"])
def test_snorm_gradient_orthogonal_to_weight(head):
    """W / sigma(W) with sigma = u^T W v (u, v constants) is homogeneous of degree 0 in W, so every pass's gradient
    w.r.t. weight_orig is orthogonal to it: <dL/dW_orig, W_orig> = 0.  The sigma term's size is
    sum_p |coef_p sigma_p|; a missing or wrong correction leaves a residual of that order.  Two LSGAN passes at
    B = 16 into one bucket (u, v of each pass in its own slot), for the fc head and the mlp head (noise floor: see
    ORTHO_TOL)."""
    B = 16
    D = _build_d(head)
    D.train()
    clean, noisy = _waves(B, 901)
    x = torch.cat((clean, noisy), 1).to(DEV)
    random.seed(9)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    with torch.no_grad():
        D(x, shifts=shifts[2])
    de = D.engine
    w0 = de.flat.detach().clone()
    recs = _record_small_sigma_terms(de)
    de.zero_grad()
    x2 = torch.cat((noisy, clean), 1).to(DEV)
    for i, (xx, tgt) in enumerate(((x, 1.0), (x2, 0.0))):
        _, cx = de.forward(xx[:, :1].contiguous(), xx[:, 1:].contiguous(), shifts[i], training=True)
        de.backward(cx, tgt, 1.0, param_grads=True)
    assert de._sn_pass == 2
    res = _orthogonality(de, w0, recs, "D/%s" % head)
    expect = {"enc_blocks.%d.conv.weight_orig" % l for l in range(5)} | set(de.HEAD_SN[head])
    assert set(res) == expect
    for nm, (ratio, missing) in res.items():
        assert ratio <= ORTHO_TOL, (nm, ratio)
        assert missing >= 10 * ORTHO_TOL, (nm, missing)


@pytest.mark.parametrize("head", ["none", "mlp"])
def test_snorm_gradient_orthogonal_to_weight_wsegan_step(head):
    """The same invariant after a WSEGAN --misalign_pair step (three accumulating D passes: real, fake, misaligned),
    read against the D weights the step's passes used."""
    from segan_pytorch_b200.segan.models import WSEGAN
    B = 4
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, opt="adam", dnorm_type="snorm", dpool_type=head)
    s = WSEGAN(opts).to(DEV)
    s.G.train()
    s.D.train()
    clean, noisy = _waves(B, 902)
    z = torch.randn(B, 1024, 16, generator=_gen(903))
    random.seed(5)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    Gopt, Dopt = s.build_optimizers(opts)
    de = s.D.engine
    de.bind()
    w0 = de.flat.detach().clone()
    recs = _record_small_sigma_terms(de)
    s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=["a"] * B, z=z.to(DEV), shifts=shifts,
                 perm=[1, 3, 0, 2])
    assert de._sn_pass == 3
    res = _orthogonality(de, w0, recs, "WSEGAN/%s" % head)
    for nm, (ratio, missing) in res.items():
        assert ratio <= ORTHO_TOL, (nm, ratio)
        assert missing >= 10 * ORTHO_TOL, (nm, missing)
