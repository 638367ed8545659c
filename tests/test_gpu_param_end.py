"""The kernels at the parameter end of a training step against fp64 (tests/step_end_model.py): the optimisers
(sg_rmsprop_step / sg_adam_step), the fp32 master import / export (sg_pack_weights / sg_unpack_wgrad with SG_F32),
the operands (sg_emit_operands), the GSkip alpha gradient (sg_alpha_grad) and the waveform-end weight-gradient folds
(sg_wave_wgrad_fold, sg_last_deconv_wgrad_fold, sg_last_deconv_wgrad_fold_1src).  The packed layers come from the
engines' own packed_layers(), not from a hand-written list.  Every destination sits between sentinel guard bands and
starts non-zero where the kernel accumulates; outputs without atomics repeat bit for bit.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16, SG_F32    # noqa: E402
from tests import step_end_model as M                          # noqa: E402
from tests.util import build_segan                             # noqa: E402

DEV = "cuda"
C_TOL = M.C_TOL
SG_DT = {"f16": SG_F16, "bf16": SG_BF16, "f32": SG_F32}
TDT = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
TWO_IN_FLIGHT = 4 * 8 * 132 * 256          # floats per grid-stride of the optimisers' float4 loop
CONFIGS = {"segan": {}, "no_skip": dict(no_skip=True), "sum_merge": dict(skip_merge="sum"),
           "snorm": dict(gnorm_type="snorm", dnorm_type="snorm"), "mlp_head": dict(dpool_type="mlp")}


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _g(pairs):
    return all(M.guards_ok(b) for b, _ in pairs)


_ENGINES = {}


def _engines(cfg):
    """(G engine, D engine) of a configuration, bound on the CPU (layer lists and bucket sizes only)."""
    if cfg not in _ENGINES:
        s = build_segan(**CONFIGS[cfg])
        _ENGINES[cfg] = (s.G.engine.bind(), s.D.engine.bind())
    return _ENGINES[cfg]


def _layers(cfg):
    """The distinct packed layers of a configuration's G and D."""
    seen, out = set(), []
    for eng in _engines(cfg):
        for l in eng.packed_layers():
            key = (l.kind, l.c_out, l.c_in, l.t_len)
            if key not in seen:
                seen.add(key)
                out.append(l)
    return out


# ------------------------------------------------------------------------------------------------------
# optimisers
# ------------------------------------------------------------------------------------------------------
def _bucket_sizes():
    g, d = _engines("segan")
    return [g.grad.numel(), d.grad.numel()]


def _opt_state(n, seed, kind):
    """Parameters with exact zeros (the update shows by itself there), gradients over 12 decades (eps matters at
    the small end), non-negative second moments."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    kw = dict(generator=g, device=DEV)
    p = torch.randn(n, **kw)
    p[::3] = 0.0
    gr = torch.sign(torch.randn(n, **kw)) * 10.0 ** (torch.rand(n, **kw) * 12 - 10)
    s1 = 1e-6 * torch.rand(n, **kw) if kind == "rmsprop" else 1e-3 * torch.randn(n, **kw)
    s2 = 1e-6 * torch.rand(n, **kw)
    return [p, gr, s1, s2]


OPT_SETTINGS = {  # (grad_scale, clear, hyper-parameters)
    "rmsprop": [(1.0, 1, dict(alpha=0.99)), (2.0 ** -10, 0, dict(alpha=0.99)), (1.0 / (3 * 1024), 1, dict(alpha=0.99))],
    "adam": [(1.0, 0, dict(betas=(0.0, 0.9), step=1)), (2.0 ** -10, 1, dict(betas=(0.5, 0.999), step=2)),
             (1.0 / (3 * 1024), 0, dict(betas=(0.5, 0.999), step=1000))],
}
OPT_N = list(range(1, 10)) + [4097, 4098, 4099, TWO_IN_FLIGHT - 1, TWO_IN_FLIGHT, TWO_IN_FLIGHT + 5,
                              2 * TWO_IN_FLIGHT + 3, "G_bucket", "D_bucket"]


def _opt_call(kind, bufs, n, lr, gscale, clear, hp):
    p, g, s1, s2 = (b[1] for b in bufs)
    if kind == "rmsprop":
        _lib.call("sg_rmsprop_step", _p(p), _p(g), _p(s1), n, lr, hp["alpha"], 1e-8, gscale, clear, _st())
    else:
        _lib.call("sg_adam_step", _p(p), _p(g), _p(s1), _p(s2), n, lr, *hp["betas"], 1e-8, hp["step"], gscale, clear,
                  _st())


@pytest.mark.parametrize("n", OPT_N)
@pytest.mark.parametrize("kind", ["rmsprop", "adam"])
def test_optimizer_step_vs_fp64(kind, n):
    """One step per setting, gated on the kernel's own state: parameters and moments at c <= C_TOL, the gradient
    zeroed exactly when `clear` is set and otherwise left bit for bit, everything past n (the G bucket's
    gradient-only tail) untouched, and the same bits from a second launch on the same state."""
    if isinstance(n, str):
        n = _bucket_sizes()[0 if n == "G_bucket" else 1]
    for i, (gscale, clear, hp) in enumerate(OPT_SETTINGS[kind]):
        st = _opt_state(n, 1000 + 7 * i + n % 1009, kind)
        runs = []
        for _ in range(2):
            bufs = [M.guarded((n,), torch.float32, DEV, t) for t in st]
            _opt_call(kind, bufs, n, 2e-4, gscale, clear, hp)
            runs.append(bufs)
        torch.cuda.synchronize()
        p0, g0, s10, s20 = st
        (p, g, s1, s2) = (b[1] for b in runs[0])
        if kind == "rmsprop":
            ref = M.rmsprop_step(p0, g0, s10, 2e-4, hp["alpha"], 1e-8, gscale)
            c = dict(p=M.c_vec(p, *ref["p"]), sq=M.c_vec(s1, *ref["sq"]))
        else:
            ref = M.adam_step(p0, g0, s10, s20, 2e-4, *hp["betas"], 1e-8, hp["step"], gscale)
            c = dict(p=M.c_vec(p, *ref["p"]), m=M.c_vec(s1, *ref["m"]), v=M.c_vec(s2, *ref["v"]))
        print("%s n=%d grad_scale %.3g clear %d %s: c" % (kind, n, gscale, clear, hp),
              {k: round(v, 2) for k, v in c.items()})
        assert all(v <= C_TOL for v in c.values()), c
        if clear:
            assert M.bits_equal(g, torch.zeros_like(g))
        else:
            assert M.bits_equal(g, g0)
        assert all(M.bits_equal(a[1], b[1]) for a, b in zip(*runs))
        assert _g(runs[0]) and _g(runs[1])
        if kind == "rmsprop":
            assert M.bits_equal(runs[0][3][1], s20)         # not an RMSprop buffer: never touched


@pytest.mark.parametrize("kind", ["rmsprop", "adam"])
def test_optimizer_20_steps_vs_torch_optim_fp64(kind):
    """20 steps on loss-scaled gradients (grad_scale = 1 / (3 * 1024) divides the scale out) against torch.optim in
    fp64 on the unscaled ones: the hyper-parameter semantics (eps outside the square root, betas) and Adam's
    bias-correction step count."""
    n, S = 4099, 3 * 1024.0
    g = _gen(77)
    p0 = torch.randn(n, generator=g, dtype=torch.float64)
    grads = [torch.randn(n, generator=g, dtype=torch.float64) * 10.0 ** (torch.rand(n, generator=g) * 4 - 3)
             for _ in range(20)]
    pr = p0.clone().requires_grad_(True)
    opt = (torch.optim.RMSprop([pr], lr=2e-4, alpha=0.99, eps=1e-8) if kind == "rmsprop"
           else torch.optim.Adam([pr], lr=2e-4, betas=(0.5, 0.999), eps=1e-8))
    bufs = [M.guarded((n,), torch.float32, DEV, t) for t in (p0.float().to(DEV), torch.zeros(n, device=DEV),
                                                             torch.zeros(n, device=DEV), torch.zeros(n, device=DEV))]
    hp = dict(alpha=0.99) if kind == "rmsprop" else dict(betas=(0.5, 0.999))
    for t, gr in enumerate(grads, 1):
        pr.grad = gr.clone()
        opt.step()
        bufs[1][1].copy_((gr * S).float().to(DEV))
        _opt_call(kind, bufs, n, 2e-4, 1.0 / S, 1, dict(hp, step=t))
    torch.cuda.synchronize()
    got = bufs[0][1].double().cpu()
    moved = (pr.detach() - p0).abs()
    err = (got - pr.detach()).abs()
    # fp32 state: the parameter's own rounding each step plus a small relative error of each update
    tol = 1e-4 * moved + 40 * M.U * p0.abs()
    print("%s 20 steps: max |p - torch fp64| %.3e, max movement %.3e" % (kind, float(err.max()), float(moved.max())))
    assert bool((err <= tol).all()), float((err - tol).max())
    assert _g(bufs)


def test_optimizers_refuse_bad_arguments():
    """Null pointers, n < 0, a buffer off 16-byte alignment (the float4 path) and Adam's step 0 (lr / 0) are refused
    before anything is launched: the buffers keep their bits."""
    n = 64
    bufs = [torch.randn(n + 8, device=DEV) for _ in range(4)]
    snap = [b.clone() for b in bufs]
    p, g, m, v = (_p(b) for b in bufs)
    off = C.c_void_p(bufs[1].data_ptr() + 4)
    for args in ((None, g, m), (p, None, m), (p, g, None), (off, g, m), (p, off, m), (p, g, off)):
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_rmsprop_step", *args, n, 1e-3, 0.99, 1e-8, 1.0, 1, _st())
    with pytest.raises(_lib.SeganB200Error):
        _lib.call("sg_rmsprop_step", p, g, m, -1, 1e-3, 0.99, 1e-8, 1.0, 1, _st())
    for args, step, nn in (((None, g, m, v), 1, n), ((p, g, m, None), 1, n), ((p, g, m, off), 1, n),
                           ((off, g, m, v), 1, n), ((p, g, m, v), 0, n), ((p, g, m, v), 1, -4)):
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_adam_step", *args, nn, 1e-3, 0.5, 0.999, 1e-8, step, 1.0, 1, _st())
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(bufs, snap))


# ------------------------------------------------------------------------------------------------------
# packed masters
# ------------------------------------------------------------------------------------------------------
def _ref_shape(l):
    return (l.c_out, l.c_in, 31) if l.kind == 0 else ((l.c_in, l.c_out, 31) if l.kind == 1 else (l.c_out, l.c_in * l.t_len))


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_master_import_export_bit_exact(cfg):
    """sg_pack_weights(kind, w, ..., SG_F32) == engine.pack_reference and sg_unpack_wgrad(..., accumulate 0) ==
    engine.unpack_reference, bit for bit, for every packed layer of the configuration's G and D."""
    for i, l in enumerate(_layers(cfg)):
        w = torch.randn(*_ref_shape(l), generator=_gen(i)).to(DEV)
        m = M.guarded((l.numel,), torch.float32, DEV)
        _lib.call("sg_pack_weights", l.kind, _p(w), l.c_out, l.c_in, l.t_len, None, 0, _p(m[1]), None, SG_F32, SG_F32,
                  _st())
        back = M.guarded(tuple(w.shape), torch.float32, DEV, torch.randn(*w.shape, generator=_gen(i + 50)))
        _lib.call("sg_unpack_wgrad", l.kind, _p(m[1]), l.c_out, l.c_in, l.t_len, None, None, 0, _p(back[1]), None, 0,
                  _st())
        torch.cuda.synchronize()
        ref = E.pack_reference(l.kind, w, l.c_out, l.c_in, l.t_len)
        assert M.bits_equal(m[1].view(ref.shape), ref), (cfg, l.name)
        assert M.bits_equal(back[1], E.unpack_reference(l.kind, ref, l.c_out, l.c_in, l.t_len)), (cfg, l.name)
        assert M.bits_equal(back[1], w) and _g([m, back]), (cfg, l.name)


def test_unpack_refuses_channel_counts_off_the_tile_grid():
    """sg_unpack_wgrad refuses what sg_pack_weights refuses (its tile grid would silently drop channels)."""
    t = torch.randn(9 * 4 * 64 * 96, device=DEV)
    dw = torch.randn(64 * 96 * 31, device=DEV)
    snap = dw.clone()
    for kind, co, ci in ((0, 64, 48), (0, 40, 64), (1, 48, 64), (1, 64, 40)):
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_unpack_wgrad", kind, _p(t), co, ci, 0, None, None, 0, _p(dw), None, 0, _st())
    torch.cuda.synchronize()
    assert torch.equal(dw, snap)


EMIT_MODES = [  # (alpha, scale, F format or None, Dg format or None)
    (False, False, "f16", "f16"), (True, False, "f16", "bf16"), (False, True, "bf16", "f16"),
    (True, True, None, "bf16"), (True, True, "f16", None), (True, True, "f32", "f32")]


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_emit_operands_bit_exact(cfg):
    """F and Dg of every packed layer from its fp32 master: alpha None or over the columns from kc / 2, the 1/sigma
    scale None or a device scalar, fp16 / bf16 / fp32 destinations, either one NULL; and the operands the
    reference-layout packer (sg_pack_weights, 16-bit) makes from the same weights."""
    for i, l in enumerate(_layers(cfg)):
        T, nc, kc = l.T, l.nc, l.kc
        w = torch.randn(*_ref_shape(l), generator=_gen(i)).to(DEV)
        m = E.pack_reference(l.kind, w, l.c_out, l.c_in, l.t_len)
        alpha = (0.5 + torch.rand(kc - kc // 2, generator=_gen(i + 1))).to(DEV)
        scale = torch.tensor([0.37], device=DEV)
        for use_a, use_s, ff, fd in EMIT_MODES:
            a, s = (alpha if use_a else None), (scale if use_s else None)
            F = M.guarded((T, nc, kc), TDT[ff], DEV) if ff else None
            D = M.guarded((T, kc, nc), TDT[fd], DEV) if fd else None
            _lib.call("sg_emit_operands", _p(m), T, nc, kc, _p(a), kc // 2, _p(F[1]) if F else None,
                      _p(D[1]) if D else None, SG_DT[ff or "f16"], SG_DT[fd or "f16"], _p(s), _st())
            torch.cuda.synchronize()
            rF, rD = M.emit(m, T, nc, kc, a, kc // 2, s, ff or "f32", fd or "f32")
            if F:
                assert M.bits_equal(F[1], rF) and _g([F]), (cfg, l.name, use_a, use_s, ff)
            if D:
                assert M.bits_equal(D[1], rD) and _g([D]), (cfg, l.name, use_a, use_s, fd)
        a = alpha if l.kind == 1 else None                   # the packer scales a ConvTranspose1d's input channels
        F0 = torch.zeros(T, nc, kc, dtype=torch.float16, device=DEV)
        D0 = torch.zeros(T, kc, nc, dtype=torch.bfloat16, device=DEV)
        _lib.call("sg_pack_weights", l.kind, _p(w), l.c_out, l.c_in, l.t_len, _p(a), l.c_in // 2, _p(F0), _p(D0),
                  SG_F16, SG_BF16, _st())
        torch.cuda.synchronize()
        rF, rD = M.emit(m, T, nc, kc, a, kc // 2, None, "f16", "bf16")
        assert M.bits_equal(F0, rF) and M.bits_equal(D0, rD), (cfg, l.name)


def _alpha_layers():
    out = []
    for cfg in CONFIGS:
        for l in _layers(cfg):
            if l.alpha_name is not None and (l.T, l.nc, l.kc, l.alpha_from) not in [x[:4] for x in out]:
                out.append((l.T, l.nc, l.kc, l.alpha_from))
    return out


@pytest.mark.parametrize("prefill", [True, False])
def test_alpha_grad_vs_fp64(prefill):
    """dW *= alpha on the columns from alpha_from (one rounding; the columns below keep their bits) and dalpha +=
    sum dW * M, for every GSkip layer of the configurations and a synthetic one with more rows (T * nc) than the
    kernel's 64-block row grid covers in one pass; dalpha NULL or pre-filled."""
    shapes = _alpha_layers() + [(9, 4096, 64, 32)]
    assert max(T * nc for T, nc, _, _ in shapes) > 64 * 8 * 64
    for i, (T, nc, kc, af) in enumerate(shapes):
        g = _gen(i + 10)
        m = torch.randn(T, nc, kc, generator=g).to(DEV)
        d0 = torch.randn(T, nc, kc, generator=g).to(DEV)
        alpha = (0.5 + torch.rand(kc - af, generator=g)).to(DEV)
        da0 = torch.randn(kc - af, generator=g).to(DEV)
        runs = []
        for _ in range(2):
            dw = M.guarded((T, nc, kc), torch.float32, DEV, d0)
            da = M.guarded((kc - af,), torch.float32, DEV, da0) if prefill else None
            _lib.call("sg_alpha_grad", _p(dw[1]), _p(m), T, nc, kc, _p(alpha), af, _p(da[1]) if da else None, _st())
            runs.append((dw, da))
        torch.cuda.synchronize()
        rD, rda = M.alpha_grad(d0, m, T, nc, kc, alpha, af, da0 if prefill else None)
        (dw, da), (dw2, _) = runs
        assert M.bits_equal(dw[1], rD) and M.bits_equal(dw2[1], dw[1]), (T, nc, kc, af)
        assert _g([dw, dw2])
        if prefill:
            c = M.c_vec(da[1], *rda)
            print("alpha_grad T=%d nc=%d kc=%d from %d: c dalpha %.2f" % (T, nc, kc, af, c))
            assert c <= C_TOL and _g([da])


@pytest.mark.parametrize("cin", [1, 2])
def test_wave_wgrad_fold_vs_fp64(cin):
    g = _gen(cin)
    dwq0 = torch.randn(2, 64, 2, 64, generator=g).to(DEV)
    dw0 = torch.randn(64, cin, 31, generator=g).to(DEV)
    dwq = M.guarded(tuple(dwq0.shape), torch.float32, DEV, dwq0)
    dw = M.guarded(tuple(dw0.shape), torch.float32, DEV, dw0)
    _lib.call("sg_wave_wgrad_fold", _p(dwq[1]), cin, _p(dw[1]), _st())
    torch.cuda.synchronize()
    (r, m), after = M.wave_wgrad_fold(dwq0, cin, dw0)
    c = M.c_vec(dw[1], r, m)
    print("wave_wgrad_fold cin=%d: c %.2f" % (cin, c))
    assert c <= C_TOL and M.bits_equal(dwq[1], after)
    once = dw[1].clone()
    _lib.call("sg_wave_wgrad_fold", _p(dwq[1]), cin, _p(dw[1]), _st())       # on the cleared blocks: adds exactly 0
    torch.cuda.synchronize()
    assert M.bits_equal(dw[1], once) and M.bits_equal(dwq[1], after) and _g([dwq, dw])


@pytest.mark.parametrize("nsrc,half,with_dalpha", [(2, 64, True), (2, 64, False), (2, 32, True), (1, 64, False),
                                                   (1, 96, False)])
def test_last_deconv_wgrad_fold_vs_fp64(nsrc, half, with_dalpha):
    """Two sources (cat(decoder, skip), alpha on the skip half; half = 64 is the default Generator's) and one
    (sg_last_deconv_wgrad_fold_1src: no skips, cin = 64 by default)."""
    g = _gen(nsrc * 1000 + half)
    dwq0 = torch.randn(2, 64, nsrc, 2, half, generator=g).to(DEV)
    w = torch.randn(nsrc * half, 1, 31, generator=g).to(DEV)
    al = (0.5 + torch.rand(half, generator=g)).to(DEV)
    dw0 = torch.randn(nsrc * half, 1, 31, generator=g).to(DEV)
    da0 = torch.randn(half, generator=g).to(DEV)
    dwq = M.guarded(tuple(dwq0.shape), torch.float32, DEV, dwq0)
    dw = M.guarded(tuple(dw0.shape), torch.float32, DEV, dw0)
    da = M.guarded((half,), torch.float32, DEV, da0) if with_dalpha else None

    def fold():
        if nsrc == 2:
            _lib.call("sg_last_deconv_wgrad_fold", _p(dwq[1]), half, _p(w), _p(al), _p(dw[1]),
                      _p(da[1]) if da else None, _st())
        else:
            _lib.call("sg_last_deconv_wgrad_fold_1src", _p(dwq[1]), half, _p(dw[1]), _st())
    fold()
    torch.cuda.synchronize()
    (r, m), rda, after = M.last_deconv_fold(dwq0, half, nsrc, w, al, dw0, da0 if with_dalpha else None)
    c = [M.c_vec(dw[1], r, m)] + ([M.c_vec(da[1], *rda)] if da else [])
    print("last_deconv_wgrad_fold nsrc=%d half=%d: c" % (nsrc, half), [round(x, 2) for x in c])
    assert all(v <= C_TOL for v in c) and M.bits_equal(dwq[1], after)
    once = (dw[1].clone(), da[1].clone() if da else None)
    fold()                                                                    # on the cleared blocks: adds exactly 0
    torch.cuda.synchronize()
    assert M.bits_equal(dw[1], once[0]) and (da is None or M.bits_equal(da[1], once[1]))
    assert _g([dwq, dw] + ([da] if da else []))
