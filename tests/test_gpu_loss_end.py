"""The kernels at the loss end of a training step against fp64 (tests/step_end_model.py): the Discriminator's fc tail
(sg_fc_tail_fwd / sg_fc_tail_bwd), the G regression losses (sg_l1_loss_bwd / sg_mse_loss_bwd) and WSEGAN's
spectral-loss glue (sg_stft_frames / sg_logpow_l1 / sg_stft_frames_fold).  Every destination sits between sentinel
guard bands and starts non-zero where the kernel accumulates into it; outputs without atomics must repeat bit for
bit.  Arithmetic is gated at c <= C_TOL (units of U * sum|terms|), data movement bit for bit.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from segan_pytorch_b200 import _lib, engine as E                # noqa: E402
from segan_pytorch_b200._lib import SG_BF16, SG_F16            # noqa: E402
from tests import step_end_model as M                          # noqa: E402

DEV = "cuda"
C_TOL = M.C_TOL
TDT = {"f16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(params=["f16", "bf16"])
def grad_dtype(request):
    """The 16-bit gradient format (sg_set_grad_dtype) for one test; the previous setting is restored after it."""
    prev = "bf16" if E.GS == SG_BF16 else "f16"
    E.set_grad_dtype(request.param)
    yield request.param
    E.set_grad_dtype(prev)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _g(buf_view_pairs):
    return all(M.guards_ok(b) for b, _ in buf_view_pairs)


# ------------------------------------------------------------------------------------------------------
# fc tail
# ------------------------------------------------------------------------------------------------------
def _fc_params(seed):
    """fc tail weights with per-channel slopes (0 = the reference init, 1, random) and exact zeros in z1 and z2:
    fc0_acc = b0 = 0 on channels 0..7 and w2 = b2 = 0 on outputs 0..3."""
    g = _gen(seed)
    b0 = 0.1 * torch.randn(256, generator=g)
    b0[:8] = 0.0
    s1 = torch.rand(256, generator=g)
    s1[:4], s1[4:6] = 0.0, 1.0
    w2 = 0.1 * torch.randn(128, 256, generator=g)
    w2[:4] = 0.0
    b2 = 0.1 * torch.randn(128, generator=g)
    b2[:4] = 0.0
    s3 = torch.rand(128, generator=g)
    s3[4:6], s3[6:8] = 0.0, 1.0
    w4 = 0.1 * torch.randn(1, 128, generator=g)
    b4 = torch.tensor([0.02])
    return [t.to(DEV) for t in (b0, s1, w2, b2, s3, w4, b4)]


def _fc_forward(B, seed):
    g = _gen(seed + 1)
    acc = torch.randn(B, 256, generator=g)
    acc[:, :8] = 0.0
    acc = acc.to(DEV)
    b0, s1, w2, b2, s3, w4, b4 = _fc_params(seed)
    outs = [M.guarded(s, torch.float32, DEV) for s in ((B, 256), (B, 128), (B,))]
    _lib.call("sg_fc_tail_fwd", _p(acc), _p(b0), _p(s1), _p(w2), _p(b2), _p(s3), _p(w4), _p(b4), B,
              *[_p(v) for _, v in outs], _st())
    return dict(acc=acc, b0=b0, s1=s1, w2=w2, b2=b2, s3=s3, w4=w4, b4=b4, outs=outs)


@pytest.mark.parametrize("B", [1, 15, 16, 17, 300])
def test_fc_tail_fwd_vs_fp64(B):
    k = _fc_forward(B, 100 + B)
    (bz1, z1), (bz2, z2), (bl, logit) = k["outs"]
    again = _fc_forward(B, 100 + B)["outs"]
    torch.cuda.synchronize()
    c = dict(z1=M.c_vec(z1, *M.fc_z1(k["acc"], k["b0"])), z2=M.c_vec(z2, *M.fc_z2(z1, k["s1"], k["w2"], k["b2"])),
             logit=M.c_vec(logit, *M.fc_logit(z2, k["s3"], k["w4"], k["b4"])))
    print("fc_tail_fwd B=%d: c" % B, {n: round(v, 2) for n, v in c.items()})
    assert all(v <= C_TOL for v in c.values()), c
    assert float((z1[:, :8] == 0).float().min()) == 1 and float((z2[:, :4] == 0).float().min()) == 1
    assert _g(k["outs"])
    assert all(M.bits_equal(a[1], b[1]) for a, b in zip(k["outs"], again))      # no atomics: the same bits


PARAM_NAMES = ("b0", "s1", "w2", "b2", "s3", "w4", "b4")


@pytest.mark.parametrize("path", ["mse_t1", "mse_t0", "g_logit_in"])
@pytest.mark.parametrize("B", [1, 15, 16, 17, 300])
def test_fc_tail_bwd_vs_fp64(B, path, grad_dtype):
    """Rows (d loss / d logit, g_z2, g_h1, g_z1 and its 16-bit copy) and parameter gradients, each stage on the
    kernel's own workspace of the stage before.  grad_scale 1024 on odd batches, else 1; loss_out NULL on the
    g_logit_in path; a second launch with g_w2 = NULL (the G step) must repeat the rows' bits and touch no parameter
    gradient."""
    fmt = grad_dtype
    k = _fc_forward(B, 200 + B)
    (_, z1), (_, z2), (_, logit) = k["outs"]
    g = _gen(300 + B)
    gscale = 1024.0 if B % 2 else 1.0
    target, weight = (0.0 if path == "mse_t0" else 1.0), 0.7
    g_in = torch.randn(B, generator=g).to(DEV) if path == "g_logit_in" else None
    shapes = dict(b0=(256,), s1=(256,), w2=(128, 256), b2=(128,), s3=(128,), w4=(128,), b4=(1,))
    p0 = {n: torch.randn(*shapes[n], generator=g).to(DEV) for n in PARAM_NAMES}
    pg = {n: M.guarded(shapes[n], torch.float32, DEV, p0[n]) for n in PARAM_NAMES}
    loss = None if g_in is not None else M.guarded((1,), torch.float32, DEV, torch.tensor([0.25]))
    ws = M.guarded((B * 641,), torch.float32, DEV)
    gz1 = M.guarded((B, 256), TDT[fmt], DEV)

    def run(ws_, gz1_, with_params):
        _lib.call("sg_fc_tail_bwd", _p(z1), _p(z2), _p(logit), _p(g_in), target, weight, _p(k["s1"]), _p(k["w2"]),
                  _p(k["s3"]), _p(k["w4"]), B, _p(loss[1]) if loss and with_params else None, _p(gz1_[1]), _p(ws_[1]),
                  *[_p(pg[n][1]) if with_params else None for n in PARAM_NAMES], gscale, _st())
    run(ws, gz1, True)
    torch.cuda.synchronize()
    after = {n: pg[n][1].clone() for n in PARAM_NAMES}
    ws2, gz1b = M.guarded((B * 641,), torch.float32, DEV), M.guarded((B, 256), TDT[fmt], DEV)
    run(ws2, gz1b, False)
    torch.cuda.synchronize()
    w = ws[1]
    gl, g_z2 = w[:B], w[B:B + B * 128].view(B, 128)
    g_z1, g_h1 = w[B + B * 128:B + B * 384].view(B, 256), w[B + B * 384:].view(B, 256)
    c = {}
    c["g_logit"] = M.c_vec(gl, *M.fc_g_logit(logit, g_in, target, weight, B, gscale))
    if loss is not None:
        lr, lm = M.fc_loss(logit, target, weight, B)
        c["loss"] = M.c_vec(loss[1], 0.25 + lr, 0.25 + lm)
    c["g_z2"] = M.c_vec(g_z2, *M.fc_g_z2(z2, gl, k["s3"], k["w4"]))
    (rh1, mh1), (rz1, mz1) = M.fc_g_h1_z1(g_z2, z1, k["s1"], k["w2"])
    c["g_h1"], c["g_z1"] = M.c_vec(g_h1, rh1, mh1), M.c_vec(g_z1, rz1, mz1)
    c["g_z1_16"] = M.c_f(gz1[1], rz1, mz1, fmt)
    ref = M.fc_params(z1, z2, gl, g_z2, g_z1, g_h1, k["s1"], k["s3"], k["w4"], p0)
    for n in PARAM_NAMES:
        c["g_" + n] = M.c_vec(after[n].reshape(ref[n][0].shape), *ref[n])
    print("fc_tail_bwd B=%d %s %s: c" % (B, path, fmt), {n: round(v, 2) for n, v in c.items()})
    assert all(v <= C_TOL for v in c.values()), c
    assert _g([ws, gz1, ws2, gz1b] + list(pg.values()) + ([loss] if loss else []))
    assert M.bits_equal(ws2[1], ws[1]) and M.bits_equal(gz1b[1], gz1[1])     # rows: no atomics
    assert all(M.bits_equal(pg[n][1], after[n]) for n in PARAM_NAMES)          # g_w2 NULL: no parameter touched


def test_fc_tail_bwd_fp16_g_z1_saturates_and_keeps_nan():
    """A loss-scaled fp16 g_z1 past 65504 stores +-65504 (not inf, which would poison fc.0's gradients), and a NaN
    gradient stays NaN (a clip with fminf / fmaxf would turn it into -65504 and hide a poisoned step)."""
    prev = "bf16" if E.GS == SG_BF16 else "f16"
    E.set_grad_dtype("f16")
    try:
        B = 3
        k = _fc_forward(B, 401)
        (_, z1), (_, z2), (_, logit) = k["outs"]
        g_in = torch.tensor([1e5, -1e5, float("nan")], device=DEV)
        ws = M.guarded((B * 641,), torch.float32, DEV)
        gz1 = M.guarded((B, 256), torch.float16, DEV)
        _lib.call("sg_fc_tail_bwd", _p(z1), _p(z2), _p(logit), _p(g_in), 1.0, 1.0, _p(k["s1"]), _p(k["w2"]),
                  _p(k["s3"]), _p(k["w4"]), B, None, _p(gz1[1]), _p(ws[1]), *[None] * 7, 1024.0, _st())
        torch.cuda.synchronize()
    finally:
        E.set_grad_dtype(prev)
    got = gz1[1].float()
    w = ws[1]
    g_z2 = w[B:B + B * 128].view(B, 128)
    _, (rz1, mz1) = M.fc_g_h1_z1(g_z2[:2], z1[:2], k["s1"], k["w2"])
    n_sat = int((got[:2].abs() == 65504).sum())
    print("fp16 g_z1: %d of 512 saturated, %d inf, row 2 NaN: %d / 256" % (n_sat, int(torch.isinf(got).sum()),
                                                                         int(torch.isnan(got[2]).sum())))
    assert not torch.isinf(got).any()
    assert n_sat > 100 and M.c_f(gz1[1][:2], rz1, mz1, "f16") <= C_TOL
    assert torch.isnan(got[2]).all() and not M.sentinel_mask(gz1[1][2]).any()    # written (the sentinel is a NaN too)
    assert _g([ws, gz1])


# ------------------------------------------------------------------------------------------------------
# regression losses
# ------------------------------------------------------------------------------------------------------
LOSS_KERNEL = {"l1": "sg_l1_loss_bwd", "mse": "sg_mse_loss_bwd"}


def _reg_inputs(n, seed):
    g = _gen(seed)
    y = torch.randn(n, generator=g)
    clean = torch.randn(n, generator=g)
    clean[::7] = y[::7]                                   # exact d = 0
    return y.to(DEV), clean.to(DEV)


@pytest.mark.parametrize("n", [1, 255, 256 * 264 - 1, 256 * 264 + 1, 300 * 16384])
@pytest.mark.parametrize("kind", ["l1", "mse"])
def test_reg_loss_vs_fp64(kind, n):
    """loss_out += w mean(term) and gy (=|+=) grad_scale * d/dy: weight 100, accumulate 0 with grad_scale 1 and
    accumulate 1 with 1024; the loss (fixed-order partial sums) and gy repeat bit for bit."""
    y, clean = _reg_inputs(n, 500 + n % 97)
    for acc, gscale in ((0, 1.0), (1, 1024.0)):
        gy0 = torch.randn(n, generator=_gen(7 + acc)).to(DEV)
        runs = []
        for _ in range(2):
            loss = M.guarded((1,), torch.float32, DEV, torch.tensor([0.25]))
            gy = M.guarded((n,), torch.float32, DEV, gy0)
            _lib.call(LOSS_KERNEL[kind], _p(y), _p(clean), n, 100.0, _p(loss[1]), _p(gy[1]), acc, gscale, _st())
            runs.append((loss, gy))
        torch.cuda.synchronize()
        ref = M.reg_loss(kind, y, clean, 100.0, gscale, gy0 if acc else None)
        (loss, gy), (loss2, gy2) = runs
        lr, lm = ref["loss"]
        c = (M.c_vec(loss[1], 0.25 + lr, 0.25 + lm), M.c_vec(gy[1], *ref["gy"]))
        print("%s n=%d accumulate %d grad_scale %g: c loss %.2f gy %.2f" % (kind, n, acc, gscale, *c))
        assert all(v <= C_TOL for v in c), c
        assert M.bits_equal(loss2[1], loss[1]) and M.bits_equal(gy2[1], gy[1])
        assert _g([loss, gy, loss2, gy2])


def test_reg_losses_interleaved_on_one_stream_repeat_bits():
    """L1, MSE, L1, MSE back to back on one stream: each kernel's arrival counter resets itself, so the repeats give
    the same loss bits (a counter left behind would end the sum early or never)."""
    n = 300 * 16384
    y, clean = _reg_inputs(n, 601)
    outs = [M.guarded((1,), torch.float32, DEV, torch.zeros(1)) for _ in range(6)]
    for i, kind in enumerate(("l1", "mse", "l1", "mse", "l1", "mse")):
        _lib.call(LOSS_KERNEL[kind], _p(y), _p(clean), n, 100.0, _p(outs[i][1]), None, 0, 1.0, _st())
    torch.cuda.synchronize()
    v = [o[1] for o in outs]
    assert M.bits_equal(v[0], v[2]) and M.bits_equal(v[0], v[4])
    assert M.bits_equal(v[1], v[3]) and M.bits_equal(v[1], v[5])
    for kind, got in (("l1", v[0]), ("mse", v[1])):
        assert M.c_vec(got, *M.reg_loss(kind, y, clean, 100.0, 1.0)["loss"]) <= C_TOL
    assert _g(outs)


def test_l1_offset_subrun():
    """WSEGAN's masked L1 (model.py:1142): one launch over the windows i..j-1 of a batch, pointers offset into the
    batch, weight w * n_run / (B L), accumulating into gy: the samples outside the run keep their bits."""
    B, L, i, j = 5, 16384, 1, 4
    y, clean = _reg_inputs(B * L, 602)
    gy0 = torch.randn(B * L, generator=_gen(9)).to(DEV)
    gy = M.guarded((B * L,), torch.float32, DEV, gy0)
    loss = M.guarded((1,), torch.float32, DEV, torch.tensor([0.5]))
    n_run = (j - i) * L
    w = 100.0 * n_run / (B * L)
    off = 4 * i * L
    _lib.call("sg_l1_loss_bwd", C.c_void_p(y.data_ptr() + off), C.c_void_p(clean.data_ptr() + off), n_run, w,
              _p(loss[1]), C.c_void_p(gy[1].data_ptr() + off), 1, 1024.0, _st())
    torch.cuda.synchronize()
    ref = M.reg_loss("l1", y[i * L:j * L], clean[i * L:j * L], w, 1024.0, gy0[i * L:j * L])
    lr, lm = ref["loss"]
    assert M.c_vec(loss[1], 0.5 + lr, 0.5 + lm) <= C_TOL
    assert M.c_vec(gy[1][i * L:j * L], *ref["gy"]) <= C_TOL
    assert M.bits_equal(gy[1][:i * L], gy0[:i * L]) and M.bits_equal(gy[1][j * L:], gy0[j * L:])
    assert _g([gy, loss])


# ------------------------------------------------------------------------------------------------------
# STFT glue
# ------------------------------------------------------------------------------------------------------
STFT_SHAPES = [(1025, 3), (16384, 300), (16384 + 159, 1), (5000, 3)]     # 5000: not a multiple of 160


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("fmt", ["f16", "bf16"])
@pytest.mark.parametrize("L,B", STFT_SHAPES)
def test_stft_frames_bit_exact(L, B, fmt, split):
    x = (0.5 * torch.randn(B, L, generator=_gen(L + B))).clamp(-1, 1).to(DEV)
    ref = M.stft_frames(x, fmt, split)
    out = M.guarded(tuple(ref.shape), TDT[fmt], DEV)
    _lib.call("sg_stft_frames", _p(x), B, L, _p(out[1]), SG_F16 if fmt == "f16" else SG_BF16, split, _st())
    torch.cuda.synchronize()
    assert M.bits_equal(out[1], ref)
    assert _g([out])


def _spectra(rows, ld, bins, half, seed, identical=False):
    """Spectra over 12 decades of power, with identical bins (d = 0 exactly), zero-power bins and a stripe of columns
    between the live ones."""
    g = _gen(seed)
    xg = torch.randn(rows, ld, generator=g) * 10.0 ** (torch.rand(rows, ld, generator=g) * 6 - 5)
    xc = xg * (1 + 0.3 * torch.randn(rows, ld, generator=g))
    for c0 in (0, half):
        xc[:, c0:c0 + 8] = xg[:, c0:c0 + 8]
        xg[:, c0 + 8:c0 + 12] = 0.0
        xc[:, c0 + 10:c0 + 14] = 0.0
    return xg.to(DEV), (xg.clone() if identical else xc).to(DEV)


def _gx_live(gx, bins, half):
    return torch.stack((gx[:, :bins], gx[:, half:half + bins]), 1)


@pytest.mark.parametrize("fmt", ["f16", "bf16"])
@pytest.mark.parametrize("rows,bins,half,ld", [(309, 1025, 1088, 2176), (300 * 103, 1025, 1088, 2176),
                                               (309, 1025, 1100, 2300)])
def test_logpow_l1_vs_fp64(rows, bins, half, ld, fmt):
    """Loss and 16-bit gradient at the production layout (bins 1025, half 1088, ld 2176) and a wider one; the pad
    columns are never written; with g_x NULL only the loss changes."""
    xg, xc = _spectra(rows, ld, bins, half, rows + ld)
    loss = M.guarded((1,), torch.float32, DEV, torch.tensor([0.5]))
    gx = M.guarded((rows, ld), TDT[fmt], DEV)
    dt = SG_F16 if fmt == "f16" else SG_BF16
    _lib.call("sg_logpow_l1", _p(xg), _p(xc), rows, bins, half, ld, 0.37, _p(loss[1]), _p(gx[1]), dt, 8.0, _st())
    loss2 = M.guarded((1,), torch.float32, DEV, torch.tensor([0.5]))
    _lib.call("sg_logpow_l1", _p(xg), _p(xc), rows, bins, half, ld, 0.37, _p(loss2[1]), None, dt, 8.0, _st())
    torch.cuda.synchronize()
    ref = M.logpow_l1(xg, xc, bins, half, 0.37, 8.0)
    lr, (budget, lm) = ref["loss"]
    got = _gx_live(gx[1], bins, half)
    c = (M.c_budget(loss[1], 0.5 + lr, budget, 0.5 + lm), M.c_budget(loss2[1], 0.5 + lr, budget, 0.5 + lm),
         M.c_logpow_gx(got, ref["gx"], ref["d"], fmt))
    print("logpow_l1 rows %d half %d ld %d %s: c loss %.2f (no g_x %.2f) g_x %.2f" % (rows, half, ld, fmt, *c))
    assert all(v <= C_TOL for v in c), c
    assert float(got[:, :, :8].abs().max()) == 0.0                 # identical bins: gradient exactly 0
    untouched = torch.cat((gx[1][:, bins:half], gx[1][:, half + bins:]), 1)
    assert M.is_sentinel(untouched)                                  # pad columns are never written
    assert _g([loss, loss2, gx])


def test_logpow_l1_identical_spectra_give_zero():
    rows, bins, half, ld = 309, 1025, 1088, 2176
    xg, _ = _spectra(rows, ld, bins, half, 77, identical=True)
    loss = M.guarded((1,), torch.float32, DEV, torch.tensor([0.5]))
    gx = M.guarded((rows, ld), torch.bfloat16, DEV)
    _lib.call("sg_logpow_l1", _p(xg), _p(xg.clone()), rows, bins, half, ld, 0.37, _p(loss[1]), _p(gx[1]), SG_BF16,
              8.0, _st())
    torch.cuda.synchronize()
    assert float(loss[1]) == 0.5
    assert float(_gx_live(gx[1], bins, half).float().abs().max()) == 0.0
    assert _g([loss, gx])


@pytest.mark.parametrize("L,B", STFT_SHAPES)
def test_stft_frames_fold_vs_fp64(L, B):
    fr = 1 + L // 160
    g = _gen(L * 3 + B)
    gf = torch.randn(B, fr, 320, generator=g).to(DEV)
    g0 = torch.randn(B, L, generator=g).to(DEV)
    gw = M.guarded((B, L), torch.float32, DEV, g0)
    _lib.call("sg_stft_frames_fold", _p(gf), B, L, 0.37, _p(gw[1]), _st())
    torch.cuda.synchronize()
    c = M.c_vec(gw[1], *M.stft_fold(gf, L, 0.37, g0))
    print("stft_frames_fold L=%d B=%d: c %.2f" % (L, B, c))
    assert c <= C_TOL
    assert _g([gw])


# ------------------------------------------------------------------------------------------------------
# argument refusals: nothing is launched, the destinations keep their bits
# ------------------------------------------------------------------------------------------------------
def test_loss_end_refuses_bad_arguments():
    B = 4
    t = torch.randn(B * 1024, device=DEV)
    d = torch.randn(B * 641, device=DEV)
    g16 = torch.randn(B, 256, device=DEV).half()
    snap = (t.clone(), d.clone(), g16.clone())
    bad_fwd = [(0, _p(t)), (B, None)]
    for batch, acc in bad_fwd:
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_fc_tail_fwd", acc, *[_p(t)] * 7, batch, _p(d), _p(d), _p(d), _st())
    pg = [_p(d)] * 7
    for batch, z1, params in ((0, _p(t), pg), (B, None, pg), (B, _p(t), [_p(d), None] + [_p(d)] * 5)):
        with pytest.raises(_lib.SeganB200Error):
            _lib.call("sg_fc_tail_bwd", z1, _p(t), _p(t), None, 1.0, 1.0, _p(t), _p(t), _p(t), _p(t), batch, _p(d),
                      _p(g16), _p(d), *params, 1.0, _st())
    for name in LOSS_KERNEL.values():
        for n, y in ((0, _p(t)), (-5, _p(t)), (16, None)):
            with pytest.raises(_lib.SeganB200Error):
                _lib.call(name, y, _p(t), n, 1.0, _p(d), _p(d), 1, 1.0, _st())
    torch.cuda.synchronize()
    assert torch.equal(t, snap[0]) and torch.equal(d, snap[1]) and torch.equal(g16, snap[2])
