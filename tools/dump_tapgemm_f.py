"""Saves what the forward-form tap-GEMM writes at the train step's shapes (batch 300) from seeded inputs, so that two
builds can be compared bit for bit:

    python tools/dump_tapgemm_f.py OUT.pt            # in each tree
    python tools/dump_tapgemm_f.py --compare A.pt B.pt

Every output buffer starts as a fixed bit pattern, so the comparison also covers what a launch must leave alone."""
import sys

import torch

from segan_pytorch_b200 import engine as E
from segan_pytorch_b200._lib import SG_BF16, SG_F16

B = 300
DEV = "cuda"
SENTINEL = 0x7E5A


def _t(g, dt, *shape):
    return (torch.randn(*shape, generator=g, device=DEV) * 0.5).to(dt)


def _buf(dt, *shape):
    t = torch.empty(*shape, device=DEV, dtype=dt)
    t.view(torch.int16).fill_(SENTINEL)
    return t


def conv_fwd(g, cin, cout, R, out2_halo=None):
    a, w = _t(g, torch.float16, B, R + 8, 4 * cin), _t(g, torch.float16, 9, cout, 4 * cin) * 0.1
    bias, slope = torch.randn(cout, generator=g, device=DEV), torch.rand(cout, generator=g, device=DEV) * 0.3
    out = _buf(torch.float16, B, R, cout)
    kw, res = {}, {"out": out}
    if out2_halo is not None:
        res["out2"] = _buf(torch.float16, B, R + 2 * out2_halo, cout)
        kw = dict(out2=res["out2"], out2_halo=out2_halo, slope=slope, slope_mod=cout)
    E.run_f(a, None, R, 4, SG_F16, w, SG_F16, 4 * cin, cout, E.tap_ranges("conv_fwd", cin, 4 * cin, cout), out, SG_F16,
            R, 0, 0, R, B, bias=bias, bias_mod=cout, backend=1, **kw)
    return res


def deconv_fwd(g, cin, cout, R, mode=None):
    """mode None: one output; "out2": raw output + PReLU output (training); "inplace": PReLU output only."""
    a0, a1 = _t(g, torch.float16, B, R, cin // 2), _t(g, torch.float16, B, R, cin // 2)
    w = _t(g, torch.float16, 9, 4 * cout, cin) * 0.1
    bias, slope = torch.randn(cout, generator=g, device=DEV), torch.rand(cout, generator=g, device=DEV) * 0.3
    out = _buf(torch.float16, B, R, 4 * cout)
    kw, res = {}, {"out": out}
    if mode == "out2":
        res["out2"] = _buf(torch.float16, B, 4 * R, cout)
        kw = dict(out2=res["out2"], slope=slope, slope_mod=cout)
    elif mode == "inplace":
        kw = dict(slope=slope, slope_mod=cout)
    E.run_f(a0, a1, R, 0, SG_F16, w, SG_F16, cin, 4 * cout, E.tap_ranges("deconv_fwd", cout, cin, 4 * cout), out,
            SG_F16, R, 0, 0, R, B, bias=bias, bias_mod=cout, a0_c=cin // 2, a1_c=cin // 2, backend=1, **kw)
    return res


def conv_dgrad(g, cin, cout, R, bf16=False):
    dt, sdt = (torch.bfloat16, SG_BF16) if bf16 else (torch.float16, SG_F16)
    gr, w = _t(g, dt, B, R, cout), _t(g, dt, 9, 4 * cin, cout) * 0.1
    out = _buf(dt, B, R + 8, 4 * cin)
    E.run_f(gr, None, R, 0, sdt, w, sdt, cout, 4 * cin, E.tap_ranges("conv_dgrad", cin, cout, 4 * cin), out, sdt, R, 4,
            -4, R + 4, B, backend=1)
    return {"out": out}


def wave0(g, out2_halo=None):
    col, w = _t(g, torch.float16, B, 4096, 64), _t(g, torch.float16, 1, 64, 64)
    bias, slope = torch.randn(64, generator=g, device=DEV), torch.rand(64, generator=g, device=DEV) * 0.3
    out = _buf(torch.float16, B, 4096, 64)
    kw, res = {}, {"out": out}
    if out2_halo is not None:
        res["out2"] = _buf(torch.float16, B, 4096 + 2 * out2_halo, 64)
        kw = dict(out2=res["out2"], out2_halo=out2_halo, slope=slope, slope_mod=64)
    E.run_f(col, None, 4096, 0, SG_F16, w, SG_F16, 64, 64, E.tap_ranges("full", 0, 64, 64), out, SG_F16, 4096, 0, 0,
            4096, B, bias=bias, bias_mod=64, d_lo=0, d_hi=0, w_tap0=4, backend=1, **kw)
    return res


def wave_dgrad(g, cin, half):
    """The last deconv's data gradient: single-tap GEMM into two column halves (n_lo > 0, out_ld = half)."""
    col, w = _t(g, torch.float16, B, 4096, 64), _t(g, torch.float16, 1, cin, 64)
    res = {}
    for n0 in (0, half):
        res["n%d" % n0] = out = _buf(torch.float16, B, 4096, half)
        E.run_f(col, None, 4096, 0, SG_F16, w, SG_F16, 64, cin, E.tap_ranges("full", 0, 64, cin), out, SG_F16, 4096,
                0, 0, 4096, B, n_lo=n0, n_hi=n0 + half, out_ld=half, out_col0=0, d_lo=0, d_hi=0, w_tap0=4, backend=1)
    return res


SHAPES = [
    ("genc0_out2_h16", lambda g: wave0(g, 16)), ("denc0", wave0),
    ("genc1_out2_h16", lambda g: conv_fwd(g, 64, 128, 1024, 16)), ("enc1", lambda g: conv_fwd(g, 64, 128, 1024)),
    ("enc2", lambda g: conv_fwd(g, 128, 256, 256)), ("genc3_out2_h16", lambda g: conv_fwd(g, 256, 512, 64, 16)),
    ("enc4", lambda g: conv_fwd(g, 512, 1024, 16)),
    ("gdec0_out2", lambda g: deconv_fwd(g, 2048, 512, 16, "out2")),
    ("gdec1_out2", lambda g: deconv_fwd(g, 1024, 256, 64, "out2")),
    ("gdec2_inplace", lambda g: deconv_fwd(g, 512, 128, 256, "inplace")),
    ("dec3", lambda g: deconv_fwd(g, 256, 64, 1024)),
    ("dgrad1", lambda g: conv_dgrad(g, 64, 128, 1024)), ("dgrad3_bf16", lambda g: conv_dgrad(g, 256, 512, 64, True)),
    ("dgrad4", lambda g: conv_dgrad(g, 512, 1024, 16)),
    ("wave_dgrad", lambda g: wave_dgrad(g, 128, 64)),
]


def main():
    if sys.argv[1] == "--compare":
        a, b = torch.load(sys.argv[2]), torch.load(sys.argv[3])
        assert sorted(a) == sorted(b), "different shape lists"
        bad = [k for k in sorted(a) if not torch.equal(a[k], b[k])]
        for k in bad:
            print("DIFFERS: %s (%d of %d elements)" % (k, int((a[k] != b[k]).sum()), a[k].numel()))
        print("%d of %d outputs bitwise equal" % (len(a) - len(bad), len(a)))
        sys.exit(1 if bad else 0)
    res = {}
    for name, fn in SHAPES:
        g = torch.Generator(device=DEV).manual_seed(1 + [n for n, _ in SHAPES].index(name))
        for k, t in fn(g).items():
            res["%s.%s" % (name, k)] = t.view(torch.int16).cpu()
        torch.cuda.synchronize()
    torch.save(res, sys.argv[1])
    print("saved %d outputs to %s" % (len(res), sys.argv[1]))


if __name__ == "__main__":
    main()
