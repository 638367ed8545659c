"""The fp64 layer references of tests/kwidth_layer_model.py against the tap form the engine runs -- packed weights
(engine.pack_reference), tap tables and spans (engine.tap_ranges, tap_span, dgrad_span) and row-shifted operands
(tests/tapgemm_model.py) -- at every kernel width 4..32, in fp64: the two differ only in summation order.  Also: the
Generator's data-gradient spans against the Discriminator's, and the GPU cases of tests/test_gpu_kwidth_layers.py
cover every partial phase range and tap-span length the tables produce.  Runs without a GPU."""
import pytest
import torch

from segan_pytorch_b200 import engine as E
from tests import kwidth_layer_model as K, tapgemm_model as M

B, R = 2, 5
CIN, COUT = 3, 2          # conv: cin -> cout; deconv: cin -> cout with the same counts
TOL = 1e-12               # relative to the magnitude: fp64 summation order only


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, dtype=torch.float64)


def _close(got, ref, mag, what):
    err = float(((got - ref).abs() / (mag + 1e-300)).max())
    assert err <= TOL, (what, err)


def _slots(packed, d_lo):
    """[d_hi - d_lo + 1][nc][kc] -> [9][nc][kc]"""
    out = packed.new_zeros((9,) + tuple(packed.shape[1:]))
    out[d_lo + 4:d_lo + 4 + packed.shape[0]] = packed
    return out


@pytest.mark.parametrize("k", K.WIDTHS)
def test_conv_references_match_the_tap_form(k):
    g = _gen(k)
    w, bias = _randn(g, COUT, CIN, k), _randn(g, COUT)
    xp, gy = _randn(g, B, CIN, 4 * R + 2 * K.HALO), _randn(g, B, COUT, R)
    a, gr = K.ncl_to_rows(xp), gy.permute(0, 2, 1)                  # [B][R + 8][4 cin], [B][R][cout]
    m = E.pack_reference(0, w, COUT, CIN, 0, k)                     # [9][cout][4 cin]
    taps = E.tap_ranges("conv_fwd", CIN, 4 * CIN, COUT, k)
    d_lo, d_hi = E.tap_span(taps)

    ref, mag = K.conv_fwd(xp, w, k, bias)
    got, _ = M.ref_f(a, None, 4, m, taps, 0, R, d_lo, d_hi, bias=bias)
    _close(got, ref.permute(0, 2, 1), mag.permute(0, 2, 1), "conv forward")

    taps_dg = E.tap_ranges("conv_dgrad", CIN, COUT, 4 * CIN, k)
    ref, mag = K.conv_dgrad(gy, w, k)
    got, _ = M.ref_f(gr, None, 0, m.flip(0).transpose(1, 2), taps_dg, -4, R + 4, *E.tap_span(taps_dg))
    _close(got, K.ncl_to_rows(ref), K.ncl_to_rows(mag), "conv data gradient")
    # the positions the conv never reads get exactly zero
    L = 4 * R
    read = torch.zeros(4 * R + 2 * K.HALO, dtype=torch.bool)
    read[K.HALO - (k // 2 - 1):K.HALO + L + k // 2] = True
    assert not ref[..., ~read].any() and not K.rows_to_ncl(got, CIN)[..., ~read].any()

    ref, mag = K.conv_wgrad(xp, gy, k)
    got, _ = M.ref_w(gr, a, None, 4, taps, d_lo, d_hi)
    _close(E.unpack_reference(0, _slots(got, d_lo), COUT, CIN, 0, k), ref, mag, "conv weight gradient")
    assert torch.equal(K.packed_live(0, k, COUT, CIN), E.pack_reference(0, torch.ones_like(w), COUT, CIN, 0, k) != 0)


@pytest.mark.parametrize("k", K.WIDTHS)
def test_deconv_references_match_the_tap_form(k):
    """Two sources (1 + 2 channels) as the decoder's concat reads them."""
    g = _gen(100 + k)
    c0 = 1
    w, bias = _randn(g, CIN, COUT, k), _randn(g, COUT)
    x, gy = _randn(g, B, CIN, R), _randn(g, B, COUT, 4 * R)
    a0, a1 = x[:, :c0].permute(0, 2, 1), x[:, c0:].permute(0, 2, 1)
    gr = K.ncl_to_rows(gy)                                          # [B][R][4 cout]
    m = E.pack_reference(1, w, COUT, CIN, 0, k)                     # [9][4 cout][cin]
    taps = E.tap_ranges("deconv_fwd", COUT, CIN, 4 * COUT, k)
    d_lo, d_hi = E.tap_span(taps)

    ref, mag = K.deconv_fwd(x, w, k, bias)
    assert ref.shape[-1] == 4 * R
    got, _ = M.ref_f(a0, a1, 0, m, taps, 0, R, d_lo, d_hi, bias=bias)
    _close(got, K.ncl_to_rows(ref), K.ncl_to_rows(mag), "deconv forward")

    taps_dg = E.tap_ranges("deconv_dgrad", COUT, 4 * COUT, CIN, k)
    ref, mag = K.deconv_dgrad(gy, w, k)
    got, _ = M.ref_f(gr, None, 0, m.flip(0).transpose(1, 2), taps_dg, 0, R, *E.dgrad_span(taps))
    _close(got, ref.permute(0, 2, 1), mag.permute(0, 2, 1), "deconv data gradient")

    ref, mag = K.deconv_wgrad(x, gy, k)
    got, _ = M.ref_w(gr, a0, a1, 0, taps, d_lo, d_hi)
    _close(E.unpack_reference(1, _slots(got, d_lo), COUT, CIN, 0, k), ref, mag, "deconv weight gradient")
    assert torch.equal(K.packed_live(1, k, COUT, CIN), E.pack_reference(1, torch.ones_like(w), COUT, CIN, 0, k) != 0)


def test_generator_and_discriminator_data_gradient_spans_agree():
    """The Generator mirrors the forward span (dgrad_span), the Discriminator takes tap_span of the data-gradient
    table: the same taps at every width, including the widths whose span is not symmetric."""
    asym = set()
    for k in K.WIDTHS:
        for base, c in (("conv", 64), ("deconv", 64)):
            fwd = E.tap_ranges(base + "_fwd", c, 4 * c, 128, k) if base == "conv" else \
                E.tap_ranges("deconv_fwd", c, 128, 4 * c, k)
            dg = E.tap_ranges("conv_dgrad", c, 128, 4 * c, k) if base == "conv" else \
                E.tap_ranges("deconv_dgrad", c, 4 * c, 128, k)
            assert E.dgrad_span(fwd) == E.tap_span(dg), (k, base)
            d_lo, d_hi = E.tap_span(fwd)
            if d_lo != -d_hi:
                asym.add(k)
    assert asym, "no width with an asymmetric span: the comparison above cannot tell a mirror from none"


def _table_features(name, c, k):
    """(partial phase ranges, span length) of one tap table: a partial range is (lo, hi) in units of c of a tap that
    reads some but not all of the four phase blocks."""
    on_k = name in ("conv_fwd", "deconv_dgrad")
    kc, nc = (4 * c, 2 * c) if on_k else (2 * c, 4 * c)
    taps = E.tap_ranges(name, c, kc, nc, k)
    lo, hi = (taps[0], taps[1]) if on_k else (taps[2], taps[3])
    full = kc if on_k else nc
    d_lo, d_hi = E.tap_span(taps)
    parts = {(lo[i] // c, hi[i] // c) for i in range(9) if 0 < hi[i] - lo[i] < full}
    return parts, d_hi - d_lo + 1


def test_gpu_cases_cover_every_partial_range_and_span():
    """For each forward-form and weight-gradient table the GPU test launches, its cases at c = 64 reach every partial
    phase range and every tap-span length that tap_ranges produces over the served widths."""
    from tests import test_gpu_kwidth_layers as L
    want, got = {}, {}
    for kind, (form, name) in L.TABLES.items():
        key = (form, name)
        for k in range(E.KW_MIN, E.KW_MAX + 1):
            parts, span = _table_features(name, 64, k)
            want.setdefault(key, (set(), set()))
            want[key][0].update(parts)
            want[key][1].add(span)
        for kk, k, c in L.CASES:
            if kk == kind and c == 64:
                parts, span = _table_features(name, 64, k)
                got.setdefault(key, (set(), set()))
                got[key][0].update(parts)
                got[key][1].add(span)
    assert set(want) == {("F", n) for n in ("conv_fwd", "conv_dgrad", "deconv_fwd", "deconv_dgrad")} | \
        {("W", "conv_fwd"), ("W", "deconv_fwd")}
    for key, (parts, spans) in want.items():
        assert parts <= got[key][0], (key, sorted(parts - got[key][0]))
        assert spans <= got[key][1], (key, sorted(spans - got[key][1]))
    # the ranges width 31 never produces are among them (the reason for the GPU test)
    assert {(0, 3), (3, 4), (1, 4), (0, 2)} <= want[("F", "conv_fwd")][0]
    assert {(0, 1), (2, 4), (0, 3), (1, 4)} <= want[("F", "deconv_fwd")][0]
    assert min(s for _, ss in want.values() for s in ss) == 1
