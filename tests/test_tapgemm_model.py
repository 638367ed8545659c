"""The tap-GEMM gate (tests/tapgemm_model.py: c <= 16 in units of 2^-24 * sum |terms|, half an output ulp taken off
16-bit stores) has teeth, shown without a GPU: an fp32-accumulated emulation of each form's sum passes it in any
summation order, and the same emulation with one defect planted fails it by orders of magnitude.

The max-abs gates of tests/test_gpu_kernels.py (form W: 2e-3 * max(1, max|ref|) per tap against an fp32 reference
and `== 0` in the structural-zero blocks of a zero-filled dw; form F: 3e-2 * max(1, max|ref|)) are evaluated on the
same planted defects, at the magnitudes those tests draw (G ~ 0.1 N(0,1), A ~ N(0,1), W ~ 0.05 N(0,1)) and with
every value 2^-10 (form W) / 2^-8 (form F) of that, which leaves c unchanged.  Asserted below:

  defect                                                   c          old gate, test magnitudes   old gate, small values
  W  one position of 2 304 dropped                         1.4e5      fails                       passes
  W  one row read from the next batch element              1.3e5      fails                       passes
  W  a tap read at row offset d + 1                        3.3e6      fails                       fails
  W  two channels swapped inside one 64-block              2.7e6      fails                       fails
  W  k-split partial sums rounded to fp16 before the add   7.0e2      passes                      passes
  W  k-split partial sums rounded to bf16 before the add   6.1e3      fails                       passes
  W  one k-split partial left unscaled by out_scale        2.8e6      not launched: test_tapgemm_w never sets out_scale
  W  0.0f added into a structural-zero block               bits       passes (a zero-filled dw absorbs it; no tap slot
                                                                      outside [d_lo, d_hi] and no guard band exist there)
  F  a tap read at row offset d + 1                        1.3e6      fails                       passes
  F  two channels swapped inside one 64-block              4.3e5      fails                       passes
  F  bias indexed n + 1                                    9.4e5      fails                       passes
  F  accumulator rounded to fp16 after every tap           2.0e3      passes                      passes

So at the magnitudes they draw, the old gates do see an index error that moves whole products; what they cannot
see is anything below 2e-3 / 3e-2 absolute -- a loss of accumulation precision three orders above the arithmetic's
own error, any defect on small values (their floor max(1, .) is absolute, c is scale-free), a stray accumulation
outside the live ranges -- and they never launch out_scale with the production format.  The clean emulation sits at
c < 7.

The paths tests/test_gpu_tapgemm_f.py adds have their own planted defects, each far outside the gate: a row read from
the neighbouring packed batch element instead of the zero fill (3.9e6), an out2 reflect-halo row mirrored one row
off (1.3e9), a bias modulus of 192 applied as a mask (3.1e7), a stream-K finisher that drops one of four partial sums
(1.3e6).  c_f takes the same per-stage truncation allowance as c_w."""
import pytest
import torch

from tests import tapgemm_model as M

INF = float("inf")


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _conv_taps(c, kc, nc):          # engine.tap_ranges("conv_fwd", ...): tap -4 reads phases 2, 3; tap +4 phase 0
    k_lo, k_hi = [0] * 9, [kc] * 9
    k_lo[0], k_hi[0], k_hi[8] = 2 * c, 4 * c, c
    return k_lo, k_hi, [0] * 9, [nc] * 9


# ------------------------------------------------------------------------------------------------------
# form W: 36 batch elements of 64 rows (2 304 positions), a_halo = 0
# ------------------------------------------------------------------------------------------------------
B, R, C_, NC = 36, 64, 64, 128
KC = 4 * C_
TAPS = _conv_taps(C_, KC, NC)
SCALE = 0.37


def _w_problem():
    g = _gen(11)
    gg = (0.1 * torch.randn(B, R, NC, generator=g)).half()
    a = torch.randn(B, R, KC, generator=g).half()
    return gg, a


def _w_operands(gg, a, row_shift=None, wrong_batch=None):
    """G [P][nc] and the row-shifted A [9][P][kc] in fp32 (products of two fp16 values are exact in fp32).
    row_shift: {tap: extra row offset}; wrong_batch: (tap, b, m) reads the next batch element's buffer instead of
    the zero fill past the end of its own."""
    G = gg.float().reshape(B * R, NC)
    A = torch.stack([M.shifted_rows(a, 0, d + (row_shift or {}).get(d, 0), R) for d in range(-4, 5)]).float()
    if wrong_batch is not None:
        d, b, m = wrong_batch
        assert m + d >= R                      # a row past the end: the flat address lands in batch element b + 1
        A[d + 4, b, m] = a[b + 1, m + d - R].float()
    return G, A.reshape(9, B * R, KC)


def _w_sum(G, A, order="forward", ksplit=1, scale=None, unscaled_split=None, skip=None, round_partials=None):
    """fp32 accumulation of sum_p G[p][n] A[d][p][kc]: `forward` / `reversed` one position at a time, `chunk64`
    64-position partial sums (one pipeline stage) added in order; ksplit > 1 adds the splits' partial sums, each
    multiplied by `scale` first (all but `unscaled_split`) or rounded to the 16-bit format `round_partials`."""
    P = [p for p in range(G.shape[0]) if p != skip]
    if order == "reversed":
        P = P[::-1]
    per = -(-len(P) // ksplit)
    total = torch.zeros(9, NC, KC)
    for sp in range(ksplit):
        acc = torch.zeros(9, NC, KC)
        idx = P[sp * per:(sp + 1) * per]
        if order == "chunk64":
            for c0 in range(0, len(idx), 64):
                ii = idx[c0:c0 + 64]
                acc += torch.einsum("pn,dpk->dnk", G[ii], A[:, ii])
        else:
            for p in idx:
                acc += G[p].view(1, NC, 1) * A[:, p].view(9, 1, KC)
        if scale is not None and sp != unscaled_split:
            acc = acc * scale
        if round_partials is not None:
            acc = acc.to(round_partials).float()
        total += acc
    mask = torch.zeros(9, NC, KC)
    for i in range(9):
        mask[i, TAPS[2][i]:TAPS[3][i], TAPS[0][i]:TAPS[1][i]] = 1
    return total * mask, mask


def _old_w_gate(got, ref32, mask):
    """test_gpu_kernels.test_tapgemm_w: per tap max-abs inside the live box, exact zeros outside (zero-filled dw)."""
    for i in range(9):
        err = float(((got[i] - ref32[i]) * mask[i]).abs().max())
        if err > 2e-3 * max(1.0, float(ref32[i].abs().max())) or float((got[i] * (1 - mask[i])).abs().max()) != 0.0:
            return False
    return True


@pytest.fixture(scope="module")
def w_case():
    gg, a = _w_problem()
    ref, mag = M.ref_w(gg, a, None, 0, TAPS)
    G, A = _w_operands(gg, a)
    ref32 = torch.einsum("pn,dpk->dnk", G, A)            # the old tests' fp32 reference (unmasked)
    return gg, a, ref, mag, G, A, ref32


@pytest.mark.parametrize("order,ksplit", [("forward", 1), ("reversed", 1), ("chunk64", 1), ("chunk64", 7),
                                          ("forward", 5)])
def test_w_clean_emulation_passes_in_any_order(w_case, order, ksplit):
    gg, a, ref, mag, G, A, ref32 = w_case
    got, mask = _w_sum(G, A, order, ksplit)
    c = M.c_w(got, ref, mag)
    print("form W emulation %s ksplit %d: c = %.2f" % (order, ksplit, c))
    assert c <= M.C_TOL / 2
    assert _old_w_gate(got, ref32, mask)
    got_s, _ = _w_sum(G, A, order, ksplit, scale=SCALE)
    assert M.c_w(got_s, ref, mag, SCALE) <= M.C_TOL / 2


SMALL_W = 2.0 ** -10
W_PLANTED = {          # name -> (the old gate of test_tapgemm_w lets it through, ... with every value SMALL_W of it)
    "position_dropped": (False, True),
    "next_batch_element_row": (False, True),
    "tap_row_offset": (False, False),
    "channels_swapped": (False, False),
    "partials_rounded_f16": (True, True),
    "partials_rounded_bf16": (False, True),
}


@pytest.mark.parametrize("name", sorted(W_PLANTED))
def test_w_planted_error_fails_the_gate(w_case, name):
    gg, a, ref, mag, G, A, ref32 = w_case
    if name == "position_dropped":
        got, mask = _w_sum(G, A, "chunk64", skip=1000)
    elif name == "next_batch_element_row":       # tap +2, last row of batch element 3: rows 64, 65 are zero fill
        G2, A2 = _w_operands(gg, a, wrong_batch=(2, 3, R - 1))
        got, mask = _w_sum(G2, A2, "chunk64")
    elif name == "tap_row_offset":
        G2, A2 = _w_operands(gg, a, row_shift={1: 1})
        got, mask = _w_sum(G2, A2, "chunk64")
    elif name == "channels_swapped":
        got, mask = _w_sum(G, A, "chunk64")
        got[:, :, [70, 85]] = got[:, :, [85, 70]]
    else:
        got, mask = _w_sum(G, A, "chunk64", ksplit=7,
                           round_partials=torch.float16 if name.endswith("_f16") else torch.bfloat16)
    c = M.c_w(got, ref, mag)
    old = (_old_w_gate(got, ref32, mask), _old_w_gate(got * SMALL_W, ref32 * SMALL_W, mask))
    print("form W planted %s: c = %.3g, old gate %s / %s on small values"
          % (name, c, *("passes" if o else "fails" for o in old)))
    assert c > 20 * M.C_TOL
    assert M.c_w(got * SMALL_W, ref * SMALL_W, mag * SMALL_W) == pytest.approx(c, rel=1e-9)      # scale-free
    assert old == W_PLANTED[name]


def test_w_planted_unscaled_split_fails_the_gate(w_case):
    """One of three k-split partial sums added without out_scale."""
    gg, a, ref, mag, G, A, ref32 = w_case
    got, _ = _w_sum(G, A, "chunk64", ksplit=3, scale=SCALE, unscaled_split=1)
    c = M.c_w(got, ref, mag, SCALE)
    print("form W planted split_unscaled: c = %.3g" % c)
    assert c > 20 * M.C_TOL


def test_w_planted_write_outside_the_live_range(w_case):
    """A stray accumulation of 0.0f into a dead block: invisible in a zero-filled dw (all the old gate looks at);
    where the pre-filled dw0 holds -0.0f it comes back as +0.0f, a bit-level difference.  Any other value there is
    infinitely far out under c_w (mag == 0)."""
    gg, a, ref, mag, G, A, ref32 = w_case
    got, mask = _w_sum(G, A, "chunk64")
    dead = mask == 0
    stray = (1 - mask) * 0.0
    assert _old_w_gate(torch.zeros_like(got) + got + stray, ref32, mask)
    dw0 = torch.full((9, NC, KC), -0.0)
    after = dw0 + stray
    assert not torch.equal(after.view(torch.int32)[dead], dw0.view(torch.int32)[dead])
    got[0, 0, 0] += 1e-6
    assert bool(dead[0, 0, 0]) and M.c_w(got, ref, mag) == INF


# ------------------------------------------------------------------------------------------------------
# form F: test_tapgemm_f's conv_fwd case (3 x 160 rows, a halo of 4, 256 -> 128 channels, fp16 out)
# ------------------------------------------------------------------------------------------------------
FB, FR, FH = 3, 160, 4


def _f_problem():
    g = _gen(12)
    w = 0.05 * torch.randn(9, NC, KC, generator=g)
    for i in range(9):
        mask = torch.zeros(NC, KC)
        mask[TAPS[2][i]:TAPS[3][i], TAPS[0][i]:TAPS[1][i]] = 1
        w[i] *= mask
    a = torch.randn(FB, FR + 2 * FH, KC, generator=g).half()
    bias = torch.randn(NC, generator=g)
    return a, w.half(), bias


def _f_sum(a, w, bias, order="forward", row_shift=None, swap=None, bias_shift=0, round_taps=False):
    """fp32 accumulation over (tap, 64-channel block) steps, bias added to the fp32 sum, one fp16 rounding."""
    steps = [(d, k0) for d in range(-4, 5) for k0 in range(TAPS[0][d + 4], TAPS[1][d + 4], 64)]
    if order == "reversed":
        steps = steps[::-1]
    elif order == "interleaved":
        steps = steps[0::2] + steps[1::2]
    acc = torch.zeros(FB, FR, NC)
    for i, (d, k0) in enumerate(steps):
        rows = M.shifted_rows(a, FH, d + (row_shift or {}).get(d, 0), FR)[..., k0:k0 + 64].float()
        if swap is not None and k0 == 64 * (swap[0] // 64):
            rows[..., [swap[0] - k0, swap[1] - k0]] = rows[..., [swap[1] - k0, swap[0] - k0]]
        acc += rows @ w[d + 4, :, k0:k0 + 64].float().t()
        if round_taps and (i + 1 == len(steps) or steps[i + 1][0] != d):
            acc = acc.half().float()
    return (acc + bias.roll(-bias_shift)).half()


def _old_f_gate(got, ref32):
    return float((got.float() - ref32).abs().max()) <= 3e-2 * max(1.0, float(ref32.abs().max()))


@pytest.mark.parametrize("order", ["forward", "reversed", "interleaved"])
def test_f_clean_emulation_passes_in_any_order(order):
    a, w, bias = _f_problem()
    ref, mag = M.ref_f(a, None, FH, w, TAPS, 0, FR, bias=bias)
    got = _f_sum(a, w, bias, order)
    c = M.c_f(got, ref, mag, "f16")
    print("form F emulation %s: c = %.2f" % (order, c))
    assert c <= M.C_TOL / 4
    assert _old_f_gate(got, ref.float())


SMALL_F = 2.0 ** -8
F_PLANTED = {          # name -> (the old gate of test_tapgemm_f lets it through, ... with every value SMALL_F of it)
    "tap_row_offset": (False, True),
    "channels_swapped": (False, True),
    "bias_shifted": (False, True),
    "accumulator_rounded_f16": (True, True),
}


@pytest.mark.parametrize("name", sorted(F_PLANTED))
def test_f_planted_error_fails_the_gate(name):
    a, w, bias = _f_problem()
    ref, mag = M.ref_f(a, None, FH, w, TAPS, 0, FR, bias=bias)
    kw = {"tap_row_offset": dict(row_shift={1: 1}), "channels_swapped": dict(swap=(70, 85)),
          "bias_shifted": dict(bias_shift=1), "accumulator_rounded_f16": dict(round_taps=True)}[name]
    got = _f_sum(a, w, bias, **kw)
    c = M.c_f(got, ref, mag, "f16")
    old = (_old_f_gate(got, ref.float()), _old_f_gate(got * SMALL_F, (ref * SMALL_F).float()))
    print("form F planted %s: c = %.3g, old gate %s / %s on small values"
          % (name, c, *("passes" if o else "fails" for o in old)))
    assert c > 20 * M.C_TOL
    assert old == F_PLANTED[name]


# ------------------------------------------------------------------------------------------------------
# form F defects of the packed-row, fused-epilogue and stream-K paths (tests/test_gpu_tapgemm_f.py's gate)
# ------------------------------------------------------------------------------------------------------
def _f_steps():
    return [(d, k0) for d in range(-4, 5) for k0 in range(TAPS[0][d + 4], TAPS[1][d + 4], 64)]


def _f_acc(a, halo, w, steps, wrong_batch=None):
    """fp32 sum over the given (tap, 64-channel block) steps.  wrong_batch = (tap, b, m): row m + d lies past the
    end of batch element b's buffer (halo 0), and is read from the next packed batch element instead of as zero."""
    acc = torch.zeros(a.shape[0], FR, NC)
    for d, k0 in steps:
        rows = M.shifted_rows(a, halo, d, FR)[..., k0:k0 + 64].float()
        if wrong_batch is not None and d == wrong_batch[0]:
            _, b, m = wrong_batch
            assert m + d >= FR
            rows[b, m] = a[b + 1, m + d - FR, k0:k0 + 64].float()
        acc += rows @ w[d + 4, :, k0:k0 + 64].float().t()
    return acc


def test_f_truncation_allowance_applies_to_c_f():
    """A 16-bit result 100 U * mag beyond half an ulp (a 300-stage sum that shrank by a third of U * mag per stage)
    passes with the stages declared (a number or one per column) and fails without."""
    got = torch.tensor([[1000.0, -1000.0]]).to(torch.bfloat16)
    mag = torch.tensor([[4000.0, 4000.0]], dtype=torch.float64)
    ref = got.double() + got.double().sign() * (M.half_ulp(got, "bf16") + 100 * M.U * mag)
    assert M.c_f(got, ref, mag, "bf16") == pytest.approx(100.0)
    assert M.c_f(got, ref, mag, "bf16", 300) <= M.C_TOL
    assert M.c_f(got, ref, mag, "bf16", torch.tensor([300.0, 300.0], dtype=torch.float64)) <= M.C_TOL
    assert M.c_f(got, ref, mag, "bf16", torch.tensor([300.0, 0.0], dtype=torch.float64)) > M.C_TOL


def test_f_stages_counts_the_taps_a_tile_reaches():
    assert M.f_stages(TAPS, -4, 4, 0, 128) == 31                 # 7 whole taps x 4 + 2 + 1
    assert M.f_stages(TAPS, -4, 4, 0, 128, split=2) == 16
    assert M.f_stages(TAPS, -4, -4, 0, 128) == 2
    dg = ([0] * 9, [256] * 9, [0] * 9, [512] * 9)
    dg[3][0] = 128                                               # tap -4 reaches columns 0..128 only
    assert M.f_stages(dg, -4, -3, 0, 256) == 8 and M.f_stages(dg, -4, -3, 256, 512) == 4


def test_f_planted_neighbouring_batch_row_fails_the_gate():
    """No halo, +-64 in the first and last row of every batch element: tap +1 of the last row of element 0 reads
    element 1's first row instead of the zero fill."""
    g = _gen(15)
    a, w, bias = _f_problem()
    a = torch.randn(FB, FR, KC, generator=g)
    a[:, 0] = torch.where(torch.rand(FB, KC, generator=g) < 0.5, -64.0, 64.0)
    a[:, -1] = torch.where(torch.rand(FB, KC, generator=g) < 0.5, -64.0, 64.0)
    a = a.half()
    ref, mag = M.ref_f(a, None, 0, w, TAPS, 0, FR, bias=bias)
    clean = (_f_acc(a, 0, w, _f_steps()) + bias).half()
    assert M.c_f(clean, ref, mag, "f16") <= M.C_TOL / 4
    got = (_f_acc(a, 0, w, _f_steps(), wrong_batch=(1, 0, FR - 1)) + bias).half()
    c = M.c_f(got, ref, mag, "f16")
    print("form F planted next_batch_element_row: c = %.3g" % c)
    assert c > 20 * M.C_TOL


def test_f_planted_out2_mirror_row_off_by_one_fails_the_gate():
    """out2 with a reflect halo of 4: row -m is PReLU(out row m); the planted kernel copies row m + 1."""
    a, w, bias = _f_problem()
    slope = 0.3 * torch.rand(NC, generator=_gen(16))
    ref, mag = M.ref_f(a, None, FH, w, TAPS, 0, FR, bias=bias)
    act, mag_act = M.prelu_ref(ref, mag, slope)
    acc = _f_acc(a, FH, w, _f_steps()) + bias
    out2 = torch.where(acc > 0, acc, acc * slope).half()
    h = 4
    want, want_mag = act[:, 1:h + 1].flip(1), mag_act[:, 1:h + 1].flip(1)       # halo rows -h .. -1
    safe = M.sign_safe(ref[:, 1:h + 1].flip(1), mag[:, 1:h + 1].flip(1))
    good = out2[:, 1:h + 1].flip(1)
    assert M.c_f(good[safe], want[safe], want_mag[safe], "f16") <= M.C_TOL / 4
    bad = out2[:, 2:h + 2].flip(1)
    c = M.c_f(bad[safe], want[safe], want_mag[safe], "f16")
    print("form F planted out2_mirror_off_by_one: c = %.3g" % c)
    assert c > 20 * M.C_TOL


def test_f_planted_bias_mod_as_a_mask_fails_the_gate():
    """bias_mod = 192 over 384 channels: n & 191 is not n % 192 (n = 64 reads bias[0])."""
    g = _gen(17)
    nc, mod = 384, 192
    a = torch.randn(2, 32, 64, generator=g).half()
    w = (0.05 * torch.randn(1, nc, 64, generator=g)).half()
    bias = torch.randn(mod, generator=g)
    taps = ([0] * 9, [64] * 9, [0] * 9, [nc] * 9)
    ref, mag = M.ref_f(a, None, 0, w, taps, 0, 32, 0, 0, 4, bias)
    acc = a.float() @ w[0].float().t()
    n = torch.arange(nc)
    clean = (acc + bias[n % mod]).half()
    assert M.c_f(clean, ref, mag, "f16") <= M.C_TOL / 4
    got = (acc + bias[n & (mod - 1)]).half()
    c = M.c_f(got, ref, mag, "f16")
    print("form F planted bias_mod_as_mask: c = %.3g" % c)
    assert c > 20 * M.C_TOL


def test_f_planted_finisher_dropping_a_partial_fails_the_gate():
    """Stream-K: the 31 k-steps split over 4 pieces, their fp32 partial sums added in slot order by the finisher;
    the planted finisher adds 3 of the 4 slots."""
    a, w, bias = _f_problem()
    ref, mag = M.ref_f(a, None, FH, w, TAPS, 0, FR, bias=bias)
    steps, S = _f_steps(), 4
    parts = [_f_acc(a, FH, w, steps[len(steps) * p // S:len(steps) * (p + 1) // S]) for p in range(S)]

    def finish(slots):
        acc = torch.zeros_like(parts[0])
        for t in slots:
            acc += t
        return (acc + bias).half()
    assert M.c_f(finish(parts), ref, mag, "f16") <= M.C_TOL / 4
    c = M.c_f(finish(parts[:-1]), ref, mag, "f16")
    print("form F planted finisher_drops_a_partial: c = %.3g" % c)
    assert c > 20 * M.C_TOL


# ------------------------------------------------------------------------------------------------------
# the yardstick itself
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,tdt", [("f16", torch.float16), ("bf16", torch.bfloat16)])
def test_half_ulp_is_the_formats_rounding_bound(fmt, tdt):
    """Rounding any fp64 value to the format moves it by at most half_ulp (normal range, fp16 subnormals,
    saturation), and by more than a quarter of it somewhere in every binade tried."""
    g = _gen(13)
    v = torch.randn(20000, generator=g, dtype=torch.float64) * torch.pow(
        2.0, torch.randint(-20 if fmt == "f16" else -40, 15, (20000,), generator=g).double())
    v = v.float().double()                 # the kernels round an fp32 value once
    r = v.to(tdt).double()
    hu = M.half_ulp(v, fmt)
    assert bool(((r - v).abs() <= hu).all())
    assert float(((r - v).abs() / hu).max()) > 0.9
    one = torch.ones(1, dtype=torch.float64)
    assert M.c_f(v.to(tdt), v, v.abs(), fmt) == 0.0
    if fmt == "f16":
        assert float(M.half_ulp(torch.tensor([1.0, 1e-7, 2.0 ** -14, 0.0]), fmt)[1]) == 2.0 ** -25
        big = torch.tensor([70000.0, -1e6], dtype=torch.float64)
        assert M.c_f(torch.tensor([65504.0, -65504.0]).half(), big, big.abs(), fmt) == 0.0
        assert M.c_f(torch.tensor([float("inf")]).half(), big[:1], big[:1].abs(), fmt) == INF
    # one whole ulp off is (half an ulp) / (U * mag) over the gate
    p = M.MANT[fmt]
    off = (one * (1.0 + 2.0 ** (1 - p))).to(tdt)
    assert M.c_f(off, one, one, fmt) == pytest.approx(2.0 ** -p / M.U)


def test_truncation_allowance_is_per_stage_and_proportional_to_the_result():
    """A sum that shrinks by 2 * U per stage passes with the stages declared and fails without; one missing product
    stays far out."""
    ref = torch.tensor([100.0, -100.0, 0.01], dtype=torch.float64)
    mag = torch.tensor([400.0, 400.0, 400.0], dtype=torch.float64)
    got = ref * (1 - 2 * M.U * 300)
    assert M.c_w(got, ref, mag) > M.C_TOL and M.c_w(got, ref, mag, trunc_stages=300) <= M.C_TOL
    got[2] += 1.0
    assert M.c_w(got, ref, mag, trunc_stages=300) > 20 * M.C_TOL


def test_ref_w_reads_zeros_outside_each_batch_elements_buffer():
    """a_halo = 0: row m + d of batch element b is zero outside [0, R), never a row of batch element b +- 1; two
    sources are one concatenated K axis; the dead part of every tap is exactly zero."""
    g = _gen(14)
    b, r, nc, kc = 3, 4, 128, 128
    gg = torch.randn(b, r, nc, generator=g).half()
    a0 = torch.randn(b, r, 64, generator=g).half()
    a1 = torch.randn(b, r, 64, generator=g).half()
    taps = [[0] * 9, [kc] * 9, [0] * 9, [nc] * 9]
    taps[0][3], taps[3][5] = 64, 64
    ref, mag = M.ref_w(gg, a0, a1, 0, taps, -1, 1)
    a = torch.cat((a0, a1), -1).double()
    for d in (-1, 0, 1):
        exp = torch.zeros(nc, kc, dtype=torch.float64)
        for bb in range(b):
            for m in range(r):
                if 0 <= m + d < r:
                    exp += gg[bb, m].double().view(nc, 1) * a[bb, m + d].view(1, kc)
        if d == -1:
            exp[:, :64] = 0
        if d == 1:
            exp[64:] = 0
        assert torch.allclose(ref[d + 1], exp, rtol=1e-12, atol=1e-12)
    assert float(ref[0, :, :64].abs().max()) == 0.0 and float(mag[2, 64:].abs().max()) == 0.0
    assert bool((mag >= ref.abs() - 1e-9).all())
