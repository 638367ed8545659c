"""The BatchNorm / PReLU yardstick (tests/bn_act_model.py) without a GPU: its reference chain is fp64 autograd of the
reference layers, an fp32 emulation of the kernels' arithmetic (per-thread fp32 partials over rows in shuffled order,
combined in double; fma rounding; saturating fp16 stores) passes every gate, and the same emulation with one defect
planted fails by orders of magnitude.  Measured c of each planted defect (problem below: B 3, L 37, H 16, roll 5,
C 16; the worst output of the stage the defect lives in):

  defect                                                     stage            c
  mirror fold missing                                        pass 0 g_pre     1.5e+07
  mirror one row off (q0 in [0, H) instead of [1, H])        pass 0 g_pre     1.4e+07
  roll sign flipped                                          forward h        1.4e+10
  roll off by one                                            forward h        2.1e+10
  roll sign flipped                                          pass 0 g_pre     6.2e+08
  skip gradient added before the activation derivative       pass 0 g_pre     2.3e+07
  PReLU branch tested with y < 0 instead of y <= 0           pass 0 g_pre     3.5e+08
  red2 not centred                                           pass 0 red2      1.1e+06
  r2 taken through fp16                                      pass 1 out       3.7e+03
  biased and unbiased variance swapped                       finalize rvar    1.4e+05
  count off by one                                           finalize mean    1.5e+05
  last tile row dropped                                      pass 0 red1      5.6e+05
  a row read from the neighbouring batch element             pass 0 g_pre     1.3e+08

The clean emulation sits at c = 1.6 at worst, in three summation orders (C_TOL = 16)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import segan_oracle as O
from tests import bn_act_model as M

B, L, H, C_, ROLL = 3, 37, 16, 16, 5
EPS, MOM = 2.0 ** -17, 0.125                       # exact in fp32: the fp64 chain and the model see the same values
TILE = 8                                           # rows per tile of the emulated tiled walk


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def f32(t):
    """Round fp64 values to fp32 (and keep them in fp64)."""
    return t.float().double()


def st16(t, fmt="f16"):
    if fmt == "f16":
        return t.clamp(-65504.0, 65504.0).half()
    return t.bfloat16()


def _seq_sum(v, perm, T):
    """fp32 partial sums of v [N][C] over rows in order `perm`, dealt to T threads row by row, combined in fp64."""
    v = v[perm]
    k = -(-v.shape[0] // T)
    v = torch.cat((v, v.new_zeros(k * T - v.shape[0], v.shape[1]))).view(k, T, -1)
    acc = torch.zeros(T, v.shape[-1], dtype=torch.float64)
    for i in range(k):
        acc = f32(acc + v[i])
    return acc.sum(0), k


# ------------------------------------------------------------------------------------------------------
# the reference chain is fp64 autograd of the reference layers
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("roll,halo", [(0, 16), (5, 16), (-5, 16), (36, 16), (-36, 0), (3, 0)])
def test_reference_chain_is_autograd(roll, halo):
    """stats -> finalize -> act_fwd -> pass 0 -> pass 1 equals fp64 autograd of O.batchnorm_train -> F.prelu ->
    O.phase_roll -> reflect F.pad, with channels 0 and 1 at gamma = 0 (y exactly 0 there: PReLU's y <= 0 branch)."""
    g = _gen(1)
    a = torch.randn(B, L, C_, generator=g).half().double()
    gamma = 1 + 0.3 * torch.randn(C_, generator=g, dtype=torch.float64)
    beta = 0.3 * torch.randn(C_, generator=g, dtype=torch.float64)
    gamma[:2] = 0.0
    beta[0] = 0.0
    slope = 0.3 * torch.randn(C_, generator=g, dtype=torch.float64)
    rm0, rv0 = torch.randn(C_, generator=g, dtype=torch.float64), 1 + torch.rand(C_, generator=g, dtype=torch.float64)
    gh = torch.randn(B, L + 2 * halo, C_, generator=g).half().double()
    # fp64 autograd on NCL
    an = a.permute(0, 2, 1).clone().requires_grad_(True)
    gm, bt, sl = (t.clone().requires_grad_(True) for t in (gamma, beta, slope))
    rm, rv = rm0.clone(), rv0.clone()
    y = O.phase_roll(F.prelu(O.batchnorm_train(an, gm, bt, rm, rv, momentum=MOM, eps=EPS), sl), roll)
    if halo:
        y = F.pad(y, (halo, halo), mode="reflect")
    y.backward(gh.permute(0, 2, 1))
    # the model chain
    ref_st, _ = M.stats(a)
    fin = M.finalize(ref_st.unsqueeze(0), B * L, gamma, beta, EPS, MOM, rm0, rv0)
    ss = torch.stack((fin["sc"][0], fin["sh"][0]))
    mi = torch.stack((fin["mean"][0], fin["invstd"][0]))
    h, _ = M.act_fwd(a, ss, slope, roll, halo)
    assert bool((M.pre_act(a, ss)[0][..., 0] == 0).all())
    assert torch.allclose(h, y.detach().permute(0, 2, 1), rtol=1e-12, atol=1e-12)
    assert torch.allclose(fin["rmean"][0], rm, rtol=1e-12, atol=1e-12)
    assert torch.allclose(fin["rvar"][0], rv, rtol=1e-12, atol=1e-12)
    p0 = M.bwd_pass0(gh, None, a, ss, mi, slope, roll, halo)
    red, rmag = p0["red"]
    for s, want in enumerate((sl.grad, bt.grad, gm.grad)):
        assert M.c_vec(want, red[s], rmag[s]) <= 1e-3, s
    out, omag = M.bwd_pass1(p0["gpre"], a, ss, mi, red.unsqueeze(0))
    assert M.c_vec(an.grad.permute(0, 2, 1), out, omag) <= 2.0      # r1, r2 rounded to fp32 as the kernels do


# ------------------------------------------------------------------------------------------------------
# an fp32 emulation of the kernels, with plantable defects
# ------------------------------------------------------------------------------------------------------
def _problem():
    g = _gen(2)
    a = 2 * torch.randn(B, L, C_, generator=g)
    sc = 1 + 0.3 * torch.randn(C_, generator=g)
    sh = 0.3 * torch.randn(C_, generator=g)
    sc[::4], sh[::4] = 0.5, -0.375                   # y = 0 exactly where a = 0.75
    a[:, ::3, ::4] = 0.75
    a = a.half()
    mu = torch.randn(C_, generator=g).float()
    inv = (0.5 + torch.rand(C_, generator=g)).float()
    slope = (0.3 * torch.randn(C_, generator=g)).float()
    gh = torch.randn(B, L + 2 * H, C_, generator=g).half()
    gadd = torch.randn(B, L, C_, generator=g).half()
    st = torch.randn(4, 2, C_, generator=g, dtype=torch.float64).abs() * 50
    st[:, 1] += st[:, 0] ** 2                        # a positive variance
    gamma, beta = (1 + 0.3 * torch.randn(C_, generator=g)).float(), (0.3 * torch.randn(C_, generator=g)).float()
    rm0, rv0 = torch.randn(C_, generator=g).float(), (1 + torch.rand(C_, generator=g)).float()
    return dict(a=a, ss=torch.stack((sc, sh)).float(), mi=torch.stack((mu, inv)), slope=slope, gh=gh, gadd=gadd,
                st=st, gamma=gamma, beta=beta, rm0=rm0, rv0=rv0, perm=torch.randperm(B * L, generator=g))


def emu_finalize(p, defect=None):
    s = p["st"].sum(0)
    n = float(B * L + (1 if defect == "count" else 0))
    mean = s[0] / n
    var = (s[1] / n - mean * mean).clamp_min(0.0)
    unb = var * n / (n - 1)
    if defect == "unbiased":
        var, unb = unb, var
    inv = f32(1.0 / torch.sqrt(var + EPS))
    sc = f32(p["gamma"].double() * inv)
    sh = f32(p["beta"].double() - f32(f32(mean) * sc))
    m = MOM
    rm = f32(f32((1 - m) * p["rm0"].double()) + f32(m * f32(mean)))
    rv = f32(f32((1 - m) * p["rv0"].double()) + f32(m * f32(unb)))
    return dict(mean=f32(mean), invstd=inv, sc=sc, sh=sh, rmean=rm, rvar=rv)


def emu_fwd(p, defect=None):
    """act_fwd_kernel's index formulation: h[b][qh] = act(a[b][unroll(reflect(qh - H))])."""
    a, sc, sh, sl = p["a"].double(), p["ss"][0].double(), p["ss"][1].double(), p["slope"].double()
    roll = {"roll_sign": -ROLL, "roll_off": ROLL + 1}.get(defect, ROLL)
    rows = []
    for qh in range(L + 2 * H):
        q = abs(qh - H)
        q = 2 * (L - 1) - q if q >= L else q
        rows.append((q - roll) % L)
    y = f32(a[:, rows] * sc + sh)
    y = torch.where(y > 0, y, f32(sl * y))
    return st16(y)


def emu_bwd(p, defect=None, skip=True, bn=True):
    """Pass 0 (tiled kernel: gather at the rolled row plus its mirror, sum(g_pre * x) centred at the flush) and pass
    1 on pass 0's own reductions; returns g_pre as stored, the fp64 reductions and the 16-bit pass-1 output."""
    a = p["a"].double()
    sc, sh = p["ss"][0].double(), p["ss"][1].double()
    mu, inv, sl = p["mi"][0].double(), p["mi"][1].double(), p["slope"].double()
    gh = p["gh"].double()
    roll = -ROLL if defect == "roll_sign" else ROLL
    g = torch.zeros(B, L, C_, dtype=torch.float64)
    live = torch.ones(B, L, dtype=torch.bool)
    for b in range(B):
        for l in range(L):
            if defect == "tail" and l % TILE == TILE - 1:
                live[b, l] = False
                continue
            q0 = (l + roll) % L
            v = gh[b, H + q0]
            lo = (0 <= q0 < H) if defect == "mirror_off" else (1 <= q0 <= H)
            if defect != "no_mirror":
                if lo:
                    v = f32(v + gh[b, H - q0])
                elif L - 1 - H <= q0 <= L - 2:
                    bb = b + 1 if defect == "wrong_batch" and b + 1 < B else b
                    v = f32(v + gh[bb, H + 2 * (L - 1) - q0])
            g[b, l] = v
    y = f32(a * sc + sh)
    neg = (y < 0) if defect == "branch_lt" else (y <= 0)
    add = p["gadd"].double() if skip else torch.zeros_like(g)
    if defect == "skip_first":
        gp = torch.where(neg, f32(f32(g + add) * sl), f32(g + add))
    else:
        gp = f32(torch.where(neg, f32(g * sl), g) + add)
    gp = torch.where(live[..., None], gp, torch.zeros_like(gp))
    t0 = torch.where(neg & live[..., None], f32(g * y), torch.zeros_like(g))
    flat = lambda t: t.reshape(B * L, C_)                                 # noqa: E731
    s0, k = _seq_sum(flat(t0), p["perm"], 8)
    s1, _ = _seq_sum(flat(gp), p["perm"], 8)
    s2, _ = _seq_sum(flat(f32(gp * a)), p["perm"], 8)
    if not bn:
        mu, inv = torch.zeros_like(mu), torch.ones_like(inv)
    red = torch.stack((s0, s1, inv * s2 if defect == "uncentred" else inv * (s2 - mu * s1)))
    # pass 1
    n = float(B * L)
    r1 = f32(red[1] / n)
    r2 = f32(red[2] / n)
    if defect == "r2_f16":
        r2 = r2.half().double()
    ka = f32(f32(-sc * r2) * inv)
    kb = f32(sc * f32(f32(f32(r2 * inv) * mu) - r1))
    out = f32(sc * gp + f32(ka * a + kb))
    return st16(gp), red, st16(out), k


def _cs(p, defect=None):
    """c of every stage of the emulation (defect planted or not) against the model."""
    c = {}
    fin = emu_finalize(p, defect)
    ref = M.finalize(p["st"], B * L, p["gamma"], p["beta"], EPS, MOM, p["rm0"], p["rv0"])
    for k in fin:
        c["finalize " + k] = M.c_vec(fin[k], *ref[k])
    c["forward h"] = M.c_f(emu_fwd(p, defect), *M.act_fwd(p["a"], p["ss"], p["slope"], ROLL, H), "f16")
    gp16, red, out16, _ = emu_bwd(p, defect)
    p0 = M.bwd_pass0(p["gh"], p["gadd"], p["a"], p["ss"], p["mi"], p["slope"], ROLL, H)
    c["pass 0 g_pre"] = M.c_f(gp16, *p0["gpre"], "f16")
    for s in range(3):
        c["pass 0 red%d" % s] = M.c_vec(red[s], p0["red"][0][s], p0["red"][1][s])
    # pass 1 is gated on the emulation's own reductions, as the GPU tests gate it on the kernel's
    c["pass 1 out"] = M.c_f(out16, *M.bwd_pass1(p0["gpre"], p["a"], p["ss"], p["mi"], red.unsqueeze(0)), "f16")
    return c


def test_fp32_emulation_passes_every_gate():
    p = _problem()
    assert bool((M.pre_act(p["a"], p["ss"])[0] == 0).any())
    for seed in (0, 1, 2):
        p["perm"] = torch.randperm(B * L, generator=_gen(10 + seed))
        c = _cs(p)
        worst = max(c.values())
        print("clean emulation, order %d: worst c = %.2f" % (seed, worst))
        assert worst <= 2.0, c


DEFECTS = [("no_mirror", "pass 0 g_pre"), ("mirror_off", "pass 0 g_pre"), ("roll_sign", "forward h"),
           ("roll_off", "forward h"), ("roll_sign", "pass 0 g_pre"), ("skip_first", "pass 0 g_pre"),
           ("branch_lt", "pass 0 g_pre"), ("uncentred", "pass 0 red2"), ("r2_f16", "pass 1 out"),
           ("unbiased", "finalize rvar"), ("count", "finalize mean"), ("tail", "pass 0 red1"),
           ("wrong_batch", "pass 0 g_pre")]


@pytest.mark.parametrize("defect,stage", DEFECTS)
def test_planted_defect_fails_far_above_the_gate(defect, stage):
    c = _cs(_problem(), defect)
    print("%-12s %-15s c = %.2g" % (defect, stage, c[stage]))
    assert c[stage] >= 100 * M.C_TOL, (defect, c)
