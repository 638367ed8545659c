"""Spectrally normalised Generators (norm_type='snorm') on the H100: the row-strided power iteration and sigma-term
kernels against fp64, the Generator's sigma / u / v, outputs and gradients against the snorm oracle
(tests/gsnorm_oracle.py) and its operand-precision control, the invariant <dL/dW_orig, W_orig> = 0, two-pass
accumulation, SEGAN and WSEGAN steps, graph replay, checkpoints and inference.
An fp32 sum must satisfy |err| <= c * 2^-24 * sum|terms| for every output (U below).
Run on an H100:  python -m pytest tests -m gpu"""
import random

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import segan_oracle as O                                          # noqa: E402
from segan_pytorch_b200 import _lib, engine as E                             # noqa: E402
from segan_pytorch_b200.segan.models import SEGAN, WSEGAN                    # noqa: E402
from tests import gsnorm_oracle as GO                                        # noqa: E402
from tests.test_gpu_parity_scale import GRAD_ABS, GRAD_VS_CONTROL           # noqa: E402
from tests.test_gsnorm import CONFIGS, snorm_generator                       # noqa: E402
from tests.util import cpu_state, load_opts, max_abs, rel_err, seed_all     # noqa: E402

DEV = "cuda"
_p, _stream = E._p, E._stream
U = 2.0 ** -24
WAVE_TOL = 1e-3


def _ratio(err, scale):
    return float((err.abs() / (U * scale.clamp_min(1e-300))).max())


def _pairs(B, seed, zc=1024):
    g = torch.Generator().manual_seed(seed)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp(-1, 1)
    return clean, noisy, torch.randn(B, zc, 16, generator=g)


def _z(G, z):
    return None if G.no_z else z[:, :G.z_dim].contiguous()


# ---- kernels ----------------------------------------------------------------------------------------------------------
# (n_taps, nc, kc, ld): a decoder master as [36][Cout][Cin], an encoder master, a tied half, the two waveform ends
LD_CASES = {"dec_kind1": (36, 512, 1024, 1024), "enc_kind0": (9, 256, 512, 512), "tied_half": (36, 128, 256, 512),
            "enc0_small": (1, 64, 31, 31), "dec_last_small": (1, 1, 128 * 31, 128 * 31)}


def _ld_case(name, seed):
    T, nc, kc, ld = LD_CASES[name]
    g = torch.Generator().manual_seed(seed)
    m = 0.05 * torch.randn(T, nc, ld, generator=g)
    if ld > kc:
        m[:, :, kc:] = m[:, :, :kc]                   # tied: [W | W]
    u0 = F.normalize(torch.randn(nc, generator=g), dim=0)
    v0 = F.normalize(torch.randn(T * kc, generator=g), dim=0)
    return m, u0, v0, (T, nc, kc, ld)


@pytest.mark.parametrize("name", list(LD_CASES))
def test_snorm_sigma_ld_training_vs_fp64(name):
    """One power iteration on M[t][n][k < kc] (rows ld apart) against fp64: v = normalize(W^T u0),
    u = normalize(W v), sigma = ||W v||, c = 32 as for sg_snorm_sigma; the same bits on a second run (fixed-order
    sums, no float atomics)."""
    m, u0, v0, (T, nc, kc, ld) = _ld_case(name, 400 + list(LD_CASES).index(name))
    md = m[:, :, :kc].double().to(DEV)
    res = []
    m = m.to(DEV)
    for _ in range(2):
        u, v = u0.to(DEV).clone(), v0.to(DEV).clone()
        scal = torch.full((4,), 5.0, device=DEV)
        work = torch.zeros(nc + T * ((kc + 255) // 256) + 4, device=DEV)
        _lib.call("sg_snorm_sigma_ld", _p(m), T, nc, kc, ld, _p(u), _p(v), _p(scal), _p(work), 1, _stream())
        torch.cuda.synchronize()
        res.append((u.clone(), v.clone(), scal.clone()))
    assert all(torch.equal(a, b) for a, b in zip(res[0], res[1]))
    u, v, scal = res[0]
    ud, vd = u0.double().to(DEV), v.double().view(T, kc)
    vr = torch.einsum("tnk,n->tk", md, ud)
    sv = torch.einsum("tnk,n->tk", md.abs(), ud.abs())
    cv = _ratio(vd - vr / vr.norm(), sv / vr.norm() + (vr / vr.norm()).abs())
    ur = torch.einsum("tnk,tk->n", md, vd)
    su = torch.einsum("tnk,tk->n", md.abs(), vd.abs())
    sig_r = float(ur.norm())
    cu = _ratio(u.double() - ur / sig_r, su / sig_r + (ur / sig_r).abs())
    cs = abs(float(scal[2]) - sig_r) / (U * (float(((ur / sig_r).abs() * su).sum()) + sig_r))
    print("snorm_sigma_ld %s (T %d nc %d kc %d ld %d): c v %.2f u %.2f sigma %.2f (tol 32)" % (name, T, nc, kc, ld, cv,
                                                                                             cu, cs))
    assert cv <= 32 and cu <= 32 and cs <= 32
    assert abs(float(scal[3]) - 1.0 / float(scal[2])) <= 2 * U / float(scal[2])


@pytest.mark.parametrize("name", ["dec_kind1", "tied_half", "enc0_small"])
def test_snorm_sigma_ld_eval_uses_stored_vectors(name):
    m, u0, v0, (T, nc, kc, ld) = _ld_case(name, 450)
    u, v, md_dev = u0.to(DEV).clone(), v0.to(DEV).clone(), m.to(DEV)
    scal = torch.zeros(4, device=DEV)
    work = torch.zeros(nc + T * ((kc + 255) // 256) + 4, device=DEV)
    _lib.call("sg_snorm_sigma_ld", _p(md_dev), T, nc, kc, ld, _p(u), _p(v), _p(scal), _p(work), 0, _stream())
    torch.cuda.synchronize()
    assert torch.equal(u.cpu(), u0) and torch.equal(v.cpu(), v0)
    md = m[:, :, :kc].double()
    wv = torch.einsum("tnk,tk->n", md, v0.double().view(T, kc))
    ref = float(torch.dot(u0.double(), wv))
    scale = float(torch.dot(u0.double().abs(), torch.einsum("tnk,tk->n", md.abs(), v0.double().abs().view(T, kc))))
    c = abs(float(scal[2]) - ref) / (U * scale)
    print("snorm_sigma_ld eval %s: c %.2f (tol 32)" % (name, c))
    assert c <= 32


@pytest.mark.parametrize("copies,P", [(1, 1), (2, 1), (2, 3), (1, 4)])
def test_snorm_rank1_ld_vs_fp64(copies, P):
    """dwp[t][n][c kc + k] -= sum_p coef_p u_p[n] v_p[t][k] on every copy c, rows ld apart; columns past the copies
    untouched.  c = 12 of 2^-24 * (|dwp| + sum_p |coef_p u_p v_p|)."""
    T, nc, kc = 36, 128, 256
    ld = copies * kc + 64
    g = torch.Generator().manual_seed(500 + 10 * copies + P)
    dwp = torch.randn(T, nc, ld, generator=g)
    u = torch.randn(P, nc, generator=g)
    v = torch.randn(P, T * kc, generator=g)
    coef = torch.randn(P, generator=g)
    d, ud, vd, cd = dwp.to(DEV).clone(), u.to(DEV), v.to(DEV), coef.to(DEV)     # held until the kernel has run
    _lib.call("sg_snorm_rank1_ld", _p(d), T, nc, kc, ld, copies, P, _p(ud), _p(vd), _p(cd), _stream())
    torch.cuda.synchronize()
    corr = torch.einsum("p,pn,ptk->tnk", coef.double(), u.double(), v.double().view(P, T, kc))
    mag = torch.einsum("p,pn,ptk->tnk", coef.double().abs(), u.double().abs(), v.double().abs().view(P, T, kc))
    d = d.cpu().double()
    for c in range(copies):
        sl = slice(c * kc, (c + 1) * kc)
        cc = _ratio(d[:, :, sl] - (dwp.double()[:, :, sl] - corr), dwp.double()[:, :, sl].abs() + mag)
        print("snorm_rank1_ld copies %d P %d copy %d: c %.2f (tol 12)" % (copies, P, c, cc))
        assert cc <= 12
    assert torch.equal(d[:, :, copies * kc:], dwp.double()[:, :, copies * kc:])


# ---- the Generator ----------------------------------------------------------------------------------------------------
def _sn_vectors(G):
    sd = G.state_dict()
    return {k: v.detach().cpu().clone() for k, v in sd.items() if k.endswith(("weight_u", "weight_v"))}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_generator_outputs_and_vectors_vs_oracle(name):
    """Training forward: u, v after the one power iteration of every normalised tensor (kind 0, kind 1, tied halves,
    both waveform ends) and the output against the fp32 oracle; eval forward: output against the oracle's eval mode,
    vectors left untouched, and a second eval forward (cached sigma) gives the same bits."""
    B = 4
    G = snorm_generator(name)
    sd = cpu_state(G)
    _, noisy, z = _pairs(B, 600)
    z = _z(G, z)
    G = G.to(DEV).train()
    with torch.no_grad():
        y_tr = G(noisy.to(DEV), z=z.to(DEV) if z is not None else None).cpu()
    vec = _sn_vectors(G)
    with O.oracle_mode(), torch.no_grad():
        ref_tr = GO.generator_forward(sd, noisy, z, training=True, skip_merge=G.skip_merge)
    for k, t in vec.items():
        assert rel_err(t, sd[k]) <= 1e-4, (k, rel_err(t, sd[k]))
    e_tr = max_abs(y_tr, ref_tr)
    G.eval()
    with torch.no_grad():
        y_ev = G(noisy.to(DEV), z=z.to(DEV) if z is not None else None).cpu()
        y_ev2 = G(noisy.to(DEV), z=z.to(DEV) if z is not None else None).cpu()
    assert torch.equal(y_ev, y_ev2)
    vec2 = _sn_vectors(G)
    assert all(torch.equal(vec[k], vec2[k]) for k in vec)
    with O.oracle_mode(), torch.no_grad():
        ref_ev = GO.generator_forward(sd, noisy, z, training=False, skip_merge=G.skip_merge)
    e_ev = max_abs(y_ev, ref_ev)
    print("gsnorm %s: train fwd max-abs %.2e, eval fwd %.2e, |u,v| rel max %.2e" % (
        name, e_tr, e_ev, max(rel_err(t, sd[k]) for k, t in vec.items())))
    assert e_tr <= WAVE_TOL and e_ev <= WAVE_TOL


def _trained_vectors(G, seed=609):
    """One training-mode forward without grad: u / v leave their random init, as after any training.  (Eval mode on
    the initial vectors is torch's semantics too, but sigma = u^T W v of two random vectors is ill-conditioned.)"""
    _, noisy, z = _pairs(2, seed)
    G.train()
    with torch.no_grad():
        G(noisy.to(DEV), z=_z(G, z).to(DEV) if not G.no_z else None)
    return G.eval()


def test_generator_forward_batch300_vs_oracle():
    """Eval mode at batch 300 against the oracle (vectors after one training iteration)."""
    B = 300
    G = _trained_vectors(snorm_generator("concat").to(DEV))
    sd = cpu_state(G)
    _, noisy, z = _pairs(B, 601)
    with torch.no_grad():
        y = G(noisy.to(DEV), z=z.to(DEV)).cpu()
    with O.oracle_mode(), torch.no_grad():
        ref = GO.generator_forward(sd, noisy, z, training=False)
    err = max_abs(y, ref)
    print("gsnorm fwd B=300: max-abs %.3e" % err)
    assert err <= WAVE_TOL


def _orthogonality(G, grads):
    """<dL/dW_orig, W_orig> of every normalised tensor relative to the size of its sigma term: for the packed layers
    sum_p |coef_p| sigma_p (the sigma term's inner product with W is coef sigma), for the small tensors |g| |W|."""
    eng = G.engine
    out = {}
    for name in eng._sn_names():
        w = dict(G.named_parameters())[name].detach().double().cpu()
        g = grads[name].double()
        dot = abs(float((g * w).sum()))
        st = eng._sn_state(name)
        if st["pl"] is not None:
            slots = sorted(eng._sn_done)
            term = sum(abs(float(st["coef"][s])) * float(st["scal"][s][2]) for s in slots) / E.LOSS_SCALE
            out[name] = dot / max(term, 1e-30)
        else:
            out[name] = dot / max(float(g.norm() * w.norm()), 1e-30) * 100.0     # held to 1e-4 below
    return out


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_generator_gradients_vs_control(name):
    """Gradients of 100 * L1 of every parameter (weight_orig, alphas, biases, slopes) against the oracle and its
    operand-precision control; the invariant <dL/dW_orig, W_orig> = 0 of every normalised tensor."""
    B = 4
    G = snorm_generator(name)
    sdG = cpu_state(G)
    G = G.to(DEV).train()
    clean, noisy, z = _pairs(B, 602)
    z = _z(G, z)
    y = G(noisy.to(DEV), z=z.to(DEV) if z is not None else None)
    out = 100 * F.l1_loss(y, clean.to(DEV))
    out.backward()
    gG = {n: p.grad.detach().cpu() for n, p in G.named_parameters() if p.grad is not None}

    def oracle():
        sd = {k: v.clone() for k, v in sdG.items()}
        pG = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd) if k in gG}
        lo = 100 * F.l1_loss(GO.generator_forward({**sd, **pG}, noisy, z, training=True, skip_merge=G.skip_merge),
                             clean)
        return float(lo.detach()), dict(zip(pG.keys(), torch.autograd.grad(lo, list(pG.values()))))
    with O.oracle_mode():
        lo, go = oracle()
        with O.operand_precision(torch.float16):
            lc, gc = oracle()
    rep = {k: rel_err(gG[k], r) for k, r in go.items()}
    ctl = {k: rel_err(gc[k], r) for k, r in go.items()}
    orth = _orthogonality(G, gG)
    print("gsnorm %s grads: loss %.5f vs %.5f | max %.3e (%s) | control max %.3e | orth max %.2e (%s)" % (
        name, float(out), lo, max(rep.values()), max(rep, key=rep.get), max(ctl.values()), max(orth.values()),
        max(orth, key=orth.get)))
    assert abs(float(out) - lo) <= max(1e-3, 3 * abs(lc - lo)) * max(1.0, abs(lo))
    assert max(rep.values()) <= GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS
    assert max(orth.values()) <= 2e-2, orth
    if name == "concat":
        assert any(k.startswith("alpha_") for k in rep)                 # dalpha is among the checked gradients


@pytest.mark.parametrize("mode", ["two_pass", "nograd_between"])
def test_two_pass_accumulation_vs_oracle(mode):
    """two_pass: two training forwards (two power iterations, two pass slots) before one backward each into the same
    bucket, against the oracle's two-pass gradient (the second pass on the vectors the first advanced).
    nograd_between: a gradient-free training forward (a third power iteration, new operands) between a forward and its
    backward.  Either way each backward must run on the operands of its own pass's sigma; held to the operand-precision
    control like the single-pass gradients."""
    B = 2
    G = snorm_generator("concat")
    sdG = cpu_state(G)
    G = G.to(DEV).train()
    eng = G.engine.bind()
    clean, noisy, z = _pairs(2 * B, 603)
    sl = [slice(0, B), slice(B, 2 * B)]
    ys, ctxs = [], []
    for i in range(2):
        grad_pass = mode == "two_pass" or i == 0
        y, ctx = eng.forward(noisy[sl[i]].to(DEV), z[sl[i]].to(DEV), fresh=True, twins=grad_pass)
        ys.append(y.clone())
        ctxs.append(ctx if grad_pass else None)
    n_pass = 2 if mode == "two_pass" else 1
    if mode == "two_pass":
        assert sorted(c["sn_slot"][0] for c in ctxs) == [0, 1]
    for i in range(n_pass):
        gy = torch.sign(ys[i] - clean[sl[i]].to(DEV)) * (100.0 / (B * 16384) * E.LOSS_SCALE)
        eng.backward(ctxs[i], gy, accumulate=(i == 1))
    assert len(eng._sn_done) == n_pass
    got = {n: eng.grad_of(n).cpu() for n, p in G.named_parameters() if p.requires_grad}
    orth = _orthogonality(G, got)

    def oracle():
        sd = {k: v.clone() for k, v in sdG.items()}
        pG = {k: sd[k].clone().requires_grad_(True) for k in O._trainable(sd)}
        tot = 0
        for i in range(2):
            yo = GO.generator_forward({**sd, **pG}, noisy[sl[i]], z[sl[i]], training=True)
            if i < n_pass:
                tot = tot + 100 * F.l1_loss(yo, clean[sl[i]], reduction="sum") / (B * 16384)
        return dict(zip(pG.keys(), torch.autograd.grad(tot, list(pG.values()))))
    with O.oracle_mode():
        go = oracle()
        with O.operand_precision(torch.float16):
            gc = oracle()
    rep = {k: rel_err(got[k], go[k]) for k in go}
    ctl = {k: rel_err(gc[k], go[k]) for k in go}
    print("gsnorm %s: grad rel max %.3e (%s) | control max %.3e | orth max %.2e" % (
        mode, max(rep.values()), max(rep, key=rep.get), max(ctl.values()), max(orth.values())))
    assert max(orth.values()) <= 2e-2, orth
    assert max(rep.values()) <= GRAD_VS_CONTROL * max(ctl.values()) + GRAD_ABS, rep


# ---- steps ------------------------------------------------------------------------------------------------------------
def _segan_with(G, B, **over):
    seed_all(111)
    opts = load_opts(batch_size=B, **over)
    return SEGAN(opts, generator=G), opts


def test_segan_steps_batch16_graph_replay_matches_eager():
    """B = 16 SEGAN steps with a snorm G: eager twice (the noise floor) and graph-replayed; losses, G gradients and
    the G's u / v of the replayed steps held to the floor."""
    B = 16
    clean, noisy, _ = _pairs(B, 604)
    clean, noisy = clean.to(DEV), noisy.to(DEV)
    random.seed(13)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(4)]
    prev_keep = E.KEEP_GRADS

    def run(graphs):
        prev = E.GRAPHS
        E.GRAPHS, E.KEEP_GRADS = graphs, True
        try:
            s, opts = _segan_with(snorm_generator("concat"), B, g_lr=5e-7, d_lr=5e-7)
            s = s.to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(opts)
            out = []
            torch.manual_seed(99)
            for i in range(4):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, shifts3=shifts[i])
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad[:s.G.engine.flat.numel()].clone(), _sn_vectors(s.G)))
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs
        finally:
            E.GRAPHS, E.KEEP_GRADS = prev, prev_keep

    (e1, n1), (e2, n2), (gr, n3) = run(False), run(False), run(True)
    assert n1 == 0 and n2 == 0 and n3 == 1
    for step in range(4):
        fl = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[step][0], e2[step][0]))
        fg = rel_err(e2[step][1], e1[step][1])
        fv = max(rel_err(e2[step][2][k], e1[step][2][k]) for k in e1[step][2])
        el = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(e1[step][0], gr[step][0]))
        eg = rel_err(gr[step][1], e1[step][1])
        ev = max(rel_err(gr[step][2][k], e1[step][2][k]) for k in e1[step][2])
        print("gsnorm SEGAN step %d: losses %s | floor loss %.2e grad %.2e u/v %.2e | graph loss %.2e grad %.2e u/v %.2e"
              % (step, [round(x, 4) for x in gr[step][0]], fl, fg, fv, el, eg, ev))
        assert all(x == x and abs(x) < 1e4 for x in gr[step][0])
        assert el <= 10 * fl + 2e-3 and eg <= 10 * fg + 5e-3 and ev <= 10 * fv + 1e-5


@pytest.mark.parametrize("opt", ["rmsprop", "adam"])
def test_wsegan_recipe_step(opt):
    """The recipe run_wsegan_train.sh intends: WSEGAN --misalign_pair with a snorm G and a snorm D, RMSprop and
    Adam.  Losses against the oracle step (both networks normalised; RMSprop, the oracle's optimiser)."""
    B = 3
    seed_all(111)
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, opt=opt, dnorm_type="snorm")
    seed_all(111)
    G = snorm_generator("concat")
    s = WSEGAN(opts, generator=G)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    clean, noisy, z = _pairs(B, 605)
    random.seed(6)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(4)]
    Gopt, Dopt = s.build_optimizers(opts)
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, z=z.to(DEV), shifts=shifts,
                          perm=[2, 0, 1]).tolist()
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    plain_fwd = O.generator_forward
    O.generator_forward = lambda sd, x, z_, ret_hid=False, skip_merge="concat": GO.generator_forward(
        sd, x, z_, training=True, skip_merge=skip_merge, ret_hid=ret_hid)
    try:
        if opt == "rmsprop":
            ref = O.wsegan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts, [2, 0, 1], pow_weight=0.001,
                                      l1_weight=100.0)
        else:
            ref = None
    finally:
        O.generator_forward = plain_fwd
    print("gsnorm WSEGAN %s: losses %s oracle %s" % (
        opt, losses, None if ref is None else [ref[k] for k in ("d_loss", "g_adv_loss", "pow_loss", "den_loss")]))
    assert all(x == x and abs(x) < 1e4 for x in losses)
    if ref is not None:
        for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
            assert abs(got - ref[k]) <= 3e-2 * max(1.0, abs(ref[k])), (k, got, ref[k])


# ---- checkpoints and inference ----------------------------------------------------------------------------------------
def test_checkpoint_round_trip_and_load_into_bound_engine(tmp_path):
    """state_dict -> a fresh Generator gives the same eval outputs and buffers; load_state_dict into an engine that
    already ran takes effect on the next forward, u / v included."""
    B = 2
    _, noisy, z = _pairs(B, 606)
    x, zz = noisy.to(DEV), z.to(DEV)
    G1 = snorm_generator("concat", seed=1).to(DEV).train()
    with torch.no_grad():
        G1(x, z=zz)                                       # one power iteration: u / v differ from their init
    path = str(tmp_path / "g.ckpt")
    torch.save(G1.state_dict(), path)
    G1.eval()
    with torch.no_grad():
        y1 = G1(x, z=zz)
    G2 = snorm_generator("concat", seed=2).to(DEV).eval()
    with torch.no_grad():
        y2_before = G2(x, z=zz)                           # bound engine, eval sigma cached
    G2.load_state_dict(torch.load(path, map_location=DEV))
    with torch.no_grad():
        y2 = G2(x, z=zz)
    assert not torch.equal(y2_before, y1)
    assert torch.equal(y2, y1)
    sd1, sd2 = G1.state_dict(), G2.state_dict()
    assert all(torch.equal(sd1[k], sd2[k]) for k in sd1)
    # only the vectors change: the next eval forward uses them
    G3 = snorm_generator("concat", seed=1).to(DEV).eval()
    with torch.no_grad():
        y3_init = G3(x, z=zz)
    G3.load_state_dict({k: v for k, v in torch.load(path, map_location=DEV).items()}, strict=True)
    with torch.no_grad():
        y3 = G3(x, z=zz)
    assert torch.equal(y3, y1) and not torch.equal(y3_init, y1)


def test_generate_and_clean_files_with_snorm_generator(tmp_path):
    """generate and clean_files run the eval-mode snorm G: the same samples as G on the windows, u / v untouched."""
    import os
    import numpy as np
    from scipy.io import wavfile
    from segan_pytorch_b200.segan.datasets import normalize_wave_minmax, pre_emphasize
    s, _ = _segan_with(snorm_generator("concat", no_z=True), 2)
    s = s.to(DEV)
    _trained_vectors(s.G)
    vec0 = _sn_vectors(s.G)
    gen = torch.Generator().manual_seed(607)
    T = 40000
    wav = 0.3 * torch.randn(1, 1, T, generator=gen)
    out, _ = s.generate(wav)
    x = torch.zeros(3, 1, 16384)
    x.view(-1)[:T] = wav.view(-1)
    with torch.no_grad():
        y = s.G(x.to(DEV)).cpu().reshape(-1)[:T].numpy()
    assert max_abs(out, O.de_emphasize(y, 0.95)) <= 1e-4
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    p = str(src / "u0.wav")
    wavfile.write(p, 16000, (np.random.RandomState(0).randn(T) * 3000).astype(np.int16))
    assert s.clean_files([p], str(dst), batch=2, group_windows=3) == 3
    rate, w = wavfile.read(p)
    ref, _ = s.generate(torch.FloatTensor(pre_emphasize(normalize_wave_minmax(w), 0.95)).view(1, 1, -1))
    _, got = wavfile.read(str(dst / os.path.basename(p)))
    assert got.shape == ref.shape and max_abs(got, ref) <= 2e-4
    vec1 = _sn_vectors(s.G)
    assert all(torch.equal(vec0[k], vec1[k]) for k in vec0)
