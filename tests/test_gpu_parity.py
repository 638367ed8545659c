"""Parity of the CUDA path with the reference, through the drop-in API:
  * against the golden vectors produced by the unmodified reference (tests/golden/*.npz)
  * against the oracle on the same seeded inputs
north_star tolerance: 1e-3 max-abs on fp32 waveforms (written below as WAVE_TOL).
Run on an H100:  python -m pytest tests -m gpu"""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import segan_oracle as O                                         # noqa: E402
from segan_pytorch_b200._lib import BACKEND_FFMA, BACKEND_TCGEN05           # noqa: E402
from tests.util import build_segan, cpu_state, golden, max_abs, rel_err, sd_sha  # noqa: E402

WAVE_TOL = 1e-3
# Gradient tolerances of the small golden step below (relative L2 over the 256 sampled entries per tensor, B = 4).
# They are upper bounds for THIS sample only; the gates that carry the parity claim are in
# tests/test_gpu_parity_scale.py, where every gradient set is held to 1.5 x the distance of the fp16-operand control
# (the oracle with fp16-rounded contractions) + 5e-3: with PReLU initialised at slope 0 the activation derivative is
# discontinuous, fp16 operands flip ~0.1-0.4 % of the masks per layer, and the D step's real / fake terms cancel
# (5-7 % at B = 16, control and kernels alike; 0.2-0.5 % with continuous activations).  G-step gradients are taken
# through the discriminator AFTER its RMSprop step; the first RMSprop step is lr*sign(g) for every one of D's 25.8 M
# weights (it moves D(fake) from +0.26 to -16.2 in the reference itself), so sign flips among near-zero gradient
# entries perturb the updated D visibly.  With an identical D the same G gradients are control-gated
# (test_generator_gradients_with_identical_discriminator).
GRAD_TOL_D = 0.2
GRAD_TOL_G_THROUGH_UPDATED_D = 0.5
DEV = "cuda"


@pytest.fixture(scope="module")
def segan():
    s = build_segan()
    assert sd_sha(s.G.state_dict()) == str(golden("g_forward_cfg1.npz")["sha_G"])
    return s.to(DEV)


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05])
def test_generator_forward_cfg1(segan, backend):
    """BASELINE config 1: G forward on 1x16384, eval, vs the reference's CPU output."""
    g = golden("g_forward_cfg1.npz")
    segan.G.eval()
    segan.G.engine.backend = backend
    with torch.no_grad():
        y, hall = segan.G(torch.from_numpy(g["x"]).to(DEV), z=torch.from_numpy(g["z"]).to(DEV), ret_hid=True)
    torch.cuda.synchronize()
    for k in hall:
        idx = torch.from_numpy(g["hall_idx." + k]).to(DEV)
        got = hall[k].reshape(-1)[idx].cpu()
        ref = torch.from_numpy(g["hall_val." + k])
        assert max_abs(got, ref) <= 4e-3 * max(1.0, float(ref.abs().max())), (k, backend)
    err = max_abs(y.cpu(), g["y"])
    print("G fwd cfg1 backend %d max-abs %.3e" % (backend, err))
    assert err <= WAVE_TOL


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05])
def test_generator_forward_batched(segan, backend):
    g = golden("g_forward_b3.npz")
    segan.G.eval()
    segan.G.engine.backend = backend
    with torch.no_grad():
        y = segan.G(torch.from_numpy(g["x"]).to(DEV), z=torch.from_numpy(g["z"]).to(DEV))
    assert max_abs(y.cpu(), g["y"]) <= WAVE_TOL


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05])
def test_discriminator_forward(backend):
    d = golden("d_forward.npz")
    s = build_segan().to(DEV)
    s.D.engine.backend = backend
    x = torch.from_numpy(d["x"]).to(DEV)
    s.D.train()
    random.seed(int(d["py_random_seed"]))
    with torch.no_grad():
        y, acts = s.D(x)
    rep = {"logit": max_abs(y.cpu(), d["y_train"])}
    for l in range(5):
        bn = s.D.enc_blocks[l].norm
        rep["rm%d" % l] = max_abs(bn.running_mean.cpu(), d["running_mean.%d" % l])
        rep["rv%d" % l] = max_abs(bn.running_var.cpu(), d["running_var.%d" % l])
        idx = torch.from_numpy(d["act_idx.%d" % l]).to(DEV)
        rep["act%d" % l] = max_abs(acts["h_%d" % l].reshape(-1)[idx].cpu(), d["act_val.%d" % l])
    print("D fwd backend %d:" % backend, {k: "%.2e" % v for k, v in rep.items()})
    # measured (fp16 operands, fp32 accumulation; deterministic): logit 1.2-1.4e-3, running mean <= 1.0e-4, running
    # var <= 3.4e-4, activations <= 3.9e-3 -- the survey's 1e-3 logit gate is the fp16 operand format's own distance
    # here (tests/test_gpu_parity_scale.py holds the batch-300 case to the gate or the control); ~2x margins:
    assert rep["logit"] <= 3e-3
    for l in range(5):
        assert rep["rm%d" % l] <= 3e-4 and rep["rv%d" % l] <= 6e-4 and rep["act%d" % l] <= 8e-3, (l, rep)
    s.D.eval()
    random.seed(8)
    with torch.no_grad():
        ye, _ = s.D(x)
    assert max_abs(ye.cpu(), d["y_eval"]) <= 2e-2          # eval mode: un-normalised activations, larger logits


def _check_sampled(t, tag, name, got, tol_rel):
    idx = torch.from_numpy(t["idx." + tag + name])
    ref = torch.from_numpy(t["val." + tag + name])
    g = got.detach().float().cpu().reshape(-1)[idx]
    norm = float(t["norm." + tag + name])
    rms = norm / max(1.0, got.numel()) ** 0.5
    # relative L2 error over the sampled entries, floored by the tensor's RMS (tiny tensors)
    return float((g - ref).norm()), float(ref.norm()) + rms


@pytest.mark.parametrize("backend", [BACKEND_FFMA, BACKEND_TCGEN05])
def test_train_step_vs_reference(backend):
    """One SEGAN+ G+D step (model.py:283-321) from the reference's seed state: losses, sampled
    gradients (norm-relative), BN running stats and the post-step parameter deltas."""
    t = golden("train_step_b4.npz")
    B = t["clean"].shape[0]
    s = build_segan(batch_size=B)
    assert sd_sha(s.G.state_dict()) == str(t["sha_G"]) and sd_sha(s.D.state_dict()) == str(t["sha_D"])
    s = s.to(DEV)
    s.G.engine.backend = backend
    s.D.engine.backend = backend
    s.G.train()
    s.D.train()
    opts = __import__("tests.util", fromlist=["load_opts"]).load_opts(batch_size=B)
    Gopt, Dopt = s.build_optimizers(opts)
    random.seed(int(t["py_random_seed"]))
    torch.manual_seed(int(t["torch_seed_z"]))
    clean = torch.from_numpy(t["clean"]).unsqueeze(1).to(DEV)
    noisy = torch.from_numpy(t["noisy"]).unsqueeze(1).to(DEV)
    pre = {("G." + k): v.detach().clone() for k, v in s.G.state_dict().items()}
    pre.update({("D." + k): v.detach().clone() for k, v in s.D.state_dict().items()})
    # capture the D-step gradients before the G step overwrites nothing (G step skips D wgrad)
    losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0)
    torch.cuda.synchronize()
    lv = losses.tolist()
    print("losses", lv, [float(t[k]) for k in ("d_real_loss", "d_fake_loss", "g_adv_loss", "g_l1_loss")])
    assert max_abs(s.G.z.cpu(), t["z"]) == 0.0          # same z as the reference drew
    for got, k in zip(lv, ("d_real_loss", "d_fake_loss", "g_adv_loss", "g_l1_loss")):
        ref = float(t[k])
        assert abs(got - ref) <= 2e-2 * max(1.0, abs(ref)), (k, got, ref)
    ge, de = s.G.engine, s.D.engine
    worst = {}
    for tag, eng in (("gD.", de), ("gG.", ge)):
        for name, p in eng.module.named_parameters():
            if tag == "gD." and name.startswith("enc_blocks") and name.endswith("conv.bias"):
                continue       # gradient is zero in exact arithmetic (bias feeds BatchNorm)
            err, rms = _check_sampled(t, tag, name, eng.grad_of(name), 0)
            worst[tag + name] = err / (rms + 1e-12)
    bad = {k: v for k, v in worst.items()
           if v > (GRAD_TOL_D if k.startswith("gD.") else GRAD_TOL_G_THROUGH_UPDATED_D)}
    print("worst sampled grad rel-L2:", sorted(worst.items(), key=lambda kv: -kv[1])[:8])
    assert not bad, bad
    for name, sd in (("G.", s.G.state_dict()), ("D.", s.D.state_dict())):
        for k, v in sd.items():
            if "running_" in k:
                assert max_abs(v.cpu(), t["post_full." + name + k]) <= 2e-2, k   # 3rd BN pass sees the updated D
            elif v.dtype.is_floating_point:
                delta = (v - pre[name + k]).detach().cpu().reshape(-1)
                idx = torch.from_numpy(t["post_idx." + name + k])
                ref = torch.from_numpy(t["post_delta." + name + k])
                # RMSprop's first step is +-lr*g/(0.1|g|+eps): sign-like, so compare loosely by count
                if "conv.bias" in k and name == "D.":
                    continue
                mism = float(((delta[idx] - ref).abs() > 2.5e-4).float().mean())
                assert mism <= (0.2 if name == "D." else 0.35), (name + k, mism)


def test_overlapped_step_matches_serial_step():
    """The side-stream schedule (weight-gradient chain and Generator forward on side streams,
    engine.OVERLAP) computes the same step as the single-stream schedule.  The weight gradients are
    summed with fp32 atomics, so two runs of the SAME schedule already differ in the last bits and
    RMSprop's sign-like first step amplifies that into the second step; the serial schedule run
    twice gives the noise floor the overlapped schedule is held to."""
    from segan_pytorch_b200 import engine as E
    from tests.util import load_opts
    t = golden("train_step_b4.npz")
    B = t["clean"].shape[0]
    clean = torch.from_numpy(t["clean"]).unsqueeze(1).to(DEV)
    noisy = torch.from_numpy(t["noisy"]).unsqueeze(1).to(DEV)
    z = torch.from_numpy(t["z"]).to(DEV)
    random.seed(7)
    shifts3 = [O.draw_phase_shifts(5, 5) for _ in range(3)]

    def run(mode):
        prev = E.OVERLAP
        E.OVERLAP = mode
        try:
            s = build_segan(batch_size=B).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B))
            out = []
            for _ in range(2):          # second step: packed weights / buffers are re-used across steps
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=z, shifts3=shifts3)
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad.clone(), s.D.engine.grad.clone()))
            return out
        finally:
            E.OVERLAP = prev

    ser1, ser2, ovl = run(False), run(False), run(True)
    for step in (0, 1):
        (l0, gG0, gD0), (l1, gG1, gD1), (l2, gG2, gD2) = ser1[step], ser2[step], ovl[step]
        floor_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l1))
        floor_g = max(rel_err(gG1, gG0), rel_err(gD1, gD0))
        err_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l2))
        err_g = max(rel_err(gG2, gG0), rel_err(gD2, gD0))
        print("step %d: serial-vs-serial loss %.2e grad %.2e | overlapped-vs-serial loss %.2e grad %.2e"
              % (step, floor_l, floor_g, err_l, err_g))
        assert err_l <= 10 * floor_l + 2e-3, (step, l0, l2)
        assert err_g <= 10 * floor_g + 5e-3, (step, err_g, floor_g)


def test_graph_replayed_steps_match_eager_steps():
    """SEGAN.train_step captures the step into CUDA graphs after engine.GRAPH_WARMUP eager steps (phase
    shifts then come from a device table) and replays it.  Four steps from the same state and inputs:
    eager vs eager gives the noise floor (fp32-atomics summation order amplified by RMSprop's sign-like
    steps), graph-replayed steps are held to it; the replayed steps must also really be replays."""
    from segan_pytorch_b200 import engine as E
    from tests.util import load_opts
    t = golden("train_step_b4.npz")
    B = t["clean"].shape[0]
    clean = torch.from_numpy(t["clean"]).unsqueeze(1).to(DEV)
    noisy = torch.from_numpy(t["noisy"]).unsqueeze(1).to(DEV)
    gen = torch.Generator().manual_seed(3)
    zs = [torch.randn(B, 1024, 16, generator=gen).to(DEV) for _ in range(4)]
    random.seed(11)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(4)]

    def run(graphs):
        prev = E.GRAPHS
        E.GRAPHS = graphs
        try:
            s = build_segan(batch_size=B).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B))
            out = []
            for i in range(4):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=zs[i], shifts3=shifts[i])
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad.clone(), s.D.engine.grad.clone()))
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs, Gopt.t
        finally:
            E.GRAPHS = prev

    (e1, n1, _), (e2, n2, _), (gr, n3, t3) = run(False), run(False), run(True)
    assert n1 == 0 and n2 == 0 and n3 == 1 and t3 == 4
    for step in range(4):
        (l0, gG0, gD0), (l1, gG1, gD1), (l2, gG2, gD2) = e1[step], e2[step], gr[step]
        floor_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l1))
        floor_g = max(rel_err(gG1, gG0), rel_err(gD1, gD0))
        err_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l2))
        err_g = max(rel_err(gG2, gG0), rel_err(gD2, gD0))
        print("step %d: eager-vs-eager loss %.2e grad %.2e | graph-vs-eager loss %.2e grad %.2e"
              % (step, floor_l, floor_g, err_l, err_g))
        # the floor is itself a random draw (two runs can land close by chance): generous multiple + absolute slack
        assert err_l <= 10 * floor_l + 2e-3, (step, l0, l2)
        assert err_g <= 10 * floor_g + 5e-3, (step, err_g, floor_g)


def test_train_loop_with_prefetcher_matches_manual_steps(tmp_path):
    """SEGAN.train (train.py:95-98 path) over a DataLoader, batches staged by DevicePrefetcher one step
    ahead on a copy stream, against the same steps fed by blocking .to(device) copies."""
    from torch.utils.data import DataLoader
    from segan_pytorch_b200.segan.datasets import SyntheticSEDataset, collate_fn
    from tests.util import load_opts, seed_all
    B, n_items = 2, 6
    dset = SyntheticSEDataset(n_items, 16384, seed=3)

    def loader():
        return DataLoader(dset, batch_size=B, shuffle=False, num_workers=0, pin_memory=True, collate_fn=collate_fn,
                          drop_last=True)
    opts = load_opts(batch_size=B, epoch=1, save_path=str(tmp_path), z_device="cuda")
    s1 = build_segan(batch_size=B, save_path=str(tmp_path), z_device="cuda").to(DEV)
    seed_all(5)
    torch.cuda.manual_seed_all(5)
    s1.train(opts, loader(), torch.nn.MSELoss(), 100.0, 1e-5, 100, log_freq=1000, device=DEV)
    torch.cuda.synchronize()
    l1 = s1.last_losses.tolist()
    s2 = build_segan(batch_size=B, z_device="cuda").to(DEV)
    s2.G.train()
    s2.D.train()
    Gopt, Dopt = s2.build_optimizers(opts)
    seed_all(5)
    torch.cuda.manual_seed_all(5)
    for _, clean, noisy, _ in loader():
        losses = s2.train_step(clean.unsqueeze(1).to(DEV), noisy.unsqueeze(1).to(DEV), Gopt, Dopt, 100.0)
    torch.cuda.synchronize()
    l2 = losses.tolist()
    print("train loop", l1, "manual", l2)
    # three GAN steps with RMSprop's sign-like first updates amplify the fp32-atomics summation order
    # (measured: losses within 3 %, parameters 1.2e-2 apart); the L1 term depends on the data and on G
    # only weakly through those steps, so it pins "same batches in the same order" tightly
    for a, b in zip(l1, l2):
        assert abs(a - b) <= 0.25 * max(1.0, abs(b)), (l1, l2)
    assert abs(l1[3] - l2[3]) <= 2e-3 * abs(l2[3]), (l1, l2)
    assert rel_err(s1.G.engine.flat, s2.G.engine.flat) <= 5e-2


def test_clear_on_read_gradients_match_explicit_zeroing():
    """Production path: the optimiser kernels zero the gradient buckets as they read them and no fill is launched;
    KEEP_GRADS (the mode the parity tests run in) zeroes explicitly.  Three steps each way from the same state:
    same losses and parameters up to the fp32-atomics noise floor (KEEP vs KEEP)."""
    from segan_pytorch_b200 import engine as E
    from tests.util import load_opts
    t = golden("train_step_b4.npz")
    B = t["clean"].shape[0]
    clean = torch.from_numpy(t["clean"]).unsqueeze(1).to(DEV)
    noisy = torch.from_numpy(t["noisy"]).unsqueeze(1).to(DEV)
    gen = torch.Generator().manual_seed(4)
    zs = [torch.randn(B, 1024, 16, generator=gen).to(DEV) for _ in range(3)]
    random.seed(12)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(3)] for _ in range(3)]

    def run(keep):
        prev = E.KEEP_GRADS, E.GRAPHS
        E.KEEP_GRADS, E.GRAPHS = keep, False
        try:
            s = build_segan(batch_size=B).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B))
            for i in range(3):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=zs[i], shifts3=shifts[i])
            torch.cuda.synchronize()
            nz = int(s.G.engine.grad.count_nonzero()) + int(s.D.engine.grad.count_nonzero())
            return losses.tolist(), s.G.engine.flat.clone(), s.D.engine.flat.clone(), nz
        finally:
            E.KEEP_GRADS, E.GRAPHS = prev
    k1, k2, c = run(True), run(True), run(False)
    assert c[3] == 0 and k1[3] > 0                      # buckets left zeroed / left in place
    floor = max(rel_err(k2[1], k1[1]), rel_err(k2[2], k1[2]))
    err = max(rel_err(c[1], k1[1]), rel_err(c[2], k1[2]))
    print("params after 3 steps: keep-vs-keep %.2e, clear-vs-keep %.2e; losses %s %s" % (floor, err, k1[0], c[0]))
    assert err <= 10 * floor + 1e-4
    lfloor = max(abs(a - b) / max(1.0, abs(b)) for a, b in zip(k2[0], k1[0]))
    for a, b in zip(c[0], k1[0]):
        assert abs(a - b) <= (10 * lfloor + 0.05) * max(1.0, abs(b)), (c[0], k1[0], k2[0])


def test_state_dict_tracks_packed_masters(tmp_path):
    """The big weights' nn.Parameters are mirrors of the packed masters: state_dict() / save() after a step return
    the UPDATED weights, load_state_dict() reaches the masters, and a forward after loading uses the loaded weights."""
    from tests.util import load_opts
    B = 2
    s = build_segan(batch_size=B).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B))
    gen = torch.Generator().manual_seed(5)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).to(DEV)
    noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=gen)).to(DEV)
    z = torch.randn(B, 1024, 16, generator=gen).to(DEV)
    sd0 = {k: v.clone() for k, v in s.G.state_dict().items()}
    s.train_step(clean, noisy, Gopt, Dopt, 100.0, z=z)
    sd1 = {k: v.clone() for k, v in s.G.state_dict().items()}
    k = "dec_blocks.1.deconv.weight"
    delta = (sd1[k] - sd0[k]).abs()
    assert 4e-4 <= float(delta.max()) <= 5.1e-4          # RMSprop first step: lr * g / (sqrt(0.01 g^2) + eps) = 10 lr sign(g)
    # the mirror equals the master, exported through the tensor-algebra twin
    from segan_pytorch_b200.engine import unpack_reference
    eng = s.G.engine
    lay = eng.by_name[k]
    assert torch.equal(sd1[k], unpack_reference(1, eng.mview(lay), lay.c_out, lay.c_in, 0).reshape(sd1[k].shape))
    s.G.eval()
    with torch.no_grad():
        y1 = s.G(noisy, z=z).clone()
        s.G.load_state_dict(sd0)                          # back to the initial weights: masters must follow
        y0 = s.G(noisy, z=z).clone()
        s.G.load_state_dict(sd1)
        y1b = s.G(noisy, z=z).clone()
    assert max_abs(y1, y1b) == 0.0 and max_abs(y1, y0) > 1e-5
    # checkpoint round trip through Saver
    s.G.save(str(tmp_path), 1)
    s2 = build_segan(seed=3, batch_size=B).to(DEV)
    import os
    s2.G.load_pretrained(os.path.join(str(tmp_path), "weights_Generator-Generator-1.ckpt"), True)
    s2.G.eval()
    with torch.no_grad():
        assert max_abs(s2.G(noisy, z=z), y1) == 0.0


def test_generate_chunked_vs_reference(segan):
    g = golden("generate_40000.npz")
    if hasattr(segan.G, "z"):
        del segan.G.z
    out, g_c = segan.generate(torch.from_numpy(g["wav"]), z=torch.from_numpy(g["z"]))
    assert out.shape == g["out"].shape
    # de-emphasis integrates the waveform error (gain 1/(1-0.95) = 20)
    assert max_abs(out, g["out"]) <= 20 * WAVE_TOL
    assert tuple(g_c.shape) == (1, 1024, 16)


def test_clean_files_streaming_matches_per_file_generate(tmp_path):
    """clean.py streaming (SEGAN.clean_files: windows batched ACROSS files, int16 -> float + whole-file pre-emphasis
    on the device, segmented de-emphasis, threaded wav I/O) against the reference loop's semantics: one
    SEGAN.generate call per normalised + pre-emphasised file (clean.py:59-82), same z stream, and against the
    oracle's chunked inference for one file."""
    from scipy.io import wavfile
    from segan_pytorch_b200.segan.datasets import normalize_wave_minmax, pre_emphasize
    rng = np.random.RandomState(9)
    lengths = [40000, 16384, 9000, 70001, 32768, 50]
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    paths = []
    for i, n in enumerate(lengths):
        w = (rng.randn(n) * 3000).clip(-32768, 32767).astype(np.int16)
        p = str(src / ("utt%02d.wav" % i))
        wavfile.write(p, 16000, w)
        paths.append(p)
    s = build_segan().to(DEV)
    sdG = cpu_state(s.G)
    torch.manual_seed(77)
    nwin = s.clean_files(paths, str(dst), batch=3, group_windows=5)        # tiny batches: groups and batches split
    assert nwin == sum((n + 16383) // 16384 for n in lengths)
    z_first = s.G.z.cpu().clone()
    # the reference's loop on a fresh model with the same RNG stream
    s2 = build_segan().to(DEV)
    torch.manual_seed(77)
    zs = torch.randn(len(lengths), 1024, 16)
    torch.manual_seed(77)
    assert torch.equal(z_first[0], zs[0])
    for i, p in enumerate(paths):
        rate, w = wavfile.read(p)
        pw = torch.FloatTensor(pre_emphasize(normalize_wave_minmax(w), 0.95)).view(1, 1, -1)
        ref, _ = s2.generate(pw)
        rate2, got = wavfile.read(str(dst / ("utt%02d.wav" % i)))
        assert rate2 == 16000 and got.dtype == np.float32 and got.shape == ref.shape == (lengths[i],)
        # same kernels, different batch composition: M-tile boundaries move, fp16 results do not
        assert max_abs(got, ref) <= 2e-4, (i, max_abs(got, ref))
    # and one file against the oracle (fp32 reference arithmetic): z of file 0 for every window of file 0
    rate, w = wavfile.read(paths[0])
    pw = torch.FloatTensor(pre_emphasize(normalize_wave_minmax(w), 0.95)).view(1, 1, -1)
    with O.oracle_mode(), torch.no_grad():
        oref = O.segan_generate(sdG, pw, zs[:1])
    rate2, got = wavfile.read(str(dst / "utt00.wav"))
    assert max_abs(got, oref) <= 20 * WAVE_TOL


def test_prefetcher_pcm16_path_matches_host_preprocessing():
    """int16 PCM batches staged by DevicePrefetcher are normalised + pre-emphasised per window on the device
    (sg_pcm16_to_wave) exactly like se_dataset.py:108-117 does on the host."""
    from segan_pytorch_b200.segan.datasets import DevicePrefetcher, normalize_wave_minmax, pre_emphasize
    rng = np.random.RandomState(4)
    batches = []
    for _ in range(3):
        c = rng.randint(-32768, 32768, size=(4, 16384)).astype(np.int16)
        n = rng.randint(-32768, 32768, size=(4, 16384)).astype(np.int16)
        batches.append([None, torch.from_numpy(c).pin_memory(), torch.from_numpy(n).pin_memory(), None])
    got = [(c.cpu().clone(), n.cpu().clone()) for _, c, n, _ in DevicePrefetcher(iter(batches), DEV, preemph=0.95)]
    assert len(got) == 3
    for (gc, gn), (_, c, n, _) in zip(got, batches):
        for g, src in ((gc, c), (gn, n)):
            ref = np.stack([pre_emphasize(normalize_wave_minmax(w.astype(np.float32)), 0.95) for w in src.numpy()])
            assert g.shape == (4, 1, 16384)
            assert max_abs(g[:, 0], ref) <= 2e-6


def test_wav_dataset_pcm16_through_prefetcher_matches_float_mode(tmp_path):
    """SEDataset(pcm16=True) -> DataLoader -> DevicePrefetcher: int16 windows + the sample before each window
    cross the link and sg_pcm16_to_wave reproduces the reference's whole-file normalise + pre-emphasise windows
    (SEDataset float mode = se_dataset.py:191-199,355-368, pinned against the reference in tests/test_dataset.py)."""
    from torch.utils.data import DataLoader
    from segan_pytorch_b200.segan.datasets import DevicePrefetcher, SEDataset, collate_fn
    from tests.test_dataset import _make_wavs
    cdir, ndir = _make_wavs(str(tmp_path), seed=5)
    kw = dict(batch_size=3, shuffle=False, num_workers=0, collate_fn=collate_fn, drop_last=False)
    ref_batches = list(DataLoader(SEDataset(cdir, ndir, 0.95), **kw))
    pcm_loader = DataLoader(SEDataset(cdir, ndir, 0.95, pcm16=True), pin_memory=True, **kw)
    n = 0
    for (names, c, nz, idx), (rn, rc, rz, ridx) in zip(DevicePrefetcher(pcm_loader, DEV, preemph=0.95), ref_batches):
        assert list(names) == list(rn) and c.shape == (rc.shape[0], 1, 16384)
        assert max_abs(c[:, 0].cpu(), rc) <= 2e-6 and max_abs(nz[:, 0].cpu(), rz) <= 2e-6
        n += 1
    assert n == len(ref_batches) == 4


def test_generate_stream_matches_direct_forward(segan):
    """Streaming inference (BASELINE config 5): batches go host -> device -> G -> host on three overlapping
    streams; every yielded batch equals the direct forward of the same windows."""
    gen = torch.Generator().manual_seed(12)
    batches = [(0.3 * torch.randn(3, 1, 16384, generator=gen)).pin_memory() for _ in range(5)]
    z = torch.randn(3, 1024, 16, generator=gen).to(DEV)
    segan.G.eval()
    outs = [o.clone() for o in segan.generate_stream(iter(batches), z=z)]
    assert len(outs) == len(batches)
    with torch.no_grad():
        for hb, o in zip(batches, outs):
            ref = segan.G(hb.to(DEV), z=z).cpu()
            assert max_abs(o, ref) <= 1e-6, max_abs(o, ref)


def test_autograd_path_matches_fused_step(segan):
    """Generator / Discriminator used as ordinary autograd modules give the same gradients as the
    fused step's engines (API compatibility path)."""
    gen = torch.Generator().manual_seed(9)
    B = 2
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).to(DEV)
    noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=gen)).to(DEV)
    z = torch.randn(B, 1024, 16, generator=gen).to(DEV)
    s = build_segan().to(DEV)
    s.G.train()
    s.D.train()
    y = s.G(noisy, z=z)
    shifts = [1, -2, 3, -4, 5]
    logit, _ = s.D(torch.cat((y, noisy), 1), shifts=shifts)
    loss = torch.nn.functional.mse_loss(logit.view(-1), torch.ones(B, device=DEV)) + \
        100 * torch.nn.functional.l1_loss(y, clean)
    loss.backward()
    gG = {n: p.grad.detach().clone() for n, p in s.G.named_parameters()}
    # oracle gradients on CPU
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    pG = {k: sdG[k].clone().requires_grad_(True) for k in O._trainable(sdG)}
    with O.oracle_mode():
        yo = O.generator_forward({**sdG, **pG}, noisy.cpu(), z.cpu())
        lo = O.discriminator_forward(dict(sdD), torch.cat((yo, noisy.cpu()), 1), shifts, training=True)
        losso = torch.nn.functional.mse_loss(lo.view(-1), torch.ones(B)) + 100 * torch.nn.functional.l1_loss(yo, clean.cpu())
        go = dict(zip(pG.keys(), torch.autograd.grad(losso, list(pG.values()))))
    assert abs(float(loss) - float(losso)) <= 2e-2 * max(1.0, abs(float(losso)))
    rep = {k: rel_err(gG[k].cpu(), ref) for k, ref in go.items()}
    print("autograd path rel errs:", {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        assert v <= 8e-2, (k, v)


@pytest.mark.parametrize("variant", ["misalign", "misalign+interf", "vanilla_gan"])
def test_wsegan_step_vs_oracle(variant):
    """WSEGAN step (model.py:572-669) with --misalign_pair, with --misalign_pair --interf_pair, and with
    --vanilla_gan (BCE-with-logits D cost).  The reference's own WSEGAN.train cannot run on CPU / torch>=2
    (SURVEY.md F4), so this compares with the oracle restatement (whose G / D / loss building blocks are
    pinned): parity of this row is 'unpinned by the reference'."""
    from segan_pytorch_b200.segan.models import WSEGAN
    from tests.util import load_opts, seed_all
    B = 3
    seed_all(111)
    misalign = variant != "vanilla_gan"
    interf_on = variant == "misalign+interf"
    vanilla = variant == "vanilla_gan"
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=misalign, interf_pair=interf_on, vanilla_gan=vanilla)
    s = WSEGAN(opts)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    s = s.to(DEV)
    s.G.train()
    s.D.train()
    gen = torch.Generator().manual_seed(21)
    clean = (0.3 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, generator=gen)).clamp(-1, 1)
    z = torch.randn(B, 1024, 16, generator=gen)
    random.seed(5)
    n_pass = 3 + int(misalign) + int(interf_on)
    shifts = [O.draw_phase_shifts(5, 5) for _ in range(n_pass)]
    perm = [2, 0, 1] if misalign else None
    interf = O.interferer_squares([(250, 0.1), (4000, 0.05), (1000, 1)], 16384) if interf_on else None
    Gopt, Dopt = s.build_optimizers(opts)
    losses = s.train_step(clean.to(DEV), noisy.to(DEV), Gopt, Dopt, 100.0, uttname=["a", "b", "c"], z=z.to(DEV),
                          shifts=shifts, perm=perm, interf=interf).tolist()
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    ref = O.wsegan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts, perm, pow_weight=0.001, l1_weight=100.0,
                              interf=interf, vanilla_gan=vanilla)
    print("wsegan", variant, "losses", losses, [ref[k] for k in ("d_loss", "g_adv_loss", "pow_loss", "den_loss")])
    for got, k in zip(losses, ("d_loss", "g_adv_loss", "pow_loss", "den_loss")):
        assert abs(got - ref[k]) <= 3e-2 * max(1.0, abs(ref[k])), (variant, k, got, ref[k])
    rep = {k: rel_err(s.D.engine.grad_of(k).cpu(), g) for k, g in ref["gradsD"].items()
           if not (k.startswith("enc_blocks") and k.endswith("conv.bias"))}
    print("wsegan D grad rel errs (max):", max(rep.values()))
    assert max(rep.values()) <= 0.2, rep


@pytest.mark.parametrize("flags", [dict(misalign_pair=True), dict(misalign_pair=True, interf_pair=True)],
                         ids=["misalign", "misalign+interf"])
def test_wsegan_graph_replayed_steps_match_eager_steps(flags):
    """WSEGAN.train_step under CUDA-graph replay (phase shifts, the misalignment permutation and the interferers are
    device tensors refreshed per step) against the eager schedule: same protocol as the SEGAN test above."""
    from segan_pytorch_b200 import engine as E
    from segan_pytorch_b200.segan.models import WSEGAN
    from tests.util import load_opts, seed_all
    B, L, n_steps = 4, 16384, 4
    g = torch.Generator().manual_seed(77)
    clean = (0.3 * torch.randn(B, 1, L, generator=g)).clamp(-1, 1).to(DEV)
    noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, L, generator=g)).clamp(-1, 1).to(DEV)
    zs = [torch.randn(B, 1024, 16, generator=g).to(DEV) for _ in range(n_steps)]
    n_pass = 3 + len(flags)
    random.seed(13)
    shifts = [[O.draw_phase_shifts(5, 5) for _ in range(n_pass)] for _ in range(n_steps)]
    perms = [torch.randperm(B, generator=g).tolist() for _ in range(n_steps)]
    interfs = [WSEGAN.interferer_squares(B, L, picks=[(250 * 4 ** (i % 3), [0.01, 0.05, 0.1, 1][(i + k) % 4])
                                                       for i in range(B)]) for k in range(n_steps)]

    def run(graphs):
        prev = E.GRAPHS
        E.GRAPHS = graphs
        try:
            opts = load_opts(batch_size=B, wsegan=True, **flags)
            seed_all(111)
            s = WSEGAN(opts).to(DEV)
            s.G.train()
            s.D.train()
            Gopt, Dopt = s.build_optimizers(opts)
            out = []
            for i in range(n_steps):
                losses = s.train_step(clean, noisy, Gopt, Dopt, 0.0, z=zs[i], shifts=shifts[i], perm=perms[i],
                                      interf=interfs[i] if flags.get("interf_pair") else None)
                torch.cuda.synchronize()
                out.append((losses.tolist(), s.G.engine.grad.clone(), s.D.engine.grad.clone()))
            n_graphs = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            return out, n_graphs, Gopt.t
        finally:
            E.GRAPHS = prev

    (e1, n1, _), (e2, n2, _), (gr, n3, t3) = run(False), run(False), run(True)
    assert n1 == 0 and n2 == 0 and n3 == 1 and t3 == n_steps
    for step in range(n_steps):
        (l0, gG0, gD0), (l1, gG1, gD1), (l2, gG2, gD2) = e1[step], e2[step], gr[step]
        floor_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l1))
        floor_g = max(rel_err(gG1, gG0), rel_err(gD1, gD0))
        err_l = max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(l0, l2))
        err_g = max(rel_err(gG2, gG0), rel_err(gD2, gD0))
        print("step %d: eager-vs-eager loss %.2e grad %.2e | graph-vs-eager loss %.2e grad %.2e"
              % (step, floor_l, floor_g, err_l, err_g))
        assert err_l <= 10 * floor_l + 2e-3, (step, l0, l2)
        assert err_g <= 10 * floor_g + 5e-3, (step, err_g, floor_g)


def test_wsegan_train_loop_on_wav_directories(tmp_path):
    """train.py --wsegan --misalign_pair on wav directories (ADVICE r1: this path used to crash on the first batch):
    SEDataset(pcm16=True) -> persistent DevicePrefetcher iterator -> WSEGAN.train for two epochs -- eager warm-up steps,
    then the captured step (no 'additive' utterance in the batch names) -- finite losses that match the same steps
    driven by hand through train_step, and end-of-epoch checkpoints on disk."""
    import glob
    from torch.utils.data import DataLoader
    from segan_pytorch_b200.segan.datasets import DevicePrefetcher, SEDataset, collate_fn
    from segan_pytorch_b200.segan.models import WSEGAN
    from tests.test_dataset import _make_wavs
    from tests.util import load_opts, seed_all
    cdir, ndir = _make_wavs(str(tmp_path), seed=9)

    def loader():
        return DataLoader(SEDataset(cdir, ndir, 0.95, pcm16=True), batch_size=3, shuffle=False, num_workers=0,
                          collate_fn=collate_fn, drop_last=True, pin_memory=True)

    def make(save):
        opts = load_opts(batch_size=3, wsegan=True, misalign_pair=True, save_path=str(save), epoch=2, z_device="cuda")
        seed_all(111)
        s = WSEGAN(opts).to(DEV)
        return s, opts
    # (a) the entry-point loop
    s, opts = make(tmp_path / "ckpt")
    random.seed(21)
    torch.manual_seed(21)
    dl = loader()
    timings = s.train(opts, dl, torch.nn.MSELoss(), 100.0, 1e-5, 100, 1, device=DEV)
    torch.cuda.synchronize()
    la = s.last_losses.tolist()
    assert len(timings) == 2 * len(dl) and all(np.isfinite(la)), la
    assert glob.glob(str(tmp_path / "ckpt" / "*EOE_G-*")) and glob.glob(str(tmp_path / "ckpt" / "*EOE_D-*"))
    assert any(getattr(v, "graph", None) is not None for v in s._step_graphs.values()), "the step was never captured"
    # (b) the same batches, the same draws, stepped by hand
    s2, opts2 = make(tmp_path / "ckpt2")
    s2.G.train()
    s2.D.train()
    Gopt, Dopt = s2.build_optimizers(opts2)
    random.seed(21)
    torch.manual_seed(21)
    lb = None
    for _ in range(2):
        for names, c, n, _ in DevicePrefetcher(loader(), DEV, preemph=0.95):
            lb = s2.train_step(c.clone(), n.clone(), Gopt, Dopt, 100.0, uttname=names).tolist()
    print("WSEGAN.train last losses", la, "manual", lb)
    for a, b in zip(la, lb):
        assert abs(a - b) <= 0.15 * max(1.0, abs(b)), (la, lb)      # fp32-atomics order, amplified over six RMSprop steps
