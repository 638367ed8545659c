"""Generates tests/golden/*.npz by EXECUTING THE UNMODIFIED REFERENCE (santi-pdp/segan_pytorch) on CPU.
Needs a checkout of the reference (SEGAN_REFERENCE_ROOT); the fixtures it writes are committed, so the
test-suite itself never needs the reference.

    SEGAN_REFERENCE_ROOT=/path/to/segan_pytorch python tests/golden/make_golden.py

Hygiene (SURVEY.md F1 / App. D): oneDNN disabled; every conv / deconv layer is first
self-checked fp32-vs-fp64 before anything is emitted.

Weights are not stored (90.6 M params): they are re-created from the seed by the same
constructor call sequence (the repo's drop-in constructors consume the torch RNG in the same
order); each fixture stores a sha256 of the state dicts so that a mismatch is caught loudly.
"""
import hashlib
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.ref_import import load_reference, reference_opts, quiet  # noqa: E402

SEED = 111
N_SAMPLE = 256


def sd_sha(sd):
    h = hashlib.sha256()
    for k in sd:
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def sample_idx(numel, tag):
    g = np.random.RandomState(abs(hash_str(tag)) % (2 ** 31))
    n = min(N_SAMPLE, numel)
    return np.sort(g.choice(numel, size=n, replace=False)).astype(np.int64)


def hash_str(s):
    return int(hashlib.md5(s.encode()).hexdigest()[:8], 16)


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def arr_sha(t):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(t, dtype=np.float32)).tobytes()).hexdigest()


def seeded_randn(seed, shape):
    torch.manual_seed(seed)
    return torch.randn(*[int(s) for s in shape])


def build_reference_segan(ref, **over):
    seed_all(SEED)                                   # train.py:22-24
    with quiet():
        return ref.SEGAN(reference_opts(**over))


def selfcheck_layers(segan):
    """F1: every conv / deconv layer fp32 vs fp64 <= 1e-5 relative before trusting the CPU path."""
    g = torch.Generator().manual_seed(5)
    worst = 0.0
    for name, mod in list(segan.G.named_modules()) + list(segan.D.named_modules()):
        if isinstance(mod, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
            cin = mod.in_channels
            x = torch.randn(2, cin, 64, generator=g)
            y32 = mod(x)
            y64 = mod.double()(x.double())
            mod.float()
            rel = float((y32.double() - y64).abs().max() / y64.abs().max())
            worst = max(worst, rel)
            assert rel < 1e-5, (name, rel)
    return worst


def golden_g_forward(ref, segan, out):
    """BASELINE config 1: G forward on 1x16384, eval / no_grad."""
    g = torch.Generator().manual_seed(SEED)
    noisy = 0.3 * torch.randn(1, 1, 16384, generator=g)
    z = torch.randn(1, 1024, 16, generator=g)
    segan.G.eval()
    with torch.no_grad():
        y, hall = segan.G(noisy, z=z, ret_hid=True)
    d = dict(x=noisy.numpy(), z=z.numpy(), y=y.numpy(), sha_G=np.array(sd_sha(segan.G.state_dict())))
    for k, v in hall.items():
        flat = v.reshape(-1)
        idx = sample_idx(flat.numel(), "hall." + k)
        d["hall_idx." + k] = idx
        d["hall_val." + k] = flat[idx].numpy()
        d["hall_absmean." + k] = np.array(float(v.abs().mean()))
    np.savez_compressed(os.path.join(out, "g_forward_cfg1.npz"), **d)
    # a batched one with B = 3 (different windows, different z per window)
    noisy3 = 0.3 * torch.randn(3, 1, 16384, generator=g)
    z3 = torch.randn(3, 1024, 16, generator=g)
    with torch.no_grad():
        y3 = segan.G(noisy3, z=z3)
    np.savez_compressed(os.path.join(out, "g_forward_b3.npz"), x=noisy3.numpy(), z=z3.numpy(),
                        y=y3.numpy(), sha_G=np.array(sd_sha(segan.G.state_dict())))


def golden_d_forward(ref, segan, out):
    g = torch.Generator().manual_seed(SEED + 1)
    x = 0.3 * torch.randn(4, 2, 16384, generator=g)
    sha = sd_sha(segan.D.state_dict())
    segan.D.train()
    random.seed(7)
    y_tr, acts = segan.D(x)
    d = dict(x=x.numpy(), y_train=y_tr.detach().numpy(), py_random_seed=np.array(7), sha_D=np.array(sha))
    for l in range(5):
        bn = segan.D.enc_blocks[l].norm
        d["running_mean.%d" % l] = bn.running_mean.numpy().copy()
        d["running_var.%d" % l] = bn.running_var.numpy().copy()
        v = acts["h_%d" % l].detach().reshape(-1)
        idx = sample_idx(v.numel(), "dact.%d" % l)
        d["act_idx.%d" % l] = idx
        d["act_val.%d" % l] = v[idx].numpy()
    # eval mode with the running stats just updated (discriminate(), model.py:159-163)
    segan.D.eval()
    random.seed(8)
    with torch.no_grad():
        y_ev, _ = segan.D(x)
    d["y_eval"] = y_ev.numpy()
    np.savez_compressed(os.path.join(out, "d_forward.npz"), **d)


def golden_train_step(ref, out, B=4):
    """One iteration of the reference's own SEGAN.train (model.py:230-321), CPU, RMSprop."""
    segan = build_reference_segan(ref, batch_size=B, epoch=1, save_freq=10 ** 9)
    shaG, shaD = sd_sha(segan.G.state_dict()), sd_sha(segan.D.state_dict())
    g = torch.Generator().manual_seed(SEED + 2)
    clean = (0.3 * torch.randn(B, 16384, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 16384, generator=g)).clamp(-1, 1)
    names = ["utt%d" % i for i in range(B)]
    dloader = [[names, clean.clone(), noisy.clone(), torch.zeros(B)]]

    pre = {("G." + k): v.detach().clone() for k, v in segan.G.state_dict().items()}
    pre.update({("D." + k): v.detach().clone() for k, v in segan.D.state_dict().items()})

    losses = []
    crit = torch.nn.MSELoss()

    def criterion(a, b):
        l = crit(a, b)
        losses.append(float(l))
        return l

    snap = {}
    orig_build = segan.build_optimizers

    def build(opts):
        Gopt, Dopt = orig_build(opts)
        dstep = Dopt.step

        def dstep_wrapped(*a, **k):
            for n, p in segan.D.named_parameters():
                snap["gD." + n] = p.grad.detach().clone()
            return dstep(*a, **k)
        Dopt.step = dstep_wrapped
        return Gopt, Dopt
    segan.build_optimizers = build
    genh = {}
    def _grab(m, i, o):                   # must return None (a value would replace G's output)
        genh.setdefault("y", o.detach().clone())
    segan.G.register_forward_hook(_grab)

    opts = reference_opts(batch_size=B, epoch=1, save_freq=10 ** 9)
    random.seed(99)
    torch.manual_seed(1234)             # z is drawn inside G.forward from the global CPU generator
    with quiet():
        segan.train(opts, dloader, criterion, 100, 1e-5, 100, 10 ** 9, device="cpu")
    z = segan.G.z.detach().clone()
    # z is stored as the seeded draw that reproduces it (tests/util.golden re-draws and checks the sha256)
    assert torch.equal(z, seeded_randn(1234, z.shape))
    d = dict(clean=clean.numpy(), noisy=noisy.numpy(), Genh=genh["y"].numpy(),
             **{"z.seed": np.array(1234), "z.shape": np.array(z.shape), "z.sha256": np.array(arr_sha(z))},
             d_real_loss=np.array(losses[0]), d_fake_loss=np.array(losses[1]),
             g_adv_loss=np.array(losses[2]),
             g_l1_loss=np.array(float(100 * torch.nn.functional.l1_loss(genh["y"], clean.unsqueeze(1)))),
             sha_G=np.array(shaG), sha_D=np.array(shaD), py_random_seed=np.array(99),
             torch_seed_z=np.array(1234))
    for n, p in segan.G.named_parameters():
        snap["gG." + n] = p.grad.detach().clone()
    for k, gten in snap.items():
        flat = gten.reshape(-1)
        idx = sample_idx(flat.numel(), k)
        d["idx." + k] = idx
        d["val." + k] = flat[idx].numpy()
        d["norm." + k] = np.array(float(flat.double().norm()))
    post = {("G." + k): v for k, v in segan.G.state_dict().items()}
    post.update({("D." + k): v for k, v in segan.D.state_dict().items()})
    for k, v in post.items():
        if not v.dtype.is_floating_point:
            d["post." + k] = v.numpy()
            continue
        delta = (v - pre[k]).reshape(-1)
        idx = sample_idx(delta.numel(), "post." + k)
        d["post_idx." + k] = idx
        d["post_delta." + k] = delta[idx].numpy()
        d["post_delta_norm." + k] = np.array(float(delta.double().norm()))
        if "running_" in k:
            d["post_full." + k] = v.numpy()
    np.savez_compressed(os.path.join(out, "train_step_b%d.npz" % B), **d)
    return segan


def golden_generate(ref, segan, out):
    """SEGAN.generate (clean.py path): 40000-sample utterance => 3 chunks, last one padded."""
    g = torch.Generator().manual_seed(SEED + 3)
    wav = 0.3 * torch.randn(1, 1, 40000, generator=g)
    z = torch.randn(1, 1024, 16, generator=g)
    with torch.no_grad():
        c_res, _ = segan.generate(wav, z=z)
    np.savez_compressed(os.path.join(out, "generate_40000.npz"), wav=wav.numpy(), z=z.numpy(),
                        out=np.asarray(c_res), sha_G=np.array(sd_sha(segan.G.state_dict())))
    ds = ref._ref_datasets
    x = (np.random.RandomState(3).randn(4000) * 3000).astype(np.int16)
    xn = ds.normalize_wave_minmax(x)
    pe = ds.pre_emphasize(xn, 0.95)
    de = ds.de_emphasize(pe.astype(np.float32), 0.95)
    np.savez_compressed(os.path.join(out, "emphasis.npz"), x=x, norm=xn, pre=pe, de=de)


def golden_wsegan_generate(ref, out):
    """WSEGAN.generate (model.py:755-766): un-chunked inference on a 20000-sample utterance (make_divN pads it
    to 20480, utils.py:26-38), xavier-initialised WSEGAN built from the seed."""
    seed_all(SEED)
    with quiet():
        w = ref.WSEGAN(reference_opts(wsegan=True, misalign_pair=True))
    g = torch.Generator().manual_seed(SEED + 4)
    wav = 0.3 * torch.randn(1, 1, 20000, generator=g)
    z = torch.randn(1, 1024, 20, generator=g)
    with torch.no_grad():
        c_res, hall = w.generate(wav, z=z)
    d = dict(wav=wav.numpy(), z=z.numpy(), out=np.asarray(c_res), sha_G=np.array(sd_sha(w.G.state_dict())),
             enc_zc_shape=np.array(hall["enc_zc"].shape))
    # and a length that already is a multiple of 1024: make_divN still appends a whole block
    wav2 = 0.3 * torch.randn(1, 1, 4096, generator=g)
    z2 = torch.randn(1, 1024, 5, generator=g)
    with torch.no_grad():
        c2, _ = w.generate(wav2, z=z2)
    d.update(wav2=wav2.numpy(), z2=z2.numpy(), out2=np.asarray(c2))
    np.savez_compressed(os.path.join(out, "wsegan_generate.npz"), **d)


def golden_oracle_direct(ref, out):
    """The reference's own SEGAN (seed 7): G forward (eval) and D forward (train) on seeded inputs."""
    seed_all(7)
    with quiet():
        rs = ref.SEGAN(reference_opts())
    sha_G, sha_D = sd_sha(rs.G.state_dict()), sd_sha(rs.D.state_dict())      # before D's BatchNorm stats move
    g = torch.Generator().manual_seed(3)
    x = 0.3 * torch.randn(2, 1, 16384, generator=g)
    z = torch.randn(2, 1024, 16, generator=g)
    rs.G.eval()
    with torch.no_grad():
        y = rs.G(x, z=z)
    xd = 0.3 * torch.randn(3, 2, 16384, generator=g)
    rs.D.train()
    random.seed(5)
    with torch.no_grad():
        yd, _ = rs.D(xd)
    np.savez_compressed(os.path.join(out, "reference_direct.npz"), y=y.numpy(), yd=yd.numpy(),
                        sha_G=np.array(sha_G), sha_D=np.array(sha_D))


SNORM_UV = ("enc_blocks.3.conv.weight_u", "enc_blocks.3.conv.weight_v", "fc.0.weight_u", "fc.3.weight_v")
SNORM_GRADS = ("enc_blocks.2.conv.weight_orig", "fc.0.weight_orig", "fc.3.weight_orig", "enc_blocks.0.conv.bias")


def golden_snorm_discriminator(ref, out):
    """norm_type='snorm' Discriminator (seed 111): two training passes and one eval pass on the same input --
    outputs, power-iteration vectors after each pass, gradients of sum(D(x)) of the training passes (sampled)."""
    seed_all(111)
    with quiet():
        D = ref.Discriminator(2, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], pool_type='none', pool_slen=16,
                              norm_type='snorm', phase_shift=5)
    d = dict(keys=np.array(list(D.state_dict().keys())), sha_D=np.array(sd_sha(D.state_dict())))
    g = torch.Generator().manual_seed(3)
    x = 0.3 * torch.randn(2, 2, 16384, generator=g)
    for i, mode in enumerate(("train", "train", "eval")):
        D.train() if mode == "train" else D.eval()
        random.seed(5)
        y, _ = D(x)
        d["y.%d" % i] = y.detach().numpy()
        for k in SNORM_UV:
            d["uv.%d.%s" % (i, k)] = D.state_dict()[k].numpy().copy()
        if mode == "train":
            D.zero_grad()
            y.sum().backward()
            for k in SNORM_GRADS:
                gr = dict(D.named_parameters())[k].grad.reshape(-1)
                idx = np.sort(np.random.RandomState(hash_str(k) % (2 ** 31)).choice(
                    gr.numel(), size=min(4096, gr.numel()), replace=False)).astype(np.int64)
                d["grad_idx.%d.%s" % (i, k)] = idx
                d["grad_val.%d.%s" % (i, k)] = gr[idx].numpy()
                d["grad_norm.%d.%s" % (i, k)] = np.array(float(gr.double().norm()))
    np.savez_compressed(os.path.join(out, "snorm_discriminator.npz"), **d)


def golden_sum_merge_generator(ref, out):
    """skip_merge='sum' Generator (seed 111) with random skip alphas, eval forward on seeded inputs."""
    seed_all(111)
    with quiet():
        G = ref.Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], z_dim=1024, skip_merge='sum',
                          skip_type='alpha', skip_init='one', bias=True)
    d = dict(sha_G_init=np.array(sd_sha(G.state_dict())))
    g = torch.Generator().manual_seed(4)
    skip_keys = []
    with torch.no_grad():
        for k, p in G.named_parameters():
            if k.endswith("skip_k"):
                p.copy_(0.5 + torch.rand(p.shape, generator=g))       # alphas that matter
                skip_keys.append(k)
    x = 0.3 * torch.randn(2, 1, 16384, generator=g)
    z = torch.randn(2, 1024, 16, generator=g)
    G.eval()
    with torch.no_grad():
        y = G(x, z=z)
    d.update(skip_keys=np.array(skip_keys), y=y.numpy(), sha_G=np.array(sd_sha(G.state_dict())),
             dec1_weight_shape=np.array(G.state_dict()["dec_blocks.1.deconv.weight"].shape))
    np.savez_compressed(os.path.join(out, "sum_merge_generator.npz"), **d)


def golden_sedataset(ref, out):
    """The reference's SEDataset windows of the wav set tests/test_dataset.py writes (seed 1), as sha256 of the
    float32 window bytes."""
    import tempfile
    from scipy.io import wavfile
    from tests.test_dataset import _make_wavs
    ds = ref._ref_datasets

    def fake_load(path, sr=16000):                 # the reference only uses librosa for the sample count
        rate, w = wavfile.read(path)
        return w.astype(np.float32) / 32768.0, rate
    ds.librosa.load = fake_load

    class SeqPool(object):                         # the detached reference module cannot be pickled for mp.Pool
        def __init__(self, n):
            pass

        def map(self, fn, args):
            return [fn(a) for a in args]
    import types
    ds.mp = types.SimpleNamespace(Pool=SeqPool)
    with tempfile.TemporaryDirectory() as tmp:
        cdir, ndir = _make_wavs(tmp, seed=1)
        with quiet():
            rds = ds.SEDataset(cdir, ndir, 0.95, cache_dir=os.path.join(tmp, "cache"), slice_size=16384, stride=0.5,
                               slice_workers=1)
        rows = [rds[i][:4] for i in range(len(rds))]
    assert all(c.dtype == torch.float32 and n.dtype == torch.float32 for _, c, n, _ in rows)
    np.savez_compressed(os.path.join(out, "sedataset_windows.npz"),
                        names=np.array([r[0] for r in rows]), slice_idx=np.array([int(r[3]) for r in rows]),
                        sha_clean=np.array([arr_sha(r[1].numpy()) for r in rows]),
                        sha_noisy=np.array([arr_sha(r[2].numpy()) for r in rows]))


def main():
    torch.set_num_threads(8)
    ref = load_reference()
    out = HERE
    segan = build_reference_segan(ref)
    print("layer self-check fp32 vs fp64, worst rel err:", selfcheck_layers(segan))
    golden_g_forward(ref, segan, out)
    golden_d_forward(ref, segan, out)
    segan = build_reference_segan(ref)       # fresh D (BN buffers untouched)
    golden_generate(ref, segan, out)
    golden_train_step(ref, out, B=4)
    golden_wsegan_generate(ref, out)
    golden_oracle_direct(ref, out)
    golden_snorm_discriminator(ref, out)
    golden_sum_merge_generator(ref, out)
    golden_sedataset(ref, out)
    for f in sorted(os.listdir(out)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(out, f)))


if __name__ == "__main__":
    main()
