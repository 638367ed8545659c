"""CPU tests of the wav-directory dataset (SURVEY.md 8(f)-N3): slicing / preprocessing parity with the
reference's SEDataset (its windows stored as checksums in tests/golden/sedataset_windows.npz) and consistency
of the int16 + previous-sample mode with the float mode."""
import os

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from segan_pytorch_b200.segan.datasets import SEDataset, collate_fn, normalize_wave_minmax, pre_emphasize
from tests.util import arr_sha, golden


def _make_wavs(root, lengths=(40000, 16384, 70001, 9000), seed=0):
    rng = np.random.RandomState(seed)
    cdir, ndir = os.path.join(root, "clean"), os.path.join(root, "noisy")
    os.makedirs(cdir)
    os.makedirs(ndir)
    for i, n in enumerate(lengths):
        c = (rng.randn(n) * 4000).clip(-32768, 32767).astype(np.int16)
        d = (c + rng.randn(n) * 800).clip(-32768, 32767).astype(np.int16)
        wavfile.write(os.path.join(cdir, "utt%02d.wav" % i), 16000, c)
        wavfile.write(os.path.join(ndir, "utt%02d.wav" % i), 16000, d)
    return cdir, ndir


def test_sedataset_windows_and_pcm16_mode_agree(tmp_path):
    cdir, ndir = _make_wavs(str(tmp_path))
    ds = SEDataset(cdir, ndir, 0.95, slice_size=16384, stride=0.5)
    # 40000 -> begs 0, 8192, 16384 ; 16384 -> beg 0 ; 70001 -> 0..49152 step 8192 (7) ; 9000 -> none
    assert len(ds) == 3 + 1 + 7
    dp = SEDataset(cdir, ndir, 0.95, slice_size=16384, stride=0.5, pcm16=True)
    assert len(dp) == len(ds)
    for i in range(len(ds)):
        name, c, n, t_i = ds[i]
        name2, cp, npcm, t2, prev = dp[i]
        assert (name, t_i) == (name2, t2) and cp.dtype == torch.int16 and prev.dtype == torch.int32
        for f, p, pv in ((c, cp, int(prev[0])), (n, npcm, int(prev[1]))):
            # numpy restatement of sg_pcm16_to_wave
            x = normalize_wave_minmax(p.numpy().astype(np.float32))
            y = x.copy()
            y[1:] = x[1:] - 0.95 * x[:-1]
            if pv != SEDataset.NO_PREV:
                y[0] = x[0] - 0.95 * normalize_wave_minmax(np.float32(pv))
            assert np.abs(y - f.numpy()).max() <= 2e-6
    # collated batch layout of the int16 mode: [names, clean(B,L) int16, noisy, slice_idx, prev(B,2) int32]
    b = collate_fn([dp[0], dp[1]])
    assert b[1].shape == (2, 16384) and b[1].dtype == torch.int16 and b[4].shape == (2, 2)
    with pytest.raises(ValueError):
        SEDataset(cdir, ndir, 0.95, pcm16=True, random_scale=[1, 0.5])


def test_sedataset_matches_reference(tmp_path):
    """Every window of the reference's SEDataset on the same files (float32 bytes, by sha256) is the window of
    ours with the same (file, slice index)."""
    cdir, ndir = _make_wavs(str(tmp_path), seed=1)
    r = golden("sedataset_windows.npz")
    ours = SEDataset(cdir, ndir, 0.95, slice_size=16384, stride=0.5)
    assert len(r["names"]) == len(ours)
    got = {(it[0], int(it[3])): it for it in (ours[i] for i in range(len(ours)))}
    for name, t_i, sc, sn in zip(r["names"], r["slice_idx"], r["sha_clean"], r["sha_noisy"]):
        mine = got[(str(name), int(t_i))]
        assert mine[1].dtype == mine[2].dtype == torch.float32
        assert arr_sha(mine[1].numpy()) == str(sc) and arr_sha(mine[2].numpy()) == str(sn)


def test_sedataset_short_noisy_file_is_trimmed_and_padded(tmp_path):
    """ADVICE r1: a noisy wav shorter than its clean twin -> the reference's extract_slice (se_dataset.py:338-347)
    cuts the pair to the common length and zero-pads to slice_size; int16 mode falls back to float windows."""
    root = str(tmp_path)
    cdir, ndir = os.path.join(root, "clean"), os.path.join(root, "noisy")
    os.makedirs(cdir)
    os.makedirs(ndir)
    rng = np.random.RandomState(2)
    c = (rng.randn(20000) * 3000).astype(np.int16)
    n = (rng.randn(19000) * 3000).astype(np.int16)          # 1000 samples short
    wavfile.write(os.path.join(cdir, "a.wav"), 16000, c)
    wavfile.write(os.path.join(ndir, "a.wav"), 16000, n)
    for pcm in (False, True):
        ds = SEDataset(cdir, ndir, 0.95, slice_size=16384, stride=1, pcm16=pcm)
        assert len(ds) == 1 and ds.pcm16 is False
        name, cw, nw, t_i = ds[0]
        assert cw.shape == nw.shape == (16384,) and cw.dtype == torch.float32
        assert np.abs(cw.numpy() - pre_emphasize(normalize_wave_minmax(c), 0.95)[:16384]).max() <= 1e-6
    # second window of a stride-0.5 slicing runs past the noisy file: trimmed to 19000-8192, padded with zeros
    c2 = (rng.randn(24576) * 3000).astype(np.int16)
    wavfile.write(os.path.join(cdir, "a.wav"), 16000, c2)
    ds = SEDataset(cdir, ndir, 0.95, slice_size=16384, stride=0.5)
    assert len(ds) == 2
    _, cw, nw, _ = ds[1]
    m = 19000 - 8192
    assert cw.shape == nw.shape == (16384,)
    assert float(cw[m:].abs().max()) == 0.0 and float(nw[m:].abs().max()) == 0.0 and float(nw[:m].abs().max()) > 0
    b = collate_fn([ds[0], ds[1]])
    assert b[1].shape == (2, 16384)
