#!/usr/bin/env python
"""train.py -- drop-in for the reference entry point (train.py:14-258): same flag names and
defaults, same seeding, writes <save_path>/train.opts, trains SEGAN+ on the H100 engine.

Additive flags only: --synthetic N (N synthetic windows instead of --clean_trainset / --noisy_trainset wav
directories), --z_device {cpu,cuda}.
Data-parallel: launch with torchrun (one process per GPU); each rank trains on its own shard and
gradients are all-reduced once per optimiser step."""
import argparse
import json
import os
import random

import numpy as np
import torch
import torch.nn as nn
from torch.utils.data import DataLoader

from segan_pytorch_b200.segan.models import SEGAN, WSEGAN
from segan_pytorch_b200.segan.datasets import SEDataset, SyntheticSEDataset, collate_fn
from segan_pytorch_b200.hostbind import bind_host_to_gpu

# (name, type, default) -- the reference's flag surface (train.py:102-245)
FLAGS = [
    ("save_path", str, "seganv1_ckpt"), ("d_pretrained_ckpt", str, None), ("g_pretrained_ckpt", str, None),
    ("cache_dir", str, "data_cache"), ("clean_trainset", str, "data/clean_trainset"),
    ("noisy_trainset", str, "data/noisy_trainset"), ("clean_valset", str, None), ("noisy_valset", str, None),
    ("h5_data_root", str, None), ("data_stride", float, 0.5), ("seed", int, 111), ("epoch", int, 100),
    ("patience", int, 100), ("batch_size", int, 100), ("save_freq", int, 50), ("slice_size", int, 16384),
    ("opt", str, "rmsprop"), ("l1_dec_epoch", int, 100), ("l1_weight", float, 100), ("l1_dec_step", float, 1e-5),
    ("g_lr", float, 0.00005), ("d_lr", float, 0.00005), ("preemph", float, 0.95), ("max_samples", int, None),
    ("eval_workers", int, 2), ("slice_workers", int, 1), ("num_workers", int, 1), ("n_fft", int, 2048),
    ("reg_loss", str, "l1_loss"), ("skip_merge", str, "concat"), ("skip_type", str, "alpha"),
    ("skip_init", str, "one"), ("skip_kwidth", int, 11), ("gkwidth", int, 31), ("z_dim", int, 1024),
    ("gdec_kwidth", int, None), ("gnorm_type", str, None), ("pow_weight", float, 0.001),
    ("dpool_type", str, "none"), ("dpool_slen", int, 16), ("dkwidth", int, None), ("dnorm_type", str, "bnorm"),
    ("phase_shift", int, 5),
]
LIST_FLAGS = [("random_scale", float, [1]), ("genc_fmaps", int, [64, 128, 256, 512, 1024]),
              ("genc_poolings", int, [4, 4, 4, 4, 4]), ("gdec_fmaps", int, None), ("gdec_poolings", int, None),
              ("denc_fmaps", int, [64, 128, 256, 512, 1024]), ("denc_poolings", int, [4, 4, 4, 4, 4])]
BOOL_FLAGS = ["h5", "no_cuda", "no_train_gen", "preemph_norm", "wsegan", "aewsegan", "vanilla_gan", "no_bias",
              "no_z", "no_skip", "misalign_pair", "interf_pair", "sinc_conv"]


def build_parser():
    p = argparse.ArgumentParser()
    for name, typ, default in FLAGS:
        p.add_argument("--" + name, type=typ, default=default)
    for name, typ, default in LIST_FLAGS:
        p.add_argument("--" + name, type=typ, nargs="+", default=default)
    for name in BOOL_FLAGS:
        p.add_argument("--" + name, action="store_true", default=False)
    p.add_argument("--synthetic", type=int, default=0, help="train on N synthetic windows (additive flag)")
    p.add_argument("--z_device", type=str, default="cpu", choices=["cpu", "cuda"])
    return p


def main(opts):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if opts.no_cuda:
        raise SystemExit("--no-cuda: this build is the H100 engine; use the reference for CPU training")
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    opts.cuda = True
    bind_host_to_gpu(device)               # pinned staging buffers (and the loader workers) on the GPU's NUMA node
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    random.seed(opts.seed)                 # identical init on every rank (train.py:22-26)
    np.random.seed(opts.seed)
    torch.manual_seed(opts.seed)
    torch.cuda.manual_seed_all(opts.seed)
    if opts.aewsegan:
        raise SystemExit("--aewsegan is out of scope (broken in the reference: SURVEY.md 2.1)")
    segan = WSEGAN(opts) if opts.wsegan else SEGAN(opts)
    segan.to(device)
    print("Total model parameters: ", segan.get_n_params())
    if opts.g_pretrained_ckpt is not None:
        segan.G.load_pretrained(opts.g_pretrained_ckpt, True)
    if opts.d_pretrained_ckpt is not None:
        segan.D.load_pretrained(opts.d_pretrained_ckpt, True)
    random.seed(opts.seed + rank)          # per-rank data / z / phase-shift streams
    torch.manual_seed(opts.seed + rank)
    sampler = None
    if opts.synthetic > 0:
        dset = SyntheticSEDataset(opts.synthetic, opts.slice_size, seed=opts.seed + rank)
    else:
        # wav directories (train.py:52-60): int16 windows over the link, normalisation + pre-emphasis on the GPU
        # whenever the options allow it (no random scaling, norm before pre-emphasis)
        pcm16 = list(opts.random_scale) == [1] and not opts.preemph_norm
        dset = SEDataset(opts.clean_trainset, opts.noisy_trainset, opts.preemph, cache_dir=opts.cache_dir,
                         split='train', stride=opts.data_stride, slice_size=opts.slice_size,
                         max_samples=opts.max_samples, preemph_norm=opts.preemph_norm,
                         random_scale=opts.random_scale, pcm16=pcm16)
        if world > 1:
            from torch.utils.data.distributed import DistributedSampler
            sampler = DistributedSampler(dset, num_replicas=world, rank=rank, shuffle=True, seed=opts.seed)
    dloader = DataLoader(dset, batch_size=opts.batch_size, shuffle=(sampler is None), sampler=sampler,
                         num_workers=opts.num_workers, pin_memory=True, collate_fn=collate_fn, drop_last=True)
    criterion = nn.MSELoss()
    segan.train(opts, dloader, criterion, opts.l1_weight, opts.l1_dec_step, opts.l1_dec_epoch, opts.save_freq,
                va_dloader=None, device=device)


if __name__ == "__main__":
    opts = build_parser().parse_args()
    opts.bias = not opts.no_bias
    if int(os.environ.get("RANK", "0")) == 0:
        os.makedirs(opts.save_path, exist_ok=True)
        with open(os.path.join(opts.save_path, "train.opts"), "w") as cfg_f:
            cfg_f.write(json.dumps(vars(opts), indent=2))
    main(opts)
