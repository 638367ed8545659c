"""A/B timing of the train-step schedules inside ONE process (machines and power states differ between
runs by several %): alternates blocks of steps between configurations and prints per-block ms/step.

    python tools/ab_step.py [--batch 300] [--steps 10] [--rounds 4]
"""
import argparse
import sys

import torch

sys.path.insert(0, ".")
from segan_pytorch_b200 import engine as E                 # noqa: E402
from tests.util import build_segan, load_opts             # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=300)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--rounds", type=int, default=4)
ap.add_argument("--sync-each-step", action="store_true", help="losses.tolist() after every step (the e2e pattern)")
args = ap.parse_args()
B = args.batch
dev = torch.device("cuda", 0)
opts = load_opts(batch_size=B, z_device="cuda")
s = build_segan(seed=111, batch_size=B, z_device="cuda").to(dev)
s.G.train()
s.D.train()
Gopt, Dopt = s.build_optimizers(opts)
g = torch.Generator().manual_seed(1)
clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp_(-1, 1).to(dev)
noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp_(-1, 1).to(dev)
losses = torch.zeros(4, device=dev)
CONFIGS = [("graph+overlap", True, True), ("eager+overlap", False, True), ("graph+serial", True, False),
           ("eager+serial", False, False)]


def block(graphs, overlap, n):
    E.GRAPHS, E.OVERLAP = graphs, overlap
    for _ in range(4):                                   # warm-up / capture for this configuration
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        ls = s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
        if args.sync_each_step:
            ls.tolist()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


res = {name: [] for name, _, _ in CONFIGS}
for r in range(args.rounds):
    for name, gr, ov in CONFIGS:
        res[name].append(block(gr, ov, args.steps))
for name, v in res.items():
    v2 = sorted(v)
    print("%-16s median %.3f ms/step   all %s" % (name, v2[len(v2) // 2], " ".join("%.2f" % x for x in v)))
