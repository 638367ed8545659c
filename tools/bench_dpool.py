"""Cost of the Discriminator's pooled heads on one GPU: the batch-300 SEGAN train step (CUDA-graph replayed, z drawn on
the device) with pool_type 'none' / 'conv' / 'gmax' / 'gavg', timed alternately in one process with CUDA events (best
of --rounds x --steps), then the WSEGAN --misalign_pair step (four D passes; graph-replayed) with 'none' and 'mlp' --
the head SEGAN cannot train -- the same way, and the head kernels' own device time per step from a separate
torch.profiler run of eager steps.  The SEGAN arms share one Generator (the head does not touch it), which keeps
four batch-300 models in memory; they are freed before the two WSEGAN arms are built.
Writes one JSON file to --out (default profiles/, git-ignored) and prints it.

    python tools/bench_dpool.py [--batch 300] [--steps 20] [--warmup 5] [--rounds 3] [--out profiles]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from segan_pytorch_b200 import engine as E                   # noqa: E402
from segan_pytorch_b200.segan.models import SEGAN, WSEGAN    # noqa: E402
from tests.util import load_opts, seed_all                   # noqa: E402
from tools.bench_conv_skip import gpu_info, timed            # noqa: E402

DEV = "cuda"
HEADS = ("none", "conv", "gmax", "gavg")


def make_arm(head, B, G):
    seed_all(111)
    opts = load_opts(batch_size=B, dpool_type=head, z_device="cuda")
    s = SEGAN(opts, generator=G).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(opts)
    g = torch.Generator(device=DEV).manual_seed(1)
    clean = (0.3 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    losses = torch.zeros(4, device=DEV)
    return dict(s=s, step=lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses))


def make_wsegan_arm(head, B):
    seed_all(111)
    opts = load_opts(batch_size=B, dpool_type=head, wsegan=True, misalign_pair=True, z_device="cuda")
    s = WSEGAN(opts).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(opts)
    g = torch.Generator(device=DEV).manual_seed(1)
    clean = (0.3 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    names = ["u%d" % i for i in range(B)]
    losses = torch.zeros(4, device=DEV)
    return dict(s=s, step=lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0, uttname=names, losses=losses))


def time_arms(arms, args):
    for a in arms.values():
        for _ in range(args.warmup):            # eager steps, graph capture, first replays
            a["step"]()
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(args.rounds):                # alternate the arms: clock / thermal drift hits all of them
        for k, a in arms.items():
            step_ms[k].append(timed(a["step"], args.steps))
    return step_ms


def head_kernel_times(arm, steps, mlp_ops=False):
    """Device time per eager step of the kernels whose names contain 'dhead' / 'fc_tail' (and, mlp_ops, the
    activation kernels, which the tower shares), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    prev = E.GRAPHS
    E.GRAPHS = False
    try:
        arm["step"]()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                arm["step"]()
            torch.cuda.synchronize()
    finally:
        E.GRAPHS = prev
    out = {}
    for ev in prof.key_averages():
        if "dhead" in ev.key or "fc_tail" in ev.key or (mlp_ops and ev.key.startswith("sg::act_")):
            us = getattr(ev, "device_time_total", None)
            if us is None:
                us = ev.cuda_time_total
            out[ev.key.split("(")[0]] = dict(ms_per_step=us / 1e3 / steps, launches_per_step=ev.count / steps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=300)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    B = args.batch
    res = dict(gpu=gpu_info(), batch=B, steps_per_round=args.steps, rounds=args.rounds, grad_dtype=str(E.GT),
               time=time.strftime("%Y-%m-%d %H:%M:%S"))
    G = SEGAN(load_opts(batch_size=B, z_device="cuda")).G
    arms = {k: make_arm(k, B, G) for k in HEADS}
    step_ms = time_arms(arms, args)
    res["gpu_after_timing"] = gpu_info()
    for k in arms:
        ms = min(step_ms[k])
        res[k] = dict(step_ms=ms, step_ms_rounds=step_ms[k], windows_per_s=B / (ms * 1e-3),
                      graph_replayed=any(v.graphs is not None for v in getattr(arms[k]["s"], "_step_graphs", {}).values()))
        if k != "none":
            res[k]["minus_none_step_ms"] = ms - min(step_ms["none"])
    res["max_memory_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    res["head_kernels"] = {k: head_kernel_times(a, 3) for k, a in arms.items()}
    del arms, G
    torch.cuda.empty_cache()
    warms = {k: make_wsegan_arm(k, B) for k in ("none", "mlp")}
    wms = time_arms(warms, args)
    res["gpu_after_wsegan_timing"] = gpu_info()
    res["wsegan"] = {k: dict(step_ms=min(wms[k]), step_ms_rounds=wms[k], windows_per_s=B / (min(wms[k]) * 1e-3),
                             graph_replayed=any(v.graphs is not None
                                                for v in getattr(warms[k]["s"], "_step_graphs", {}).values()))
                     for k in warms}
    res["wsegan"]["mlp_minus_none_step_ms"] = res["wsegan"]["mlp"]["step_ms"] - res["wsegan"]["none"]["step_ms"]
    res["wsegan_max_memory_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    res["wsegan_head_kernels"] = {k: head_kernel_times(a, 2, mlp_ops=True) for k, a in warms.items()}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "bench_dpool.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
