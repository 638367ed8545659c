"""Cost of the Generator topologies on one GPU: the batch-300 G+D train step (CUDA-graph replayed) and G-only
inference for the default Generator, --no_z, --no_skip, --z_dim 256 and the default with --reg_loss mse_loss, timed
alternately in one process with CUDA events (best of --rounds rounds of --steps steps).  z is drawn on the device
(train steps) or passed in device-resident (inference): nothing on the host is timed.  Writes one JSON file to --out
(default profiles/, git-ignored) and prints it.

    python tools/bench_gtopo.py [--batch 300] [--steps 20] [--warmup 5] [--rounds 3] [--out profiles]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from segan_pytorch_b200 import engine as E              # noqa: E402
from tests.util import build_segan, load_opts           # noqa: E402

DEV = "cuda"
# arm -> train.py options
ARMS = {"default": {}, "no_z": dict(no_z=True), "no_skip": dict(no_skip=True), "z256": dict(z_dim=256),
        "mse": dict(reg_loss="mse_loss")}


def gpu_info():
    info = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        pl, sm, smax = [v.strip() for v in q.strip().split(",")]
        info.update(power_limit_w=float(pl), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(smax))
    except Exception as e:                  # the numbers stay valid without the context; say why it is missing
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def make_arm(over, B):
    """One SEGAN at batch B, set up as bench.py sets up its step: z drawn on the device (z_device='cuda'), so the
    timed region holds no host work."""
    s = build_segan(batch_size=B, z_device="cuda", **over).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B, z_device="cuda", **over))
    g = torch.Generator(device=DEV).manual_seed(1)
    clean = (0.3 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    z = None if s.G.no_z else torch.randn(B, s.G.z_dim, 16, device=DEV, generator=g)   # inference: reused
    losses = torch.zeros(4, device=DEV)
    return dict(s=s, step=lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses), noisy=noisy, z=z)


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
    arms = {k: make_arm(over, B) for k, over in ARMS.items()}
    for a in arms.values():
        for _ in range(args.warmup):            # eager steps, graph capture, first replays
            a["step"]()
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(args.rounds):                # alternate the arms: clock / thermal drift hits all of them
        for k, a in arms.items():
            step_ms[k].append(timed(a["step"], args.steps))
    inf_ms = {k: [] for k in arms}
    for a in arms.values():
        a["s"].G.eval()
    for _ in range(args.rounds):
        for k, a in arms.items():
            with torch.no_grad():
                G, x, z = a["s"].G, a["noisy"], a["z"]
                inf_ms[k].append(timed(lambda: G(x, z=z), max(2, args.steps // 4)))
    res["gpu_after_timing"] = gpu_info()
    for k in arms:
        ms = min(step_ms[k])
        res[k] = dict(step_ms=ms, step_ms_rounds=step_ms[k], windows_per_s=B / (ms * 1e-3),
                      g_infer_ms=min(inf_ms[k]), g_infer_windows_per_s=B / (min(inf_ms[k]) * 1e-3),
                      graph_replayed=any(v.graphs is not None for v in getattr(arms[k]["s"], "_step_graphs", {}).values()))
    res["max_memory_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "bench_gtopo.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
