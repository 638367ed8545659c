"""Cost of spectrally normalised Generators (norm_type='snorm') on one GPU: the batch-300 SEGAN G+D train step
(CUDA-graph replayed) with the default Generator and with the snorm Generator, the WSEGAN recipe of
run_wsegan_train.sh (snorm G and D, --misalign_pair, Adam: eager, as Adam steps are not graph-replayed), and G-only
eval inference, timed alternately in one process with CUDA events (best of --rounds rounds of --steps steps).  z is
drawn on the device (train steps) or passed in device-resident (inference): nothing on the host is timed.  Writes one
JSON file to --out (default profiles/, git-ignored) and prints it.

    python tools/bench_gsnorm.py [--batch 300] [--steps 20] [--warmup 5] [--rounds 3] [--out profiles]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from segan_pytorch_b200 import engine as E              # noqa: E402
from segan_pytorch_b200.segan.models import SEGAN, WSEGAN, Generator   # noqa: E402
from tests.util import load_opts, seed_all              # noqa: E402
from tools.bench_gtopo import gpu_info, timed           # noqa: E402

DEV = "cuda"
# arm -> (model class, train.py options, Generator norm_type)
ARMS = {"segan_default": (SEGAN, {}, None), "segan_snorm_g": (SEGAN, {}, "snorm"),
        "wsegan_recipe": (WSEGAN, dict(wsegan=True, misalign_pair=True, opt="adam", dnorm_type="snorm"), "snorm")}


def make_arm(cls, over, norm, B):
    """One model at batch B with z drawn on the device (z_device='cuda'), so the timed region holds no host work."""
    opts = load_opts(batch_size=B, z_device="cuda", **over)
    seed_all(111)
    G = Generator(1, opts.genc_fmaps, opts.gkwidth, opts.genc_poolings, opts.gdec_fmaps, opts.gdec_kwidth,
                  opts.gdec_poolings, z_dim=opts.z_dim, no_z=opts.no_z, skip=not opts.no_skip, bias=opts.bias,
                  skip_init=opts.skip_init, skip_type=opts.skip_type, skip_merge=opts.skip_merge,
                  skip_kwidth=opts.skip_kwidth, norm_type=norm)
    s = cls(opts, generator=G).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(opts)
    g = torch.Generator(device=DEV).manual_seed(1)
    clean = (0.3 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    z = torch.randn(B, s.G.z_dim, 16, device=DEV, generator=g)          # inference: reused
    if cls is SEGAN:
        losses = torch.zeros(4, device=DEV)
        step = lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)     # noqa: E731
    else:
        step = lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0)                   # noqa: E731
    return dict(s=s, step=step, noisy=noisy, z=z)


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
    arms = {k: make_arm(cls, over, norm, B) for k, (cls, over, norm) in ARMS.items()}
    for a in arms.values():
        for _ in range(args.warmup):            # eager steps, graph capture, first replays
            a["step"]()
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(args.rounds):                # alternate the arms: clock / thermal drift hits all of them
        for k, a in arms.items():
            step_ms[k].append(timed(a["step"], args.steps))
    inf_ms = {k: [] for k in ("segan_default", "segan_snorm_g")}
    for k in inf_ms:
        arms[k]["s"].G.eval()
    for _ in range(args.rounds):
        for k in inf_ms:
            with torch.no_grad():
                G, x, z = arms[k]["s"].G, arms[k]["noisy"], arms[k]["z"]
                inf_ms[k].append(timed(lambda: G(x, z=z), max(2, args.steps // 4)))
    res["gpu_after_timing"] = gpu_info()
    for k in arms:
        ms = min(step_ms[k])
        res[k] = dict(step_ms=ms, step_ms_rounds=step_ms[k], windows_per_s=B / (ms * 1e-3),
                      graph_replayed=any(v.graphs is not None or getattr(v, "graph", None) is not None
                                         for v in getattr(arms[k]["s"], "_step_graphs", {}).values()))
        if k in inf_ms:
            res[k].update(g_infer_ms=min(inf_ms[k]), g_infer_windows_per_s=B / (min(inf_ms[k]) * 1e-3))
    res["snorm_g_extra_step_ms"] = res["segan_snorm_g"]["step_ms"] - res["segan_default"]["step_ms"]
    res["max_memory_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "bench_gsnorm.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
