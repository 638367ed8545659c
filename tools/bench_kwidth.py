"""Cost of the kernel width on one GPU: the batch-300 SEGAN G+D train step (CUDA-graph replayed) and G-only eval
inference with every conv and transposed conv of width k (--gkwidth = --gdec_kwidth = --dkwidth = k) for
k in --widths, timed alternately in one process with CUDA events (best of --rounds rounds of --steps steps).  z is drawn
on the device (train steps) or passed in device-resident (inference): nothing on the host is timed.

Besides the times it reports the algorithmic FLOPs of one Generator forward -- 2 x rows x the valid (tap, phase) blocks
of every tap-GEMM layer at that width (engine.tap_ranges) plus the waveform-end layers' 2 x positions x Cin x k x Cout --
and the rate G inference achieves on them, so that one can see whether time tracks the block count.  Writes one JSON
file to --out (default profiles/, git-ignored) and prints it.

    python tools/bench_kwidth.py [--batch 300] [--steps 20] [--warmup 5] [--rounds 3] [--widths 11,15,21,31]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from segan_pytorch_b200 import engine as E              # noqa: E402
from segan_pytorch_b200.segan.models import SEGAN       # noqa: E402
from tests.util import load_opts, seed_all              # noqa: E402
from tools.bench_gtopo import gpu_info, timed           # noqa: E402

DEV = "cuda"


def g_forward_flops(opts, k, B, L=16384):
    """Algorithmic FLOPs of one Generator forward at width k (valid blocks only; bias / activations not counted)."""
    fm = list(opts.genc_fmaps)
    nl = len(fm)
    Lq = [L // 4 ** (l + 1) for l in range(nl)]
    f = 2 * B * Lq[0] * 1 * k * fm[0]                                  # enc0: Cin = 1
    for l in range(1, nl):
        cin, cout = fm[l - 1], fm[l]
        taps = E.tap_ranges("conv_fwd", cin, 4 * cin, cout, k)
        f += E._tap_flops(taps, -4, 4, 0, cout, B * Lq[l])
    dec_in = fm[-1] + (0 if opts.no_z else opts.z_dim)
    lin = Lq[-1]
    for l in range(nl - 1):
        cout = fm[nl - 2 - l]
        taps = E.tap_ranges("deconv_fwd", cout, dec_in, 4 * cout, k)
        f += E._tap_flops(taps, -4, 4, 0, 4 * cout, B * lin)
        lin *= 4
        dec_in = 2 * cout                                              # concat skip
    f += 2 * B * lin * dec_in * k                                      # last deconv: Cout = 1, lin = L / 4 inputs
    return f


def make_arm(k, B):
    opts = load_opts(batch_size=B, z_device="cuda", gkwidth=k, gdec_kwidth=k, dkwidth=k)
    seed_all(111)
    s = SEGAN(opts).to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(opts)
    g = torch.Generator(device=DEV).manual_seed(1)
    clean = (0.3 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    z = torch.randn(B, s.G.z_dim, 16, device=DEV, generator=g)
    losses = torch.zeros(4, device=DEV)
    step = lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)     # noqa: E731
    return dict(s=s, step=step, noisy=noisy, z=z, flops=g_forward_flops(opts, k, B))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=300)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--widths", default="11,15,21,31")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    B = args.batch
    widths = [int(w) for w in args.widths.split(",")]
    res = dict(gpu=gpu_info(), batch=B, steps_per_round=args.steps, rounds=args.rounds, grad_dtype=str(E.GT),
               time=time.strftime("%Y-%m-%d %H:%M:%S"))
    arms = {k: make_arm(k, B) for k in widths}
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
    for k, a in arms.items():
        ms, ims = min(step_ms[k]), min(inf_ms[k])
        res["k%d" % k] = dict(step_ms=ms, step_ms_rounds=step_ms[k], windows_per_s=B / (ms * 1e-3),
                              graph_replayed=any(v.graphs is not None or getattr(v, "graph", None) is not None
                                                 for v in getattr(a["s"], "_step_graphs", {}).values()),
                              g_infer_ms=ims, g_forward_gflop=a["flops"] / 1e9,
                              g_infer_tflops=a["flops"] / (ims * 1e-3) / 1e12)
    res["max_memory_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "bench_kwidth.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
