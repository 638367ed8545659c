"""Cost of skip_type='conv' on one GPU: the batch-300 G+D train step (CUDA-graph replayed) and G-only inference for
skip_type 'alpha' and 'conv', timed alternately in one process with CUDA events, and the skip convs' own launches
per layer (forward, data gradient, weight gradient + fold) with algorithmic TFLOP/s (2 B Lq C^2 K per launch).
z is drawn on the device (train steps) or passed in device-resident (inference): nothing on the host is timed.
Writes one JSON file to --out (default profiles/, git-ignored) and prints it.

    python tools/bench_conv_skip.py [--batch 300] [--steps 20] [--warmup 5] [--rounds 3] [--out profiles]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from segan_pytorch_b200 import _lib, engine as E        # noqa: E402
from segan_pytorch_b200._lib import SG_F16              # noqa: E402
from tests.util import build_segan, load_opts           # noqa: E402

DEV = "cuda"


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


def make_arm(skip_type, B):
    """One SEGAN at batch B, set up as bench.py sets up its step: z drawn on the device (z_device='cuda'), so the
    timed region holds no host work."""
    s = build_segan(batch_size=B, skip_type=skip_type, z_device="cuda").to(DEV)
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(load_opts(batch_size=B, skip_type=skip_type, z_device="cuda"))
    g = torch.Generator(device=DEV).manual_seed(1)
    clean = (0.3 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 1, 16384, device=DEV, generator=g)).clamp(-1, 1)
    z = torch.randn(B, 1024, 16, device=DEV, generator=g)        # inference: one device-resident z, reused
    losses = torch.zeros(4, device=DEV)
    return dict(s=s, step=lambda: s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses), noisy=noisy, z=z)


def skip_layer_launches(B, K, reps):
    """The skip convs' launches at the batch-B shapes of the four skip levels, in the current gradient format
    (engine.GT: the weight gradient's activation operand is converted to it, as the engine's bf16 twins are)."""
    out = []
    fm, L = [64, 128, 256, 512], 16384
    for l, c in enumerate(fm):
        lq = L // 4 ** (l + 1)
        rows = lq // 4
        D = (K // 2 + 3) // 4
        g = torch.Generator(device=DEV).manual_seed(l)
        w = 0.05 * torch.randn(c, c, K, device=DEV, generator=g)
        a = torch.randn(B, lq, c, device=DEV, generator=g).half()
        gs = torch.randn(B, lq, c, device=DEV, generator=g).to(E.GT)
        a_w = a if E.GT == torch.float16 else a.to(E.GT)       # wgmma needs one 16-bit type on both operands
        wf = torch.empty(2 * D + 1, 4 * c, 4 * c, dtype=torch.float16, device=DEV)
        wd = torch.empty(2 * D + 1, 4 * c, 4 * c, dtype=E.GT, device=DEV)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        d_lo, d_hi, tap0, taps, taps_dg = E.skipconv_geometry(c, K)
        o = torch.empty(B, lq, c, dtype=torch.float16, device=DEV)
        ga = torch.empty(B, lq, c, dtype=E.GT, device=DEV)
        dwq = torch.zeros((2 * D + 1) * 16 * c * c, device=DEV)
        dw = torch.zeros(c, c, K, device=DEV)
        ks = E.wgrad_ksplit(B * rows, 0, taps, 4 * c, 4 * c, d_lo, d_hi)
        emit = lambda: _lib.call("sg_skipconv_emit", C.c_void_p(w.data_ptr()), c, K, C.c_void_p(wf.data_ptr()),
                                 C.c_void_p(wd.data_ptr()), SG_F16, E.GS, st)
        fwd = lambda: E.run_f(a, None, rows, 0, SG_F16, wf, SG_F16, 4 * c, 4 * c, taps, o, SG_F16, rows, 0, 0, rows, B,
                              d_lo=d_lo, d_hi=d_hi, w_tap0=tap0)
        dgrad = lambda: E.run_f(gs, None, rows, 0, E.GS, wd, E.GS, 4 * c, 4 * c, taps_dg, ga, E.GS, rows, 0, 0, rows, B,
                                d_lo=d_lo, d_hi=d_hi, w_tap0=tap0)
        wgrad = lambda: E.run_w(gs, rows, E.GS, a_w, None, rows, 0, E.GS, 4 * c, 4 * c, taps, dwq, B, d_lo=d_lo,
                                d_hi=d_hi, dw_tap0=tap0, ksplit=ks)
        fold = lambda: _lib.call("sg_skipconv_wgrad_fold", C.c_void_p(dwq.data_ptr()), c, K, C.c_void_p(dw.data_ptr()), st)
        for f in (emit, fwd, dgrad, wgrad, fold):
            f()
        flops = 2.0 * B * lq * c * c * K
        ent = dict(level=l, C=c, Lq=lq, K=K, algorithmic_gflop=flops / 1e9, wgrad_ksplit=ks)
        for name, f in (("emit", emit), ("fwd", fwd), ("dgrad", dgrad), ("wgrad", wgrad), ("fold", fold)):
            ms = timed(f, reps)
            ent[name + "_ms"] = ms
            if name in ("fwd", "dgrad", "wgrad"):
                ent[name + "_tflops"] = flops / (ms * 1e-3) / 1e12
        out.append(ent)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=300)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip_kwidth", type=int, default=11)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    B = args.batch
    res = dict(gpu=gpu_info(), batch=B, steps_per_round=args.steps, rounds=args.rounds, skip_kwidth=args.skip_kwidth,
               grad_dtype=str(E.GT), time=time.strftime("%Y-%m-%d %H:%M:%S"))
    arms = {k: make_arm(k, B) for k in ("alpha", "conv")}
    for a in arms.values():
        for _ in range(args.warmup):            # eager steps, graph capture, first replays
            a["step"]()
    torch.cuda.synchronize()
    step_ms = {k: [] for k in arms}
    for _ in range(args.rounds):                # alternate the two arms: clock / thermal drift hits both
        for k, a in arms.items():
            step_ms[k].append(timed(a["step"], args.steps))
    inf_ms = {k: [] for k in arms}
    for k, a in arms.items():
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
    res["conv_minus_alpha_step_ms"] = res["conv"]["step_ms"] - res["alpha"]["step_ms"]
    res["max_memory_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    del arms
    torch.cuda.empty_cache()
    res["skip_layers"] = skip_layer_launches(B, args.skip_kwidth, 20)
    res["skip_layers_total_ms"] = {n: sum(e[n + "_ms"] for e in res["skip_layers"])
                                   for n in ("emit", "fwd", "dgrad", "wgrad", "fold")}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "bench_conv_skip.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
