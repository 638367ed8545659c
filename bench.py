#!/usr/bin/env python
"""bench.py -- headline benchmark of BASELINE.json: 16384-sample windows/s of one full SEGAN+
G+D train step (batch 300 per GPU, synthetic clean/noisy pairs, RMSprop, LSGAN + L1).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python bench.py --gpus 1 --steps 20 --warmup 5 --dump-outputs DIR   # + what the last timed step computed
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...
    python bench.py --impl reference ...        # the reference's CPU path (oracle port), host cores

A "step" = the hot path over one batch: G fwd, D(real) fwd+bwd, D(fake) fwd+bwd, D RMSprop,
D(fake) fwd + dgrad through the updated D, L1, G bwd, G RMSprop (segan/models/model.py:283-321).
`value`  : device-timed (CUDA events), inputs already resident in HBM.
`e2e`    : same step through SEGAN.train's per-batch path with pinned HOST buffers: H2D copy of the
           batch and D2H read of the four losses inside the timed region.
`roofline`: the dominant kernel (wgmma forward-form tap-GEMM), algorithmic FLOPs / CUDA-event time.
`cpu_baseline`: the oracle (CPU restatement of the reference step) on this box's host cores.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
import zlib

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

ALG_GFLOP_PER_WINDOW = 35.8          # SURVEY.md 8(d): algorithmic FLOPs of one G+D step per window
ALG_GFLOP_F_PER_WINDOW = 25.2        # ... of which the forward-form tap-GEMM launches (fwd + data gradients)
WORKLOAD = "SEGAN+ G+D train step, batch 300/GPU, 16384-sample windows, synthetic pairs (BASELINE configs[1])"


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return dict(tflops=float(d.get("bf16_tflops_sustained", d.get("bf16_tflops", 1590.0))),
                    hbm=float(d.get("hbm_gbs", 6650.0)), src="measured (MEASURED_PEAKS.json, sustained)")
    # NVIDIA H100 SXM data sheet (700 W): dense FP16 tensor rate, HBM3 bandwidth -- not reached figures
    return dict(tflops=989.0, hbm=3350.0, src="H100 SXM data sheet (dense FP16, 700 W)")


def ncu_traffic(path=None):
    """DRAM bytes per launch of the dominant kernel (dram__bytes_read.sum + dram__bytes_write.sum, average over the
    launches of one train step) from a step-level ncu capture summarised by tools/ncu_step_summary.py (default:
    profiles/step_traffic.json, see tools/step_traffic.py), or None when there is none."""
    p = path or os.path.join(ROOT, "profiles", "step_traffic.json")
    try:
        with open(p) as f:
            ks = json.load(f)["kernels"]
        hits = [v for k, v in ks.items() if k.startswith("tapgemm_f_tc")]
        n = sum(v["launches"] for v in hits)
        return sum(v["dram_read_bytes"] + v["dram_write_bytes"] for v in hits) / n if n else None
    except Exception:
        return None


class ClockSampler(object):
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "20"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return dict(sm_mhz=None, sm_max_mhz=None, reasons=["nvidia-smi unavailable"])
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            pass
        sm, smax, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            parts = [p.strip() for p in ln.split(",")]
            if len(parts) < 6:
                continue
            try:
                sm.append(float(parts[0]))
                smax = float(parts[1])
            except ValueError:
                continue
            for n, v in zip(names, parts[2:6]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return dict(sm_mhz=(sm[len(sm) // 2] if sm else None), sm_max_mhz=smax, reasons=sorted(reasons),
                    samples=len(sm))


DUMP_SAMPLE = 4096     # entries kept per state tensor by --dump-outputs (fixed, seeded positions)


def dump_outputs(out_dir, s, losses):
    """What the timed path hands its caller after its last step: the step's four losses and the updated G / D
    state (reference-layout state_dict, as a checkpoint would hold it), the latter as a fixed, seeded sample of
    DUMP_SAMPLE entries per tensor, concatenated in state_dict order."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "losses.npy"), losses.detach().float().cpu().numpy())
    for name, mod in (("G", s.G), ("D", s.D)):
        parts = []
        for k, v in mod.state_dict().items():
            if not v.dtype.is_floating_point:
                continue
            flat = v.detach().float().reshape(-1).cpu().numpy()
            if flat.size > DUMP_SAMPLE:
                rs = np.random.RandomState(zlib.crc32(k.encode()))
                flat = flat[np.sort(rs.choice(flat.size, DUMP_SAMPLE, replace=False))]
            parts.append(flat)
        np.save(os.path.join(out_dir, "%s_state_sample.npy" % name), np.concatenate(parts).astype(np.float32))


def synth_batch(B, seed):
    """SURVEY.md 8(d): clean = 0.3*randn, noisy = clean + 0.1*randn, clamped to [-1, 1]."""
    g = torch.Generator().manual_seed(seed)
    clean = (0.3 * torch.randn(B, 16384, generator=g)).clamp_(-1, 1)
    noisy = (clean + 0.1 * torch.randn(B, 16384, generator=g)).clamp_(-1, 1)
    return clean, noisy


# ----------------------------------------------------------------------------------------------
# reference arm / cpu_baseline: the oracle (CPU restatement of model.py:283-321) on host cores
# ----------------------------------------------------------------------------------------------
def cpu_reference_steps(steps, warmup, B):
    import random
    from oracle import segan_oracle as O
    from tests.util import build_segan, cpu_state
    s = build_segan(batch_size=B)
    # "all the host threads it can use": the reference's CPU convs (slow_conv2d / im2col) stop scaling
    # well before 128 threads; probe a few thread counts on one G forward and keep the fastest
    ncpu = os.cpu_count() or 1
    best_nt, best_t = 1, None
    xs = torch.randn(2, 1, 16384)
    zs = torch.randn(2, 1024, 16)
    sd_probe = cpu_state(s.G)
    for nt in sorted(set(min(ncpu, n) for n in (8, 16, 32, 64, 128))):
        torch.set_num_threads(nt)
        with O.oracle_mode(), torch.no_grad():
            O.generator_forward(sd_probe, xs, zs)
            t0 = time.perf_counter()
            O.generator_forward(sd_probe, xs, zs)
            dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best_nt, best_t = nt, dt
    torch.set_num_threads(best_nt)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    clean, noisy = synth_batch(B, 111)
    clean, noisy = clean.unsqueeze(1), noisy.unsqueeze(1)
    random.seed(111)
    times = []
    for it in range(warmup + steps):
        z = torch.randn(B, 1024, 16)
        shifts3 = [O.draw_phase_shifts(5, 5) for _ in range(3)]
        t0 = time.perf_counter()
        O.segan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts3, l1_weight=100.0)
        if it >= warmup:
            times.append(time.perf_counter() - t0)
    total = sum(times)
    return B * len(times) / total, total / len(times), torch.get_num_threads()


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            for ln in f:
                if ln.lower().startswith("model name"):
                    return ln.split(":", 1)[1].strip()
    except Exception:
        pass
    import platform
    return platform.processor() or "unknown"


def cpu_baseline_section4(nthreads):
    """BASELINE.md section 4 on this box's host cores: (i) config 1 -- Generator forward on 1 x 16384, eval / no_grad,
    median of 20 after 3 warm-ups; (ii) the train-step analogue at B=16, 1 warm-up + 3 timed steps; both with oneDNN
    off (the correctness oracle, SURVEY.md F1) and as configured by default (what a reference user gets)."""
    import contextlib
    import random
    from oracle import segan_oracle as O
    from tests.util import build_segan, cpu_state
    torch.set_num_threads(nthreads)
    out = {"cpu_model": cpu_model(), "nproc": os.cpu_count(), "torch_threads": torch.get_num_threads(),
           "torch": torch.__version__, "impl": "oracle port of generator.py:180-230 / model.py:283-321"}
    s = build_segan(batch_size=16)
    sdG, sdD = cpu_state(s.G), cpu_state(s.D)
    g = torch.Generator().manual_seed(111)
    x1 = 0.3 * torch.randn(1, 1, 16384, generator=g)
    z1 = torch.randn(1, 1024, 16, generator=g)
    clean, noisy = synth_batch(16, 111)
    clean, noisy = clean.unsqueeze(1), noisy.unsqueeze(1)
    ref_y = None
    for tag, ctx in (("onednn_off", contextlib.nullcontext), ("onednn_default", O.onednn_as_configured)):
        with ctx():
            with torch.no_grad():
                ts = []
                for i in range(23):
                    t0 = time.perf_counter()
                    y = O.generator_forward(sdG, x1, z1)
                    if i >= 3:
                        ts.append(time.perf_counter() - t0)
            ts.sort()
            med = ts[len(ts) // 2]
            if ref_y is None:
                ref_y = y
            sG = {k: v.clone() for k, v in sdG.items()}
            sD = {k: v.clone() for k, v in sdD.items()}
            sqG = {k: torch.zeros_like(sG[k]) for k in O._trainable(sG)}
            sqD = {k: torch.zeros_like(sD[k]) for k in O._trainable(sD)}
            random.seed(111)
            tt = []
            for it in range(4):
                z = torch.randn(16, 1024, 16)
                sh = [O.draw_phase_shifts(5, 5) for _ in range(3)]
                t0 = time.perf_counter()
                O.segan_train_step(sG, sD, sqG, sqD, clean, noisy, z, sh, l1_weight=100.0)
                if it >= 1:
                    tt.append(time.perf_counter() - t0)
        out[tag] = {"g_forward_1x16384_ms_median20": med * 1e3, "g_forward_windows_per_s": 1.0 / med,
                    "g_forward_max_abs_vs_onednn_off": float((y - ref_y).abs().max()),
                    "train_step_b16_s": sum(tt) / len(tt), "train_step_windows_per_s": 16 * len(tt) / sum(tt)}
    return out


def run_reference_arm(args, emit=print):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    B = args.ref_batch
    wps, spstep, cores = cpu_reference_steps(args.steps, max(1, min(args.warmup, 2)), B)
    line = {
        "impl": "reference", "metric": "16384-sample windows/sec (G+D train step)", "value": wps,
        "unit": "windows/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": spstep * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD, "note": "reference CPU path = oracle port of segan/models/model.py:283-321 "
                   "(the Python reference is not installable on the GPU box); each step is a bounded sample of "
                   "%d windows of the batch-300 workload; windows/s is batch-normalised" % B},
        "cpu_baseline": {"value": wps, "unit": "windows/s", "cores": cores, "kind": "port",
                         "sample": "%d timed steps of a %d-window batch, oneDNN off (SURVEY.md F1)" % (args.steps, B)},
        "e2e": {"value": wps, "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    emit(json.dumps(line))


def gpu_extras(dev, B, s_plus):
    """BASELINE.json configs 4 and 5 as extra keys (rank 0, N=1; not the headline):
    config 4 -- WSEGAN (--wsegan --misalign_pair) train step at batch B, device-resident inputs;
    config 5 -- clean.py streaming inference over 10 000 windows incl. de-emphasis: (a) device-resident int16 PCM ->
    enhanced float windows (pre-emphasis, G, segmented de-emphasis), (b) SEGAN.clean_files over wav files on disk
    (decode, upload, G, de-emphasis, download, float32 wav writing: the host I/O included, wall clock)."""
    import random
    import shutil
    import tempfile
    import numpy as np
    from scipy.io import wavfile
    from segan_pytorch_b200 import _lib, engine as E
    from segan_pytorch_b200.engine import _p, _stream
    from segan_pytorch_b200.segan.models import WSEGAN
    from tests.util import load_opts, seed_all
    out = {}
    # ---- config 4
    opts = load_opts(batch_size=B, wsegan=True, misalign_pair=True, z_device="cuda")
    seed_all(111)
    w = WSEGAN(opts).to(dev)
    w.G.train()
    w.D.train()
    Gopt, Dopt = w.build_optimizers(opts)
    clean_h, noisy_h = synth_batch(B, 211)
    clean, noisy = clean_h.to(dev).unsqueeze(1), noisy_h.to(dev).unsqueeze(1)
    random.seed(211)
    losses = torch.zeros(4, device=dev)
    names = ["utt_%d.wav" % i for i in range(B)]
    for _ in range(4):
        w.train_step(clean, noisy, Gopt, Dopt, 0.0, uttname=names, losses=losses)
    torch.cuda.synchronize()
    n4 = 10
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n4):
        w.train_step(clean, noisy, Gopt, Dopt, 0.0, uttname=names, losses=losses)
    e1.record()
    torch.cuda.synchronize()
    ms4 = e0.elapsed_time(e1) / n4
    out["config4_wsegan_step"] = {
        "value": B / (ms4 * 1e-3), "unit": "windows/s", "ms_per_step": ms4, "batch": B, "steps": n4,
        "what": "WSEGAN --misalign_pair step (D on real / fake / misaligned pairs, RMSprop, G loss = adversarial + "
                "STFT log-power L1 as a tensor-core GEMM), device-resident synthetic pairs, %s"
                % ("step replayed from one CUDA graph" if any(getattr(v, "graph", None) is not None
                                                              for v in getattr(w, "_step_graphs", {}).values())
                   else "eager launches"),
        "last_losses": losses.tolist()}
    del w, Gopt, Dopt
    torch.cuda.empty_cache()
    # ---- config 5
    N, n_files, per_file = 16384, 40, 250                       # 40 files x 250 windows = 10 000 windows
    rng = np.random.RandomState(5)
    s_plus.G.eval()
    total = n_files * per_file
    pcm = torch.from_numpy(rng.randint(-9000, 9000, size=(per_file * N,)).astype(np.int16))
    # (a) device-resident: one file's int16 PCM on the device, processed n_files times in batches of B windows
    pcm_d = pcm.view(per_file, N).to(dev)
    prev = torch.full((per_file,), 0x7fffffff, dtype=torch.int32)
    prev[1:] = pcm.view(per_file, N)[:-1, -1].to(torch.int32)
    prev_d = prev.to(dev)
    valid_d = torch.full((per_file,), N, dtype=torch.int32, device=dev)
    seg = torch.tensor([[0, per_file * N]], dtype=torch.int64, device=dev)
    x = torch.empty(per_file, 1, N, device=dev)
    y = torch.empty(per_file, N, device=dev)
    o = torch.empty_like(y)
    zb = torch.randn(per_file, 1024, 16, device=dev)
    coef = float(s_plus.preemph)

    def one_file():
        _lib.call("sg_pcm16_to_wave", _p(pcm_d), _p(prev_d), per_file, N, coef, _p(x), _p(valid_d), _stream())
        with torch.no_grad():
            for b0 in range(0, per_file, B):
                b1 = min(per_file, b0 + B)
                y[b0:b1] = s_plus.G(x[b0:b1], z=zb[b0:b1]).view(b1 - b0, N)
        _lib.call("sg_deemphasis_segments", _p(y), _p(seg), 1, coef, _p(o), _stream())
    for _ in range(2):
        one_file()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_files):
        one_file()
    e1.record()
    torch.cuda.synchronize()
    ms5a = e0.elapsed_time(e1)
    # (b) through wav files on disk
    # wavs on tmpfs when the box has one: the figure is the software path (decode, staging, G, encode), not the disk
    shm = "/dev/shm" if os.path.isdir("/dev/shm") and os.access("/dev/shm", os.W_OK) else None
    tmp = tempfile.mkdtemp(prefix="segan_b200_bench_", dir=shm)
    try:
        src, dst = os.path.join(tmp, "in"), os.path.join(tmp, "out")
        os.makedirs(src)
        paths = []
        for i in range(n_files):
            pth = os.path.join(src, "f%03d.wav" % i)
            wavfile.write(pth, 16000, np.roll(pcm.numpy(), 977 * i))
            paths.append(pth)
        s_plus.clean_files(paths[:4], dst, batch=B)                # warm-up (allocator, pinned pools)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        nwin = s_plus.clean_files(paths, dst, batch=B)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    s_plus.G.train()
    out["config5_clean_streaming"] = {
        "windows": total, "unit": "windows/s",
        "device_resident": {"value": total / (ms5a * 1e-3), "ms_total": ms5a,
                            "what": "int16 PCM in HBM -> float + pre-emphasis -> G (fp16 operands, batches of %d) -> "
                                    "segmented de-emphasis, CUDA events" % B},
        "with_host_io": {"value": nwin / dt, "s_total": dt, "files": n_files,
                         "what": "SEGAN.clean_files: %d int16 wav files of %d windows under %s -> float32 wavs; reader "
                                 "thread (decode), copy streams, 4 writer threads; wall clock"
                                 % (n_files, per_file, "/dev/shm (tmpfs)" if shm else "the local temp dir")}}
    return out


# ----------------------------------------------------------------------------------------------
# our arm
# ----------------------------------------------------------------------------------------------
def _claim_stdout():
    """A caller reads ONE JSON line from stdout: native libraries (NCCL prints its version banner
    there) are pointed at stderr for the whole run; the returned writer emits on the real stdout."""
    sys.stdout.flush()
    real = os.dup(1)
    os.dup2(2, 1)

    def emit(text):
        sys.stdout.flush()
        os.write(real, (text + "\n").encode())
    return emit


def _guard(fn, *a):
    try:
        return fn(*a)
    except Exception as e:
        return {"error": "%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")}


def _leave(world):
    """End of a data-parallel run: the step's CUDA graph holds captured NCCL kernels, and tearing the process group
    down under it was seen to block (2 GPUs: the JSON line was out, destroy_process_group() never returned).  Every
    rank has passed its last collective when it gets here, all device work is drained, so the process simply ends."""
    if world > 1:
        import torch.distributed as dist
        dist.barrier()                       # rank 0 is last (it prints): nobody leaves while a peer still computes
        torch.cuda.synchronize()
        time.sleep(0.2)
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)


def main():
    t_start = time.time()
    emit = _claim_stdout()
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--batch", type=int, default=300, help="windows per GPU (BASELINE: 300)")
    ap.add_argument("--ref-batch", type=int, default=8, help="bounded CPU sample size of the reference arm")
    ap.add_argument("--cpu-baseline-steps", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip BASELINE configs 4 / 5 (extra keys)")
    ap.add_argument("--backend", default=None, help="tcgen05 (default: the wgmma tensor-core kernels) | ffma")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed as DIR/<name>.npy")
    args = ap.parse_args()
    if args.warmup < 3 and args.impl == "b200":
        args.warmup = 3
    if args.impl == "reference":
        return run_reference_arm(args, emit)

    if args.backend:
        os.environ["SEGAN_B200_BACKEND"] = args.backend
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        # NCCL_DEBUG is left as the launcher set it: fd 1 already points at stderr (_claim_stdout), so NCCL's INFO
        # lines (communicator / rank evidence) cannot pollute the one JSON line
        dist.init_process_group("nccl", device_id=dev)
    from segan_pytorch_b200 import _lib, engine as E
    from segan_pytorch_b200.hostbind import bind_host_to_gpu
    from tests.util import build_segan, load_opts
    numa_cpus = bind_host_to_gpu(dev)          # before any pinned staging buffer is allocated
    if not _lib.device_ok():
        raise SystemExit("bench.py needs an H100 (sm_90) GPU and libsegan_b200.so (no fallback path)")
    B = args.batch
    opts = load_opts(batch_size=B, z_device="cuda")
    s = build_segan(seed=111, batch_size=B, z_device="cuda").to(dev)      # identical init on every rank
    s.G.train()
    s.D.train()
    Gopt, Dopt = s.build_optimizers(opts)
    clean_h, noisy_h = synth_batch(B, 111 + rank)                          # per-rank data shard
    clean_h, noisy_h = clean_h.pin_memory(), noisy_h.pin_memory()
    clean = clean_h.to(dev).unsqueeze(1)
    noisy = noisy_h.to(dev).unsqueeze(1)
    import random
    random.seed(111 + rank)
    torch.manual_seed(111 + rank)
    losses = torch.zeros(4, device=dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    trace = os.environ.get("SEGAN_B200_BENCH_TRACE", "0") not in ("0", "")

    def mark(msg):
        if trace:
            sys.stderr.write("[bench rank %d +%.1fs] %s\n" % (rank, time.time() - t_start, msg))
            sys.stderr.flush()

    # ---- warm-up
    mark("models built, process group up")
    for i in range(args.warmup):
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
        if trace:
            torch.cuda.synchronize()
            mark("warm-up step %d done" % i)
    barrier()
    mark("warm-up barrier passed")
    # ---- timed region 1: device-resident inputs (the headline `value`)
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    launches0 = _lib.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for _ in range(args.steps):
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    mark("timed region done: %.3f ms/step" % (ms / args.steps))
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, s, losses)
    launches = _lib.launch_count - launches0
    ngraphs = [len(v.graphs) for v in getattr(s, "_step_graphs", {}).values() if getattr(v, "graphs", None) is not None]
    clocks = sampler.stop() if rank == 0 else None
    # ---- timed region 1b: the same steps again with a CUDA-event pair around every C-ABI call
    #      (live per-kernel times for the roofline object; the ~600 extra event records per step
    #      are why this is not the region `value` is taken from)
    #      This region runs the SERIAL schedule (engine.OVERLAP off: everything on one stream) so that
    #      the per-kernel times are exclusive; the headline region above overlaps the HBM-bound glue
    #      kernels with the tap-GEMMs on side streams.
    overlap_on, graphs_on = E.OVERLAP, E.GRAPHS
    E.OVERLAP = False
    E.GRAPHS = False
    for _ in range(2):
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    s0.record()
    for _ in range(args.steps):
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
    s1.record()
    barrier()
    ms_serial = s0.elapsed_time(s1)
    mark("serial region done")
    E.PROFILE = []
    _lib.call_profile = []
    p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    p0.record()
    for _ in range(args.steps):
        s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
    p1.record()
    barrier()
    ms_prof = p0.elapsed_time(p1)
    mark("profiled region done")
    prof = E.PROFILE
    E.PROFILE = None
    calls = _lib.call_profile
    _lib.call_profile = None
    E.OVERLAP, E.GRAPHS = overlap_on, graphs_on
    # ---- timed region 2: end to end through the public data path with HOST buffers: every step's batch
    #      is copied from pinned host memory by segan.datasets.DevicePrefetcher (the loader wrapper
    #      SEGAN.train uses: batch n+1 is staged on a copy stream while batch n trains) and the step's
    #      four losses are read back to the host, all inside the timed region
    from segan_pytorch_b200.segan.datasets import DevicePrefetcher

    def to_pcm(x):      # inverse of normalize_wave_minmax (se_dataset.py:108-109): what a wav file holds
        return torch.round((x - 1.0) * (65535.0 / 2.0) + 32767.0).clamp_(-32768, 32767).to(torch.int16).pin_memory()
    clean_p, noisy_p = to_pcm(clean_h), to_pcm(noisy_h)

    def host_batches(n):
        for _ in range(n):
            yield [None, clean_p, noisy_p, None]                             # pinned (B, 16384) int16 PCM pair
    # preemph=0: the synthetic pairs are defined in the network-input domain, so the device side only
    # de-quantises them (the step sees the headline region's signals to within 1.5e-5)
    pre = DevicePrefetcher(host_batches(args.steps), dev, preemph=0.0)
    barrier()
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    # the four losses of EVERY step are read back into pinned host memory by an asynchronous copy ordered after the
    # step (SEGAN.train reads them every log_freq steps, model.py:336-348); the host is synchronised once, at the end
    host_losses = torch.zeros(args.steps, 4).pin_memory()
    for i, (_, cbuf, nbuf, _) in enumerate(pre):
        ls = s.train_step(cbuf, nbuf, Gopt, Dopt, 100.0, losses=losses)
        host_losses[i].copy_(ls, non_blocking=True)                        # D2H read of the step's losses
    f1.record()
    barrier()
    ms_e2e = f0.elapsed_time(f1)
    mark("e2e region done")
    host_loss = host_losses[-1].tolist()
    assert all(abs(v) > 0 for v in host_losses[:, 3].tolist()), "a step's losses never reached the host"
    h2d_per_step = pre.h2d_bytes // args.steps
    cbuf = torch.empty(B, 1, 16384, device=dev)
    nbuf = torch.empty(B, 1, 16384, device=dev)
    # ---- BASELINE config 5 (secondary metric): G-only streaming inference, fp16, batches of B windows,
    #      host->device copy of every batch and device->host copy of the enhanced windows included
    s.G.eval()
    n_inf = 8
    zinf = torch.randn(B, 1024, 16, device=dev)
    with torch.no_grad():
        for _ in range(2):
            s.G(cbuf, z=zinf)
    for _ in s.generate_stream([noisy_h.unsqueeze(1)] * 2, z=zinf):       # warm the pinned output buffers
        pass
    barrier()
    g0, g1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g0.record()
    n_out = 0
    for out_h in s.generate_stream((noisy_h.unsqueeze(1) for _ in range(n_inf)), z=zinf):
        n_out += out_h.shape[0]                                            # enhanced windows, in pinned host memory
    g1.record()
    barrier()
    assert n_out == B * n_inf
    ms_inf = g0.elapsed_time(g1)
    with torch.no_grad():                  # the same batches without the host copies (device-resident)
        h0, h1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        h0.record()
        for _ in range(n_inf):
            y = s.G(nbuf, z=zinf)
        h1.record()
        barrier()
    ms_inf_dev = h0.elapsed_time(h1)
    mark("inference regions done")
    s.G.train()
    extras = None
    if world == 1 and not args.no_extras:
        try:
            extras = gpu_extras(dev, B, s)
        except Exception as e:                       # secondary figures must never cost the headline line
            extras = {"error": "%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")}
            torch.cuda.synchronize()
            s.G.train()
    t = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)                           # max over ranks
    ms, ms_e2e = float(t[0]), float(t[1])
    if rank != 0:
        _leave(world)
        return
    total_windows = B * world * args.steps
    value = total_windows / (ms * 1e-3)
    e2e_value = total_windows / (ms_e2e * 1e-3)
    # ---- roofline of the dominant kernel from the live CUDA-event profile
    peaks = measured_peaks()
    agg = {}
    for kind, s_ev, e_ev, flops in prof:
        a = agg.setdefault(kind, [0.0, 0.0, 0])
        a[0] += s_ev.elapsed_time(e_ev) * 1e-3
        a[1] += flops
        a[2] += 1
    if os.environ.get("SEGAN_B200_DUMP_CALLS"):
        per = len(prof) // args.steps
        with open(os.environ["SEGAN_B200_DUMP_CALLS"], "w") as f:
            for i, (kind, s_ev, e_ev, flops) in enumerate(prof[-per:]):
                t = s_ev.elapsed_time(e_ev)
                f.write("%3d %-10s %8.3f ms %9.2f GFLOP %7.1f TFLOP/s\n" % (i, kind, t, flops / 1e9, flops / t / 1e9))
    step_s = ms * 1e-3 / args.steps
    dom = max(agg.items(), key=lambda kv: kv[1][0])[0] if agg else None
    roof = None
    kern = {}
    for kind, (sec, fl, n) in agg.items():
        kern[kind] = {"launches_per_step": n / args.steps, "ms_per_step": sec * 1e3 / args.steps,
                      "share_of_step": sec / (ms_prof * 1e-3), "tflops": fl / sec / 1e12 if sec > 0 else None}
    by_call = {}
    for name, s_ev, e_ev, _ in calls:
        c = by_call.setdefault(name, [0.0, 0])
        c[0] += s_ev.elapsed_time(e_ev)
        c[1] += 1
    call_ms = {k: {"ms_per_step": round(v[0] / args.steps, 4), "calls_per_step": v[1] / args.steps}
               for k, v in sorted(by_call.items(), key=lambda kv: -kv[1][0])}
    if dom:
        sec, fl, n = agg[dom]
        ach_exec = fl / sec / 1e12
        # ALGORITHMIC FLOPs of the dominant kernel's launches (SURVEY.md App. A): the executed count above also holds the
        # data-gradient launches' halo rows (+12 % on the short layers) and the 64-wide padding of the waveform-end
        # single-tap GEMMs (K = 31 / 62 real): 26.2 vs 25.2 GFLOP per window for form F
        alg_fl = ALG_GFLOP_F_PER_WINDOW * 1e9 * B * args.steps if dom == "tapgemm_f" else fl
        alg_fl = min(alg_fl, fl)
        ach = alg_fl / sec / 1e12
        roof = {"kernel": dom + "_tc (wgmma tap-GEMM)", "bound": "tensor", "achieved": ach,
                "peak": peaks["tflops"], "unit": "TFLOP/s", "frac": ach / peaks["tflops"], "traffic": ncu_traffic(),
                "peak_source": peaks["src"], "avg_launch_ms": sec * 1e3 / n,
                "alg_flops_per_launch": alg_fl / n, "executed_flops_per_launch": fl / n,
                "achieved_executed": ach_exec, "kernels": kern, "abi_calls": call_ms,
                "profiled_ms_per_step": ms_prof / args.steps,
                "serial_ms_per_step": ms_serial / args.steps,
                "whole_step_tflops": ALG_GFLOP_PER_WINDOW * 1e9 * B / step_s / 1e12}
    cpu = None
    if not args.no_cpu_baseline and world == 1:        # reported on rank 0 at N=1 only
        wps, spstep, cores = cpu_reference_steps(args.cpu_baseline_steps, 1, args.ref_batch)
        cpu = {"value": wps, "unit": "windows/s", "cores": cores, "kind": "port",
               "sample": "%d timed steps of a %d-window batch of the same workload (oracle, oneDNN off)"
                         % (args.cpu_baseline_steps, args.ref_batch),
               "baseline_md_section4": _guard(cpu_baseline_section4, cores)}
    line = {
        "metric": "16384-sample windows/sec (G+D train step)", "value": value, "unit": "windows/s",
        "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f16 operands / f32 accumulate (%s gradient tensors%s)" % (("f16", ", loss scale %g" % E.LOSS_SCALE) if E.GS == 1 else ("bf16", "")), "data": "synthetic",
        "config": {"workload": WORKLOAD, "global_batch": B * world, "window": 16384,
                   "parallelism": "dp%d" % world, "optimizer": "rmsprop lr 5e-5", "l1_weight": 100,
                   "z": "device RNG (opts.z_device='cuda')", "backend": args.backend or "tcgen05",
                   "schedule": (("side streams (wgrad chains, D(real) pass next to G forward + D(fake) pass)"
                                 if overlap_on else "single stream") +
                                (", step replayed from %s CUDA graph(s)%s" % (
                                    "/".join(str(n) for n in ngraphs) or "?",
                                    " (NCCL all-reduce chunks captured inside)" if world > 1 and ngraphs == [1] else "")
                                 if graphs_on else ", eager launches")),
                   "l2": "per-step working set (packed weights 0.4 GB + activations > 2 GB) exceeds the 50 MB L2"},
        "clocks": clocks,
        "e2e": {"value": e2e_value, "unit": "windows/s", "ms_per_step": ms_e2e / args.steps,
                "h2d_bytes_per_step": h2d_per_step, "d2h_bytes_per_step": 16, "last_losses": host_loss,
                "path": "DevicePrefetcher (pinned int16 PCM host batch -> copy stream one step ahead -> sg_pcm16_to_wave "
                        "on the device) + train_step + async D2H copy of the step's four losses into pinned memory "
                        "(host synchronised once, after the last step)",
                "host_cpus_bound_to_gpu_numa": sorted(numa_cpus)[:4] + ["..."] if numa_cpus else None},
        "g_only_inference": {"value": B * n_inf / (ms_inf * 1e-3), "unit": "windows/s per GPU",
                             "what": "SEGAN.generate_stream: G forward (clean.py path), fp16 operands, %d batches of %d "
                                     "windows from pinned host memory back to pinned host memory; H2D of batch n+1, G "
                                     "on batch n and D2H of batch n-1 overlap on three streams" % (n_inf, B),
                             "ms_per_batch": ms_inf / n_inf, "ms_per_batch_device_resident": ms_inf_dev / n_inf},
        "gpu_launches": launches,
        "roofline": roof,
        "cpu_baseline": cpu,
        "extra_configs": extras,
    }
    emit(json.dumps(line))
    _leave(world)


if __name__ == "__main__":
    main()
