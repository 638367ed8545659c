"""Per-call timeline of one SEGAN+ train step under the side-stream schedule: every C-ABI call with its
stream, start and end (CUDA events, microseconds from the start of the step), plus a utilisation
summary (time with >= 1 tap-GEMM in flight, time with only HBM-bound kernels in flight, idle time).

    python tools/timeline.py [--batch 300] > profiles/timeline.txt
"""
import argparse
import sys

import torch

sys.path.insert(0, ".")
from segan_pytorch_b200 import _lib, engine as E          # noqa: E402
from tests.util import build_segan, load_opts             # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=300)
ap.add_argument("--serial", action="store_true")
args = ap.parse_args()
B = args.batch
dev = torch.device("cuda", 0)
if args.serial:
    E.OVERLAP = False
opts = load_opts(batch_size=B, z_device="cuda")
s = build_segan(seed=111, batch_size=B, z_device="cuda").to(dev)
s.G.train()
s.D.train()
Gopt, Dopt = s.build_optimizers(opts)
g = torch.Generator().manual_seed(1)
clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp_(-1, 1).to(dev)
noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp_(-1, 1).to(dev)
losses = torch.zeros(4, device=dev)
for _ in range(4):
    s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
torch.cuda.synchronize()
_lib.call_profile = []
t0 = torch.cuda.Event(enable_timing=True)
t1 = torch.cuda.Event(enable_timing=True)
t0.record()
s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
t1.record()
torch.cuda.synchronize()
calls = _lib.call_profile
_lib.call_profile = None
streams = {}
rows = []
for name, a, b, st in calls:
    sid = streams.setdefault(st, len(streams))
    rows.append((t0.elapsed_time(a) * 1e3, t0.elapsed_time(b) * 1e3, sid, name))
rows.sort()
print("# step %.1f us, %d calls, %d streams (0 = caller's stream)" % (t0.elapsed_time(t1) * 1e3, len(rows), len(streams)))
for a, b, sid, name in rows:
    print("%9.1f %9.1f %7.1f  s%d %s%s" % (a, b, b - a, sid, "    " * sid, name))
# utilisation summary on a 1 us grid
end = int(t0.elapsed_time(t1) * 1e3) + 1
gemm = [0] * (end + 1)
other = [0] * (end + 1)
for a, b, sid, name in rows:
    tgt = gemm if name.startswith("sg_tapgemm") else other
    for t in range(max(0, int(a)), min(end, int(b) + 1)):
        tgt[t] += 1
both = sum(1 for t in range(end) if gemm[t] and other[t])
only_g = sum(1 for t in range(end) if gemm[t] and not other[t])
only_o = sum(1 for t in range(end) if other[t] and not gemm[t])
idle = sum(1 for t in range(end) if not gemm[t] and not other[t])
multi_g = sum(1 for t in range(end) if gemm[t] > 1)
print("# us with GEMM+other %d, GEMM only %d (of which >1 GEMM queued %d), other only %d, no call in flight %d"
      % (both, only_g, multi_g, only_o, idle))
