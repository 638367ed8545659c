"""One eager SEGAN+ train step (batch 300) inside a cudaProfilerStart/Stop range, for a step-level ncu pass:

    ncu --profile-from-start off --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum \\
        --clock-control none --csv --log-file profiles/step_traffic.csv python tools/step_traffic.py
    python tools/ncu_step_summary.py profiles/step_traffic.csv profiles/step_traffic

(the graphs are off: every kernel of the step is its own launch; times under ncu are serialised and cold-cache: the
kernels' SHARES and their DRAM bytes are what this capture is for, not the absolute times)."""
import os
import random
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["SEGAN_B200_GRAPH"] = "0"
from segan_pytorch_b200 import engine as E                # noqa: E402
from tests.util import build_segan, load_opts             # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 300
dev = torch.device("cuda", 0)
E.GRAPHS = False
E.OVERLAP = False                                         # one stream: the launch list reads in program order
opts = load_opts(batch_size=B, z_device="cuda")
s = build_segan(seed=111, batch_size=B, z_device="cuda").to(dev)
s.G.train()
s.D.train()
Gopt, Dopt = s.build_optimizers(opts)
g = torch.Generator().manual_seed(111)
clean = (0.3 * torch.randn(B, 1, 16384, generator=g)).clamp_(-1, 1).to(dev)
noisy = (clean.cpu() + 0.1 * torch.randn(B, 1, 16384, generator=g)).clamp_(-1, 1).to(dev)
random.seed(111)
losses = torch.zeros(4, device=dev)
for _ in range(3):
    s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
torch.cuda.synchronize()
torch.cuda.profiler.start()
s.train_step(clean, noisy, Gopt, Dopt, 100.0, losses=losses)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("losses", losses.tolist())
