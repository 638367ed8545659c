"""CPU-only checks: the C-ABI library loads and exports every symbol the header declares, the
ctypes structs mirror the C structs, and the host-side logic of the drop-in (state-dict keys,
checkpoint format, RNG order, tap tables, flat buckets) behaves like the reference."""
import ctypes
import json
import os
import random
import re
import subprocess
import tempfile

import pytest
import torch

from tests.util import build_segan, load_opts, sd_sha, golden

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, "include", "segan_b200.h")


@pytest.fixture(scope="module")
def lib():
    from segan_pytorch_b200 import build, _lib
    build.build()
    return _lib.load()


def test_header_symbols_exported(lib):
    src = open(HEADER).read()
    names = sorted(set(re.findall(r"\b(sg_[a-z0-9_]+)\s*\(", src)))
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), "header declares %s but the library does not export it" % n
    from segan_pytorch_b200 import _lib
    assert sorted(set(_lib.EXPORTS)) == names
    assert lib.sg_abi_version() == 3


def test_ctypes_structs_match_c_layout(lib):
    from segan_pytorch_b200._lib import TapGemmF, TapGemmW
    code = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "segan_b200.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu %zu\n", sizeof(sg_tapgemm_f), offsetof(sg_tapgemm_f, out), offsetof(sg_tapgemm_f, backend),
             sizeof(sg_tapgemm_w), offsetof(sg_tapgemm_w, dw), offsetof(sg_tapgemm_w, backend));
      return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(REPO, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")]).decode().split()
    got = [ctypes.sizeof(TapGemmF), TapGemmF.out.offset, TapGemmF.backend.offset,
           ctypes.sizeof(TapGemmW), TapGemmW.dw.offset, TapGemmW.backend.offset]
    assert [int(v) for v in out] == got


def test_state_dict_keys_and_seed_parity():
    s = build_segan()
    g = golden("g_forward_cfg1.npz")
    assert sd_sha(s.G.state_dict()) == str(g["sha_G"])
    keys = list(s.G.state_dict().keys())
    assert keys[:3] == ["enc_blocks.0.conv.weight", "enc_blocks.0.conv.bias", "enc_blocks.0.act.weight"]
    assert "alpha_3.skip_k" in keys and "dec_blocks.4.deconv.bias" in keys and "dec_blocks.4.act.weight" not in keys
    dk = list(s.D.state_dict().keys())
    assert "enc_blocks.0.norm.running_var" in dk and "fc.4.bias" in dk
    assert s.G.get_n_params() == 64770561 and s.D.get_n_params() == 25825793
    nb = build_segan(bias=False)
    assert "enc_blocks.0.conv.bias" not in nb.G.state_dict() and "dec_blocks.0.deconv.bias" in nb.G.state_dict()


def test_missing_reg_loss_tolerated():
    o = load_opts()
    del o.reg_loss
    from segan_pytorch_b200.segan.models import SEGAN
    assert SEGAN(o).reg_loss_name == "l1_loss"        # SURVEY.md F5


def test_phase_shift_draw_order_matches_oracle():
    from oracle import segan_oracle as O
    from segan_pytorch_b200.segan.models.discriminator import draw_phase_shifts
    random.seed(99)
    a = [draw_phase_shifts(5, 5) for _ in range(3)]
    random.seed(99)
    b = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    assert a == b


def test_flat_buckets_and_checkpoint_roundtrip(tmp_path):
    s = build_segan()
    eng = s.G.engine.bind()
    # packed masters (36 of 31 tap slots) + small parameters in one bucket
    assert sum(l.numel for l in eng.layers) == 75202560          # 64 757 760 packed weights x 36 / 31
    assert 75202560 + (64770561 - 64757760) <= eng.flat.numel() <= 75202560 + (64770561 - 64757760) + 4 * 40
    w = dict(s.G.named_parameters())["enc_blocks.1.conv.weight"]
    assert w.data_ptr() == eng.pview("enc_blocks.1.conv.weight").data_ptr()
    sha = sd_sha(s.G.state_dict())
    s.G.save(str(tmp_path), 7)
    files = os.listdir(str(tmp_path))
    assert "weights_Generator-Generator-7.ckpt" in files and "Generator-checkpoints" in files
    st = torch.load(os.path.join(str(tmp_path), "weights_Generator-Generator-7.ckpt"))
    assert set(st.keys()) >= {"step", "state_dict"}
    s2 = build_segan(seed=5)
    assert sd_sha(s2.G.state_dict()) != sha
    s2.G.load_pretrained(os.path.join(str(tmp_path), "weights_Generator-Generator-7.ckpt"), True)
    assert sd_sha(s2.G.state_dict()) == sha


def test_tap_tables_cover_31_taps():
    from segan_pytorch_b200.engine import tap_ranges
    for kind, c, kc, nc in (("conv_fwd", 64, 256, 128), ("conv_dgrad", 64, 128, 256),
                            ("deconv_fwd", 64, 256, 256), ("deconv_dgrad", 64, 256, 256)):
        k_lo, k_hi, n_lo, n_hi = tap_ranges(kind, c, kc, nc)
        blocks = 0
        for i in range(9):
            blocks += ((k_hi[i] - k_lo[i]) // c if "conv_fwd" == kind or kind == "deconv_dgrad" else 4) * \
                      ((n_hi[i] - n_lo[i]) // c if kind in ("conv_dgrad", "deconv_fwd") else 4) // 4
        assert blocks == 31, (kind, blocks)


def test_cpu_forward_fails_loudly():
    s = build_segan()
    with pytest.raises(RuntimeError):
        s.G(torch.zeros(1, 1, 16384))
    with pytest.raises(RuntimeError):
        s.D(torch.zeros(1, 2, 16384))


def test_saver_index_rolls_and_partial_load(tmp_path):
    """Checkpoint format of core.py: JSON index with 'latest' / 'current', the oldest file dropped once the index
    lists more than max_ckpts entries, load_pretrained skipping the file's last two keys unless load_last."""
    import json
    from segan_pytorch_b200.segan.models.core import Saver
    s = build_segan()
    d = str(tmp_path)
    sv = Saver(s.D, d, max_ckpts=2, prefix="EOE_D-")
    for step in (1, 2, 3, 4):
        sv.save("Discriminator", step)
    idx = json.load(open(os.path.join(d, "EOE_D-checkpoints")))
    assert idx["current"] == "EOE_D-Discriminator-4.ckpt"
    assert idx["latest"] == ["EOE_D-Discriminator-%d.ckpt" % i for i in (2, 3, 4)]
    assert not os.path.exists(os.path.join(d, "weights_EOE_D-Discriminator-1.ckpt"))
    assert sv.read_latest_checkpoint() == "EOE_D-Discriminator-4.ckpt"
    sv.save("Discriminator", 9, best_val=True)
    assert os.path.exists(os.path.join(d, "weights_EOE_D-best_Discriminator-9.ckpt"))
    # partial load: everything but the last two keys (fc.4.weight / fc.4.bias)
    s2 = build_segan(seed=7)
    before = {k: v.clone() for k, v in s2.D.state_dict().items()}
    s2.D.load_pretrained(os.path.join(d, "weights_EOE_D-Discriminator-4.ckpt"), load_last=False)
    after, src = s2.D.state_dict(), s.D.state_dict()
    assert torch.equal(after["fc.4.weight"], before["fc.4.weight"]) and torch.equal(after["fc.4.bias"], before["fc.4.bias"])
    assert torch.equal(after["fc.0.weight"], src["fc.0.weight"]) and torch.equal(after["enc_blocks.3.conv.weight"], src["enc_blocks.3.conv.weight"])
    # legacy file = bare state dict
    torch.save(s.D.state_dict(), os.path.join(d, "legacy.ckpt"))
    s3 = build_segan(seed=9)
    s3.D.load_pretrained(os.path.join(d, "legacy.ckpt"), load_last=True)
    assert sd_sha(s3.D.state_dict()) == sd_sha(s.D.state_dict())


@pytest.mark.parametrize("kind", ["rmsprop", "adam"])
def test_fused_optimizer_state_dict_is_torch_compatible(kind):
    """ADVICE r1: FusedOptimizer.state_dict() must load into torch.optim.RMSprop / Adam built over
    Model.parameters() (trainable parameters only, full param_groups) and back, lr included."""
    from segan_pytorch_b200.segan.models.model import FusedOptimizer
    s = build_segan(skip_type="constant")             # frozen alphas: indices must skip them
    eng = s.G.engine.bind()
    opt = FusedOptimizer(eng, kind, 5e-5, betas=(0, 0.9))
    opt._state()
    opt.t = 3
    opt.s1.uniform_(0.1, 1.0)
    if kind == "adam":
        opt.s2.uniform_(0.1, 1.0)
    sd = opt.state_dict()
    import copy
    sd0 = copy.deepcopy(sd)                           # torch's load_state_dict adopts the tensors and step() mutates them
    params = list(s.G.parameters())
    assert len(sd["state"]) == len(params) == len(sd["param_groups"][0]["params"])
    assert all(not n.startswith("alpha_") for n, _ in opt._trainable())
    ref = torch.optim.RMSprop(params, lr=1e-3) if kind == "rmsprop" else torch.optim.Adam(params, lr=1e-3, betas=(0.0, 0.9))
    ref.load_state_dict(sd)
    assert ref.param_groups[0]["lr"] == 5e-5
    for p in params:
        p.grad = torch.zeros_like(p)
    ref.step()                                        # KeyError here if a hyper-parameter were missing
    key = "square_avg" if kind == "rmsprop" else "exp_avg"
    names = [k for k, _ in opt._trainable()]
    i = names.index("enc_blocks.1.conv.weight")          # a packed layer: its state is exported to reference layout
    j = names.index("dec_blocks.2.act.weight")           # a small parameter: a view of the bucket
    assert ref.state_dict()["state"][i][key].shape == torch.Size([128, 64, 31])
    from segan_pytorch_b200.engine import unpack_reference
    lay = eng.by_name["enc_blocks.1.conv.weight"]
    assert torch.equal(sd0["state"][i][key], unpack_reference(0, opt.s1[lay.off:lay.off + lay.numel], 128, 64, 0))
    # and back, with a changed lr
    sd2 = ref.state_dict()
    sd2["param_groups"][0]["lr"] = 2e-5
    opt2 = FusedOptimizer(eng, kind, 5e-5, betas=(0, 0.9))
    opt2.load_state_dict(sd2)
    assert opt2.param_groups[0]["lr"] == 2e-5 and opt2.t == 4
    assert torch.allclose(unpack_reference(0, opt2.s1[lay.off:lay.off + lay.numel], 128, 64, 0),
                          ref.state_dict()["state"][i][key])
    off, n, shape = eng.index["dec_blocks.2.act.weight"]
    assert torch.allclose(opt2.s1[off:off + n].view(shape), ref.state_dict()["state"][j][key])


def test_hostbind_cpulist_and_noop_without_gpu():
    from segan_pytorch_b200 import hostbind
    assert hostbind.parse_cpulist("0-3,8,10-11\n") == {0, 1, 2, 3, 8, 10, 11}
    assert hostbind.parse_cpulist("") == set()
    import os
    before = os.sched_getaffinity(0) if hasattr(os, "sched_getaffinity") else None
    if not torch.cuda.is_available():
        assert hostbind.bind_host_to_gpu(0) is None              # no sysfs entry for a GPU: nothing is changed
        assert before is None or os.sched_getaffinity(0) == before


def _ncu_step_csv(path):
    """A step-level ncu CSV in the format tools/step_traffic.py's ncu command writes (banner lines, one row per
    (launch, metric)): 60 tap-GEMM launches of 100 us / 96 MB read + 34 MB written, 60 fill launches."""
    import csv
    with open(path, "w", newline="") as f:
        f.write("==PROF== Connected to process 1 (python)\n")
        w = csv.writer(f, quoting=csv.QUOTE_ALL)
        w.writerow(["ID", "Process ID", "Process Name", "Host Name", "Kernel Name", "Context", "Stream", "Block Size",
                    "Grid Size", "Device", "CC", "Section Name", "Metric Name", "Metric Unit", "Metric Value"])
        for i in range(120):
            name = ("void sg::tapgemm_f_tc<256, false>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, sg::FTcParams)"
                    if i % 2 == 0 else "void at::vectorized_elementwise_kernel<4, at::FillFunctor<float>>(int)")
            vals = (("gpu__time_duration.sum", "ns", "100,000"), ("dram__bytes_read.sum", "Mbyte", "96.00"),
                    ("dram__bytes_write.sum", "Mbyte", "34.00")) if i % 2 == 0 else \
                   (("gpu__time_duration.sum", "us", "5.5"), ("dram__bytes_read.sum", "byte", "0"),
                    ("dram__bytes_write.sum", "Kbyte", "512"))
            for m, u, v in vals:
                w.writerow([str(i), "1", "python", "127.0.0.1", name, "1", "7", "(384, 1, 1)", "(132, 1, 1)", "0",
                            "9.0", "Command line profiler metrics", m, u, v])


def test_step_traffic_summary_tool_and_bench_traffic(tmp_path):
    """tools/ncu_step_summary.py on a step-level ncu CSV (per-kernel aggregation), and bench.ncu_traffic() on its
    summary (DRAM bytes per launch of the dominant kernel)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, out = str(tmp_path / "launches.csv"), str(tmp_path / "s")
    _ncu_step_csv(src)
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "ncu_step_summary.py"), src, out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    js = json.load(open(out + ".json"))
    k = "tapgemm_f_tc<256, false>"
    assert js["total_launches"] > 100 and k in js["kernels"] and js["kernels"][k]["ms"] > 0
    assert abs(js["kernels"][k]["ms"] - 6.0) < 1e-9 and js["kernels"][k]["dram_bytes_per_launch"] == 130e6
    sys.path.insert(0, root)
    import bench
    t = bench.ncu_traffic(out + ".json")
    assert t is not None and 1e7 < t < 1e9, t          # 130 MB per tap-GEMM launch
