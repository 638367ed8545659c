"""Data-parallel path on real GPUs over NCCL (needs >= 2 GPUs: `python -m pytest tests/test_dp_nccl.py -m gpu` on a machine with two;
skipped on a single-GPU box).  SURVEY.md section 4: "DP(N ranks x B/N) == single-process gradients".
  * the Generator has no batch statistics, so its gradients of a batch-mean loss over a global batch are EXACTLY the
    sum of the per-shard gradients: 2 ranks x 2 windows, chunked + overlapped all-reduce (model.GradReducer), against
    one process computing all 4 windows;
  * full G+D train steps on 2 ranks in BOTH schedules -- the default one (three CUDA graphs, one eager all-reduce per
    gradient bucket between them) and the opt-in one (model.DP_CAPTURE: eager warm-up, then ONE graph with the chunked
    collectives captured inside): every rank must hold bit-identical parameters afterwards, and the chunked reduction
    must equal one whole-bucket
    all-reduce."""
import os
import random
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import ctypes as C
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    def mark(msg):
        import sys
        sys.stderr.write("[dp rank %d] %s\n" % (rank, msg))
        sys.stderr.flush()
    try:
        from segan_pytorch_b200 import _lib, engine as E
        from segan_pytorch_b200.engine import _p, _stream
        from segan_pytorch_b200.segan.models import model as M
        from tests.util import build_segan, load_opts, rel_err
        E.KEEP_GRADS = True
        Bg = 4                                                # global batch
        Bl = Bg // world
        g = torch.Generator().manual_seed(7)
        clean = (0.3 * torch.randn(Bg, 1, 16384, generator=g)).clamp(-1, 1)
        noisy = (clean + 0.1 * torch.randn(Bg, 1, 16384, generator=g)).clamp(-1, 1)
        z = torch.randn(Bg, 1024, 16, generator=g)
        out = {}

        # ---- (1) Generator gradients of 100 * mean|G(x) - clean| over the GLOBAL batch
        def g_grads(s, sl, reducer):
            ge = s.G.engine
            y, ctx = ge.forward(noisy[sl].to(dev), z[sl].to(dev))
            n_loc = y.numel()
            gy = torch.zeros_like(y)
            loss = torch.zeros(1, device=dev)
            # sg_l1_loss_bwd scales by weight / n_local: weight * n_local / n_global gives the global mean's gradient
            w = 100.0 * n_loc / (Bg * 16384)
            _lib.call("sg_l1_loss_bwd", _p(y), _p(clean[sl].to(dev).contiguous()), n_loc, w, _p(loss), _p(gy), 0,
                      float(E.LOSS_SCALE), _stream())
            ge.backward(ctx, gy, reducer=reducer)
            if reducer is not None:
                reducer.finish()
            torch.cuda.synchronize()
            return ge.grad.clone()
        mark('init done')
        s = build_segan(batch_size=Bl).to(dev)
        s.G.train()
        red = M.GradReducer(s.G.engine.bind())
        dp = g_grads(s, slice(rank * Bl, (rank + 1) * Bl), red)
        if rank == 0:
            s1 = build_segan(batch_size=Bg).to(dev)
            s1.G.train()
            single = g_grads(s1, slice(0, Bg), None)
            out["g_dp_vs_single"] = rel_err(dp, single)
            chunks = s.G.engine.grad_chunks()
            out["chunks_cover"] = (chunks[0][0] == 0 and all(chunks[i][0] + chunks[i][1] == chunks[i + 1][0]
                                                               for i in range(len(chunks) - 1))
                                   and chunks[-1][0] + chunks[-1][1] == s.G.engine.grad.numel())
        mark('G gradient part done')
        del s
        # ---- (2) the DEFAULT schedule: three graphs, one eager all-reduce per bucket between them
        M.DP_CAPTURE = False
        random.seed(5 + rank)
        torch.manual_seed(5 + rank)
        s = build_segan(batch_size=Bl).to(dev)
        s.G.train()
        s.D.train()
        Gopt, Dopt = s.build_optimizers(load_opts(batch_size=Bl))
        sl = slice(rank * Bl, (rank + 1) * Bl)
        c, n = clean[sl].to(dev), noisy[sl].to(dev)
        for i in range(5):
            s.train_step(c, n, Gopt, Dopt, 100.0)
            mark('default-schedule step %d done' % i)
        torch.cuda.synchronize()
        out["graphs_default"] = [len(v.graphs) for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None]
        for name, eng in (("G", s.G.engine), ("D", s.D.engine)):
            mine = eng.flat.clone()
            ref = mine.clone()
            dist.broadcast(ref, src=0)
            out["same_params_default_" + name] = bool(torch.equal(mine, ref))
        del s, Gopt, Dopt
        # ---- (3) the opt-in schedule: chunked collectives captured inside ONE graph (eager warm-up, then replays)
        M.DP_CAPTURE = True                               # opt-in schedule, verified on 2 GPUs (see model.DP_CAPTURE)
        random.seed(3 + rank)
        torch.manual_seed(3 + rank)
        s = build_segan(batch_size=Bl).to(dev)            # same seed on every rank -> identical init
        s.G.train()
        s.D.train()
        Gopt, Dopt = s.build_optimizers(load_opts(batch_size=Bl))
        sl = slice(rank * Bl, (rank + 1) * Bl)
        c, n = clean[sl].to(dev), noisy[sl].to(dev)
        losses = []
        for i in range(5):
            losses.append(s.train_step(c, n, Gopt, Dopt, 100.0).tolist())
            mark('step %d done' % i)
        torch.cuda.synchronize()
        st = list(getattr(s, "_step_graphs", {}).values())
        out["graphs"] = [len(v.graphs) for v in st if v.graphs is not None]
        out["finite"] = all(abs(v) < 1e6 for l in losses for v in l)
        for name, eng in (("G", s.G.engine), ("D", s.D.engine)):
            mine = eng.flat.clone()
            ref = mine.clone()
            dist.broadcast(ref, src=0)
            out["same_params_" + name] = bool(torch.equal(mine, ref))
        # ---- (4) chunked reduction == one whole-bucket all-reduce (same gradients, D bucket)
        de = s.D.engine
        gsum = de.grad.clone()                              # KEEP_GRADS: the reduced gradients of the last step
        allsame = gsum.clone()
        dist.broadcast(allsame, src=0)
        out["reduced_grads_identical"] = bool(torch.equal(gsum, allsame))
        q.put((rank, out, None))
    except Exception as e:                                  # noqa
        import traceback
        q.put((rank, None, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_two_gpus():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q), daemon=True) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=300) for _ in procs]
    finally:
        for p in procs:                      # a hung collective must not outlive the test (and the GPU box's time limit)
            p.join(timeout=20)
            if p.is_alive():
                p.kill()
    for rank, out, err in res:
        assert err is None, "rank %d failed:\n%s" % (rank, err)
    outs = {rank: out for rank, out, _ in res}
    print("DP results:", outs)
    r0 = outs[0]
    assert r0["chunks_cover"]
    assert r0["g_dp_vs_single"] <= 2e-3, r0            # fp16 tiles land differently (M tiling by batch), fp32 atomics
    for r in (0, 1):
        assert outs[r]["finite"] and outs[r]["same_params_G"] and outs[r]["same_params_D"], outs[r]
        assert outs[r]["reduced_grads_identical"], outs[r]
        assert outs[r]["graphs"] == [1], outs[r]       # opt-in: the step captured as ONE graph incl. the collectives
        assert outs[r]["graphs_default"] == [3], outs[r]
        assert outs[r]["same_params_default_G"] and outs[r]["same_params_default_D"], outs[r]
