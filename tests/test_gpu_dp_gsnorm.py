"""Data parallelism with a spectrally normalised Generator (norm_type='snorm'), two ranks.
  * The Generator's weight_orig gradients of a batch-mean loss over the global batch, after the chunked + overlapped
    all-reduce (model.GradReducer) and finish_grads, equal one process computing the whole batch: the sigma terms
    applied after the all-reduce must use the coefficients summed over the ranks (they ride in the bucket's
    gradient-only tail), not the local ones.
  * The power iteration does not depend on the batch: u / v after the first pass are the same bits on both ranks and
    in the single process.
  * Full SEGAN steps: every rank ends with bit-identical G parameters and weight_u / weight_v (sg_snorm_sigma_ld sums
    in a fixed order, and every rank steps the same all-reduced bucket).  A whole step is not compared with the
    single-process step: the default Discriminator's BatchNorm statistics are per rank, as in tests/test_dp_nccl.py.
Two ranks on ONE GPU over gloo, which runs on a single-GPU box: the gradient and first-pass checks.  Over gloo with both
ranks on one GPU even the plain Generator's ranks do not stay bit-identical through whole steps, so the step checks run
over NCCL on two GPUs, in the default three-graph schedule, eagerly, and with the collectives captured inside one graph
(skipped with fewer than two GPUs)."""
import os
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


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    gpu = rank if backend == "nccl" else 0
    torch.cuda.set_device(gpu)
    dev = torch.device("cuda", gpu)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from segan_pytorch_b200 import _lib, engine as E
        from segan_pytorch_b200.engine import _p, _stream
        from segan_pytorch_b200.segan.models import SEGAN, model as M
        from tests.test_gsnorm import snorm_generator
        from tests.util import load_opts, rel_err, seed_all
        E.KEEP_GRADS = True
        Bg = 4
        Bl = Bg // world
        g = torch.Generator().manual_seed(7)
        clean = (0.3 * torch.randn(Bg, 1, 16384, generator=g)).clamp(-1, 1)
        noisy = (clean + 0.1 * torch.randn(Bg, 1, 16384, generator=g)).clamp(-1, 1)
        z = torch.randn(Bg, 1024, 16, generator=g)
        out = {}

        def segan(B):
            seed_all(111)
            opts = load_opts(batch_size=B, g_lr=5e-5, d_lr=5e-5)
            s = SEGAN(opts, generator=snorm_generator("concat")).to(dev)
            s.G.train()
            s.D.train()
            return s, opts

        def vectors(G):
            return torch.cat([v.reshape(-1) for k, v in G.state_dict().items() if k.endswith(("weight_u", "weight_v"))])

        def same_on_all_ranks(t):
            ref = t.clone()
            dist.broadcast(ref, src=0)
            return bool(torch.equal(t, ref))

        # ---- (1) weight_orig gradients of 100 * mean|G(x) - clean| over the GLOBAL batch
        def g_grads(s, sl, reducer):
            ge = s.G.engine.bind()
            y, ctx = ge.forward(noisy[sl].to(dev), z[sl].to(dev))
            n_loc = y.numel()
            gy = torch.zeros_like(y)
            loss = torch.zeros(1, device=dev)
            w = 100.0 * n_loc / (Bg * 16384)
            _lib.call("sg_l1_loss_bwd", _p(y), _p(clean[sl].to(dev).contiguous()), n_loc, w, _p(loss), _p(gy), 0,
                      float(E.LOSS_SCALE), _stream())
            ge.backward(ctx, gy, reducer=reducer)
            if reducer is not None:
                reducer.finish()
            ge.finish_grads()
            torch.cuda.synchronize()
            return {n: ge.grad_of(n).cpu() for n, p in s.G.named_parameters() if p.requires_grad}, vectors(s.G)
        s, _ = segan(Bl)
        dp, v_dp = g_grads(s, slice(rank * Bl, (rank + 1) * Bl), M.GradReducer(s.G.engine.bind()))
        out["same_vectors_first_pass"] = same_on_all_ranks(v_dp)
        if rank == 0:
            s1, _ = segan(Bg)
            single, v_single = g_grads(s1, slice(0, Bg), None)
            out["vectors_dp_vs_single"] = bool(torch.equal(v_dp, v_single))
            out["g_dp_vs_single"] = max(rel_err(dp[k], single[k]) for k in single)
            out["g_dp_vs_single_orig"] = max(rel_err(dp[k], single[k]) for k in single if k.endswith("weight_orig"))
            del s1
        del s
        # ---- (2) SEGAN steps: identical parameters and vectors on every rank
        schedules = [(False, False), (True, False), (True, True)] if backend == "nccl" else []
        shifts = [[[2, -1, 0, 3, 1], [0, 0, -2, 1, 4], [1, -3, 2, 0, 0]] for _ in range(3)]
        for graphs, capture in schedules:
            tag = "%s%s" % ("graph" if graphs else "eager", "_capture" if capture else "")
            E.GRAPHS, M.DP_CAPTURE = graphs, capture
            s, opts = segan(Bl)
            Gopt, Dopt = s.build_optimizers(opts)
            sl = slice(rank * Bl, (rank + 1) * Bl)
            for i in range(4):
                s.train_step(clean[sl].to(dev), noisy[sl].to(dev), Gopt, Dopt, 100.0, z=z[sl].to(dev),
                             shifts3=shifts[min(i, 2)])
            torch.cuda.synchronize()
            out["same_params_" + tag] = same_on_all_ranks(s.G.engine.flat)
            out["same_vectors_" + tag] = same_on_all_ranks(vectors(s.G))
            out["graphs_" + tag] = sum(1 for v in getattr(s, "_step_graphs", {}).values() if v.graphs is not None)
            del s, Gopt, Dopt
        q.put((rank, out, None))
    except Exception:                                       # noqa
        import traceback
        q.put((rank, None, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _run(backend):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, q), daemon=True) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=400) for _ in procs]
    finally:
        for p in procs:                      # a hung collective must not outlive the test
            p.join(timeout=20)
            if p.is_alive():
                p.kill()
    for rank, out, err in res:
        assert err is None, "rank %d failed:\n%s" % (rank, err)
    outs = {rank: out for rank, out, _ in res}
    print("snorm-G DP (%s):" % backend, outs)
    r0 = outs[0]
    # the per-shard gradients sum exactly up to fp16 tiles landing differently and fp32 atomics (tests/test_dp_nccl.py
    # holds the plain G to 2e-3); a rank-local sigma-term coefficient is off by half the term: 0.5-23 % of a gradient
    assert r0["g_dp_vs_single"] <= 2e-3, r0
    assert r0["vectors_dp_vs_single"], r0
    for r in (0, 1):
        o = outs[r]
        assert o["same_vectors_first_pass"], o
        if backend == "nccl":
            assert all(v for k, v in o.items() if k.startswith(("same_params_", "same_vectors_"))), o
            assert len([k for k in o if k.startswith("same_params_")]) == 3, o
            assert o["graphs_eager"] == 0 and o["graphs_graph"] == 1 and o["graphs_graph_capture"] == 1, o


def test_snorm_generator_two_ranks_one_gpu_gloo():
    _run("gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_snorm_generator_two_gpus_nccl():
    _run("nccl")
