"""Drop-in `SEGAN` / `WSEGAN` (reference: segan/models/model.py:28-766).

Constructor, `generate`, `discriminate`, `infer_G`, `infer_D`, `build_optimizers` and `train` keep
the reference's signatures and step order (model.py:283-321); the step itself is the fused kernel
pipeline of segan_pytorch_b200.engine plus one gradient all-reduce per optimiser step when
torch.distributed is initialised (one process per GPU; SURVEY.md 8e)."""
import ctypes as C
import os
import random
import timeit
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .core import Model, Saver
from .discriminator import Discriminator, draw_phase_shifts
from .generator import Generator
from ..datasets.se_dataset import DevicePrefetcher
from ... import _lib
from ... import engine as _engine
from ...engine import _p, _stream

try:  # optional, absent in this image (SURVEY.md section 5)
    from tensorboardX import SummaryWriter
except Exception:  # pragma: no cover
    class SummaryWriter(object):
        def __init__(self, *a, **k):
            pass

        def add_scalar(self, *a, **k):
            pass

        def add_histogram(self, *a, **k):
            pass


def weights_init(m):
    """model.py:28-43 -- matches class names containing 'Conv1d' / 'Linear' only
    (nn.ConvTranspose1d keeps torch's default init)."""
    classname = m.__class__.__name__
    if classname.find('Conv1DResBlock') != -1:
        for k, p in m.named_parameters():
            if 'weight' in k and 'conv' in k:
                p.data.normal_(0.0, 0.02)
    elif classname.find('Conv1d') != -1:
        m.weight.data.normal_(0.0, 0.02)
        if hasattr(m, 'bias') and m.bias is not None:
            m.bias.data.fill_(0)
    elif classname.find('Linear') != -1:
        nn.init.xavier_uniform_(m.weight.data)


def wsegan_weights_init(m):
    """model.py:45-60 -- xavier on Conv1d, ConvTranspose1d and Linear."""
    classname = m.__class__.__name__
    if classname.find('Conv1DResBlock') != -1:
        for k, p in m.named_parameters():
            if 'weight' in k and 'conv' in k:
                nn.init.xavier_uniform_(p.data)
    elif classname.find('Conv1d') != -1:
        nn.init.xavier_uniform_(m.weight.data)
    elif classname.find('ConvTranspose1d') != -1:
        nn.init.xavier_uniform_(m.weight.data)
    elif classname.find('Linear') != -1:
        nn.init.xavier_uniform_(m.weight.data)


class FusedOptimizer(object):
    """torch.optim.RMSprop / Adam semantics (model.py:221-225) as ONE kernel over the flat fp32
    parameter bucket of a network.  state_dict() is torch-compatible (per-parameter tensors)."""

    def __init__(self, eng, kind, lr, betas=(0.0, 0.9), alpha=0.99, eps=1e-8):
        self.eng, self.kind, self.lr, self.betas, self.alpha, self.eps = eng, kind, lr, betas, alpha, eps
        self.t = 0
        self.s1 = None
        self.s2 = None
        self.param_groups = [dict(lr=lr)]

    def _state(self):
        flat = self.eng.bind().flat
        if self.s1 is None or self.s1.shape != flat.shape or self.s1.device != flat.device:
            self.s1 = torch.zeros_like(flat)
            self.s2 = torch.zeros_like(flat) if self.kind == 'adam' else None
        return flat

    def zero_grad(self):
        """The bucket is cleared by step() as it is read: this only fills when gradients were left behind."""
        self.eng.bind()
        self.eng.zero_grad()

    def step(self, grad_scale=1.0):
        flat = self._state()
        lr = self.param_groups[0]['lr']
        self.t += 1
        n = flat.numel()
        grad_scale = float(grad_scale) / _engine.LOSS_SCALE      # the bucket carries the fp16 loss scale
        self.eng.finish_grads()                                  # dWeff -> dW, dalpha (decoder skip halves)
        clear = 0 if _engine.KEEP_GRADS else 1
        if self.kind == 'rmsprop':
            _lib.call("sg_rmsprop_step", _p(flat), _p(self.eng.grad), _p(self.s1), n, lr, self.alpha, self.eps,
                      float(grad_scale), clear, _stream())
        else:
            _lib.call("sg_adam_step", _p(flat), _p(self.eng.grad), _p(self.s1), _p(self.s2), n, lr, self.betas[0],
                      self.betas[1], self.eps, self.t, float(grad_scale), clear, _stream())
        self.eng.grads_consumed(bool(clear))
        self.eng.master_updated()

    def _trainable(self):
        """(name, parameter) in torch's optimiser order: the requires_grad parameters only (core.py:196-197)."""
        return [(n, p) for n, p in self.eng.module.named_parameters() if p.requires_grad]

    def state_dict(self):
        """Same structure as torch.optim.RMSprop / Adam .state_dict() over Model.parameters(): per-parameter state
        tensors in reference layout, indices over the trainable parameters, full hyper-parameter groups -- a
        checkpoint written here loads into the reference's optimiser and vice versa."""
        self._state()
        state = {}
        names = self._trainable()
        for i, (name, p) in enumerate(names):
            view = lambda t, name=name: self._state_view(t, name)
            step = torch.tensor(float(self.t))
            if self.kind == 'rmsprop':
                state[i] = {'step': step, 'square_avg': view(self.s1)}
            else:
                state[i] = {'step': step, 'exp_avg': view(self.s1), 'exp_avg_sq': view(self.s2)}
        lr = self.param_groups[0]['lr']
        if self.kind == 'rmsprop':
            group = dict(lr=lr, momentum=0, alpha=self.alpha, eps=self.eps, centered=False, weight_decay=0,
                         capturable=False, foreach=None, maximize=False, differentiable=False)
        else:
            group = dict(lr=lr, betas=tuple(float(b) for b in self.betas), eps=self.eps, weight_decay=0, amsgrad=False, maximize=False,
                         foreach=None, capturable=False, differentiable=False, fused=None)
        group['params'] = list(range(len(names)))
        return {'state': state if self.t > 0 else {}, 'param_groups': [group]}

    def _state_view(self, t, name):
        """Per-parameter state tensor in reference layout on the CPU (the state lives in the bucket's layout)."""
        eng = self.eng
        l = eng.by_name.get(name)
        if l is None:
            off, n, shape = eng.index[name]
            return t[off:off + n].view(shape).detach().to('cpu', copy=True)
        out = torch.empty_like(eng._param(name).data)
        eng._export(l, t[l.off:l.off + l.numel], out)
        return out.cpu()

    def _state_load(self, t, name, value):
        eng = self.eng
        l = eng.by_name.get(name)
        if l is None:
            off, n, shape = eng.index[name]
            t[off:off + n].copy_(value.reshape(-1))
        else:
            eng._import(l, src=value.to(t.device).float().contiguous(), dst=t[l.off:l.off + l.numel])

    def load_state_dict(self, sd):
        self._state()
        groups = sd.get('param_groups') or [{}]
        if 'lr' in groups[0]:
            self.param_groups[0]['lr'] = float(groups[0]['lr'])
        for i, (name, p) in enumerate(self._trainable()):
            st = sd.get('state', {}).get(i)
            if st is None:
                continue
            self.t = int(st.get('step', self.t))
            if 'square_avg' in st:
                self._state_load(self.s1, name, st['square_avg'])
            if 'exp_avg' in st:
                self._state_load(self.s1, name, st['exp_avg'])
                self._state_load(self.s2, name, st['exp_avg_sq'])


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist
    return None


def allreduce_grads(eng):
    """The single gradient collective of an optimiser step: one all-reduce (SUM) over the flat
    bucket the weight-gradient kernels wrote into (no pack pass).  Returns the grad scale."""
    dist = _dist()
    if dist is None:
        return 1.0
    dist.all_reduce(eng.grad, op=dist.ReduceOp.SUM)
    return 1.0 / dist.get_world_size()


# Data-parallel gradient exchange (SURVEY.md 8e): one all-reduce per optimiser step over the network's gradient
# bucket.  DP_OVERLAP (default on) sends the bucket in the 2-3 chunks of engine.grad_chunks() -- bucket order is
# gradient-completion order -- on a communication stream as the backward pass produces them, so only the last,
# small chunk is exposed; with CUDA graphs the collectives are captured into the step's single graph.
DP_OVERLAP = os.environ.get("SEGAN_B200_DP_OVERLAP", "1").lower() not in ("0", "off", "no", "false")
# SEGAN_B200_DP_CAPTURE=1 captures the chunked collectives INSIDE the step's single CUDA graph.  Opt-in: with 4 GPUs
# the replays following the first one were seen to hang (NCCL 2.28.9, eager collectives -- barriers -- mixed with
# the captured ones).  Default: three graphs with one eager all-reduce per bucket between them.
DP_CAPTURE = os.environ.get("SEGAN_B200_DP_CAPTURE", "0").lower() not in ("0", "off", "no", "false")
# SEGAN's regression term (--reg_loss, model.py:79,318) -> its fused loss + gradient kernel.  WSEGAN's denoising term
# is always L1 (model.py:663).
REG_LOSS_KERNELS = {'l1_loss': 'sg_l1_loss_bwd', 'mse_loss': 'sg_mse_loss_bwd'}


class GradReducer(object):
    """Chunked, overlapped all-reduce (SUM) of one engine's gradient bucket."""

    def __init__(self, eng):
        self.eng = eng
        self.comm = torch.cuda.Stream(device=eng.flat.device)
        self.events = {}

    def ready(self, i, launch):
        """Called on the stream that just enqueued the last writer of chunk `i` for the current pass."""
        ev = torch.cuda.Event()
        ev.record()
        self.events.setdefault(i, []).append(ev)
        if launch:
            dist = _dist()
            off, n = self.eng.grad_chunks()[i]
            for e in self.events.pop(i):
                self.comm.wait_event(e)
            with torch.cuda.stream(self.comm):
                dist.all_reduce(self.eng.grad[off:off + n], op=dist.ReduceOp.SUM)

    def finish(self):
        """The optimiser's stream waits for every chunk; returns the gradient scale."""
        assert not self.events, "gradient chunks marked ready but never reduced: %r" % list(self.events)
        torch.cuda.current_stream().wait_stream(self.comm)
        return 1.0 / _dist().get_world_size()


class SEGAN(Model):

    def __init__(self, opts, name='SEGAN', generator=None, discriminator=None):
        super(SEGAN, self).__init__(name)
        self.save_path = opts.save_path
        self.preemph = opts.preemph
        # SURVEY.md F5: the shipped ckpt_segan+/train.opts has no reg_loss key
        self.reg_loss_name = getattr(opts, 'reg_loss', 'l1_loss')
        self.reg_loss = getattr(F, self.reg_loss_name)
        if generator is None:
            self.G = Generator(1, opts.genc_fmaps, opts.gkwidth, opts.genc_poolings, opts.gdec_fmaps,
                               opts.gdec_kwidth, opts.gdec_poolings, z_dim=opts.z_dim, no_z=opts.no_z,
                               skip=(not opts.no_skip), bias=opts.bias, skip_init=opts.skip_init,
                               skip_type=opts.skip_type, skip_merge=opts.skip_merge,
                               skip_kwidth=opts.skip_kwidth)
        else:
            self.G = generator
        self.G.apply(weights_init)
        if discriminator is None:
            dkwidth = opts.gkwidth if opts.dkwidth is None else opts.dkwidth
            self.D = Discriminator(2, opts.denc_fmaps, dkwidth, poolings=opts.denc_poolings,
                                   pool_type=opts.dpool_type, pool_slen=opts.dpool_slen,
                                   norm_type=opts.dnorm_type, phase_shift=opts.phase_shift,
                                   sinc_conv=opts.sinc_conv)
        else:
            self.D = discriminator
        self.D.apply(weights_init)
        self.z_device = getattr(opts, 'z_device', 'cpu')

    # ------------------------------------------------------------------------------------------
    # inference (model.py:116-175)
    # ------------------------------------------------------------------------------------------
    def generate(self, inwav, z=None, device=None):
        """Chunked enhancement of one utterance (1,1,T).  All 16384-sample windows are run as ONE
        batch (they are independent), with the reference's z semantics: the given z (or the z drawn
        for the first window) for window 0 and `G.z` -- the first z G ever saw -- afterwards
        (model.py:144-146).  De-emphasis runs on the GPU as a scan (se_dataset.py:119-126)."""
        self.G.eval()
        N = 16384
        dev = next(super(Model, self.G).parameters()).device
        inwav = torch.as_tensor(inwav).float()
        T = inwav.shape[2]
        nchunks = (T + N - 1) // N
        x = torch.zeros(nchunks, 1, N, dtype=torch.float32, device=dev)
        flat = inwav[0, 0].to(dev)
        x.view(-1)[:T].copy_(flat)
        code_len = N // (4 ** len(self.G.enc_blocks))
        if self.G.no_z:
            zb = None                                      # generator.py:193-208: no z drawn, G.z never set
        elif z is None:
            z0 = torch.randn(1, self.G.z_dim, code_len).to(dev)
            if not hasattr(self.G, 'z'):
                self.G.z = z0
            zrest = self.G.z
        else:
            z0 = z.to(dev)
            if not hasattr(self.G, 'z'):
                self.G.z = z0
            zrest = z0
        if not self.G.no_z:
            zb = torch.cat([z0[:1]] + [zrest[:1]] * (nchunks - 1), 0) if nchunks > 1 else z0[:1]
        last = 'enc_{}'.format(len(self.G.enc_blocks) - 1)
        with torch.no_grad():
            y, hall = self.G(x, z=zb, ret_hid=(last,))     # only the code of model.py:149 is converted to NCL
        g_c = hall[last][-1:]
        c = y.reshape(-1)[:T].contiguous()
        out = torch.empty_like(c)
        if self.preemph > 0:
            _lib.call("sg_deemphasis", _p(c), T, float(self.preemph), _p(out), _stream())
        else:
            out = c
        return out.cpu().numpy(), g_c

    def generate_batch(self, windows, z=None):
        """Streaming inference (BASELINE config 5): (N,1,16384) pre-emphasised windows -> enhanced
        windows, no de-emphasis (windows of different utterances)."""
        self.G.eval()
        with torch.no_grad():
            return self.G(windows, z=z)

    def generate_stream(self, host_batches, z=None):
        """Streaming inference over HOST batches (BASELINE config 5; the clean.py:59-82 loop batched across
        files): yields one pinned host tensor of enhanced windows per input batch of (N,1,16384) pre-emphasised
        windows.  Three streams: the H2D copy of batch n+1, G on batch n and the D2H copy of batch n-1 overlap,
        so a slow host link hides behind the Generator.  A yielded tensor is valid only until the NEXT batch is
        requested (two pinned output buffers alternate and the following iteration already copies into the
        other slot's successor): consume or copy it before calling next() again."""
        self.G.eval()
        dev = next(super(Model, self.G).parameters()).device
        main = torch.cuda.current_stream(dev)
        h2d, d2h = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        slots = [dict(), dict()]

        def stage(hb, slot):
            hb = torch.as_tensor(hb).float()
            if slot.get("x") is None or slot["x"].shape != hb.shape:
                slot["x"] = torch.empty(hb.shape, dtype=torch.float32, device=dev)
                slot["out"] = torch.empty(hb.shape, dtype=torch.float32).pin_memory()
            with torch.cuda.stream(h2d):
                if slot.get("free") is not None:
                    h2d.wait_event(slot["free"])
                slot["x"].copy_(hb, non_blocking=True)
                slot["ready"] = torch.cuda.Event()
                slot["ready"].record(h2d)
            return slot

        it = iter(host_batches)
        try:
            cur = stage(next(it), slots[0])
        except StopIteration:
            return
        n, prev = 0, None
        while cur is not None:
            n += 1
            try:
                nxt = stage(next(it), slots[n % 2])
            except StopIteration:
                nxt = None
            main.wait_event(cur["ready"])
            if cur.get("out_done") is not None:
                cur["out_done"].synchronize()          # its previous output has been handed out and copied
            with torch.no_grad():
                y = self.G(cur["x"], z=z)
            cur["free"] = torch.cuda.Event()
            cur["free"].record(main)
            d2h.wait_event(cur["free"])
            with torch.cuda.stream(d2h):
                cur["out"].copy_(y, non_blocking=True)
                y.record_stream(d2h)
                cur["out_done"] = torch.cuda.Event()
                cur["out_done"].record(d2h)
            if prev is not None:
                prev["out_done"].synchronize()
                yield prev["out"]
            prev, cur = cur, nxt
        if prev is not None:
            prev["out_done"].synchronize()
            yield prev["out"]

    def clean_files(self, wav_paths, out_dir, batch=256, group_windows=None, on_done=None):
        """Streaming enhancement of many wav files -- the clean.py:59-82 loop batched ACROSS files (SURVEY.md 8f-N1,
        BASELINE config 5).  Per file the result equals `generate` on the normalised + pre-emphasised file
        (model.py:116-157): 16384-sample windows, the last one zero-padded, z semantics of the reference (a fresh
        z for the first window of every file, `G.z` -- the first z G ever saw -- for the others), de-emphasis.

        Pipeline: a reader thread decodes wavs into pinned int16 window groups (whole files, about `group_windows`
        windows); the copy stream uploads group n+1 while the main stream runs group n -- int16 -> float +
        whole-file pre-emphasis on the device (sg_pcm16_to_wave), G in batches of `batch` windows, one
        segmented de-emphasis launch for all files of the group -- and a third stream downloads group n-1 into
        pinned memory, from which a writer thread saves float32 wavs (scipy, like clean.py:79).
        Returns the number of windows processed.  on_done(path, n_samples) is called per written file."""
        import queue
        import threading
        from scipy.io import wavfile
        self.G.eval()
        N = 16384
        dev = next(super(Model, self.G).parameters()).device
        code_len = N // (4 ** len(self.G.enc_blocks))
        zdim = None if self.G.no_z else self.G.z_dim
        group_windows = int(group_windows or 2 * batch)
        coef = float(self.preemph)
        os.makedirs(out_dir, exist_ok=True)
        q_in, q_out = queue.Queue(maxsize=2), queue.Queue(maxsize=2)
        errors = []

        def reader():
            """Groups of whole files as pinned int16 windows + per-window side tables."""
            try:
                group, nwin = [], 0

                def flush():
                    nonlocal group, nwin
                    if not group:
                        return
                    pcm = torch.zeros(nwin, N, dtype=torch.int16).pin_memory()
                    prev = torch.full((nwin,), 0x7fffffff, dtype=torch.int32)
                    valid = torch.full((nwin,), N, dtype=torch.int32)
                    first, files, w0 = [], [], 0
                    for path, wav in group:
                        T = wav.shape[0]
                        n = (T + N - 1) // N
                        flat = pcm[w0:w0 + n].view(-1)
                        flat[:T] = torch.from_numpy(wav)
                        if n > 1:
                            prev[w0 + 1:w0 + n] = torch.from_numpy(wav[N - 1:(n - 1) * N:N].astype(np.int32))
                        valid[w0 + n - 1] = T - (n - 1) * N
                        first.append(w0)
                        files.append((path, w0, T))
                        w0 += n
                    # one fresh z per file, drawn in file order from torch's CPU generator (generator.py:197-199);
                    # none with no_z
                    zf = torch.randn(len(files), zdim, code_len).pin_memory() if zdim is not None else None
                    q_in.put(dict(pcm=pcm, prev=prev.pin_memory(), valid=valid.pin_memory(), files=files,
                                  first=torch.tensor(first, dtype=torch.long), zf=zf, nwin=nwin))
                    group, nwin = [], 0
                for path in wav_paths:
                    rate, wav = wavfile.read(path)
                    if wav.ndim != 1 or wav.dtype != np.int16:
                        raise ValueError('mono 16-bit PCM wavs expected: %s' % path)
                    n = (wav.shape[0] + N - 1) // N
                    if group and nwin + n > group_windows:
                        flush()
                    group.append((path, wav))
                    nwin += n
                flush()
            except Exception as e:            # surfaced in the main thread
                errors.append(e)
            finally:
                q_in.put(None)

        def writer():
            # files of a group are independent: a few threads keep several write() system calls in flight (scipy's
            # wavfile.write releases the GIL inside them)
            from concurrent.futures import ThreadPoolExecutor

            def save(arr, path, w0, T):
                wavfile.write(os.path.join(out_dir, os.path.basename(path)), 16000, arr[w0 * N:w0 * N + T])
                if on_done is not None:
                    on_done(path, T)
            try:
                with ThreadPoolExecutor(max_workers=4) as pool:
                    while True:
                        item = q_out.get()
                        if item is None:
                            return
                        ev, host, files = item
                        ev.synchronize()
                        arr = host.numpy()
                        for f in [pool.submit(save, arr, *fl) for fl in files]:
                            f.result()
            except Exception as e:
                errors.append(e)

        tr, tw = threading.Thread(target=reader, daemon=True), threading.Thread(target=writer, daemon=True)
        tr.start()
        tw.start()
        main = torch.cuda.current_stream(dev)
        h2d, d2h = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        total = 0
        pending = []                                   # (host buffer, done event) kept alive until written

        def upload(g):
            with torch.cuda.stream(h2d):
                d = {k: (g[k].to(dev, non_blocking=True) if g[k] is not None else None)
                     for k in ('pcm', 'prev', 'valid', 'zf')}
                d['ready'] = torch.cuda.Event()
                d['ready'].record(h2d)
            return d
        nxt = q_in.get()
        nxt_dev = upload(nxt) if nxt is not None else None
        while nxt is not None and not errors:
            g, d = nxt, nxt_dev
            nxt = q_in.get()                               # decode of the following group ran meanwhile
            nxt_dev = upload(nxt) if nxt is not None else None
            main.wait_event(d['ready'])
            nw = g['nwin']
            x = torch.empty(nw, 1, N, dtype=torch.float32, device=dev)
            _lib.call("sg_pcm16_to_wave", _p(d['pcm']), _p(d['prev']), nw, N, coef, _p(x), _p(d['valid']), _stream())
            if zdim is not None and not hasattr(self.G, 'z'):
                self.G.z = d['zf'][:1].clone()             # generator.py:203-204: the first z ever
            first = g['first'].to(dev)
            y = torch.empty(nw, N, dtype=torch.float32, device=dev)
            with torch.no_grad():
                for b0 in range(0, nw, batch):
                    b1 = min(nw, b0 + batch)
                    zb = None
                    if zdim is not None:
                        zb = self.G.z[:1].expand(b1 - b0, -1, -1).clone()
                        sel = (first >= b0) & (first < b1)
                        if bool(sel.any()):
                            zb[first[sel] - b0] = d['zf'][sel]
                    y[b0:b1] = self.G(x[b0:b1], z=zb).view(b1 - b0, N)
            out = torch.empty_like(y)
            if coef > 0:
                seg = torch.tensor([[w0 * N, T] for _, w0, T in g['files']], dtype=torch.int64).to(dev)
                _lib.call("sg_deemphasis_segments", _p(y), _p(seg), len(g['files']), coef, _p(out), _stream())
            else:
                out = y
            done = torch.cuda.Event()
            done.record(main)
            for t_ in (d['pcm'], d['prev'], d['valid'], d['zf']):
                if t_ is not None:
                    t_.record_stream(main)
            host = torch.empty(nw * N, dtype=torch.float32).pin_memory()
            with torch.cuda.stream(d2h):
                d2h.wait_event(done)
                host.copy_(out.view(-1), non_blocking=True)
                out.record_stream(d2h)
                copied = torch.cuda.Event()
                copied.record(d2h)
            q_out.put((copied, host, g['files']))
            total += nw
        q_out.put(None)
        tw.join()
        tr.join(timeout=1.0)
        if errors:
            raise errors[0]
        return total

    def discriminate(self, cwav, nwav):
        self.D.eval()
        d_in = torch.cat((cwav, nwav), dim=1)
        d_veredict, _ = self.D(d_in)
        return d_veredict

    def infer_G(self, nwav, cwav=None, z=None, ret_hid=False):
        if ret_hid:
            Genh, hall = self.G(nwav, z=z, ret_hid=ret_hid)
            return Genh, hall
        return self.G(nwav, z=z, ret_hid=ret_hid)

    def infer_D(self, x_, ref):
        D_in = torch.cat((x_, ref), dim=1)
        return self.D(D_in)

    def build_optimizers(self, opts):
        ge, de = self.G.engine.bind(), self.D.engine.bind()
        if opts.opt == 'rmsprop':
            Gopt = FusedOptimizer(ge, 'rmsprop', opts.g_lr)
            Dopt = FusedOptimizer(de, 'rmsprop', opts.d_lr)
        elif opts.opt == 'adam':
            Gopt = FusedOptimizer(ge, 'adam', opts.g_lr, betas=(0, 0.9))
            Dopt = FusedOptimizer(de, 'adam', opts.d_lr, betas=(0, 0.9))
        else:
            raise ValueError('Unrecognized optimizer {}'.format(opts.opt))
        return Gopt, Dopt

    # ------------------------------------------------------------------------------------------
    # one LSGAN + L1 step (model.py:283-321) on device-resident (B,1,L) tensors
    # ------------------------------------------------------------------------------------------
    def _sample_z(self, B, code_len, dev):
        if self.G.no_z:
            return None                  # the reference draws no z (and consumes no random numbers) with no_z
        if self.z_device == 'cpu':
            z = torch.randn(B, self.G.z_dim, code_len).to(dev)        # generator.py:197-199
        else:
            z = torch.randn(B, self.G.z_dim, code_len, device=dev)
        if not hasattr(self.G, 'z'):
            self.G.z = z
        return z

    def _reducers(self):
        """(D reducer, G reducer) of an overlapped data-parallel step, or (None, None)."""
        if _dist() is None or not DP_OVERLAP:
            return None, None
        r = self.__dict__.get('_grad_reducers')
        ge, de = self.G.engine, self.D.engine
        if r is None or r[0].eng.grad is not de.grad or r[1].eng.grad is not ge.grad:
            r = self.__dict__['_grad_reducers'] = (GradReducer(de), GradReducer(ge))
        return r

    def _check_d_logits(self, B):
        """SEGAN's losses compare D's logits, flattened, with B labels (model.py:298,305,316).  pool_type='mlp' gives
        B * Lq logits, which the reference rejects in its first step; refuse it before training anything."""
        if getattr(self.D, 'pool_type', 'none') == 'mlp':
            lq = self.D.pool_slen
            raise RuntimeError("SEGAN cannot train a Discriminator with pool_type='mlp': it gives one logit per "
                               "position, B * Lq = %d logits against B = %d labels (the reference fails at "
                               "model.py:298 with 'The size of tensor a (%d) must match the size of tensor b (%d)'); "
                               "WSEGAN (--wsegan) trains it" % (B * lq, B, B * lq, B))

    def train_step(self, clean, noisy, Gopt, Dopt, l1_weight, z=None, shifts3=None, losses=None):
        """clean / noisy: (B,1,L) fp32 cuda.  Returns the device tensor of the four losses
        [d_real, d_fake, g_adv, g_l1] (no host sync).

        After `engine.GRAPH_WARMUP` eager steps of the same shape the step is captured once into three
        CUDA graphs (D phase | D optimiser + G phase | G optimiser; the two gradient all-reduces of a
        data-parallel run sit between them) and replayed: the ~300 launches of a step then cost no host
        time and the side-stream schedule (engine.OVERLAP) becomes real concurrency on the device.  The
        per-step phase shifts live in a small device table the host rewrites before each replay."""
        self._check_d_logits(clean.shape[0])
        ge, de = self.G.engine, self.D.engine
        B, _, L = clean.shape
        dev = clean.device
        nl = len(self.D.enc_blocks)
        if self.reg_loss_name not in REG_LOSS_KERNELS:
            raise NotImplementedError("reg_loss %r is not built: the G regression term runs as a fused kernel for %s"
                                      % (self.reg_loss_name, " / ".join(repr(k) for k in REG_LOSS_KERNELS)))
        if shifts3 is None:        # python `random` draw order of the reference: real, fake, G-step pass
            shifts3 = [draw_phase_shifts(nl, self.D.phase_shift) for _ in range(3)]
        if self.G.no_z:
            z = None
        elif z is None and self.z_device == 'cpu':
            z = self._sample_z(B, L // (4 ** len(self.G.enc_blocks)), dev)
        sample_z = z is None and not self.G.no_z          # z drawn on the device inside the step
        st = self._graph_state(clean, noisy, Gopt, Dopt, l1_weight, sample_z)
        if st is None:
            # ---- eager schedule
            if losses is None:
                losses = torch.zeros(4, dtype=torch.float32, device=dev)
            if z is None:
                z = self._sample_z(B, L // (4 ** len(self.G.enc_blocks)), dev)
            rd, rg = self._reducers()
            Genh, gctx = self._seg_d(clean, noisy, z, shifts3, None, losses, Dopt, sample_z=False, reducer=rd)
            dscale = rd.finish() if rd is not None else allreduce_grads(de)      # before model.py:308
            self._seg_g(clean, noisy, Genh, gctx, shifts3, None, losses, l1_weight, Gopt, Dopt, dscale, reducer=rg)
            gscale = rg.finish() if rg is not None else allreduce_grads(ge)      # before model.py:321
            Gopt.step(gscale)                                              # model.py:321
            return losses
        # ---- CUDA-graph schedule: refresh the static inputs, replay
        if st.clean.data_ptr() != clean.data_ptr():
            st.clean.copy_(clean, non_blocking=True)
        if st.noisy.data_ptr() != noisy.data_ptr():
            st.noisy.copy_(noisy, non_blocking=True)
        if z is not None:
            st.z.copy_(z, non_blocking=True)
            if not hasattr(self.G, 'z'):
                self.G.z = z
        # this step's phase shifts -> device table, through a ring of pinned rows (a fresh pinned allocation
        # per step would hit cudaHostAlloc whenever the host runs ahead of the device)
        i = st.ring_i % st.ring.shape[0]
        st.ring_i += 1
        if st.ring_ev[i] is not None:
            st.ring_ev[i].synchronize()        # the copy that last used this row (ring-size steps ago) is done
        st.ring[i].copy_(torch.tensor([int(v) for sh in shifts3 for v in sh], dtype=torch.int32))
        st.shifts.copy_(st.ring[i], non_blocking=True)
        st.ring_ev[i] = torch.cuda.Event()
        st.ring_ev[i].record()
        if st.graphs is None:
            self._capture_step(st, sample_z, shifts3, l1_weight, Gopt, Dopt)
        else:
            # parameters touched outside the step (checkpoint load ...): import them; D's operands of graph 1 were
            # emitted by the previous replay of graph 2, so they are refreshed here
            ge.notice_external_writes()
            de.ensure_packed()
            if len(st.graphs) == 1:            # data-parallel with the collectives captured inside
                st.graphs[0].replay()
            else:
                st.graphs[0].replay()
                allreduce_grads(de)
                st.graphs[1].replay()
                allreduce_grads(ge)
                st.graphs[2].replay()
            Dopt.t += 1
            Gopt.t += 1
            ge.master_updated()                # the replayed optimiser steps changed the masters in place
            de._mirror_stale = True
            _lib.launch_count += st.launches
        if losses is not None and losses.data_ptr() != st.losses.data_ptr():
            losses.copy_(st.losses, non_blocking=True)
            return losses
        return st.losses

    # -- step segments (shared by the eager and the graph schedule) -------------------------------
    def _seg_d(self, clean, noisy, z, shifts3, shifts_dev, losses, Dopt, sample_z, reducer=None):
        """G forward (model.py:295), D real (model.py:297-299) and D fake (model.py:303-306) passes.
        Schedule (engine.OVERLAP): the D(real) pass depends on neither G nor the fake pass, so it runs as
        lane 1 of the D engine (own workspace + gradient bucket) on side stream 2, concurrently with the
        G forward and the D(fake) pass on the caller's stream."""
        ge, de = self.G.engine, self.D.engine
        dev = clean.device
        nl = len(self.D.enc_blocks)
        lptr = lambda i: C.c_void_p(losses.data_ptr() + 4 * i)
        sdev = (lambda i: None) if shifts_dev is None else (lambda i: shifts_dev[i * nl:(i + 1) * nl])
        losses.zero_()
        if sample_z:
            z.normal_()                                                    # generator.py:197-199 on the device
        Dopt.zero_grad()
        # (a spectrally normalised D re-emits its operands for every pass: its passes cannot overlap)
        rside = None if de.snorm else _engine.side_stream(dev, 2)
        lane = 1 if rside is not None else 0
        fwd_real_done = None
        with _engine.on_side(rside):
            _, c = de.forward(clean, noisy, shifts3[0], training=True, lane=lane, shifts_dev=sdev(0))
            if rside is not None:
                fwd_real_done = torch.cuda.Event()
                fwd_real_done.record()
            de.backward(c, 1.0, 1.0, param_grads=True, loss_out=lptr(0), reducer=reducer, reduce_now=False)
        Genh, gctx = ge.forward(noisy, z)
        if fwd_real_done is not None:
            # BatchNorm running statistics are updated real pass first, fake pass second (model.py:297,303)
            torch.cuda.current_stream().wait_event(fwd_real_done)
        _, c = de.forward(Genh, noisy, shifts3[1], training=True, shifts_dev=sdev(1))
        # the real lane's pass was enqueued above (python order), so its "ready" events exist: the fake pass launches
        # each chunk once its own and the real lane's weight gradients of that chunk are enqueued
        de.backward(c, 0.0, 1.0, param_grads=True, loss_out=lptr(1), reducer=reducer, reduce_now=True)
        _engine.join_side(rside)
        return Genh, gctx

    def _seg_g(self, clean, noisy, Genh, gctx, shifts3, shifts_dev, losses, l1_weight, Gopt, Dopt, dscale, reducer=None):
        """D optimiser step (model.py:308), then the G update against the UPDATED D (model.py:313-320)."""
        ge, de = self.G.engine, self.D.engine
        B, _, L = clean.shape
        dev = clean.device
        nl = len(self.D.enc_blocks)
        lptr = lambda i: C.c_void_p(losses.data_ptr() + 4 * i)
        Dopt.step(dscale)
        Gopt.zero_grad()
        sdev = None if shifts_dev is None else shifts_dev[2 * nl:3 * nl]
        _, c = de.forward(Genh, noisy, shifts3[2], training=True, twins=False, shifts_dev=sdev)   # no weight gradients here
        gy = ge.buf.get("g.gy", (B, 1, L), torch.float32, dev, zero=True)
        de.backward(c, 1.0, 1.0, param_grads=False, input_grad=gy, loss_out=lptr(2))
        # model.py:318: l1_weight * reg_loss(Genh, clean) -- logged as g_l1 whatever reg_loss is
        _lib.call(REG_LOSS_KERNELS[self.reg_loss_name], _p(Genh), _p(clean.contiguous()), B * L, float(l1_weight),
                  lptr(3), _p(gy), 1, float(_engine.LOSS_SCALE), _stream())
        ge.backward(gctx, gy, reducer=reducer)

    # -- CUDA graphs ------------------------------------------------------------------------------
    def _graph_state(self, clean, noisy, Gopt, Dopt, l1_weight, sample_z):
        """Static tensors + graphs of the step for this (shape, hyper-parameter) key, or None while the
        eager schedule should run (graphs disabled, profiling active, optimiser with a per-step scalar,
        or fewer than GRAPH_WARMUP eager steps seen for the key)."""
        if not _engine.GRAPHS or _engine.PROFILE is not None or _lib.call_profile is not None:
            return None
        if Gopt.kind != 'rmsprop' or Dopt.kind != 'rmsprop' or not _engine.wave_on_tensor_cores():
            return None                         # Adam passes its step count by value
        if torch.cuda.is_current_stream_capturing():
            return None
        ge, de = self.G.engine, self.D.engine
        world = _dist().get_world_size() if _dist() is not None else 1
        B, _, L = clean.shape
        key = (B, L, float(l1_weight), Gopt.param_groups[0]['lr'], Dopt.param_groups[0]['lr'], world,
               ge.flat.data_ptr() if ge.flat is not None else 0, de.flat.data_ptr() if de.flat is not None else 0,
               _engine.OVERLAP, self.z_device, bool(sample_z), ge.backend, de.backend, _engine.GS,
               _engine.LOSS_SCALE)
        cache = self.__dict__.setdefault('_step_graphs', {})
        st = cache.get(key)
        if st is None:
            if len(cache) >= 4:
                cache.clear()                   # hyper-parameters that change every step: stay eager-ish
            st = cache[key] = types.SimpleNamespace(seen=0, graphs=None)
        st.seen += 1
        if st.seen <= _engine.GRAPH_WARMUP:
            return None
        if st.graphs is None and not hasattr(st, 'clean'):
            dev = clean.device
            nl = len(self.D.enc_blocks)
            st.clean = torch.empty_like(clean)
            st.noisy = torch.empty_like(noisy)
            st.z = (None if self.G.no_z else
                    torch.empty(B, self.G.z_dim, L // (4 ** len(self.G.enc_blocks)), device=dev))
            st.losses = torch.zeros(4, dtype=torch.float32, device=dev)
            st.shifts = torch.zeros(3 * nl, dtype=torch.int32, device=dev)
            st.ring = torch.zeros(32, 3 * nl, dtype=torch.int32).pin_memory()
            st.ring_ev = [None] * 32
            st.ring_i = 0
            st.launches = 0
        return st

    def _capture_step(self, st, sample_z, shifts3, l1_weight, Gopt, Dopt):
        """Runs one step under stream capture (the captured work is NOT executed: the three graphs are
        replayed right after) -- see train_step."""
        ge, de = self.G.engine, self.D.engine
        dscale = 1.0 / (_dist().get_world_size() if _dist() is not None else 1)
        torch.cuda.synchronize()
        # the pack kernels of BOTH networks must be part of the captured step: a G forward between the last eager
        # step and this capture (generate(), sample logging) would otherwise leave G "clean" here, nothing would be
        # captured and every replay would run on the stale 16-bit operands (D is re-packed after Dopt.step anyway)
        ge.mark_dirty()
        de.mark_dirty()
        n0 = _lib.launch_count
        t_d, t_g = Dopt.t, Gopt.t
        rd, rg = self._reducers()
        graphs = None
        if rd is not None and DP_CAPTURE and not getattr(self, '_dp_capture_failed', False):
            # data parallel: ONE graph with the chunked all-reduces captured on the communication stream
            # (thread-local capture mode: NCCL's watchdog thread keeps polling its events meanwhile)
            g1 = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(g1, capture_error_mode="thread_local"):
                    Genh, gctx = self._seg_d(st.clean, st.noisy, st.z, shifts3, st.shifts, st.losses, Dopt,
                                             sample_z=sample_z, reducer=rd)
                    rd.finish()
                    self._seg_g(st.clean, st.noisy, Genh, gctx, shifts3, st.shifts, st.losses, l1_weight, Gopt, Dopt,
                                dscale, reducer=rg)
                    rg.finish()
                    Gopt.step(dscale)
                graphs = (g1,)
            except Exception as e:              # fall back to collectives between three graphs
                print("segan_b200: capturing the NCCL all-reduces failed (%s): using eager collectives between graphs"
                      % (str(e).splitlines()[0] if str(e) else type(e).__name__))
                self._dp_capture_failed = True
                rd.events.clear()
                rg.events.clear()
                torch.cuda.synchronize()
                ge.mark_dirty()
                de.mark_dirty()
                Dopt.t, Gopt.t = t_d, t_g
                _lib.launch_count = n0
        if graphs is None and _dist() is None:
            # single GPU: nothing separates the three segments -- one graph, one launch per step
            g1 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g1):
                Genh, gctx = self._seg_d(st.clean, st.noisy, st.z, shifts3, st.shifts, st.losses, Dopt, sample_z=sample_z)
                self._seg_g(st.clean, st.noisy, Genh, gctx, shifts3, st.shifts, st.losses, l1_weight, Gopt, Dopt, dscale)
                Gopt.step(dscale)
            graphs = (g1,)
        if graphs is None:
            g1, g2, g3 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(g1):
                Genh, gctx = self._seg_d(st.clean, st.noisy, st.z, shifts3, st.shifts, st.losses, Dopt, sample_z=sample_z)
            with torch.cuda.graph(g2, pool=g1.pool()):
                self._seg_g(st.clean, st.noisy, Genh, gctx, shifts3, st.shifts, st.losses, l1_weight, Gopt, Dopt, dscale)
            with torch.cuda.graph(g3, pool=g1.pool()):
                Gopt.step(dscale)
            graphs = (g1, g2, g3)
        Dopt.t, Gopt.t = t_d, t_g               # capture only recorded the launches
        st.launches = _lib.launch_count - n0
        _lib.launch_count = n0
        st.keep = (Genh, gctx)                  # tensors of the graphs' private pool referenced by later nodes
        st.graphs = graphs
        # the step itself: replay
        if len(graphs) == 1:
            graphs[0].replay()
        else:
            graphs[0].replay()
            allreduce_grads(de)
            graphs[1].replay()
            allreduce_grads(ge)
            graphs[2].replay()
        Dopt.t += 1
        Gopt.t += 1
        ge.master_updated()
        de._mirror_stale = True
        _lib.launch_count += st.launches
        if sample_z and not hasattr(self.G, 'z'):
            self.G.z = st.z

    def train(self, opts, dloader, criterion, l1_init, l1_dec_step, l1_dec_epoch, log_freq, va_dloader=None,
              device='cuda'):
        """Train the SEGAN (model.py:230-437): same loop structure, logging line and checkpoint
        cadence.  `criterion` must be nn.MSELoss (LSGAN); it is fused into the D head backward."""
        self._check_d_logits(opts.batch_size)
        if not isinstance(criterion, nn.MSELoss):
            raise NotImplementedError("SEGAN.train is built for the LSGAN criterion nn.MSELoss (train.py:94)")
        rank0 = _dist() is None or _dist().get_rank() == 0
        self.writer = SummaryWriter(os.path.join(self.save_path, 'train')) if rank0 else SummaryWriter()
        self.z_device = getattr(opts, 'z_device', self.z_device)
        Gopt, Dopt = self.build_optimizers(opts)
        self.G.optim = Gopt
        self.D.optim = Dopt
        eoe_g_saver = Saver(self.G, opts.save_path, max_ckpts=3, optimizer=self.G.optim, prefix='EOE_G-')
        eoe_d_saver = Saver(self.D, opts.save_path, max_ckpts=3, optimizer=self.D.optim, prefix='EOE_D-')
        l1_weight = l1_init
        iteration = 1
        timings = []
        losses = None
        for epoch in range(1, opts.epoch + 1):
            beg_t = timeit.default_timer()
            self.G.train()
            self.D.train()
            if hasattr(getattr(dloader, 'sampler', None), 'set_epoch'):
                dloader.sampler.set_epoch(epoch)                 # DistributedSampler: a new shuffle every epoch
            # batch n+1 is staged on the GPU (copy stream) while batch n trains
            for bidx, batch in enumerate(DevicePrefetcher(dloader, device, preemph=getattr(opts, 'preemph', 0.95)),
                                         start=1):
                if epoch >= l1_dec_epoch:
                    if l1_weight > 0:
                        l1_weight -= l1_dec_step
                        l1_weight = max(0, l1_weight)
                if len(batch) != 4:
                    raise ValueError('Returned {} elements per sample?'.format(len(batch)))
                uttname, clean, noisy, slice_idx = batch
                losses = self.train_step(clean, noisy, Gopt, Dopt, l1_weight, losses=losses)
                end_t = timeit.default_timer()
                timings.append(end_t - beg_t)
                beg_t = timeit.default_timer()
                if bidx % log_freq == 0 or bidx >= len(dloader):
                    lv = losses.tolist()                                   # the only host sync
                    if rank0:
                        print('(Iter {}) Batch {}/{} (Epoch {}) d_real:{:.4f}, d_fake:{:.4f}, g_adv:{:.4f}, '
                              'g_l1:{:.4f} l1_w: {:.2f}, btime: {:.4f} s, mbtime: {:.4f} s'
                              ''.format(iteration, bidx, len(dloader), epoch, lv[0], lv[1], lv[2], lv[3],
                                        l1_weight, timings[-1], np.mean(timings)))
                        self.writer.add_scalar('D_real', lv[0], iteration)
                        self.writer.add_scalar('D_fake', lv[1], iteration)
                        self.writer.add_scalar('G_adv', lv[2], iteration)
                        self.writer.add_scalar('G_l1', lv[3], iteration)
                iteration += 1
            if va_dloader is not None:
                raise NotImplementedError("validation with composite objective metrics (model.py:394-433) is "
                                          "out of the hot-path scope (SURVEY.md 2.1)")
            if rank0:
                self.G.save(self.save_path, iteration, saver=eoe_g_saver)
                self.D.save(self.save_path, iteration, saver=eoe_d_saver)
        self.last_losses = losses
        return timings


class WSEGAN(SEGAN):
    """Whisper-SEGAN (model.py:509-766): xavier init, one weighted D loss over real / fake /
    [misaligned] pairs, G loss = adversarial + STFT log-power L1 + masked L1."""

    def __init__(self, opts, name='WSEGAN', generator=None, discriminator=None):
        self.lbd = 1
        self.critic_iters = 1
        self.misalign_pair = opts.misalign_pair
        self.interf_pair = opts.interf_pair
        self.pow_weight = opts.pow_weight
        self.vanilla_gan = opts.vanilla_gan
        self.n_fft = opts.n_fft
        super(WSEGAN, self).__init__(opts, name, None, None)
        self.G.apply(wsegan_weights_init)
        self.D.apply(wsegan_weights_init)

    def infer_G(self, nwav, cwav=None, z=None, ret_hid=False):
        return self.G(nwav, z=z, ret_hid=ret_hid)

    def sample_dloader(self, dloader, device='cuda'):
        """model.py:526-535 -- one batch from a FRESH iterator of the loader (the reference's per-step behaviour),
        staged like every other batch: float windows as they are, int16 PCM windows (SEDataset(pcm16=True), five
        fields) normalised + pre-emphasised on the device.  `train` does not use this: it keeps one persistent
        prefetching iterator (SURVEY.md 8f-N3)."""
        uttname, clean, noisy, slice_idx = next(iter(DevicePrefetcher(dloader, device, preemph=self.preemph)))
        return uttname, clean.clone(), noisy.clone(), slice_idx

    @staticmethod
    def _endless(dloader):
        """Epoch after epoch of `dloader` (a shuffling loader reshuffles each pass; DistributedSampler gets its
        epoch set) -- the persistent replacement of the reference's `next(iter(dloader))` per step."""
        epoch = 0
        while True:
            epoch += 1
            if hasattr(getattr(dloader, 'sampler', None), 'set_epoch'):
                dloader.sampler.set_epoch(epoch)
            n = 0
            for batch in dloader:
                n += 1
                yield batch
            if n == 0:
                raise ValueError('empty data loader')

    @staticmethod
    def stft_logpow(x, n_fft):
        """model.py:640-646: |STFT| (n_fft 2048, hop 160, win 320 rectangular, normalized) -> 10 log10(.^2+1e-19).
        Library-backed (cuFFT through torch.stft): the spectral term is <1 % of the step's FLOPs."""
        st = torch.stft(x.squeeze(1), n_fft=min(x.size(-1), n_fft), hop_length=160, win_length=320,
                        normalized=True, return_complex=True)
        mod = torch.norm(torch.view_as_real(st), 2, dim=3)
        return 10 * torch.log10(mod ** 2 + 10e-20)

    def _d_pass(self, x0, x1, shifts, target, weight, losses, slot, input_grad=None, param_grads=True,
                twins=True, reducer=None, reduce_now=True):
        """One D forward + backward of `weight * cost(D(x0 | x1), target)`: LSGAN (MSE, fused into the head
        backward kernel) or, with --vanilla_gan, BCE with logits (model.py:583-586; its gradient
        (sigmoid(logit) - target) * weight / B is handed to the same backward)."""
        de = self.D.engine
        lptr = C.c_void_p(losses.data_ptr() + 4 * slot)
        shifts, shifts_dev = shifts if isinstance(shifts, tuple) else (shifts, None)
        logit, c = de.forward(x0, x1, shifts, training=True, twins=twins, shifts_dev=shifts_dev)
        red = dict(reducer=reducer, reduce_now=reduce_now) if param_grads else {}
        if not self.vanilla_gan:
            de.backward(c, target, weight, param_grads=param_grads, input_grad=input_grad, loss_out=lptr, **red)
            return
        lg = logit.detach().view(-1)
        tg = torch.full_like(lg, float(target))
        losses[slot] += weight * F.binary_cross_entropy_with_logits(lg, tg)
        g_logit = ((torch.sigmoid(lg) - tg) * (float(weight) / lg.numel())).contiguous()
        de.backward(c, target, weight, param_grads=param_grads, input_grad=input_grad, loss_out=None, g_logit=g_logit,
                    **red)

    @staticmethod
    def interferer_squares(B, L, picks=None):
        """model.py:606-622: per sample a square wave of random frequency {250, 1000, 4000} Hz and amplitude
        {0.01, 0.05, 0.1, 1} (python `random.choice`, frequency first), t = linspace(0, 2, 32000), cut to L."""
        from scipy import signal
        freqs, amps = [250, 1000, 4000], [0.01, 0.05, 0.1, 1]
        t = np.linspace(0, 2, 32000)
        rows = []
        for i in range(B):
            f_, a_ = picks[i] if picks is not None else (random.choice(freqs), random.choice(amps))
            rows.append(torch.FloatTensor((a_ * signal.square(2 * np.pi * f_ * t))[:L].reshape((1, -1))))
        return torch.cat(rows, dim=0).unsqueeze(1)

    def train_step(self, clean, noisy, Gopt, Dopt, l1_weight, uttname=None, z=None, shifts=None, perm=None,
                   losses=None, interf=None):
        """One WSEGAN step (model.py:572-669) with optional --misalign_pair / --interf_pair / --vanilla_gan.
        Returns the device tensor [d_loss, g_adv, pow_loss, den_loss].  Draw order of python `random` as in the
        reference: D(real) shifts, [z], D(fake) shifts, [shuffle, D(misaligned) shifts], [per sample: interferer
        frequency, amplitude; D(interfered) shifts], D(fake) shifts.  `perm` / `interf` (the squares, (B,1,L))
        override the draws (tests).

        Like SEGAN.train_step, after `engine.GRAPH_WARMUP` eager steps of a shape the step is captured into ONE CUDA
        graph and replayed (RMSprop, LSGAN, no masked L1 term in the batch): the phase shifts, the misalignment
        permutation and the interferers are device tensors the host refreshes before each replay."""
        B, _, L = clean.shape
        dev = clean.device
        nl = len(self.D.enc_blocks)
        # ---- host draws, in the reference's order
        nsh = iter(shifts) if shifts is not None else None
        draw = (lambda: next(nsh)) if nsh is not None else (lambda: draw_phase_shifts(nl, self.D.phase_shift))
        sh = [draw()]                                                      # D(real)
        if self.G.no_z:
            z = None
        sample_z = z is None and self.z_device != 'cpu' and not self.G.no_z
        if z is None and not sample_z:
            z = self._sample_z(B, L // (4 ** len(self.G.enc_blocks)), dev)
        sh.append(draw())                                                  # D(fake)
        if self.misalign_pair:
            if perm is None:
                perm = list(range(B))
                random.shuffle(perm)                                       # model.py:598-600
            sh.append(draw())
        if self.interf_pair:
            if interf is None:
                interf = self.interferer_squares(B, L)                     # model.py:606-622
            sh.append(draw())
        sh.append(draw())                                                  # D(fake) of the G step
        masked = bool(l1_weight > 0 and uttname is not None and any('additive' in u for u in uttname))
        st = None if masked else self._wgraph_state(clean, noisy, Gopt, Dopt, sample_z, len(sh))
        if st is None:
            losses = torch.zeros(4, dtype=torch.float32, device=dev) if losses is None else losses
            if sample_z:
                z = self._sample_z(B, L // (4 ** len(self.G.enc_blocks)), dev)
            perm_d = torch.as_tensor(perm, device=dev) if self.misalign_pair else None
            interf_d = interf.to(dev) if self.interf_pair else None
            return self._wstep(clean, noisy, z, sh, None, perm_d, interf_d, losses, Gopt, Dopt, l1_weight, uttname,
                               False)
        # ---- CUDA-graph schedule: refresh the static inputs, replay
        ge, de = self.G.engine, self.D.engine
        if st.clean.data_ptr() != clean.data_ptr():
            st.clean.copy_(clean, non_blocking=True)
        if st.noisy.data_ptr() != noisy.data_ptr():
            st.noisy.copy_(noisy, non_blocking=True)
        if z is not None:
            st.z.copy_(z, non_blocking=True)
        i = st.ring_i % st.ring.shape[0]
        st.ring_i += 1
        if st.ring_ev[i] is not None:
            st.ring_ev[i].synchronize()
        row = [int(v) for one in sh for v in one] + ([int(v) for v in perm] if self.misalign_pair else [])
        st.ring[i].copy_(torch.tensor(row, dtype=torch.int32))
        st.table.copy_(st.ring[i], non_blocking=True)
        st.ring_ev[i] = torch.cuda.Event()
        st.ring_ev[i].record()
        if self.interf_pair:
            st.interf.copy_(interf.to(dev, non_blocking=True))
        if st.graph is None:
            self._wcapture(st, sh, sample_z, Gopt, Dopt, l1_weight)
        else:
            ge.notice_external_writes()
            de.ensure_packed()
            st.graph.replay()
            Dopt.t += 1
            Gopt.t += 1
            ge.master_updated()
            de._mirror_stale = True
            _lib.launch_count += st.launches
        if losses is not None and losses.data_ptr() != st.losses.data_ptr():
            losses.copy_(st.losses, non_blocking=True)
            return losses
        return st.losses

    def _wstep(self, clean, noisy, z, sh, table, perm_d, interf_d, losses, Gopt, Dopt, l1_weight, uttname, sample_z):
        """The step's device work (shared by the eager and the captured schedule).  sh: the host's phase shifts per D
        pass; table: device int32 copy of the same (then the kernels read the shifts from memory), or None."""
        ge, de = self.G.engine, self.D.engine
        B, _, L = clean.shape
        dev = clean.device
        nl = len(self.D.enc_blocks)
        losses.zero_()
        if sample_z:
            z.normal_()
        ip = iter(range(len(sh)))

        def nxt():
            i = next(ip)
            return sh[i], (None if table is None else table[i * nl:(i + 1) * nl])
        # model.py:595,603,626: 1/2, 1/3 with the misaligned pair, 1/4 whenever the interferer pair is on
        d_weight = 0.25 if self.interf_pair else ((1.0 / 3) if self.misalign_pair else 0.5)
        # the G forward (model.py:583) does not depend on the D(real) pass before it: side stream 1
        gside = _engine.side_stream(dev, 1)
        with _engine.on_side(gside):
            Genh, gctx = ge.forward(noisy, z)
        Dopt.zero_grad()
        rd, rg = self._reducers()
        n_d = 2 + int(bool(self.misalign_pair)) + int(bool(self.interf_pair))      # the last D pass launches the chunks
        self._d_pass(clean, noisy, nxt(), 1.0, d_weight, losses, 0, reducer=rd, reduce_now=False)
        _engine.join_side(gside)
        self._d_pass(Genh, noisy, nxt(), 0.0, d_weight, losses, 0, reducer=rd, reduce_now=(n_d == 2))
        if self.misalign_pair:
            clean_shuf = torch.index_select(clean, 0, perm_d)              # model.py:598-600
            self._d_pass(clean, clean_shuf, nxt(), 0.0, d_weight, losses, 0, reducer=rd,
                         reduce_now=not self.interf_pair)
        if self.interf_pair:
            self._d_pass(clean + interf_d, noisy, nxt(), 0.0, d_weight, losses, 0, reducer=rd, reduce_now=True)
        Dopt.step(rd.finish() if rd is not None else allreduce_grads(de))
        Gopt.zero_grad()
        gy = ge.buf.get("g.gy", (B, 1, L), torch.float32, dev, zero=True)
        self._d_pass(Genh, noisy, nxt(), 1.0, 1.0, losses, 1, input_grad=gy, param_grads=False, twins=False)
        # spectral power loss (model.py:638-653): one tensor-core GEMM over the frames of both signals
        # (engine.SpectralLoss); other n_fft / windows shorter than a frame keep the library transform
        lscale = _engine.LOSS_SCALE
        if self.n_fft == 2048 and L >= 2048:
            if getattr(self, '_spectral', None) is None or self._spectral.dev != dev:
                self._spectral = _engine.SpectralLoss(dev)
            self._spectral(Genh, clean, self.pow_weight, C.c_void_p(losses.data_ptr() + 8), g_wave=gy, g_scale=lscale)
        else:
            gt = Genh.detach().requires_grad_(True)
            with torch.enable_grad():
                pow_loss = self.pow_weight * F.l1_loss(self.stft_logpow(gt, self.n_fft),
                                                       self.stft_logpow(clean, self.n_fft))
                pow_loss.backward()
            losses[2] += pow_loss.detach()
            gy.add_(gt.grad, alpha=lscale)
        if l1_weight > 0 and uttname is not None and any('additive' in u for u in uttname):
            # model.py:655-665: l1_weight * mean over ALL B*L samples of |mask (G - clean)|, mask = 1 on the samples of
            # 'additive' utterances: one fused loss + gradient launch per run of consecutive masked windows
            i = 0
            while i < B:
                if 'additive' not in uttname[i]:
                    i += 1
                    continue
                j = i
                while j < B and 'additive' in uttname[j]:
                    j += 1
                n_run = (j - i) * L
                _lib.call("sg_l1_loss_bwd", C.c_void_p(Genh.data_ptr() + 4 * i * L), C.c_void_p(clean.data_ptr() + 4 * i * L),
                          n_run, float(l1_weight) * n_run / (B * L), C.c_void_p(losses.data_ptr() + 12),
                          C.c_void_p(gy.data_ptr() + 4 * i * L), 1, float(lscale), _engine._stream())
                i = j
        ge.backward(gctx, gy, reducer=rg)
        Gopt.step(rg.finish() if rg is not None else allreduce_grads(ge))
        return losses

    def _wgraph_state(self, clean, noisy, Gopt, Dopt, sample_z, n_pass):
        """Static tensors + graph of the WSEGAN step for this key, or None while the eager schedule should run."""
        if not _engine.GRAPHS or _engine.PROFILE is not None or _lib.call_profile is not None:
            return None
        if Gopt.kind != 'rmsprop' or Dopt.kind != 'rmsprop' or not _engine.wave_on_tensor_cores() or self.vanilla_gan:
            return None                         # Adam passes its step count by value; BCE runs through torch ops
        if self.n_fft != 2048 or clean.shape[-1] < 2048 or torch.cuda.is_current_stream_capturing():
            return None
        if getattr(self, '_wgraph_failed', False):
            return None
        if _dist() is not None and not DP_CAPTURE:
            return None                         # data parallel: the collectives stay eager (see DP_CAPTURE)
        ge, de = self.G.engine, self.D.engine
        world = _dist().get_world_size() if _dist() is not None else 1
        B, _, L = clean.shape
        key = ('w', B, L, Gopt.param_groups[0]['lr'], Dopt.param_groups[0]['lr'], world,
               ge.flat.data_ptr() if ge.flat is not None else 0, de.flat.data_ptr() if de.flat is not None else 0,
               _engine.OVERLAP, self.z_device, bool(sample_z), ge.backend, de.backend, _engine.GS, _engine.LOSS_SCALE,
               bool(self.misalign_pair), bool(self.interf_pair), float(self.pow_weight), n_pass)
        cache = self.__dict__.setdefault('_step_graphs', {})
        st = cache.get(key)
        if st is None:
            if len(cache) >= 4:
                cache.clear()
            st = cache[key] = types.SimpleNamespace(seen=0, graph=None, graphs=None)
        st.seen += 1
        if st.seen <= _engine.GRAPH_WARMUP:
            return None
        if st.graph is None and not hasattr(st, 'clean'):
            dev = clean.device
            nl = len(self.D.enc_blocks)
            ntab = n_pass * nl + (B if self.misalign_pair else 0)
            st.clean = torch.empty_like(clean)
            st.noisy = torch.empty_like(noisy)
            st.z = (None if self.G.no_z else
                    torch.empty(B, self.G.z_dim, L // (4 ** len(self.G.enc_blocks)), device=dev))
            st.losses = torch.zeros(4, dtype=torch.float32, device=dev)
            st.table = torch.zeros(ntab, dtype=torch.int32, device=dev)     # phase shifts of every pass [+ permutation]
            st.interf = torch.zeros_like(clean) if self.interf_pair else None
            st.ring = torch.zeros(32, ntab, dtype=torch.int32).pin_memory()
            st.ring_ev = [None] * 32
            st.ring_i = 0
            st.launches = 0
            st.n_shift = n_pass * nl
        return st

    def _wcapture(self, st, sh, sample_z, Gopt, Dopt, l1_weight):
        """Captures one step (not executed) and replays it; on failure the key falls back to eager steps."""
        ge, de = self.G.engine, self.D.engine
        torch.cuda.synchronize()
        ge.mark_dirty()
        de.mark_dirty()
        n0 = _lib.launch_count
        t_d, t_g = Dopt.t, Gopt.t
        perm_d = st.table[st.n_shift:].to(torch.int64) if self.misalign_pair else None
        g = torch.cuda.CUDAGraph()
        mode = dict(capture_error_mode="thread_local") if _dist() is not None and DP_OVERLAP else {}
        try:
            with torch.cuda.graph(g, **mode):
                pd = st.table[st.n_shift:].to(torch.int64) if self.misalign_pair else None    # inside: follows the table
                self._wstep(st.clean, st.noisy, st.z, sh, st.table, pd, st.interf, st.losses, Gopt, Dopt, l1_weight,
                            None, sample_z)
        except Exception as e:
            print("segan_b200: capturing the WSEGAN step failed (%s): eager steps from here on"
                  % (str(e).splitlines()[0] if str(e) else type(e).__name__))
            self._wgraph_failed = True
            for r in (self._reducers() if _dist() is not None else ()):
                if r is not None:
                    r.events.clear()
            torch.cuda.synchronize()
            ge.mark_dirty()
            de.mark_dirty()
            Dopt.t, Gopt.t = t_d, t_g
            _lib.launch_count = n0
            losses = st.losses
            return self._wstep(st.clean, st.noisy, st.z, sh, None, perm_d, st.interf, losses, Gopt, Dopt, l1_weight,
                               None, sample_z)
        Dopt.t, Gopt.t = t_d, t_g
        st.launches = _lib.launch_count - n0
        _lib.launch_count = n0
        st.graph = g
        st.graphs = (g,)
        g.replay()
        Dopt.t += 1
        Gopt.t += 1
        ge.master_updated()
        de._mirror_stale = True
        _lib.launch_count += st.launches
        if sample_z and not hasattr(self.G, 'z'):
            self.G.z = st.z

    def train(self, opts, dloader, criterion, l1_init, l1_dec_step, l1_dec_epoch, log_freq, va_dloader=None,
              device='cuda'):
        """model.py:537-753: iteration-based loop (a fresh loader iterator per step), EOE checkpoints."""
        rank0 = _dist() is None or _dist().get_rank() == 0
        self.writer = SummaryWriter(os.path.join(opts.save_path, 'train')) if rank0 else SummaryWriter()
        self.z_device = getattr(opts, 'z_device', self.z_device)
        Gopt, Dopt = self.build_optimizers(opts)
        self.G.optim, self.D.optim = Gopt, Dopt
        eoe_g_saver = Saver(self.G, opts.save_path, max_ckpts=3, optimizer=self.G.optim, prefix='EOE_G-')
        eoe_d_saver = Saver(self.D, opts.save_path, max_ckpts=3, optimizer=self.D.optim, prefix='EOE_D-')
        l1_weight = l1_init
        timings = []
        losses = None
        self.G.train()
        self.D.train()
        # one persistent iterator, the next batch staged on a copy stream while this one trains (the reference
        # builds a new DataLoader iterator -- and its worker processes -- every step, model.py:527)
        batches = iter(DevicePrefetcher(self._endless(dloader), device, preemph=getattr(opts, 'preemph', 0.95)))
        for iteration in range(1, opts.epoch * len(dloader) + 1):
            beg_t = timeit.default_timer()
            uttname, clean, noisy, slice_idx = next(batches)
            losses = self.train_step(clean, noisy, Gopt, Dopt, l1_weight, uttname=uttname, losses=losses)
            timings.append(timeit.default_timer() - beg_t)
            if iteration % log_freq == 0:
                lv = losses.tolist()
                if rank0:
                    print('Iter {}/{} ({} bpe) d_loss:{:.4f}, g_loss: {:.4f}, pow_loss: {:.4f}, den_loss: {:.4f} '
                          'btime: {:.4f} s, mbtime: {:.4f} s'.format(iteration, len(dloader) * opts.epoch, len(dloader),
                                                                     lv[0], lv[1] + lv[2] + lv[3], lv[2], lv[3],
                                                                     timings[-1], np.mean(timings)))
            if iteration % len(dloader) == 0 and rank0:
                self.G.save(self.save_path, iteration, saver=eoe_g_saver)
                self.D.save(self.save_path, iteration, saver=eoe_d_saver)
        self.last_losses = losses
        return timings

    def generate(self, inwav, z=None):
        """model.py:755-766: un-chunked inference on the utterance zero-padded to a multiple of 1024
        (make_divN pads a full extra block when already divisible, utils.py:26-38)."""
        self.G.eval()
        dev = next(super(Model, self.G).parameters()).device
        inwav = torch.as_tensor(inwav).float()
        ori_len = inwav.size(2)
        pad_num = (ori_len + 1024) - (ori_len % 1024) - ori_len
        p_wav = torch.cat((inwav, torch.zeros(inwav.size(0), inwav.size(1), pad_num)), dim=2).to(dev)
        with torch.no_grad():
            c_res, hall = self.infer_G(p_wav, z=z, ret_hid=True)
        c = c_res[0, 0, :ori_len].contiguous()
        out = torch.empty_like(c)
        if self.preemph > 0:
            _lib.call("sg_deemphasis", _p(c), ori_len, float(self.preemph), _p(out), _stream())
        else:
            out = c
        return out.cpu().numpy(), hall
