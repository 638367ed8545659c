"""Drop-in `Discriminator` (reference: segan/models/discriminator.py:65-194).

conv -> BatchNorm1d -> PReLU tower with the random circular phase shift before every layer
(two python-`random` draws per layer, also in eval mode -- discriminator.py:160-172) and the
16384-256-128-1 PReLU head (pool_type 'none'), or one of the pooled heads 'conv' / 'gmax' / 'gavg' / 'mlp'
(discriminator.py:122-146; 'mlp' gives one logit per position, (B, 1, L / 4^n_layers)).  Arithmetic: segan_pytorch_b200.engine.DiscriminatorEngine."""
import random

import torch
import torch.nn as nn

from .core import Model
from .modules import GConv1DBlock
from ... import engine as _engine


def draw_phase_shifts(n_layers, phase_shift):
    """Signed shifts (+ right / - left) in the reference's draw order (discriminator.py:161-163)."""
    out = []
    for _ in range(n_layers):
        if phase_shift is None:
            out.append(0)
            continue
        shift = random.randint(1, phase_shift)
        right = random.random() > 0.5
        out.append(shift if right else -shift)
    return out


class _DiscriminatorFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, eng, x, shifts, training, *params):
        x0 = x[:, 0:1, :].contiguous()
        x1 = x[:, 1:2, :].contiguous()
        logit, ectx = eng.forward(x0, x1, shifts, training=training, fresh=True)
        ctx.eng, ctx.ectx = eng, ectx
        eng._last_ctx = ectx
        return logit

    @staticmethod
    def backward(ctx, g_logit):
        eng, ectx = ctx.eng, ctx.ectx
        gx = None
        g0 = g1 = None
        ctx.need_x = ctx.needs_input_grad[1]
        if ctx.need_x:
            B, L = ectx["B"], ectx["L"]
            g0 = torch.zeros(B, 1, L, dtype=torch.float32, device=g_logit.device)
            g1 = torch.zeros(B, 1, L, dtype=torch.float32, device=g_logit.device)
        eng.grad.zero_()
        eng._alpha_fixed = False
        eng.backward(ectx, 0.0, 1.0, param_grads=True, input_grad=g0, input_grad1=g1,
                     g_logit=g_logit.contiguous().float().view(-1))
        inv = 1.0 / _engine.LOSS_SCALE            # the engine's gradients carry the fp16 loss scale
        if ctx.need_x:
            gx = torch.cat((g0, g1), dim=1) * inv
        grads = []
        for n, p in eng.module.named_parameters():
            grads.append(eng.grad_of(n) if p.requires_grad else None)      # reference layout, true units
        return (None, gx, None, None) + tuple(grads)


class Discriminator(Model):

    def __init__(self, ninputs, fmaps, kwidth, poolings, pool_type='none', pool_slen=None, norm_type='bnorm',
                 bias=True, phase_shift=None, sinc_conv=False):
        super().__init__(name='Discriminator')
        self.phase_shift = phase_shift
        if phase_shift is not None:
            assert isinstance(phase_shift, int), type(phase_shift)
            assert phase_shift > 1, phase_shift
        if pool_slen is None:
            raise ValueError('Please specify D network pool seq len (pool_slen) in the end of the conv '
                             'stack: [inp_len // (total_pooling_factor)]')
        if sinc_conv:
            raise NotImplementedError("--sinc_conv is a SURVEY.md 8(f)-N4 'next' row; not built yet")
        ninp = ninputs
        self.enc_blocks = nn.ModuleList()
        for pi, (fmap, pool) in enumerate(zip(fmaps, poolings), start=1):
            self.enc_blocks.append(GConv1DBlock(ninp, fmap, kwidth, stride=pool, bias=bias, norm_type=norm_type))
            ninp = fmap
        self.pool_type = pool_type
        self.pool_slen = pool_slen                     # positions after the tower (16 for L = 16384)
        if pool_type == 'none':
            pool_slen *= fmaps[-1]
            self.fc = nn.Sequential(
                nn.Linear(pool_slen, 256),
                nn.PReLU(256),
                nn.Linear(256, 128),
                nn.PReLU(128),
                nn.Linear(128, 1)
            )
            if norm_type == 'snorm':                   # discriminator.py:118-121 (incl. the PReLU(128) slope vector)
                torch.nn.utils.spectral_norm(self.fc[0])
                torch.nn.utils.spectral_norm(self.fc[2])
                torch.nn.utils.spectral_norm(self.fc[3])
        elif pool_type == 'conv':                      # discriminator.py:122-127: pool_slen is NOT scaled by C here
            self.pool_conv = nn.Conv1d(fmaps[-1], 1, 1)
            self.fc = nn.Linear(pool_slen, 1)
            if norm_type == 'snorm':
                torch.nn.utils.spectral_norm(self.pool_conv)
                torch.nn.utils.spectral_norm(self.fc)
        elif pool_type in ('gmax', 'gavg'):            # discriminator.py:128-137 (Linear's third argument: bias)
            if pool_type == 'gmax':
                self.gmax = nn.AdaptiveMaxPool1d(1)
            else:
                self.gavg = nn.AdaptiveAvgPool1d(1)
            self.fc = nn.Linear(fmaps[-1], 1, 1)
            if norm_type == 'snorm':
                torch.nn.utils.spectral_norm(self.fc)
        elif pool_type == 'mlp':                       # discriminator.py:138-146: mlp.2 is not normalised
            self.mlp = nn.Sequential(
                nn.Conv1d(fmaps[-1], fmaps[-1], 1),
                nn.PReLU(fmaps[-1]),
                nn.Conv1d(fmaps[-1], 1, 1)
            )
            if norm_type == 'snorm':
                torch.nn.utils.spectral_norm(self.mlp[0])
                torch.nn.utils.spectral_norm(self.mlp[1])
        else:
            raise TypeError('Unrecognized pool type: ', pool_type)
        self.fmaps = list(fmaps)
        self.bias = bias
        self.norm_type = norm_type
        self._served = (ninputs == 2 and norm_type in ('bnorm', 'snorm') and bias and _engine.kwidth_served(kwidth)
                        and all(p == 4 for p in poolings)
                        and fmaps[0] == 64 and all(f % 64 == 0 for f in fmaps) and len(fmaps) >= 2)
        self._unserved = ("this Discriminator configuration is outside the built hot path "
                          "(SEGAN+ defaults: 2 input channels, bnorm or snorm, kernel width 4-32, stride 4)")
        if not _engine.kwidth_served(kwidth):
            self._unserved = ("kernel width kwidth=%r is not served: it must be an integer in 4-32 (the first layer's "
                              "im2col holds 32 taps per input channel)" % (kwidth,))
        self._engine = None

    @property
    def engine(self):
        if not self._served:
            raise NotImplementedError(self._unserved)
        if self._engine is None:
            self._engine = _engine.DiscriminatorEngine(self)
        return self._engine

    # The big weights' nn.Parameters are reference-layout mirrors of the engine's packed fp32 masters: anything that
    # reads or moves the parameters wholesale first refreshes them (a no-op unless an optimiser step intervened).
    def state_dict(self, *args, **kwargs):
        if self._engine is not None:
            self._engine.sync_to_reference()
        return super().state_dict(*args, **kwargs)

    def _apply(self, fn, *args, **kwargs):
        if getattr(self, '_engine', None) is not None:
            self._engine.sync_to_reference()
        return super()._apply(fn, *args, **kwargs)

    def forward(self, x, shifts=None):
        eng = self.engine
        _engine._require_cuda(x)
        if shifts is None:
            shifts = draw_phase_shifts(len(self.enc_blocks), self.phase_shift)
        eng.bind()
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad
                                                                         for p in super().parameters()))
        if needs_grad:
            params = [p for _, p in self.named_parameters()]
            y = _DiscriminatorFn.apply(eng, x, shifts, self.training, *params)
            ectx = eng._last_ctx
            eng._last_ctx = None
        else:
            y, ectx = eng.forward(x[:, 0:1, :].contiguous(), x[:, 1:2, :].contiguous(), shifts,
                                  training=self.training)
        int_act = _LazyActs(eng, ectx)
        if self.pool_type == 'conv':        # pool_conv output (B, Lq), discriminator.py:176-178; its buffer is reused
            int_act['avg_conv_h'] = ectx["pooled"].clone()
        int_act['logit'] = y
        return y, int_act


class _LazyActs(dict):
    """`int_act` of discriminator.py:158-193: h_{i} converted to fp32 NCL only when looked up."""

    def __init__(self, eng, ectx):
        super().__init__()
        self._eng, self._ectx = eng, ectx

    def __missing__(self, key):
        if key.startswith('h_'):
            import ctypes as C
            from ... import _lib
            l = int(key[2:])
            ectx, eng = self._ectx, self._eng
            B, Lq, C_ = ectx["B"], ectx["Lq"][l], eng.fmaps[l]
            halo = 16 if l < eng.nl - 1 else 0
            hp = ectx["hp"][l][:, halo:halo + Lq, :].contiguous()
            roll = ectx["shifts"][l + 1] if l < eng.nl - 1 else 0
            out = torch.empty(B, C_, Lq, dtype=torch.float32, device=hp.device)
            _lib.call("sg_nlc_to_ncl", C.c_void_p(hp.data_ptr()), _lib.SG_F16, B, C_, Lq,
                      C.c_void_p(out.data_ptr()), _engine._stream())
            out = torch.roll(out, -roll, dims=2)      # hp is stored already shifted for the next layer
            self[key] = out
            return out
        raise KeyError(key)
