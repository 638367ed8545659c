"""Drop-in `Generator` (reference: segan/models/generator.py:18-230).

Same constructor signature, same `forward(x, z=None, ret_hid=False)` contract, same state-dict
keys; the arithmetic runs in libsegan_b200.so (segan_pytorch_b200.engine.GeneratorEngine).  Served: alpha / constant /
conv skips with concat or sum merge, skip=False, no_z=True, any z_dim that is a positive multiple of 64,
norm_type None or 'snorm' (spectrally normalised encoder convs and decoder deconvs), and every kernel width
4 <= k <= 32 for each encoder conv (kwidth) and decoder deconv (dec_kwidth)."""
import torch
import torch.nn as nn

from .core import Model
from .modules import GConv1DBlock, GDeconv1DBlock
from ... import engine as _engine


class GSkip(nn.Module):
    """Skip connection of one encoder level (generator.py:18-78): a learnable per-channel scale (skip_type 'alpha',
    or 'constant' = frozen) or a stride-1 Conv1d(C, C, kwidth, padding kwidth//2) (skip_type 'conv'), with merge
    'concat' (ckpt_segan+/train.opts) or 'sum' (generator.py:72-74).  All three are served by the kernels; the
    conv needs an odd kwidth <= 33."""

    def __init__(self, skip_type, size, skip_init, skip_dropout=0, merge_mode='sum', kwidth=11, bias=True):
        super().__init__()
        self.merge_mode = merge_mode
        if skip_type in ('alpha', 'constant'):
            if skip_init == 'zero':
                alpha_ = torch.zeros(size)
            elif skip_init == 'randn':
                alpha_ = torch.randn(size)
            elif skip_init == 'one':
                alpha_ = torch.ones(size)
            else:
                raise TypeError('Unrecognized alpha init scheme: ', skip_init)
            self.skip_k = nn.Parameter(alpha_.view(1, -1, 1))
            if skip_type == 'constant':
                self.skip_k.requires_grad = False
        elif skip_type == 'conv':
            if not _engine.skipconv_served(kwidth):
                raise NotImplementedError(
                    "skip_type='conv' needs an odd skip_kwidth <= 33 (got %r): an even width makes the skip one "
                    "sample longer than the decoder input it is merged with (padding kwidth//2 on both ends), and "
                    "wider kernels do not fit the tap-GEMMs' 9-tap table" % (kwidth,))
            self.skip_k = nn.Conv1d(size, size, kwidth, stride=1, padding=kwidth // 2 if kwidth > 1 else 0,
                                    bias=bias)
        else:
            raise TypeError('Unrecognized GSkip scheme: ', skip_type)
        self.skip_type = skip_type
        if skip_dropout > 0:
            raise NotImplementedError("skip_dropout > 0 is not built yet (non-default)")

    def __repr__(self):
        if self.skip_type == 'conv':
            return super().__repr__()
        return self._get_name() + ('(Alpha(1))' if self.skip_type == 'alpha' else '(Constant(1))')


class _GeneratorFn(torch.autograd.Function):
    """Whole-network autograd node: forward / backward are the fused kernel pipelines."""

    @staticmethod
    def forward(ctx, eng, x, z, training, *params):
        y, ectx = eng.forward(x, z, fresh=True, training=training)
        ctx.eng, ctx.ectx = eng, ectx
        eng._last_ctx = ectx
        ctx.names = [n for n, p in eng.module.named_parameters()]
        return y

    @staticmethod
    def backward(ctx, gy):
        eng = ctx.eng
        scale = _engine.LOSS_SCALE                # the engine's gradient tensors carry the fp16 loss scale
        eng.backward(ctx.ectx, gy * scale if scale != 1.0 else gy)
        grads = []
        for n, p in eng.module.named_parameters():
            grads.append(eng.grad_of(n) if p.requires_grad else None)      # reference layout, true units
        return (None, None, None, None) + tuple(grads)


class Generator(Model):

    def __init__(self, ninputs, fmaps, kwidth, poolings, dec_fmaps=None, dec_kwidth=None, dec_poolings=None,
                 z_dim=None, no_z=False, skip=True, bias=False, skip_init='one', skip_dropout=0,
                 skip_type='alpha', norm_type=None, skip_merge='sum', skip_kwidth=11, name='Generator'):
        super().__init__(name=name)
        self.skip = skip
        self.bias = bias
        self.no_z = no_z
        self.z_dim = z_dim
        self.enc_blocks = nn.ModuleList()
        assert isinstance(fmaps, list), type(fmaps)
        assert isinstance(poolings, list), type(poolings)
        if isinstance(kwidth, int):
            kwidth = [kwidth] * len(fmaps)
        assert isinstance(kwidth, list), type(kwidth)
        skips = {}
        ninp = ninputs
        for pi, (fmap, pool, kw) in enumerate(zip(fmaps, poolings, kwidth), start=1):
            if skip and pi < len(fmaps):
                gskip = GSkip(skip_type, fmap, skip_init, skip_dropout, merge_mode=skip_merge,
                              kwidth=skip_kwidth, bias=bias)
                l_i = pi - 1
                skips[l_i] = {'alpha': gskip}
                setattr(self, 'alpha_{}'.format(l_i), skips[l_i]['alpha'])
            self.enc_blocks.append(GConv1DBlock(ninp, fmap, kw, stride=pool, bias=bias, norm_type=norm_type))
            ninp = fmap
        self.skips = skips
        if not no_z and z_dim is None:
            z_dim = fmaps[-1]
        if not no_z:
            ninp += z_dim
        if dec_fmaps is None:
            dec_fmaps = fmaps[::-1][1:] + [1]
        else:
            assert isinstance(dec_fmaps, list), type(dec_fmaps)
        if dec_poolings is None:
            dec_poolings = poolings[:]
        else:
            assert isinstance(dec_poolings, list), type(dec_poolings)
        self.dec_poolings = dec_poolings
        if dec_kwidth is None:
            dec_kwidth = kwidth[:]
        elif isinstance(dec_kwidth, int):
            dec_kwidth = [dec_kwidth] * len(dec_fmaps)
        assert isinstance(dec_kwidth, list), type(dec_kwidth)
        self.dec_blocks = nn.ModuleList()
        for pi, (fmap, pool, kw) in enumerate(zip(dec_fmaps, dec_poolings, dec_kwidth), start=1):
            if skip and pi > 1 and pool > 1:
                if skip_merge == 'concat':
                    ninp *= 2
            act = 'Tanh' if pi >= len(dec_fmaps) else None
            if pool > 1:
                dec_block = GDeconv1DBlock(ninp, fmap, kw, stride=pool, norm_type=norm_type, bias=bias, act=act)
            else:
                dec_block = GConv1DBlock(ninp, fmap, kw, stride=1, bias=bias, norm_type=norm_type)
            self.dec_blocks.append(dec_block)
            ninp = fmap
        # ---- what the kernels serve (everything else is a "next" row, SURVEY.md 8f-N4)
        self.enc_fmaps = list(fmaps)
        self.skip_merge = skip_merge
        self.skip_type, self.skip_kwidth = skip_type, skip_kwidth
        # no_z / skip=False / z_dim only change the channel counts the decoder's GEMMs contract over; z must be a
        # whole number of 64-channel K blocks so that the z / code split of block 0 falls on a block boundary
        self._served = (ninputs == 1 and (not skip or (skip_merge in ('concat', 'sum')
                                                       and (skip_type in ('alpha', 'constant')
                                                            or (skip_type == 'conv'
                                                                and _engine.skipconv_served(skip_kwidth)))))
                        and norm_type in (None, 'snorm')
                        and all(_engine.kwidth_served(k) for k in list(kwidth) + list(dec_kwidth))
                        and all(p == 4 for p in poolings) and all(p == 4 for p in dec_poolings)
                        and list(dec_fmaps) == fmaps[::-1][1:] + [1]
                        and all(f % 64 == 0 for f in fmaps) and fmaps[0] == 64)
        self.norm_type = norm_type
        self._unserved = None if self._served else ("this Generator configuration is outside the built hot path "
                                                     "(SEGAN+ layout: kernel widths 4-32, stride 4, norm_type None "
                                                     "or 'snorm', fmaps 64..)")
        if not all(_engine.kwidth_served(k) for k in list(kwidth) + list(dec_kwidth)):
            self._unserved = ("kernel widths kwidth=%r / dec_kwidth=%r are not served: every width must be an integer "
                              "in 4-32 (the waveform-end im2col holds 32 taps per channel; below 4 the transposed "
                              "conv does not give 4x its input length)" % (list(kwidth), list(dec_kwidth)))
        if norm_type == 'bnorm':
            self._unserved = ("norm_type='bnorm' is not served for the Generator: the Generator's kernels have no "
                              "BatchNorm between a convolution and its PReLU (norm_type None and 'snorm' are served)")
        if self.z_dim is None and not no_z:
            self.z_dim = fmaps[-1]
        if self._served and not no_z and not (isinstance(self.z_dim, int) and self.z_dim > 0 and self.z_dim % 64 == 0):
            self._served = False
            self._unserved = ("z_dim=%r is not served: it must be a positive multiple of 64, so that the split "
                              "between z and the code in decoder block 0 falls on a 64-channel K block of the "
                              "tensor-core GEMM" % (self.z_dim,))
        self.z_device = 'cpu'   # 'cpu' = draw z on the CPU generator like generator.py:197-199; 'cuda' = on device
        self._engine = None

    # -- engine ---------------------------------------------------------------------------------
    @property
    def engine(self):
        if not self._served:
            raise NotImplementedError(self._unserved)
        if self._engine is None:
            self._engine = _engine.GeneratorEngine(self)
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

    def forward(self, x, z=None, ret_hid=False):
        eng = self.engine
        _engine._require_cuda(x)
        B, _, L = x.shape
        if self.no_z:
            z = None                     # generator.py:193-208: a passed z is ignored, none is drawn, self.z never set
        else:
            if z is None:
                code_len = L // (4 ** len(self.enc_blocks))
                if self.z_device == 'cpu':
                    z = torch.randn(B, self.z_dim, code_len).to(x.device)      # generator.py:197-199
                else:
                    z = torch.randn(B, self.z_dim, code_len, device=x.device)
            if len(z.size()) != 3:
                raise ValueError('len(z.size) {} != len(hi.size) {}'.format(len(z.size()), 3))
            if not hasattr(self, 'z'):
                self.z = z                                                   # generator.py:203-204
        eng.bind()
        if torch.is_grad_enabled() and any(p.requires_grad for p in super().parameters()):
            params = [p for _, p in self.named_parameters()]
            y = _GeneratorFn.apply(eng, x, z, self.training, *params)
            ectx = eng._last_ctx          # hidden activations are exposed detached (inspection only)
            eng._last_ctx = None
        else:
            # inference: no bf16 twins for weight gradients
            y, ectx = eng.forward(x, z, twins=False, training=self.training)
        if ret_hid:
            # ret_hid may be an iterable of keys (additive): only those activations are converted to NCL
            only = None if ret_hid is True else set(ret_hid)
            return y, eng.hidden_ncl(ectx, only)
        return y
