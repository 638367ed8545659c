"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the SEGAN+ hot path of santi-pdp/segan_pytorch.

This file is the *oracle*: a functional, dependency-free (torch CPU + numpy) restatement of the
reference algorithm, used exclusively by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs as the checker.  The product path (segan_pytorch_b200)
never imports it.

Parity status: PINNED.  tests/test_oracle_pinned.py checks every function here against
(a) the unmodified reference executed in the authoring container (oracle/ref_import.py) and
(b) the golden vectors that tests/golden/make_golden.py generated from that same reference
(the reference itself ships no tests / golden vectors -- SURVEY.md section 4).

All `file:line` citations are into santi-pdp/segan_pytorch (commit 0522387).

oneDNN is switched off for every call made here (SURVEY.md finding F1: the multi-threaded
oneDNN fp32 conv_transpose1d forward is wrong for the dec_blocks.0-2 shapes in this image).
"""
import contextlib
import math
import random as _pyrandom

import numpy as np
import torch
import torch.nn.functional as F

KWIDTH = 31
STRIDE = 4
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


_KEEP_ONEDNN = False


@contextlib.contextmanager
def oracle_mode():
    prev = torch.backends.mkldnn.enabled
    torch.backends.mkldnn.enabled = bool(_KEEP_ONEDNN and prev)
    try:
        yield
    finally:
        torch.backends.mkldnn.enabled = prev


@contextlib.contextmanager
def onednn_as_configured():
    """TIMING ONLY (bench.py cpu_baseline, BASELINE.md section 4): leave torch.backends.mkldnn as the user has it --
    what a reference user gets by default -- instead of switching it off.  Never used as the parity oracle: the
    oneDNN transposed convolution of this torch build is numerically wrong multi-threaded (SURVEY.md F1)."""
    global _KEEP_ONEDNN
    prev = _KEEP_ONEDNN
    _KEEP_ONEDNN = True
    try:
        yield
    finally:
        _KEEP_ONEDNN = prev


# --------------------------------------------------------------------------------------
# operand-precision control (tests only).  The CUDA path feeds its tensor cores 16-bit operands (fp16
# activations and weights, fp32 accumulation) and stores layer outputs in fp16.  Inside
# `with operand_precision(torch.float16):` the three contraction primitives below round their inputs, weights
# and outputs the same way while everything else stays the fp32 reference arithmetic: the distance between this
# control and the plain oracle is what the 16-bit operand FORMAT costs, independent of any kernel.  The parity
# tests print it next to the kernels' own error (DESIGN.md section 4).
# --------------------------------------------------------------------------------------
_OPERAND_DTYPE = None


@contextlib.contextmanager
def operand_precision(dtype):
    global _OPERAND_DTYPE
    prev = _OPERAND_DTYPE
    _OPERAND_DTYPE = dtype
    try:
        yield
    finally:
        _OPERAND_DTYPE = prev


def _q(t):
    """Round-trip through the control's operand dtype (straight-through for autograd)."""
    if _OPERAND_DTYPE is None or t is None:
        return t
    return t + (t.detach().to(_OPERAND_DTYPE).to(t.dtype) - t.detach())


# --------------------------------------------------------------------------------------
# blocks (segan/models/modules.py)
# --------------------------------------------------------------------------------------
def gconv_linear(x, weight, bias, stride=STRIDE):
    """GConv1DBlock up to the conv: reflect-pad then strided Conv1d.
    modules.py:91-99 -- P = (k//2 - 1, k//2) for stride > 1, (k//2, k//2) otherwise."""
    k = weight.shape[2]
    pad = (k // 2 - 1, k // 2) if stride > 1 else (k // 2, k // 2)
    xp = F.pad(_q(x), pad, mode="reflect")
    return _q(F.conv1d(xp, _q(weight), bias, stride=stride))


def prelu(a, w):
    """nn.PReLU(C): per-channel slope (modules.py:81,101; init 0)."""
    return F.prelu(a, w)


def batchnorm_train(a, gamma, beta, running_mean=None, running_var=None,
                    momentum=BN_MOMENTUM, eps=BN_EPS):
    """nn.BatchNorm1d in train mode (modules.py:11,100): biased variance normalises,
    unbiased variance feeds the running estimate.  Buffers are updated in place."""
    return F.batch_norm(a, running_mean, running_var, gamma, beta, True, momentum, eps)


def batchnorm_eval(a, gamma, beta, running_mean, running_var, eps=BN_EPS):
    return F.batch_norm(a, running_mean, running_var, gamma, beta, False, 0.0, eps)


def gdeconv_linear(x, weight, bias, stride=STRIDE):
    """GDeconv1DBlock up to the activation (modules.py:115-119,135-138):
    pad = max(0, (stride - k)//-2) (python floor division => 13 for k=31,s=4); bias always on;
    the last output sample is dropped when k is odd."""
    k = weight.shape[2]
    pad = max(0, (stride - k) // -2)
    h = F.conv_transpose1d(_q(x), _q(weight), bias, stride=stride, padding=pad)
    if weight.shape[1] > 1:
        h = _q(h)                             # hidden layers are stored in fp16; the waveform output is fp32
    if k % 2 != 0:
        h = h[:, :, :-1]
    return h


# --------------------------------------------------------------------------------------
# Generator (segan/models/generator.py:180-230), SEGAN+ defaults:
# skip_type='alpha', skip_merge='concat', no norm, PReLU, Tanh on the last decoder block
# --------------------------------------------------------------------------------------
def generator_forward(sd, x, z, ret_hid=False, skip_merge="concat"):
    """sd: state_dict with the reference key names (SURVEY.md App. B).  x: (B,1,T) z: (B,1024,T/1024).
    skip_merge: 'concat' (train.py default) or 'sum' (generator.py:72-74)."""
    n_enc = len([k for k in sd if k.startswith("enc_blocks.") and k.endswith("conv.weight")])
    n_dec = len([k for k in sd if k.startswith("dec_blocks.") and k.endswith("deconv.weight")])
    hall = {}
    skips = {}
    hi = x
    for l in range(n_enc):
        a = gconv_linear(hi, sd["enc_blocks.%d.conv.weight" % l], sd.get("enc_blocks.%d.conv.bias" % l))
        hi = prelu(a, sd["enc_blocks.%d.act.weight" % l])
        if l < n_enc - 1:
            skips[l] = a                      # PRE-activation (generator.py:185,191)
        if ret_hid:
            hall["enc_%d" % l] = hi
    hi = torch.cat((z, hi), dim=1)            # z first (generator.py:205)
    if ret_hid:
        hall["enc_zc"] = hi
    enc_idx = n_enc - 1
    for l in range(n_dec):
        if enc_idx in skips:                  # generator.py:212-219
            alpha = sd["alpha_%d.skip_k" % enc_idx]
            hj = skips[enc_idx]
            sk = alpha.repeat(hj.size(0), 1, hj.size(2)) * hj     # generator.py:68-69
            if skip_merge == "sum":
                hi = sk + hi                                      # generator.py:72-74
            else:
                hi = torch.cat((hi, sk), dim=1)                   # decoder first (generator.py:76)
        h = gdeconv_linear(hi, sd["dec_blocks.%d.deconv.weight" % l], sd["dec_blocks.%d.deconv.bias" % l])
        if l == n_dec - 1:
            hi = torch.tanh(h)                # act='Tanh' on the last block (generator.py:165-166)
        else:
            hi = prelu(h, sd["dec_blocks.%d.act.weight" % l])
        enc_idx -= 1
        if ret_hid:
            hall["dec_%d" % l] = hi
    return (hi, hall) if ret_hid else hi


# --------------------------------------------------------------------------------------
# Discriminator (segan/models/discriminator.py:150-194), pool_type='none', norm 'bnorm'
# --------------------------------------------------------------------------------------
def draw_phase_shifts(n_layers=5, phase_shift=5, rng=_pyrandom):
    """The two python-`random` draws per layer, in program order (discriminator.py:161-163).
    Returns a list of signed shifts: +s = roll right by s, -s = roll left by s."""
    out = []
    for _ in range(n_layers):
        shift = rng.randint(1, phase_shift)
        right = rng.random() > 0.5
        out.append(shift if right else -shift)
    return out


def phase_roll(h, s):
    """discriminator.py:165-172 -- circular shift along time, whole batch alike."""
    if s > 0:
        return torch.cat((h[:, :, -s:], h[:, :, :-s]), dim=2)
    if s < 0:
        s = -s
        return torch.cat((h[:, :, s:], h[:, :, :s]), dim=2)
    return h


def spectral_weight(sd, prefix, training, eps=1e-12):
    """torch.nn.utils.spectral_norm's weight (SpectralNorm.compute_weight), which build_norm_layer applies for
    norm_type='snorm' (modules.py:12-14; discriminator.py:118-121 for the head): parameters `weight_orig`, buffers
    `weight_u`, `weight_v` over weight.reshape(dim0, -1).  Training: ONE power iteration in place, without grad,
    v = normalize(W^T u), u = normalize(W v); then weight = weight_orig / sigma with sigma = u^T W v, differentiated
    with u, v held constant."""
    w, u, v = sd[prefix + "weight_orig"], sd[prefix + "weight_u"], sd[prefix + "weight_v"]
    wm = w.reshape(w.shape[0], -1)
    if training:
        with torch.no_grad():
            v.copy_(F.normalize(torch.mv(wm.detach().t(), u), dim=0, eps=eps))
            u.copy_(F.normalize(torch.mv(wm.detach(), v), dim=0, eps=eps))
        u, v = u.clone(), v.clone()
    sigma = torch.dot(u, torch.mv(wm, v))
    return w / sigma


def _weight(sd, prefix, training):
    """`<prefix>weight`, spectrally normalised when the layer carries weight_orig (norm_type='snorm')."""
    if prefix + "weight_orig" in sd:
        return spectral_weight(sd, prefix, training)
    return sd[prefix + "weight"]


def discriminator_forward(sd, x, shifts, training=True, ret_act=False):
    """x: (B,2,16384) = cat(candidate, noisy).  `sd` buffers running_mean/var/num_batches_tracked (bnorm) or
    weight_u / weight_v (snorm) are updated in place when training.  Returns logits (B,1).
    norm_type is read off the state dict: 'bnorm' layers carry norm.* keys, 'snorm' layers weight_orig/u/v and no
    norm layer (build_norm_layer returns None for it, modules.py:12-14)."""
    n_enc = len([k for k in sd if k.startswith("enc_blocks.") and (k.endswith("conv.weight") or
                                                                   k.endswith("conv.weight_orig"))])
    h = x
    acts = {}
    for l in range(n_enc):
        h = phase_roll(h, shifts[l])
        p = "enc_blocks.%d." % l
        a = gconv_linear(h, _weight(sd, p + "conv.", training), sd.get(p + "conv.bias"))
        if p + "norm.weight" not in sd:
            pass                                        # snorm / no norm: conv -> PReLU
        elif training:
            a = batchnorm_train(a, sd[p + "norm.weight"], sd[p + "norm.bias"],
                                sd[p + "norm.running_mean"], sd[p + "norm.running_var"])
            if p + "norm.num_batches_tracked" in sd:
                sd[p + "norm.num_batches_tracked"] += 1
        else:
            a = batchnorm_eval(a, sd[p + "norm.weight"], sd[p + "norm.bias"],
                               sd[p + "norm.running_mean"], sd[p + "norm.running_var"])
        h = prelu(a, sd[p + "act.weight"])
        acts["h_%d" % l] = h
    h = h.view(h.size(0), -1)                                     # discriminator.py:180-182
    h = F.linear(_q(h), _q(_weight(sd, "fc.0.", training)), sd["fc.0.bias"])
    h = F.prelu(h, sd["fc.1.weight"])
    h = F.linear(h, _weight(sd, "fc.2.", training), sd["fc.2.bias"])
    h = F.prelu(h, _weight(sd, "fc.3.", training))      # discriminator.py:121 normalises the PReLU(128) slope vector
    y = F.linear(h, sd["fc.4.weight"], sd["fc.4.bias"])
    acts["logit"] = y
    return (y, acts) if ret_act else y


# --------------------------------------------------------------------------------------
# optimiser (torch.optim.RMSprop defaults used at model.py:221-222)
# --------------------------------------------------------------------------------------
def rmsprop_step(param, grad, square_avg, lr, alpha=0.99, eps=1e-8):
    square_avg.mul_(alpha).addcmul_(grad, grad, value=1 - alpha)
    param.addcdiv_(grad, square_avg.sqrt().add_(eps), value=-lr)


def adam_step(param, grad, state, lr, betas=(0.0, 0.9), eps=1e-8):
    """torch.optim.Adam (amsgrad False, no weight decay) as used at model.py:224-225 (betas (0, 0.9)).
    state: dict with 'step', 'exp_avg', 'exp_avg_sq' (created on first use)."""
    if "step" not in state:
        state["step"], state["exp_avg"], state["exp_avg_sq"] = 0, torch.zeros_like(param), torch.zeros_like(param)
    state["step"] += 1
    b1, b2 = betas
    state["exp_avg"].mul_(b1).add_(grad, alpha=1 - b1)
    state["exp_avg_sq"].mul_(b2).addcmul_(grad, grad, value=1 - b2)
    bc1 = 1 - b1 ** state["step"]
    bc2 = 1 - b2 ** state["step"]
    denom = (state["exp_avg_sq"].sqrt() / math.sqrt(bc2)).add_(eps)
    param.addcdiv_(state["exp_avg"], denom, value=-lr / bc1)


# --------------------------------------------------------------------------------------
# SEGAN+ train step (segan/models/model.py:283-321)
# --------------------------------------------------------------------------------------
TRAINABLE_SUFFIXES = ("weight", "weight_orig", "bias", "skip_k")


def _trainable(sd):
    return [k for k in sd if k.endswith(TRAINABLE_SUFFIXES) and sd[k].dtype.is_floating_point
            and "running_" not in k]


def segan_train_step(sdG, sdD, sqG, sqD, clean, noisy, z, shifts3, l1_weight=100.0,
                     g_lr=5e-5, d_lr=5e-5):
    """One LSGAN + L1 step.  sdG/sdD: state dicts (updated in place), sqG/sqD: RMSprop
    square_avg dicts (updated in place), clean/noisy: (B,1,16384), z: (B,1024,16),
    shifts3: three lists of 5 signed shifts (D(real), D(fake.detach), D(fake) -- the order in
    which the reference consumes python `random`).
    Returns dict(losses..., gradsD, gradsG, Genh)."""
    with oracle_mode():
        pD = {k: sdD[k].detach().clone().requires_grad_(True) for k in _trainable(sdD)}
        pG = {k: sdG[k].detach().clone().requires_grad_(True) for k in _trainable(sdG)}

        def fullD():
            d = dict(sdD)
            d.update(pD)
            return d

        def fullG():
            d = dict(sdG)
            d.update(pG)
            return d

        B = clean.size(0)
        # model.py:295
        Genh = generator_forward(fullG(), noisy, z)
        # (1) D real, model.py:297-299
        d_real = discriminator_forward(fullD(), torch.cat((clean, noisy), 1), shifts3[0])
        d_real_loss = F.mse_loss(d_real.view(-1), torch.ones(B))
        # (2) D fake, model.py:303-306
        d_fake = discriminator_forward(fullD(), torch.cat((Genh.detach(), noisy), 1), shifts3[1])
        d_fake_loss = F.mse_loss(d_fake.view(-1), torch.zeros(B))
        gD = torch.autograd.grad(d_real_loss + d_fake_loss, list(pD.values()))
        gradsD = dict(zip(pD.keys(), gD))
        with torch.no_grad():                 # Dopt.step(), model.py:308
            for k in pD:
                rmsprop_step(pD[k], gradsD[k], sqD[k], d_lr)
        # (3) G update with the UPDATED D, model.py:313-321
        d_fake_ = discriminator_forward(fullD(), torch.cat((Genh, noisy), 1), shifts3[2])
        g_adv_loss = F.mse_loss(d_fake_.view(-1), torch.ones(B))
        g_l1_loss = l1_weight * F.l1_loss(Genh, clean)
        gG = torch.autograd.grad(g_adv_loss + g_l1_loss, list(pG.values()))
        gradsG = dict(zip(pG.keys(), gG))
        with torch.no_grad():
            for k in pG:
                rmsprop_step(pG[k], gradsG[k], sqG[k], g_lr)
            for k in pD:
                sdD[k].copy_(pD[k])
            for k in pG:
                sdG[k].copy_(pG[k])
        return dict(d_real_loss=float(d_real_loss), d_fake_loss=float(d_fake_loss),
                    g_adv_loss=float(g_adv_loss), g_l1_loss=float(g_l1_loss),
                    gradsD=gradsD, gradsG=gradsG, Genh=Genh.detach())


# --------------------------------------------------------------------------------------
# WSEGAN step (segan/models/model.py:572-669) with --misalign_pair, device agnostic.
# --------------------------------------------------------------------------------------
def stft_logpow(x, n_fft=2048):
    """model.py:640-646: torch.stft(n_fft, hop 160, win 320 (rectangular, centre-padded to
    n_fft), normalized=True) -> |X| (norm over re/im) -> 10*log10(|X|^2 + 10e-20)."""
    n_fft = min(x.size(-1), n_fft)
    st = torch.stft(x.squeeze(1), n_fft=n_fft, hop_length=160, win_length=320, normalized=True,
                    return_complex=True)
    mod = torch.norm(torch.view_as_real(st), 2, dim=3)
    return 10 * torch.log10(mod ** 2 + 10e-20)


def interferer_squares(picks, length):
    """model.py:606-622: per sample a square wave a * square(2 pi f t), t = linspace(0, 2, 32000), cut to
    `length`; picks = [(f, a), ...] in the order `random.choice(freqs)`, `random.choice(amps)` are drawn."""
    from scipy import signal
    t = np.linspace(0, 2, 32000)
    sq = [torch.FloatTensor((a_ * signal.square(2 * np.pi * f_ * t))[:length].reshape((1, -1))) for f_, a_ in picks]
    return torch.cat(sq, dim=0).unsqueeze(1)


def wsegan_train_step(sdG, sdD, optG, optD, clean, noisy, z, shifts4, perm, pow_weight=0.001,
                      l1_weight=100.0, additive_mask=None, lr=5e-5, betas=(0.0, 0.9), opt="rmsprop",
                      interf=None, vanilla_gan=False):
    """One WSEGAN step (model.py:572-669).  shifts4: the D passes in the order model.py consumes python `random`:
    D(real), D(fake.detach), [D(clean, shuffled) when perm is given (misalign_pair, :598-604)],
    [D(clean + interf, noisy) when `interf` (the squares of :606-622) is given], D(fake).  vanilla_gan: BCE with
    logits instead of MSE (:583-586).  optG/optD: dict name -> state (the square_avg tensor for rmsprop; a dict
    filled by adam_step for opt='adam', model.py:224-225)."""
    cost = F.binary_cross_entropy_with_logits if vanilla_gan else F.mse_loss

    def opt_step(p, g, states, k):
        if opt == "adam":
            adam_step(p, g, states.setdefault(k, {}), lr, betas)
        else:
            rmsprop_step(p, g, states[k], lr)
    with oracle_mode():
        pD = {k: sdD[k].detach().clone().requires_grad_(True) for k in _trainable(sdD)}
        pG = {k: sdG[k].detach().clone().requires_grad_(True) for k in _trainable(sdG)}
        fullD = lambda: {**sdD, **pD}
        fullG = lambda: {**sdG, **pG}
        sh = iter(shifts4)
        d_real = discriminator_forward(fullD(), torch.cat((clean, noisy), 1), next(sh))
        d_real_loss = cost(d_real, torch.ones_like(d_real))
        Genh = generator_forward(fullG(), noisy, z)
        d_fake = discriminator_forward(fullD(), torch.cat((Genh.detach(), noisy), 1), next(sh))
        d_fake_loss = cost(d_fake, torch.zeros_like(d_fake))
        d_weight = 0.5
        d_loss = d_fake_loss + d_real_loss
        if perm is not None:
            clean_shuf = clean[perm]
            d_shuf = discriminator_forward(fullD(), torch.cat((clean, clean_shuf), 1), next(sh))
            d_weight = 1.0 / 3
            d_loss = d_loss + cost(d_shuf, torch.zeros_like(d_shuf))
        if interf is not None:
            d_int = discriminator_forward(fullD(), torch.cat((clean + interf, noisy), 1), next(sh))
            d_weight = 1.0 / 4                         # model.py:626: set to 1/4 whether or not misalign is on
            d_loss = d_loss + cost(d_int, torch.zeros_like(d_int))
        d_loss = d_weight * d_loss
        gD = dict(zip(pD.keys(), torch.autograd.grad(d_loss, list(pD.values()))))
        with torch.no_grad():
            for k in pD:
                opt_step(pD[k], gD[k], optD, k)
        d_fake_ = discriminator_forward(fullD(), torch.cat((Genh, noisy), 1), next(sh))
        g_adv = cost(d_fake_, torch.ones_like(d_fake_))
        pow_loss = pow_weight * F.l1_loss(stft_logpow(Genh), stft_logpow(clean))
        G_cost = g_adv + pow_loss
        den_loss = torch.zeros(1)
        if l1_weight > 0:
            mask = torch.zeros(clean.size(0), 1, clean.size(2)) if additive_mask is None else additive_mask
            den_loss = l1_weight * F.l1_loss(Genh * mask, clean * mask)
            G_cost = G_cost + den_loss
        gG = dict(zip(pG.keys(), torch.autograd.grad(G_cost, list(pG.values()))))
        with torch.no_grad():
            for k in pG:
                opt_step(pG[k], gG[k], optG, k)
            for k in pD:
                sdD[k].copy_(pD[k])
            for k in pG:
                sdG[k].copy_(pG[k])
        return dict(d_loss=float(d_loss), g_adv_loss=float(g_adv), pow_loss=float(pow_loss),
                    den_loss=float(den_loss), gradsD=gD, gradsG=gG, Genh=Genh.detach())


# --------------------------------------------------------------------------------------
# waveform contract (segan/datasets/se_dataset.py:108-126) and chunked inference
# --------------------------------------------------------------------------------------
def normalize_wave_minmax(x):
    return (2. / 65535.) * (x - 32767.) + 1.        # se_dataset.py:108-109


def pre_emphasize(x, coef=0.95):
    if coef <= 0:
        return x
    x0 = np.reshape(x[0], (1,))
    diff = x[1:] - coef * x[:-1]
    return np.concatenate((x0, diff), axis=0)        # se_dataset.py:111-117


def de_emphasize(y, coef=0.95):
    """se_dataset.py:119-126: first-order IIR, float32 state, sequential."""
    if coef <= 0:
        return y
    x = np.zeros(y.shape[0], dtype=np.float32)
    x[0] = y[0]
    c = np.float32(coef)
    prev = x[0]
    yl = y.astype(np.float32)
    for n in range(1, y.shape[0]):
        prev = np.float32(c * prev + yl[n])
        x[n] = prev
    return x


def segan_generate(sdG, inwav, z, preemph=0.95, N=16384):
    """SEGAN.generate (model.py:116-157): chunk into N-sample windows (zero-pad the last),
    same z for every chunk, strip pad, concatenate, de-emphasise.  inwav: (1,1,T) tensor."""
    with oracle_mode():
        outs = []
        T = inwav.shape[2]
        for beg in range(0, T, N):
            length = min(N, T - beg)
            x = torch.zeros(1, 1, N)
            x[0, 0, :length] = inwav[0, 0, beg:beg + length]
            y = generator_forward(sdG, x, z)
            outs.append(y[0, 0, :length].detach().numpy())
        c_res = np.concatenate(outs)
        return de_emphasize(c_res, preemph)


# --------------------------------------------------------------------------------------
# algorithmic work (SURVEY.md App. A): used by bench.py for the roofline arithmetic
# --------------------------------------------------------------------------------------
def flops_per_window():
    fm = [64, 128, 256, 512, 1024]
    L = 16384
    conv = []
    cin = 1
    l = L
    for c in fm:
        l //= 4
        conv.append(2 * cin * c * KWIDTH * l)
        cin = c
    g_enc = sum(conv)
    d_enc = sum(conv) + conv[0]           # Cin = 2 on the first D layer
    dec_in = [2048, 1024, 512, 256, 128]
    dec_out = [512, 256, 128, 64, 1]
    lin = 16
    g_dec = 0
    for ci, co in zip(dec_in, dec_out):
        g_dec += 2 * ci * co * KWIDTH * lin
        lin *= 4
    fc = 2 * (16384 * 256 + 256 * 128 + 128)
    return dict(G_fwd=g_enc + g_dec, D_fwd=d_enc + fc)
