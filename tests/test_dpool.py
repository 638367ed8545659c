"""Discriminators with a pooled head (pool_type 'conv' / 'gmax' / 'gavg' / 'mlp', discriminator.py:122-146) on the CPU:
the head-aware oracle against the reference's golden logits, avg_conv_h and gradients (tests/golden/dpool_heads.npz),
seeded construction of the drop-in modules, the engine's gradient-bucket layout for each head, and SEGAN's refusal
of the mlp head's per-position logits."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import segan_oracle as O
from segan_pytorch_b200 import engine as E
from segan_pytorch_b200.segan.models import Discriminator
from tests import dpool_oracle as DO
from tests.util import build_segan, cpu_state, golden, load_opts, max_abs, sd_sha, seed_all

GOLD = "dpool_heads.npz"
HEADS = ("conv", "gmax", "gavg", "mlp")
NORMS = ("bnorm", "snorm")
TRAIN_SEED, EVAL_SEED = 5, 6


def pooled_discriminator(head, norm, seed=111):
    seed_all(seed)
    return Discriminator(2, [64, 128, 256, 512, 1024], 31, [4] * 5, pool_type=head, pool_slen=16, norm_type=norm,
                         phase_shift=5)


def golden_input(g):
    return 0.3 * torch.from_numpy(g["xr"])


@pytest.fixture(scope="module", autouse=True)
def _threads():
    torch.set_num_threads(max(1, min(8, torch.get_num_threads())))


@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("head", HEADS)
def test_discriminator_matches_reference_keys_and_init(head, norm):
    g = golden(GOLD)
    p = "%s.%s." % (head, norm)
    D = pooled_discriminator(head, norm)
    sd = D.state_dict()
    assert list(sd.keys()) == [str(k) for k in g[p + "keys"]]
    assert np.array_equal(np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()]), g[p + "shapes"])
    assert sd_sha(sd) == str(g[p + "sha_D"])
    assert D._served
    # the head is built after the tower (the order fixes the seeded init)
    names = [n for n, _ in D.named_parameters()]
    assert names.index("enc_blocks.4.act.weight") < names.index("mlp.2.bias" if head == "mlp" else "fc.bias")


@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("head", HEADS)
def test_segan_and_wsegan_discriminators_match_reference_init(head, norm):
    from segan_pytorch_b200.segan.models import WSEGAN
    g = golden(GOLD)
    p = "%s.%s." % (head, norm)
    s = build_segan(dpool_type=head, dnorm_type=norm)
    assert sd_sha(s.D.state_dict()) == str(g[p + "sha_segan_D"])
    seed_all(111)
    w = WSEGAN(load_opts(wsegan=True, misalign_pair=True, dpool_type=head, dnorm_type=norm))
    assert sd_sha(w.D.state_dict()) == str(g[p + "sha_wsegan_D"])


def oracle_pass(sd, x, head, training, seed):
    random.seed(seed)
    shifts = O.draw_phase_shifts(5, 5)
    return DO.discriminator_forward(sd, x, shifts, training=training, ret_act=True, pool_type=head)


@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("head", HEADS)
def test_oracle_vs_golden(head, norm):
    """Train pass (logits, avg_conv_h, sampled gradients of mse(logits, 1)) then eval pass, as the fixture ran them."""
    g = golden(GOLD)
    p = "%s.%s." % (head, norm)
    x = golden_input(g)
    sd = cpu_state(pooled_discriminator(head, norm))
    keys = [str(k) for k in g[p + "grad_keys"]]
    sfx = "_orig" if norm == "snorm" else ""
    if head == "mlp":       # mlp.2 is not normalised (discriminator.py:144-146)
        assert {"mlp.0.weight" + sfx, "mlp.1.weight" + sfx, "mlp.2.weight", "mlp.2.bias"} <= set(keys)
    else:
        assert "fc.weight" + sfx in keys and "fc.bias" in keys
    assert (head == "conv") == any(k.startswith("pool_conv.") for k in keys)
    with O.oracle_mode():
        pr = {k: sd[k].clone().requires_grad_(True) for k in keys}
        y, act = oracle_pass({**sd, **pr}, x, head, True, TRAIN_SEED)
        assert tuple(y.shape) == ((3, 1, 16) if head == "mlp" else (3, 1))
        loss = F.mse_loss(y, torch.ones_like(y))          # mlp: a mean over the B * Lq logits
        grads = dict(zip(keys, torch.autograd.grad(loss, [pr[k] for k in keys])))
        assert max_abs(y.detach(), g[p + "y_train"]) <= 1e-5
        assert abs(float(loss.detach()) - float(g[p + "loss"])) <= 1e-5 * max(1.0, float(g[p + "loss"]))
        if head == "conv":
            assert tuple(act["avg_conv_h"].shape) == (3, 16)
            assert max_abs(act["avg_conv_h"].detach(), g[p + "avg_conv_h_train"]) <= 1e-5
        for k in keys:
            got = grads[k].reshape(-1)[torch.from_numpy(g[p + "grad_idx." + k])]
            ref = torch.from_numpy(g[p + "grad_val." + k])
            assert float((got - ref).norm()) <= 1e-4 * float(ref.norm()) + 1e-7, k
            assert abs(float(grads[k].double().norm()) - float(g[p + "grad_norm." + k])) <= \
                1e-4 * float(g[p + "grad_norm." + k]) + 1e-9, k
        with torch.no_grad():
            y, act = oracle_pass(sd, x, head, False, EVAL_SEED)
        assert max_abs(y, g[p + "y_eval"]) <= 1e-5
        if head == "conv":
            assert max_abs(act["avg_conv_h"], g[p + "avg_conv_h_eval"]) <= 1e-5


def test_oracle_routes_train_steps_through_pooled_heads():
    sd = cpu_state(pooled_discriminator("gmax", "bnorm"))
    x = torch.zeros(1, 2, 16384)
    shifts = [1, 1, 1, 1, 1]
    with pytest.raises(KeyError):
        O.discriminator_forward(sd, x, shifts, training=False)
    with DO.pooled_heads("gmax"):
        assert tuple(O.discriminator_forward(sd, x, shifts, training=False).shape) == (1, 1)
    assert O.discriminator_forward is DO._plain_discriminator_forward
    with pytest.raises(ValueError):
        DO.discriminator_forward(sd, x, shifts, training=False)       # gmax and gavg look alike: name it


@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("head", ("none",) + HEADS)
def test_grad_chunks_cover_the_bucket_once(head, norm):
    """The data-parallel gradient chunks: [fc.0 | mlp.0 +] the last tower layer first (complete when its weight
    gradient is enqueued), then everything else -- disjoint, in order, covering the bucket."""
    D = pooled_discriminator(head, norm)
    eng = E.DiscriminatorEngine(D).bind()
    names = [l.name for l in eng.layers]
    sfx = "_orig" if norm == "snorm" else ""
    assert ("fc.0.weight" + sfx in names) == (head == "none")
    assert ("mlp.0.weight" + sfx in names) == (head == "mlp")
    first = 1 if head in ("none", "mlp") else 0
    assert names[first] == "enc_blocks.4.conv.weight" + sfx
    chunks = eng.grad_chunks()
    off = 0
    for o, n in chunks:
        assert o == off and n > 0
        off += n
    assert off == eng.grad.numel()
    assert chunks[0][1] == sum(l.numel for l in eng.layers[:first + 1])
    if norm == "snorm":              # every spectrally normalised tensor of the head is one of the module's
        assert set(eng._sn_names()) <= set(n for n, _ in D.named_parameters())


def test_segan_refuses_mlp_head_before_the_first_step():
    """The reference's SEGAN compares D's flattened logits with B labels (model.py:298): with mlp's B * Lq logits its
    first step fails.  Ours says so before anything runs, quoting the reference's error for the same shapes."""
    g = golden(GOLD)
    s = build_segan(dpool_type="mlp")
    assert tuple(s.D.mlp[2].weight.shape) == (1, 1024, 1)
    clean = torch.zeros(3, 1, 16384)
    ref_text = str(g["segan_mlp_error"]).split(" at non-singleton")[0]
    with pytest.raises(RuntimeError, match="mlp") as e:
        s.train_step(clean, clean, None, None, 100.0)
    assert ref_text in str(e.value)
    with pytest.raises(RuntimeError, match="B \\* Lq"):
        s.train(load_opts(batch_size=3, dpool_type="mlp"), None, torch.nn.MSELoss(), 100.0, 0, 0, 1)


def test_sinc_conv_raises():
    with pytest.raises(NotImplementedError, match="sinc_conv"):
        Discriminator(2, [64, 128, 256, 512, 1024], 31, [4] * 5, pool_type="conv", pool_slen=16, sinc_conv=True)
