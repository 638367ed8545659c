"""Generator topologies --no_z / --no_skip / --z_dim and SEGAN's --reg_loss mse_loss on the CPU: the topology
oracle (tests/gtopo_oracle.py) against the reference's golden outputs, gradients and step losses
(tests/golden/g_topology.npz), seeded construction of the drop-in modules, and which configurations are served."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import segan_oracle as O
from segan_pytorch_b200.segan.models import Generator
from tests import gtopo_oracle as TO
from tests.util import build_segan, cpu_state, golden, load_opts, max_abs, sd_sha, seed_all

GOLD = "g_topology.npz"
# configuration -> train.py options (tests/golden/make_golden_gtopo.py)
CONFIGS = {
    "no_z": dict(no_z=True),
    "no_skip": dict(no_skip=True),
    "no_z_no_skip": dict(no_z=True, no_skip=True),
    "z256": dict(z_dim=256),
    "no_z_sum": dict(no_z=True, skip_merge="sum"),
    "no_z_conv": dict(no_z=True, skip_type="conv"),
    "no_skip_no_bias": dict(no_skip=True, bias=False),
}


def generator_kwargs(over):
    o = load_opts(**over)
    return dict(z_dim=o.z_dim, no_z=o.no_z, skip=not o.no_skip, bias=o.bias, skip_init=o.skip_init,
                skip_type=o.skip_type, skip_merge=o.skip_merge, skip_kwidth=o.skip_kwidth)


def topo_generator(name, seed=111):
    seed_all(seed)
    return Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], **generator_kwargs(CONFIGS[name]))


def golden_inputs(g, name):
    """(x, z or None, clean) of the fixture's two windows."""
    x = 0.3 * torch.from_numpy(g["xr"])
    z = torch.from_numpy(g["zr.%s" % name]) if ("zr.%s" % name) in g else None
    return x, z, (0.3 * torch.from_numpy(g["cr"])).clamp(-1, 1)


@pytest.fixture(scope="module", autouse=True)
def _threads():
    torch.set_num_threads(max(1, min(8, torch.get_num_threads())))


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_seeded_generator_matches_reference(name):
    g = golden(GOLD)
    G = topo_generator(name)
    sd = G.state_dict()
    assert list(sd.keys()) == [str(k) for k in g["keys.%s" % name]]
    shapes = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()])
    assert np.array_equal(shapes, g["shapes.%s" % name])
    assert sd_sha(sd) == str(g["sha_G_init.%s" % name])
    assert G._served
    s = build_segan(**CONFIGS[name])
    assert sd_sha(s.G.state_dict()) == str(g["sha_segan_G.%s" % name])


def test_topology_shapes():
    assert tuple(topo_generator("no_z").dec_blocks[0].deconv.weight.shape) == (1024, 512, 31)
    assert tuple(topo_generator("no_skip").dec_blocks[4].deconv.weight.shape) == (64, 1, 31)
    assert tuple(topo_generator("z256").dec_blocks[0].deconv.weight.shape) == (1280, 512, 31)
    assert not any(k.startswith("alpha_") for k in topo_generator("no_z_no_skip").state_dict())


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oracle_forward_vs_golden(name):
    g = golden(GOLD)
    x, z, _ = golden_inputs(g, name)
    G = topo_generator(name)
    sd = cpu_state(G)
    with O.oracle_mode(), torch.no_grad():
        y, hall = TO.generator_forward(sd, x, z, ret_hid=True, skip_merge=G.skip_merge)
    yv = y.reshape(-1)[torch.from_numpy(g["y_idx.%s" % name])]
    assert max_abs(yv, g["y_val.%s" % name]) <= 1e-5
    assert abs(float(y.double().norm()) - float(g["y_norm.%s" % name])) <= 1e-5 * float(g["y_norm.%s" % name])
    assert sorted(hall) == [str(k) for k in g["hall_keys.%s" % name]]


@pytest.mark.parametrize("loss", ["l1", "mse"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oracle_gradients_vs_golden(name, loss):
    g = golden(GOLD)
    x, z, clean = golden_inputs(g, name)
    G = topo_generator(name)
    sd = cpu_state(G)
    pre = "grad_idx.%s.%s." % (loss, name)
    keys = [k[len(pre):] for k in g if k.startswith(pre)]
    assert len(keys) == (3 if "no_skip" in name else 4)
    fn = F.l1_loss if loss == "l1" else F.mse_loss
    with O.oracle_mode():
        p = {k: sd[k].clone().requires_grad_(True) for k in keys}
        out = 100 * fn(TO.generator_forward({**sd, **p}, x, z, skip_merge=G.skip_merge), clean)
        grads = dict(zip(keys, torch.autograd.grad(out, [p[k] for k in keys])))
    ref_loss = float(g["%s_loss.%s" % (loss, name)])
    assert abs(float(out.detach()) - ref_loss) <= 1e-5 * ref_loss
    for k in keys:
        tag = "%s.%s.%s" % (loss, name, k)
        got = grads[k].reshape(-1)[torch.from_numpy(g["grad_idx." + tag])]
        ref = torch.from_numpy(g["grad_val." + tag])
        assert float((got - ref).norm()) <= 1e-4 * float(ref.norm()) + 1e-7, tag
        assert abs(float(grads[k].double().norm()) - float(g["grad_norm." + tag])) <= \
            1e-4 * float(g["grad_norm." + tag]), tag


def test_oracle_mse_step_vs_golden():
    """The reference's SEGAN step with reg_loss='mse_loss' on the inputs of train_step_b4.npz."""
    g, t = golden(GOLD), golden("train_step_b4.npz")
    B = t["clean"].shape[0]
    segan = build_segan(batch_size=B, reg_loss="mse_loss")
    assert segan.reg_loss is F.mse_loss
    sdG, sdD = cpu_state(segan.G), cpu_state(segan.D)
    sqG = {k: torch.zeros_like(sdG[k]) for k in O._trainable(sdG)}
    sqD = {k: torch.zeros_like(sdD[k]) for k in O._trainable(sdD)}
    random.seed(int(t["py_random_seed"]))
    shifts3 = [O.draw_phase_shifts(5, 5) for _ in range(3)]
    clean = torch.from_numpy(t["clean"]).unsqueeze(1)
    noisy = torch.from_numpy(t["noisy"]).unsqueeze(1)
    with TO.gtopo("mse_loss"):
        out = O.segan_train_step(sdG, sdD, sqG, sqD, clean, noisy, torch.from_numpy(t["z"]), shifts3, l1_weight=100.0)
    assert O.F is F and O.generator_forward is not TO.generator_forward
    for k, gk in (("d_real_loss", "d_real_loss"), ("d_fake_loss", "d_fake_loss"), ("g_adv_loss", "g_adv_loss"),
                  ("g_l1_loss", "g_reg_loss")):
        ref = float(g["mse_step." + gk])
        assert abs(out[k] - ref) <= 1e-4 * max(1.0, abs(ref)), k
    assert abs(out["g_l1_loss"] - 100 * float(F.mse_loss(out["Genh"], clean))) <= 1e-4


@pytest.mark.parametrize("over", [dict(), dict(skip_merge="sum"), dict(skip_type="constant"),
                                  dict(skip_type="conv"), dict(z_dim=64), dict(z_dim=512), dict(z_dim=2048)])
@pytest.mark.parametrize("topo", [dict(no_z=True), dict(no_skip=True), dict(no_z=True, no_skip=True),
                                  dict(z_dim=256)])
def test_served_combinations(topo, over):
    seed_all(0)
    G = Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], **generator_kwargs({**over, **topo}))
    assert G._served


@pytest.mark.parametrize("z_dim", [100, 1000, 32, 0])
def test_z_dim_not_multiple_of_64_refused(z_dim):
    seed_all(0)
    if z_dim == 0:
        z_dim = -64
    G = Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], z_dim=z_dim, skip_merge="concat")
    assert not G._served
    with pytest.raises(NotImplementedError, match="positive multiple of 64"):
        G.engine


def test_z_dim_ignored_with_no_z():
    seed_all(0)
    G = Generator(1, [64, 128, 256, 512, 1024], 31, [4, 4, 4, 4, 4], z_dim=100, no_z=True, skip_merge="concat")
    assert G._served


def test_unknown_reg_loss_fails_at_construction():
    with pytest.raises(AttributeError):
        build_segan(reg_loss="not_a_loss")


def test_wsegan_keeps_l1_with_mse_reg_loss():
    """model.py:663: WSEGAN's denoising term is F.l1_loss whatever --reg_loss says: its step never dispatches to the
    MSE kernel."""
    import inspect
    from segan_pytorch_b200.segan.models import model as M
    src = inspect.getsource(M.WSEGAN)
    assert "sg_l1_loss_bwd" in src and "sg_mse_loss_bwd" not in src and "REG_LOSS_KERNELS" not in src
    assert M.REG_LOSS_KERNELS == {"l1_loss": "sg_l1_loss_bwd", "mse_loss": "sg_mse_loss_bwd"}
    from segan_pytorch_b200.segan.models import WSEGAN
    seed_all(111)
    w = WSEGAN(load_opts(reg_loss="mse_loss", wsegan=True, misalign_pair=True))
    assert w.reg_loss_name == "mse_loss"
