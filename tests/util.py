"""Shared helpers for the test-suite (not collected)."""
import hashlib
import json
import os
import random
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def load_opts(**over):
    """ckpt_segan+/train.opts (copied verbatim to tests/golden/train_opts.json) + reg_loss (F5)."""
    with open(os.path.join(GOLDEN, "train_opts.json")) as f:
        d = json.load(f)
    d.setdefault("reg_loss", "l1_loss")
    d["save_path"] = over.pop("save_path", "/tmp/segan_b200_ckpt")
    d.update(over)
    return types.SimpleNamespace(**d)


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def build_segan(seed=111, **over):
    from segan_pytorch_b200.segan.models import SEGAN
    seed_all(seed)                       # train.py:22-24
    return SEGAN(load_opts(**over))


def sd_sha(sd):
    h = hashlib.sha256()
    for k in sd:
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def arr_sha(a):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a, dtype=np.float32)).tobytes()).hexdigest()


def golden(name):
    """A fixture as a dict of arrays.  An array stored as a seeded draw (keys `<k>.seed`, `<k>.shape`,
    `<k>.sha256`: torch.manual_seed(seed); torch.randn(shape)) is re-drawn and checked against its sha256."""
    with np.load(os.path.join(GOLDEN, name)) as f:
        d = {k: f[k] for k in f.files}
    for k in [k[:-len(".seed")] for k in d if k.endswith(".seed")]:
        torch.manual_seed(int(d[k + ".seed"]))
        a = torch.randn(*[int(s) for s in d[k + ".shape"]]).numpy()
        assert arr_sha(a) == str(d[k + ".sha256"]), "seeded draw %s of %s does not reproduce" % (k, name)
        d[k] = a
    return d


def cpu_state(module):
    return {k: v.detach().cpu().clone() for k, v in module.state_dict().items()}


def rel_err(a, b):
    a = torch.as_tensor(a).double().reshape(-1)
    b = torch.as_tensor(b).double().reshape(-1)
    return float((a - b).norm() / (b.norm() + 1e-30))


def max_abs(a, b):
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())
