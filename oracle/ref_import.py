"""TEST INFRASTRUCTURE ONLY -- loader for the *unmodified* reference (santi-pdp/segan_pytorch).

Used only by tests/golden/make_golden.py, which executes the reference to write the committed fixtures
under tests/golden/; the location of a reference checkout comes from SEGAN_REFERENCE_ROOT.  Nothing in
the test-suite, smoke() or bench.py calls this.

Recipe = SURVEY.md App. D: six stub modules for un-installed, un-needed dependencies, oneDNN
disabled (finding F1: the multi-threaded oneDNN fp32 conv_transpose1d forward is numerically
wrong in this image), Saver.save patched to a no-op.
"""
import contextlib
import importlib.machinery
import io
import json
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("SEGAN_REFERENCE_ROOT", "")


def reference_available():
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "segan", "models"))


def _stub(name, **kw):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__dict__.update(kw)
    sys.modules[name] = m
    return m


class _Writer:  # tensorboardX.SummaryWriter stand-in
    def __init__(self, *a, **k):
        pass

    def add_scalar(self, *a, **k):
        pass

    def add_histogram(self, *a, **k):
        pass


_loaded = None


def load_reference():
    """Returns the imported reference `segan.models` module (SEGAN, WSEGAN, Generator, ...)."""
    global _loaded
    if _loaded is not None:
        return _loaded
    if not reference_available():
        raise RuntimeError("no reference checkout: set SEGAN_REFERENCE_ROOT (got %r)" % REFERENCE_ROOT)
    import torch
    torch.backends.mkldnn.enabled = False  # F1
    for n in ("librosa", "soundfile", "h5py", "ahoproc_tools", "ahoproc_tools.io",
              "ahoproc_tools.interpolate", "matplotlib.pyplot"):
        if n not in sys.modules:
            _stub(n)
    if "tensorboardX" not in sys.modules:
        _stub("tensorboardX", SummaryWriter=_Writer)
    if "matplotlib" not in sys.modules:
        _stub("matplotlib", use=lambda *a, **k: None)
    # our repo ships a drop-in package that is also called `segan`; make sure the reference wins
    for k in [k for k in sys.modules if k == "segan" or k.startswith("segan.")]:
        del sys.modules[k]
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            import segan.models as ref_models
            import segan.models.core as ref_core
            import segan.datasets.se_dataset as ref_ds
    finally:
        sys.path.remove(REFERENCE_ROOT)
    ref_core.Saver.save = lambda *a, **k: None
    ref_models._ref_datasets = ref_ds
    # detach the reference from the name `segan` so that the repo's own drop-in can be imported
    ref_mods = {k: sys.modules.pop(k) for k in list(sys.modules)
                if k == "segan" or k.startswith("segan.")}
    ref_models._ref_modules = ref_mods
    _loaded = ref_models
    return ref_models


def reference_opts(**over):
    """ckpt_segan+/train.opts + reg_loss='l1_loss' (finding F5), as an attribute namespace."""
    with open(os.path.join(REFERENCE_ROOT, "ckpt_segan+", "train.opts")) as f:
        d = json.load(f)
    d.setdefault("reg_loss", "l1_loss")
    d["save_path"] = over.pop("save_path", "/tmp/segan_ref_ckpt")
    d.update(over)
    return types.SimpleNamespace(**d)


@contextlib.contextmanager
def quiet():
    with contextlib.redirect_stdout(io.StringIO()):
        yield
