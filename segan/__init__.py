"""Top-level alias so that the reference's entry points (`from segan.models import SEGAN`,
train.py:5 / clean.py:5) resolve to the H100 engine unchanged."""
import sys

from segan_pytorch_b200.segan import models, datasets  # noqa: F401

sys.modules[__name__ + ".models"] = models
sys.modules[__name__ + ".datasets"] = datasets
