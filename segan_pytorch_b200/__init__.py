"""segan_pytorch_b200 -- H100-native (sm_90a) engine for the SEGAN+ hot path of
santi-pdp/segan_pytorch: Generator / Discriminator conv stacks, the G+D LSGAN train step and
G-only streaming inference, behind the reference's Python API (`segan_pytorch_b200.segan`,
also importable as top-level `segan`).  Compute lives in libsegan_b200.so (C ABI:
include/segan_b200.h); there is no CPU fallback."""
__version__ = "0.1.0"
