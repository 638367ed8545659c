"""Every C-ABI compute entry point (segan_pytorch_b200._lib._SIGS) has a direct GPU test: its name appears in some
tests/test_gpu_*.py, or EXEMPT names the test that reaches it through a Python wrapper.  The non-kernel exports
(EXPORTS minus _SIGS: ABI version, error string, tuning switches) are exempt.  Runs without a GPU."""
import glob
import os
import re

from segan_pytorch_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))

# entry point -> the GPU test that checks it through a wrapper (its name does not appear in the test itself)
EXEMPT = {
    "sg_tapgemm_w_run": "tests/test_gpu_tapgemm_w.py::test_tapgemm_w_vs_fp64 (through engine.run_w)",
}


def _gpu_test_sources():
    return {os.path.basename(f): open(f).read() for f in sorted(glob.glob(os.path.join(HERE, "test_gpu_*.py")))}


def test_every_kernel_entry_point_has_a_direct_gpu_test():
    src = _gpu_test_sources()
    uncovered = [n for n in _lib._SIGS if n not in EXEMPT
                 and not any(re.search(r"\b%s\b" % n, t) for t in src.values())]
    assert not uncovered, "C-ABI entry points without a direct GPU test: %s" % ", ".join(uncovered)


def test_exemptions_name_existing_tests():
    src = _gpu_test_sources()
    for name, where in EXEMPT.items():
        assert name in _lib._SIGS, "stale exemption: %s is not an entry point" % name
        path, test = where.split(" ")[0].split("::")
        assert re.search(r"^def %s\(" % test, src[os.path.basename(path)], re.M), (name, where)


def test_non_kernel_exports_are_not_in_sigs():
    extra = set(_lib.EXPORTS) - set(_lib._SIGS)
    assert extra == {"sg_abi_version", "sg_last_error", "sg_device_ok", "sg_set_cta_pair", "sg_set_ew_variant",
                     "sg_set_grad_dtype", "sg_set_stream_k", "sg_tapgemm_f_workspace_bytes", "sg_debug_timeline"}
