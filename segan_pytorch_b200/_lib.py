"""ctypes binding of libsegan_b200.so (the C ABI declared in include/segan_b200.h).

The library is the product: if it is missing, not loadable, or the device is not an H100 (sm_90),
every compute entry point raises -- there is no CPU / ATen fallback behind this module.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsegan_b200.so")

SG_F32, SG_F16, SG_BF16 = 0, 1, 2
ACT_NONE, ACT_PRELU, ACT_TANH = 0, 1, 2
EW_ACT_FWD, EW_BN_STATS, EW_BWD_REDUCE, EW_BWD_APPLY = 1, 2, 3, 4
PCM_NO_PREV = 0x7fffffff
BACKEND_FFMA, BACKEND_TCGEN05 = 0, 1
SG_DHEAD_CONV, SG_DHEAD_GMAX, SG_DHEAD_GAVG, SG_DHEAD_MLP = 1, 2, 3, 4

_vp, _i, _f, _i64 = C.c_void_p, C.c_int, C.c_float, C.c_int64
I9 = C.c_int32 * 9


class TapGemmF(C.Structure):
    _fields_ = [
        ("a0", _vp), ("a1", _vp), ("a0_c", C.c_int32), ("a1_c", C.c_int32),
        ("a_rows", C.c_int32), ("a_halo", C.c_int32), ("a_dtype", C.c_int32),
        ("w", _vp), ("w_dtype", C.c_int32), ("w_tap0", C.c_int32),
        ("kc", C.c_int32), ("nc", C.c_int32), ("d_lo", C.c_int32), ("d_hi", C.c_int32),
        ("tap_k_lo", I9), ("tap_k_hi", I9), ("tap_n_lo", I9), ("tap_n_hi", I9),
        ("out", _vp), ("out_ld", C.c_int32), ("out_col0", C.c_int32),
        ("out_dtype", C.c_int32), ("out_rows", C.c_int32), ("out_halo", C.c_int32),
        ("m_lo", C.c_int32), ("m_hi", C.c_int32), ("n_lo", C.c_int32), ("n_hi", C.c_int32),
        ("bias", _vp), ("bias_mod", C.c_int32), ("batch", C.c_int32), ("ksplit", C.c_int32),
        ("backend", C.c_int32), ("tile_n", C.c_int32), ("bn_stats", _vp),
        ("out2", _vp), ("out2_halo", C.c_int32), ("slope", _vp), ("slope_mod", C.c_int32), ("sk_ws", _vp),
    ]


class TapGemmW(C.Structure):
    _fields_ = [
        ("g", _vp), ("g_rows", C.c_int32), ("g_dtype", C.c_int32),
        ("a0", _vp), ("a1", _vp), ("a0_c", C.c_int32), ("a1_c", C.c_int32),
        ("a_rows", C.c_int32), ("a_halo", C.c_int32), ("a_dtype", C.c_int32),
        ("kc", C.c_int32), ("nc", C.c_int32), ("d_lo", C.c_int32), ("d_hi", C.c_int32),
        ("tap_k_lo", I9), ("tap_k_hi", I9), ("tap_n_lo", I9), ("tap_n_hi", I9),
        ("dw", _vp), ("dw_tap0", C.c_int32),
        ("batch", C.c_int32), ("ksplit", C.c_int32), ("backend", C.c_int32), ("out_scale", _vp),
    ]


# name -> argtypes (all return int status)
_SIGS = {
    "sg_tapgemm_f_run": [C.POINTER(TapGemmF), _vp],
    "sg_tapgemm_w_run": [C.POINTER(TapGemmW), _vp],
    "sg_pack_weights": [_i, _vp, _i, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp],
    "sg_unpack_wgrad": [_i, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _i, _vp],
    "sg_wave_conv_fwd": [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp],
    "sg_wave_conv_wgrad": [_vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp],
    "sg_wave_conv_dgrad": [_vp, _i, _i, _i, _vp, _i, _i, _vp, _i, _vp],
    "sg_wave_deconv_fwd": [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _vp],
    "sg_wave_deconv_bwd": [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "sg_wave_im2col": [_vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp],
    "sg_wave_shiftadd_tanh": [_vp, _i, _i, _vp, _vp, _vp],
    "sg_wave_col2im_fold": [_vp, _i, _i, _i, _i, _vp, _vp, _vp],
    "sg_tanh_bwd": [_vp, _vp, _i64, _vp, _vp, _vp],
    "sg_bn_stats": [_vp, _i, _i64, _i, _vp, _vp],
    "sg_bn_finalize": [_vp, _i64, _i, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp],
    "sg_act_fwd": [_vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp],
    "sg_act_bwd_reduce": [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp],
    "sg_act_bwd_apply": [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp],
    "sg_stat_grads": [_vp, _i, _i, _vp, _vp, _vp, _vp],
    "sg_convert_f32_rows": [_vp, _vp, _i, _i64, _i, _i, _i, _vp],
    "sg_ncl_to_nlc": [_vp, _i, _i, _i, _vp, _i, _vp],
    "sg_nlc_to_ncl": [_vp, _i, _i, _i, _i, _vp, _vp],
    "sg_colsum": [_vp, _i, _i64, _i, _i, _vp, _i, _vp, _vp],
    "sg_fc_tail_fwd": [_vp] * 8 + [_i, _vp, _vp, _vp, _vp],
    "sg_fc_tail_bwd": [_vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp] + [_vp] * 7 + [_f, _vp],
    "sg_l1_loss_bwd": [_vp, _vp, _i64, _f, _vp, _vp, _i, _f, _vp],
    "sg_mse_loss_bwd": [_vp, _vp, _i64, _f, _vp, _vp, _i, _f, _vp],
    "sg_rmsprop_step": [_vp, _vp, _vp, _i64, _f, _f, _f, _f, _i, _vp],
    "sg_adam_step": [_vp, _vp, _vp, _vp, _i64, _f, _f, _f, _f, _i, _f, _i, _vp],
    "sg_emit_operands": [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp],
    "sg_snorm_sigma": [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp],
    "sg_snorm_grad": [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp],
    "sg_snorm_coef": [_vp, _vp, _i, _vp, _vp, _vp],
    "sg_snorm_rank1": [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp],
    "sg_alpha_grad": [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp],
    "sg_wave_wgrad_fold": [_vp, _i, _vp, _vp],
    "sg_last_deconv_wgrad_fold": [_vp, _i, _vp, _vp, _vp, _vp, _vp],
    "sg_last_deconv_wgrad_fold_1src": [_vp, _i, _vp, _vp],
    "sg_deemphasis": [_vp, _i64, _f, _vp, _vp],
    "sg_preemphasis": [_vp, _i64, _f, _vp, _vp],
    "sg_pcm16_to_wave": [_vp, _vp, _i64, _i, _f, _vp, _vp, _vp],
    "sg_deemphasis_segments": [_vp, _vp, _i, _f, _vp, _vp],
    "sg_stft_frames": [_vp, _i, _i, _vp, _i, _i, _vp],
    "sg_logpow_l1": [_vp, _vp, _i64, _i, _i, _i, _f, _vp, _vp, _i, _f, _vp],
    "sg_stft_frames_fold": [_vp, _i, _i, _f, _vp, _vp],
    "sg_skipconv_emit": [_vp, _i, _i, _vp, _vp, _i, _i, _vp],
    "sg_skipconv_wgrad_fold": [_vp, _i, _i, _vp, _vp],
    "sg_dhead_fwd": [_i, _vp, _i, _i, _i] + [_vp] * 8,
    "sg_dhead_bwd": [_i, _vp, _i, _i, _i] + [_vp] * 6 + [_f, _f, _vp, _vp] + [_vp] * 4 + [_f, _vp],
}
EXPORTS = ["sg_abi_version", "sg_last_error", "sg_device_ok", "sg_set_cta_pair", "sg_set_ew_variant",
           "sg_set_grad_dtype", "sg_set_stream_k", "sg_tapgemm_f_workspace_bytes", "sg_debug_timeline"] + list(_SIGS)

_lib = None


class SeganB200Error(RuntimeError):
    pass


def load():
    """Loads the shared library (building nothing: see segan_pytorch_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SeganB200Error(
            "libsegan_b200.so not found at %s -- build it with `python -m segan_pytorch_b200.build` "
            "(there is no fallback path)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.sg_abi_version.restype = C.c_int
    lib.sg_last_error.restype = C.c_char_p
    lib.sg_device_ok.restype = C.c_int
    lib.sg_set_cta_pair.restype = C.c_int
    lib.sg_set_cta_pair.argtypes = [C.c_int]
    lib.sg_set_ew_variant.restype = C.c_int
    lib.sg_set_ew_variant.argtypes = [C.c_int] * 4
    lib.sg_tapgemm_f_workspace_bytes.restype = C.c_int64
    lib.sg_tapgemm_f_workspace_bytes.argtypes = []
    lib.sg_set_stream_k.restype = C.c_int
    lib.sg_set_stream_k.argtypes = [C.c_int, C.c_float]
    lib.sg_set_grad_dtype.restype = C.c_int
    lib.sg_set_grad_dtype.argtypes = [C.c_int]
    for name, args in _SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    if lib.sg_abi_version() != 3:
        raise SeganB200Error("ABI version mismatch")
    if os.environ.get("SEGAN_B200_CTA_PAIR", "") in ("0", "1", "2"):
        lib.sg_set_cta_pair(int(os.environ["SEGAN_B200_CTA_PAIR"]))
    lib.sg_set_grad_dtype(SG_BF16 if os.environ.get("SEGAN_B200_GRAD_DTYPE", "f16").lower() == "bf16" else SG_F16)
    _lib = lib
    return lib


# kernels launched per C-ABI call (memsets not counted); used for bench.py's gpu_launches claim
LAUNCHES_PER_CALL = {"sg_colsum": 2, "sg_wave_deconv_bwd": 3, "sg_fc_tail_bwd": 2}
launch_count = 0


# optional live timing of every C-ABI call (bench.py, tools/timeline.py): list of
# (name, start_event, end_event, stream handle)
call_profile = None


def call(name, *args):
    global launch_count
    lib = load()
    launch_count += LAUNCHES_PER_CALL.get(name, 1)
    if call_profile is not None:
        import torch
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rc = getattr(lib, name)(*args)
        e.record()
        call_profile.append((name, s, e, torch.cuda.current_stream().cuda_stream))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        raise SeganB200Error("%s failed (%d): %s" % (name, rc, lib.sg_last_error().decode(errors="replace")))


def device_ok():
    return bool(load().sg_device_ok())
