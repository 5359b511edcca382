"""ctypes binding of the C-ABI library (include/b200audio.h).  No fallback: if the library is
missing this module raises, and every op raises if its return code is non-zero."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200audio.so")

c_f = C.c_void_p   # device pointers travel as void*
i32, i64, f32 = C.c_int32, C.c_int64, C.c_float


class Conv1dParams(C.Structure):
    """Mirror of b2a_conv1d_t."""
    _fields_ = [
        ("x", C.c_void_p), ("x_bs", i64), ("x_ld", i64),
        ("B", i32), ("L", i32), ("Cin", i32),
        ("w", C.c_void_p), ("bias", C.c_void_p),
        ("y", C.c_void_p), ("y_bs", i64), ("y_ld", i64),
        ("Lout", i32), ("Cout", i32),
        ("K", i32), ("stride", i32), ("dilation", i32), ("pad_left", i32), ("groups", i32), ("pad_mode", i32),
        ("pre_scale", C.c_void_p), ("pre_shift", C.c_void_p),
        ("pre_act", i32), ("pre_p0", f32), ("pre_a", C.c_void_p), ("pre_b", C.c_void_p),
        ("post_act", i32), ("post_p0", f32),
        ("post_cscale", C.c_void_p), ("post_cscale_bs", i64),
        ("res", C.c_void_p), ("res_bs", i64), ("res_ld", i64), ("res_div", i32),
        ("out_scale", f32), ("accumulate", i32),
        ("emit_hi", C.c_void_p), ("emit_lo", C.c_void_p), ("emit_ld", i64),
        ("emit_act", i32), ("emit_p0", f32), ("emit_a", C.c_void_p), ("emit_b", C.c_void_p),
    ]


class AttnParams(C.Structure):
    """Mirror of b2a_attn_t."""
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("o", C.c_void_p),
        ("q_bs", i64), ("q_ld", i64), ("k_bs", i64), ("k_ld", i64), ("v_bs", i64), ("v_ld", i64), ("o_bs", i64), ("o_ld", i64),
        ("B", i32), ("Tq", i32), ("Tk", i32), ("H", i32), ("Hkv", i32), ("D", i32),
        ("scale", f32), ("causal", i32), ("q_offset", i32), ("window", i32),
        ("k_len", C.c_void_p),
        ("emit_hi", C.c_void_p), ("emit_lo", C.c_void_p), ("emit_ld", i64), ("operands_ready", i32),
    ]


class ConvFParams(C.Structure):
    """Mirror of b2a_convf_t (one problem of a fused tensor-core conv launch)."""
    _fields_ = [
        ("x", C.c_void_p), ("x1", C.c_void_p), ("x2", C.c_void_p), ("x_bs", i64), ("x_ld", i64), ("in_scale", f32),
        ("B", i32), ("L", i32), ("Cin", i32),
        ("pre_mode", i32), ("pre_scale", C.c_void_p), ("pre_shift", C.c_void_p), ("pre_stats", C.c_void_p), ("pre_gb", C.c_void_p),
        ("pre_gb_bs", i64), ("pre_eps", f32),
        ("pre_act", i32), ("pre_p0", f32), ("pre_a", C.c_void_p), ("pre_b", C.c_void_p),
        ("w_hi", C.c_void_p), ("w_lo", C.c_void_p), ("cin_pad", i32), ("taps", i32), ("N", i32), ("shifts", i32 * 32),
        ("Lout", i32), ("bias", C.c_void_p), ("post_act", i32), ("post_p0", f32), ("cscale", C.c_void_p), ("cscale_bs", i64),
        ("res", C.c_void_p), ("res_bs", i64), ("res_ld", i64), ("res_div", i32), ("out_scale", f32), ("accumulate", i32),
        ("y", C.c_void_p), ("y_bs", i64), ("y_ld", i64),
        ("up_stride", i32), ("up_crop", i32),
        ("stats_out", C.c_void_p),
    ]


class AlbertParams(C.Structure):
    """b2a_albert_t"""
    _fields_ = [("T", i32), ("layers", i32), ("heads", i32), ("hidden", i32), ("inter", i32), ("planes", i32),
                ("w", C.c_void_p * 4), ("bias", C.c_void_p * 4), ("ln_w", C.c_void_p * 2), ("ln_b", C.c_void_p * 2),
                ("eps", f32), ("scale", f32), ("h", C.c_void_p), ("h_hi", C.c_void_p), ("h_lo", C.c_void_p)]


class RowOp(C.Structure):
    """Mirror of b2a_rowop_t."""
    _fields_ = [("src", C.c_void_p), ("src_bs", i64), ("src_ld", i64), ("dst", C.c_void_p), ("dst_bs", i64), ("dst_ld", i64),
                ("B", i32), ("rows", i32), ("C", i32), ("op", i32)]


class DacLevel(C.Structure):
    """Mirror of b2a_dac_level_t."""
    _fields_ = [("w_in", C.c_void_p), ("b_in", C.c_void_p), ("cbn", C.c_void_p), ("c2", C.c_void_p), ("cb", C.c_void_p),
                ("w_out", C.c_void_p), ("b_out", C.c_void_p), ("cd", i32), ("lat_off", i32)]


ROWOPS_MAX = 32      # B2A_ROWOPS_MAX


# name -> (restype, argtypes); every symbol include/b200audio.h declares
PROTOTYPES = {
    "b2a_last_error": (C.c_char_p, []),
    "b2a_version": (i32, []),
    "b2a_device_sm_count": (i32, []),
    "b2a_conv1d_cl": (i32, [C.POINTER(Conv1dParams), C.c_void_p]),
    "b2a_convtr1d_cl": (i32, [C.POINTER(Conv1dParams), C.c_void_p]),
    "b2a_conv1d_cl_last_path": (i32, [C.POINTER(i32)]),
    "b2a_kokoro_source_conv": (i32, [c_f, i32, i32, c_f, c_f, c_f, i32, i32, i32, i32, i32, C.c_void_p]),
    "b2a_prep_bf16": (i32, [c_f, i64, i64, i32, i32, i32, i32, c_f, c_f, i32, f32, c_f, c_f, c_f, c_f, i32, C.c_void_p]),
    "b2a_conv1d_tc": (i32, [c_f, c_f, i32, i32, i32, i32, c_f, c_f, i32, C.POINTER(i32), i32, i32, c_f, i32, f32, c_f, i64, c_f, i64, i64, i32, f32, i32,
                            c_f, i64, i64, i32, i32, c_f, c_f, i64, c_f, i32, f32, C.c_void_p]),
    "b2a_conv1d_tc_debug": (i32, [c_f]),
    "b2a_conv1d_tc_last_config": (i32, [C.POINTER(i32)]),
    "b2a_conv1d_fused_debug": (i32, [c_f]),
    "b2a_conv1d_fused_last_config": (i32, [C.POINTER(i32)]),
    "b2a_conv1d_fused": (i32, [C.POINTER(ConvFParams), i32, i32, i32, c_f, i64, C.c_void_p]),
    "b2a_conv1d_fused_fits": (i32, [i32, i32, i32, i32, i32]),
    "b2a_copy2d": (i32, [c_f, i64, c_f, i64, i64, i32, C.c_void_p]),
    "b2a_gather_rows": (i32, [c_f, i64, c_f, c_f, i64, i64, i32, i64, c_f, i64, i64, C.c_void_p]),
    "b2a_durations_to_index": (i32, [c_f, c_f, i32, f32, c_f, c_f, i64, c_f, C.c_void_p]),
    "b2a_adain_ws_bytes": (i64, [i32, i32, i32]),
    "b2a_adain_coeffs": (i32, [c_f, i64, i64, i32, i32, i32, c_f, f32, c_f, c_f, c_f, C.c_void_p]),
    "b2a_channel_stats": (i32, [c_f, i64, i64, i32, i32, i32, C.POINTER(C.c_void_p), C.POINTER(i64), i32, C.c_void_p]),
    "b2a_coeffs_from_stats": (i32, [c_f, i32, i32, i32, c_f, f32, c_f, c_f, C.c_void_p]),
    "b2a_layernorm": (i32, [c_f, i64, c_f, i64, c_f, i64, i64, i32, c_f, c_f, c_f, f32, i32, i32, f32, c_f, c_f, i64, C.c_void_p]),
    "b2a_attention": (i32, [C.POINTER(AttnParams), C.c_void_p]),
    "b2a_attention_tc_ws_bytes": (i64, [i32, i32, i32, i32]),
    "b2a_attention_tc": (i32, [C.POINTER(AttnParams), C.c_void_p, C.c_void_p]),
    "b2a_albert_ws_bytes": (i64, [i32, i32, i32, i32]),
    "b2a_albert_encoder": (i32, [C.POINTER(AlbertParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2a_rope": (i32, [c_f, i64, i64, i32, i32, i32, i32, i32, f32, i32, C.c_void_p]),
    "b2a_lstm_bidir": (i32, [c_f, c_f, c_f, i64, i32, i32, i32, C.c_void_p]),
    "b2a_stft": (i32, [c_f, i64, i32, i64, c_f, i32, i32, i32, i64, c_f, c_f, C.c_void_p]),
    "b2a_whisper_logmel": (i32, [c_f, i64, i32, i64, i64, c_f, c_f, i32, i64, c_f, c_f, C.c_void_p]),
    "b2a_istft": (i32, [c_f, c_f, i32, i32, i32, i32, c_f, i32, i32, i64, i64, c_f, c_f, C.c_void_p]),
    "b2a_resample_poly": (i32, [c_f, i64, i32, i64, c_f, i32, i32, i32, i64, i64, c_f, i64, C.c_void_p]),
    "b2a_kokoro_source": (i32, [c_f, i32, i32, i32, c_f, c_f, c_f, c_f, c_f, c_f, C.c_void_p]),
    "b2a_kokoro_istft_head": (i32, [c_f, i64, i64, i32, i32, c_f, C.c_void_p]),
    "b2a_randn": (i32, [c_f, i64, C.c_uint64, C.c_uint64, C.c_void_p]),
    "b2a_randn_dev": (i32, [c_f, i64, c_f, C.c_void_p]),
    "b2a_whisper_greedy_step": (i32, [c_f, i64, c_f, i64, i32, i32, i32, i32, c_f, c_f, i32, i32, i32, i32, i32, c_f, c_f, c_f, f32, c_f, C.c_void_p]),
    "b2a_sample_token": (i32, [c_f, i64, i32, i32, c_f, c_f, i64, i32, f32, f32, i32, f32, f32, c_f, c_f, i64, c_f, c_f, i32, C.c_void_p]),
    "b2a_gemv_bf16": (i32, [c_f, i64, i32, i32, c_f, i64, i32, c_f, c_f, f32, i32, c_f, i64, c_f, i64, c_f, i64, C.c_void_p]),
    "b2a_qknorm_rope_cache": (i32, [c_f, i64, i64, i32, i32, i32, i32, i32, c_f, c_f, f32, c_f, c_f, i32, i32, i32, f32, c_f, i64, i64,
                                    c_f, c_f, i64, i64, i32, c_f, c_f, c_f, C.c_void_p]),
    "b2a_attn_decode": (i32, [c_f, i64, i64, c_f, c_f, i64, i64, c_f, i64, i64, i32, i32, i32, i32, i32, f32, c_f, i32, c_f, i32, c_f, c_f,
                              C.c_void_p]),
    "b2a_attn_prefill": (i32, [c_f, i64, i64, c_f, c_f, i64, i64, c_f, i64, i64, i32, i32, i32, i32, i32, f32, c_f, i32, c_f, i32, c_f, c_f,
                               C.c_void_p]),
    "b2a_swiglu": (i32, [c_f, i64, i64, i32, i32, c_f, i64, C.c_void_p]),
    "b2a_embed_sum": (i32, [c_f, i64, i32, i32, i32, c_f, c_f, c_f, i64, i64, i32, c_f, c_f, i64, c_f, c_f, c_f, C.c_void_p]),
    "b2a_incr_i32": (i32, [c_f, i32, C.c_void_p]),
    "b2a_slot_advance": (i32, [c_f, c_f, c_f, c_f, c_f, i32, c_f, i64, c_f, i64, c_f, i32, C.c_void_p]),
    "b2a_rvq_decode": (i32, [c_f, i64, i64, i32, i32, i64, c_f, i32, i32, c_f, i64, c_f, C.c_void_p]),
    "b2a_rvq_encode": (i32, [c_f, i64, i64, i32, c_f, c_f, i32, i32, i32, c_f, i64, i64, C.c_void_p]),
    "b2a_snac_from_codes": (i32, [C.POINTER(C.c_void_p), C.POINTER(i32), i32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                  C.POINTER(C.c_void_p), i32, i64, i32, i32, i32, c_f, c_f, C.c_void_p]),
    "b2a_dac_rvq_encode_smem_bytes": (i64, [i32]),
    "b2a_dac_rvq_encode": (i32, [c_f, i64, i32, i64, i32, c_f, i32, i32, i32, c_f, c_f, c_f, c_f, C.c_void_p]),
    "b2a_dac_from_codes": (i32, [c_f, i64, i64, i32, i32, i64, c_f, i32, i32, i32, c_f, c_f, c_f, C.c_void_p]),
    "b2a_aa_snakebeta": (i32, [c_f, i64, i64, i32, i32, i32, c_f, c_f, c_f, c_f, i32, i32, c_f, i64, i64, c_f, c_f, i32, C.c_void_p]),
    "b2a_stream_rows": (i32, [C.POINTER(RowOp), i32, C.c_void_p]),
    "b2a_conv1d_stream": (i32, [C.POINTER(Conv1dParams), c_f, i64, i32, c_f, i32, C.c_void_p]),
    "b2a_convtr1d_stream": (i32, [C.POINTER(Conv1dParams), c_f, i64, C.c_void_p]),
    "b2a_ring_rope_kv": (i32, [c_f, i64, i64, i32, i32, i32, i32, f32, c_f, c_f, i64, i32, c_f, C.c_void_p]),
    "b2a_ring_attn": (i32, [c_f, i64, i64, c_f, c_f, i64, i32, c_f, i64, i64, i32, i32, i32, i32, f32, i32, c_f, C.c_void_p]),
    "b2a_stream_advance": (i32, [c_f, i32, C.c_void_p]),
    "b2a_spk_logmel": (i32, [c_f, i64, i32, i64, c_f, c_f, i32, i64, c_f, C.c_void_p]),
    "b2a_spk_reflect_pad": (i32, [c_f, i64, i64, i32, i32, i32, i32, c_f, c_f, c_f, i32, C.c_void_p]),
    "b2a_spk_res2net_smem_bytes": (i64, [i32, i32, i32, i32, i32]),
    "b2a_spk_res2net": (i32, [c_f, i64, i64, c_f, i64, i64, c_f, c_f, i32, i32, i32, i32, i32, i32, i32, C.c_void_p]),
    "b2a_spk_channel_stats": (i32, [c_f, i64, i64, i32, i32, i32, i32, f32, c_f, i64, C.c_void_p]),
    "b2a_spk_se_gate": (i32, [c_f, i64, i32, i32, i32, c_f, c_f, c_f, c_f, c_f, C.c_void_p]),
    "b2a_spk_se_apply": (i32, [c_f, i64, i64, c_f, c_f, i64, i64, c_f, i64, i64, i32, i32, i32, C.c_void_p]),
    "b2a_spk_gemv": (i32, [c_f, i64, i32, i32, c_f, i64, i32, c_f, i32, c_f, i64, C.c_void_p]),
    "b2a_spk_asp_act": (i32, [c_f, i64, i64, c_f, i32, i32, i32, C.c_void_p]),
    "b2a_spk_asp_pool": (i32, [c_f, i64, i64, c_f, i64, i64, i32, i32, i32, f32, c_f, i64, C.c_void_p]),
    "b2a_vocos_dwnorm": (i32, [c_f, i64, i64, i32, i32, i32, c_f, c_f, i32, c_f, c_f, c_f, i64, f32, c_f, i64, i64, c_f, c_f, C.c_void_p]),
    "b2a_vocos_istft_head": (i32, [c_f, i64, i64, i32, i32, i32, i32, c_f, c_f, i64, C.c_void_p]),
    "b2a_vocos_logmel": (i32, [c_f, i64, i32, i64, c_f, c_f, i32, i64, c_f, C.c_void_p]),
    "b2a_encodec_lstm": (i32, [c_f, c_f, c_f, c_f, i32, i32, i32, c_f, C.c_void_p]),
    "b2a_encodec_pad": (i32, [c_f, i64, i64, i32, i32, i32, i32, i32, i32, c_f, c_f, i32, c_f, i64, i64, c_f, i64, i64, C.c_void_p]),
    "b2a_encodec_gn_ws_bytes": (i64, [i32]),
    "b2a_encodec_gn_coeffs": (i32, [c_f, i64, i64, i32, i32, i32, c_f, c_f, f32, c_f, c_f, c_f, C.c_void_p]),
    "b2a_encodec_normalize": (i32, [c_f, i64, i64, i32, i32, i32, c_f, i64, c_f, c_f, C.c_void_p]),
    "b2a_encodec_ola": (i32, [c_f, i32, i32, i32, i32, c_f, i32, i32, c_f, C.c_void_p]),
    "b2a_lm_sample_mlx": (i32, [c_f, i64, i32, i32, f32, C.c_double, c_f, i64, c_f, c_f, c_f, i64, c_f, i32, i32, C.c_void_p]),
    "b2a_soprano_upsample": (i32, [c_f, i64, i64, i32, i32, i32, i32, c_f, i64, i64, c_f, c_f, i32, C.c_void_p]),
    "b2a_soprano_store_rows": (i32, [c_f, i64, i32, i32, c_f, i64, i64, c_f, i32, i32, C.c_void_p]),
}

E_INVALID, E_CUDA, E_UNSUPPORTED = -1, -2, -3


def load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m mlx_audio_b200.build` "
            "(there is no CPU or PyTorch fallback for the hot path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)       # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = load()
    return _LIB


def check(rc: int) -> None:
    """Map C status codes to the Python exceptions the reference raises (SURVEY.md section 8b)."""
    if rc == 0:
        return
    msg = lib().b2a_last_error().decode("utf-8", "replace")
    if rc == E_INVALID:
        raise ValueError(msg)
    if rc == E_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(msg)
