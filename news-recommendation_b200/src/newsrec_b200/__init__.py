"""ctypes binding of the newsrec_b200 C ABI (include/newsrec_b200.h).

Host glue only: PyTorch supplies device memory, streams and autograd bookkeeping; every arithmetic
step of the hot path runs in the sm_90a kernels behind ``libnewsrec_b200.so``.  There is NO CPU or
PyTorch fallback: if the library is missing or no CUDA device is present the ops raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnewsrec_b200.so")

_vp, _i, _ll, _f, _ull = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_ulonglong


class MhsaEncoderFwdArgs(C.Structure):
    """nr_mhsa_encoder_fwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("n_seq", _ll), ("T", _i), ("d", _i), ("heads", _i), ("q", _i), ("ldx", _i), ("ld3", _i),
        ("ids", _vp), ("table_bf16", _vp), ("V", _i),
        ("dense", _vp), ("dense_s_seq", _ll), ("dense_s_tok", _ll), ("dense_s_col", _ll),
        ("wqkv_bf16", _vp), ("bqkv", _vp), ("wa_bf16", _vp), ("ba", _vp), ("qv", _vp),
        ("p_drop", _f), ("seed", _ull),
        ("X_bf16", _vp), ("QKV_bf16", _vp), ("C_bf16", _vp), ("w", _vp), ("out", _vp), ("bad_id_flag", _vp),
        ("C_lo_bf16", _vp),
        ("wqkv_kcat_bf16", _vp), ("X_kcat_bf16", _vp), ("QKV_f32", _vp),
        ("V_lo_bf16", _vp),
        ("dense_pos", _vp),
    ]


class MhsaEncoderBwdArgs(C.Structure):
    """nr_mhsa_encoder_bwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("n_seq", _ll), ("T", _i), ("d", _i), ("heads", _i), ("q", _i), ("ldx", _i), ("ld3", _i), ("ldq", _i),
        ("ids", _vp), ("V", _i),
        ("wqkvT_bf16", _vp), ("wa_bf16", _vp), ("waT_bf16", _vp), ("ba", _vp), ("qv", _vp),
        ("p_drop", _f), ("seed", _ull),
        ("X_bf16", _vp), ("QKV_bf16", _vp), ("C_bf16", _vp), ("w", _vp), ("dout", _vp),
        ("dWqkv_ext", _vp), ("dWa_ext", _vp), ("dqv", _vp), ("demb", _vp), ("ddense", _vp),
        ("workspace", _vp), ("workspace_bytes", _ll),
        ("wqkv_bf16", _vp), ("bqkv", _vp), ("emb_grad_ready_event", _vp),
        ("dpos", _vp), ("table_bf16", _vp),
    ]


class CnnEncoderFwdArgs(C.Structure):
    """nr_cnn_encoder_fwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("n_seq", _ll), ("T", _i), ("d", _i), ("F", _i), ("q", _i), ("ldx", _i), ("ldf", _i),
        ("ids", _vp), ("table_bf16", _vp), ("V", _i),
        ("wconv_bf16", _vp), ("bconv", _vp), ("wa_bf16", _vp), ("ba", _vp), ("qv", _vp),
        ("p_drop", _f), ("seed", _ull),
        ("Xp_bf16", _vp), ("Y_bf16", _vp), ("w", _vp), ("out", _vp), ("bad_id_flag", _vp),
        ("Y_lo_bf16", _vp), ("window", _i),
    ]


class CnnEncoderBwdArgs(C.Structure):
    """nr_cnn_encoder_bwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("n_seq", _ll), ("T", _i), ("d", _i), ("F", _i), ("q", _i), ("ldx", _i), ("ldf", _i), ("ldq", _i),
        ("ids", _vp), ("V", _i),
        ("wconvT_bf16", _vp), ("wa_bf16", _vp), ("waT_bf16", _vp), ("ba", _vp), ("qv", _vp),
        ("p_drop", _f), ("seed", _ull),
        ("Xp_bf16", _vp), ("Y_bf16", _vp), ("w", _vp), ("dout", _vp),
        ("dWconv_ext", _vp), ("dWa_ext", _vp), ("dqv", _vp), ("demb", _vp),
        ("workspace", _vp), ("workspace_bytes", _ll), ("window", _i),
    ]


class KcnnEncoderFwdArgs(C.Structure):
    """nr_kcnn_encoder_fwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("n_seq", _ll), ("T", _i), ("d", _i), ("de", _i), ("F", _i), ("q", _i), ("n_win", _i), ("win", _i * 4),
        ("ldx", _i), ("lde", _i), ("ldf", _i), ("ldo", _i),
        ("word_ids", _vp), ("entity_ids", _vp), ("word_table_bf16", _vp), ("V", _i), ("entity_table_bf16", _vp), ("Ve", _i),
        ("mT_bf16", _vp), ("mb", _vp), ("wconv_bf16", _vp), ("bconv", _vp), ("wa_bf16", _vp), ("ba", _vp), ("qv", _vp),
        ("X2_bf16", _vp), ("E_bf16", _vp), ("Y_bf16", _vp), ("w", _vp), ("out", _vp), ("bad_id_flag", _vp),
    ]


class KcnnEncoderBwdArgs(C.Structure):
    """nr_kcnn_encoder_bwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("n_seq", _ll), ("T", _i), ("d", _i), ("de", _i), ("F", _i), ("q", _i), ("n_win", _i), ("win", _i * 4),
        ("ldx", _i), ("lde", _i), ("ldf", _i), ("ldo", _i), ("ldq", _i),
        ("word_ids", _vp), ("entity_ids", _vp), ("V", _i), ("Ve", _i),
        ("wT_word_bf16", _vp), ("wT_entity_bf16", _vp), ("m_bf16", _vp), ("wa_bf16", _vp), ("waT_bf16", _vp), ("ba", _vp),
        ("qv", _vp), ("X2_bf16", _vp), ("E_bf16", _vp), ("Y_bf16", _vp), ("w", _vp), ("dout", _vp),
        ("dWconv_ext", _vp), ("dM_ext", _vp), ("dWa_ext", _vp), ("dqv", _vp), ("dword", _vp), ("dentity", _vp),
        ("workspace", _vp), ("workspace_bytes", _ll),
    ]


class GruFwdArgs(C.Structure):
    """nr_gru_fwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("B", _i), ("S", _i), ("D", _i), ("Hd", _i),
        ("x", _vp), ("x_s_b", _ll), ("x_s_t", _ll), ("x_s_c", _ll),
        ("len", _vp), ("h0", _vp), ("wih_bf16", _vp), ("whh_bf16", _vp), ("bih", _vp), ("bhh", _vp),
        ("xb", _vp), ("gi", _vp), ("gh", _vp), ("hs", _vp), ("hb", _vp), ("out", _vp),
        ("x_lo_bf16", _vp),
    ]


class GruBwdArgs(C.Structure):
    """nr_gru_bwd_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("B", _i), ("S", _i), ("D", _i), ("Hd", _i),
        ("len", _vp), ("wihT_bf16", _vp), ("whhT_bf16", _vp),
        ("xb", _vp), ("gi", _vp), ("gh", _vp), ("hs", _vp), ("hb", _vp),
        ("dout", _vp), ("dWih_ext", _vp), ("dWhh_ext", _vp), ("dx", _vp), ("dh0", _vp),
        ("workspace", _vp), ("workspace_bytes", _ll),
    ]


class GemmStoreArgs(C.Structure):
    """nr_gemm_store_args (include/newsrec_b200.h)."""
    _fields_ = [
        ("A", _vp), ("M", _i), ("lda", _i), ("W", _vp), ("N", _i), ("ldw", _i), ("K", _i), ("taps", _i), ("w_tap_rows", _i),
        ("tap_origin", _i),
        ("out", _vp), ("ld_out", _i), ("out_bf16", _i), ("relu", _i), ("tanh", _i), ("dtanh_src", _vp), ("dtanh_ld", _i),
        ("bias", _vp),
        ("rm_seg_in", _i), ("rm_in_off", _i), ("rm_seg_len", _i), ("rm_seg_out", _i), ("rm_out_off", _i),
        ("p_drop", _f), ("seed", _ull),
        ("ones_col", _i), ("ones_zero_upto", _i), ("lo_out", _vp), ("ld_lo", _i), ("lo_col0", _i), ("accumulate", _i),
        ("rows_per_tile", _i),
    ]


class FeedField(C.Structure):
    """nr_feed_field (include/newsrec_b200.h)."""
    _fields_ = [("table", _vp), ("width", _i), ("out", _vp)]


# name -> (restype, argtypes).  Must list EVERY symbol include/newsrec_b200.h declares
# (tests/test_abi_symbols.py cross-checks this table against the header and the built .so).
SIGNATURES = {
    "nr_version": (_i, []),
    "nr_last_error": (C.c_char_p, []),
    "nr_device_error": (_i, [C.POINTER(_i * 4)]),
    "nr_launch_count": (_ll, []),
    "nr_num_sms": (_i, []),
    "nr_debug_set_simt_gemm": (None, [_i]),
    "nr_debug_set_gru_stepwise": (None, [_i]),
    "nr_debug_gemm_store": (_i, [C.POINTER(GemmStoreArgs), _vp]),
    "nr_has_triage_backends": (_i, []),
    "nr_reserve_sms_for_comm": (None, [_i]),
    "nr_debug_set_gemm_timing": (None, [_vp, _i]),
    "nr_debug_live_tokens": (_i, [_vp, _ll, _i, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nr_profile_enable": (None, [_i]),
    "nr_profile_context": (None, [C.c_char_p]),
    "nr_profile_report": (_i, [C.c_char_p, _i]),
    "nr_cast_pad_bf16": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp]),
    "nr_cast_pad_bf16_many": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nr_rows_to_bf16": (_i, [_vp, _ll, _i, _ll, _ll, _vp, _i, _vp]),
    "nr_rows_to_bf16_hilo": (_i, [_vp, _ll, _i, _ll, _ll, _vp, _vp, _i, _vp]),
    "nr_gather_rows": (_i, [_vp, _ll, _i, _vp, _i, _i, _i, _vp, _i, _f, _ull, _vp, _vp]),
    "nr_linear": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _vp]),
    "nr_gemm_tn": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "nr_mhsa_core_fwd": (_i, [_vp, _i, _i, _ll, _i, _i, _i, _vp, _i, _f, _ull, _vp]),
    "nr_mhsa_core_bwd": (_i, [_vp, _i, _i, _vp, _i, _ll, _i, _i, _i, _vp, _i, _vp]),
    "nr_additive_attention_fwd": (_i, [_vp, _ll, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _vp]),
    "nr_additive_attention_fwd_hilo": (_i, [_vp, _vp, _ll, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _vp]),
    "nr_additive_attention_bwd_workspace": (_ll, [_ll, _i, _i]),
    "nr_additive_attention_bwd": (_i, [_vp, _ll, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i,
                                        _vp, _vp, _vp, _ll, _vp]),
    "nr_dot_score_fwd": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "nr_slots_device_readable": (_i, [_vp, _i]),
    "nr_pack_slots": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "nr_feed_gather": (_i, [C.POINTER(FeedField), _i, _vp, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "nr_sample_negatives": (_i, [_vp, _vp, _vp, _ll, _vp, _i, _ull, _ll, _vp, _i, _vp]),
    "nr_segment_dot": (_i, [_vp, _ll, _i, _vp, _ll, _vp, _ll, _vp, _vp, _vp, _vp]),
    "nr_impression_metrics": (_i, [_vp, _vp, _vp, _ll, _vp, _vp, _vp]),
    "nr_impression_ranks": (_i, [_vp, _vp, _ll, _vp, _vp, _vp]),
    "nr_topk_dot_workspace": (_ll, [_ll, _ll, _i, _i]),
    "nr_topk_dot": (_i, [_vp, _ll, _i, _vp, _ll, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "nr_topk_dot_capped": (_i, [_vp, _ll, _i, _vp, _ll, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "nr_pool_ranks_workspace": (_ll, [_ll, _ll, _i]),
    "nr_pool_ranks": (_i, [_vp, _ll, _i, _vp, _ll, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "nr_prediction_line_offsets_workspace": (_ll, [_ll]),
    "nr_prediction_line_offsets": (_i, [_vp, _vp, _vp, _ll, _vp, _vp, _ll, _vp]),
    "nr_prediction_text": (_i, [_vp, _vp, _vp, _ll, _vp, _vp, _vp]),
    "nr_accumulate_ext_grad": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "nr_dot_score_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "nr_mhsa_accurate_supported": (_i, [_i, _i, _i]),
    "nr_mhsa_encoder_fwd": (_i, [C.POINTER(MhsaEncoderFwdArgs), _vp]),
    "nr_mhsa_encoder_bwd_workspace": (_ll, [_ll, _i, _i, _i]),
    "nr_mhsa_encoder_bwd": (_i, [C.POINTER(MhsaEncoderBwdArgs), _vp]),
    "nr_cnn_encoder_fwd": (_i, [C.POINTER(CnnEncoderFwdArgs), _vp]),
    "nr_cnn_encoder_bwd_workspace": (_ll, [_ll, _i, _i, _i]),
    "nr_cnn_encoder_bwd": (_i, [C.POINTER(CnnEncoderBwdArgs), _vp]),
    "nr_kcnn_encoder_fwd": (_i, [C.POINTER(KcnnEncoderFwdArgs), _vp]),
    "nr_kcnn_encoder_bwd_workspace": (_ll, [_ll, _i, _i, _i, _i, _i]),
    "nr_kcnn_encoder_bwd": (_i, [C.POINTER(KcnnEncoderBwdArgs), _vp]),
    "nr_linear_rows_fwd": (_i, [_vp, _ll, _i, _ll, _ll, _vp, _i, _vp, _i, _i, _vp, _i, _vp, _i, _vp]),
    "nr_linear_rows_bwd": (_i, [_vp, _vp, _ll, _i, _i, _vp, _i, _vp, _i, _i, _vp, _i, _vp, _vp, _i, _vp]),
    "nr_embedding_f32_fwd": (_i, [_vp, _ll, _vp, _i, _i, _vp, _vp, _vp]),
    "nr_embedding_f32_bwd": (_i, [_vp, _ll, _vp, _i, _i, _vp, _vp]),
    "nr_element_encoder_fwd": (_i, [_vp, _ll, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "nr_element_encoder_bwd": (_i, [_vp, _ll, _vp, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "nr_gru_fwd": (_i, [C.POINTER(GruFwdArgs), _vp]),
    "nr_gru_persistent_supported": (_i, [_i, _i]),
    "nr_gru_bwd_workspace": (_ll, [_i, _i, _i, _i]),
    "nr_gru_bwd": (_i, [C.POINTER(GruBwdArgs), _vp]),
    "nr_archive_user_fwd": (_i, [_vp, _ll, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "nr_archive_user_bwd_workspace": (_ll, [_ll, _i, _i]),
    "nr_archive_user_bwd": (_i, [_vp, _ll, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "nr_archive_score_fwd": (_i, [_vp, _ll, _i, _vp, _ll, _vp, _ll, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "nr_archive_score_bwd_workspace": (_ll, [_ll, _i, _i]),
    "nr_archive_score_bwd": (_i, [_vp, _ll, _i, _vp, _ll, _vp, _ll, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp,
                                   _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "nr_dkn_user_fwd": (_i, [_vp, _ll, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "nr_dkn_user_bwd_workspace": (_ll, [_ll, _i]),
    "nr_dkn_user_bwd": (_i, [_vp, _ll, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
}

_lib = None


class NewsrecError(RuntimeError):
    pass


def load_library(path: str | None = None):
    """dlopen the C-ABI library and attach signatures.  Raises if it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise NewsrecError(
            f"{p} not found: build it with `python __graft_entry__.py build` (or `make -C news-recommendation_b200/csrc`). "
            "There is no CPU / PyTorch fallback for the hot path.")
    lib = C.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def check(rc: int, what: str = ""):
    """Turn a non-zero ABI return code into an exception carrying nr_last_error()."""
    if rc != 0:
        lib = load_library()
        msg = lib.nr_last_error().decode(errors="replace")
        raise NewsrecError(f"{what} failed (code {rc}): {msg}")


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise NewsrecError("newsrec_b200 needs a CUDA (sm_90a) device: the hot path has no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def profile_report() -> dict:
    """Drain the live per-kernel timing records: {name: (launches, total_ms)}."""
    import json
    buf = C.create_string_buffer(1 << 16)
    n = load_library().nr_profile_report(buf, len(buf))
    if n < 0:
        raise NewsrecError("profile report does not fit the buffer")
    return {k: tuple(v) for k, v in json.loads(buf.value.decode()).items()}


def launch_count() -> int:
    return int(load_library().nr_launch_count())
