"""ctypes binding of libwts.so — the C-ABI declared in include/wts.h.

PyTorch tensors are only the memory carrier: every call passes raw device pointers, sizes and
the current CUDA stream.  There is NO CPU fallback: if the library is missing or cannot be
loaded the import of the product fails loudly.
"""
import ctypes
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwts.so")


class WtsError(RuntimeError):
    pass


class SegDesc(ctypes.Structure):
    """Mirror of `WtsSegDesc` (include/wts.h)."""
    _fields_ = [
        ("window", ctypes.c_int32), ("row0", ctypes.c_int32), ("last_row", ctypes.c_int32),
        ("T", ctypes.c_int32), ("f0", ctypes.c_int32), ("F", ctypes.c_int32),
        ("max_dur", ctypes.c_int32), ("flags", ctypes.c_int32),
        ("cost_off", ctypes.c_int64), ("jumps_off", ctypes.c_int64),
        ("dir_off", ctypes.c_int64), ("bnd_off", ctypes.c_int64),
    ]


SEG_DTYPE = np.dtype([
    ("window", "<i4"), ("row0", "<i4"), ("last_row", "<i4"), ("T", "<i4"), ("f0", "<i4"),
    ("F", "<i4"), ("max_dur", "<i4"), ("flags", "<i4"), ("cost_off", "<i8"), ("jumps_off", "<i8"),
    ("dir_off", "<i8"), ("bnd_off", "<i8")])
assert SEG_DTYPE.itemsize == ctypes.sizeof(SegDesc) == 64


class Gemm(ctypes.Structure):
    """Mirror of `WtsGemm` (include/wts.h)."""
    _fields_ = [
        ("a", ctypes.c_void_p), ("lda", ctypes.c_int64), ("a_plane", ctypes.c_int64), ("a_bo", ctypes.c_int64), ("a_bi", ctypes.c_int64),
        ("b", ctypes.c_void_p), ("ldb", ctypes.c_int64), ("b_plane", ctypes.c_int64), ("b_bo", ctypes.c_int64), ("b_bi", ctypes.c_int64),
        ("M", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32), ("batch_outer", ctypes.c_int32), ("batch_inner", ctypes.c_int32),
        ("alpha", ctypes.c_float),
        ("bias", ctypes.c_void_p), ("bias_on_m", ctypes.c_int32), ("act", ctypes.c_int32),
        ("residual", ctypes.c_void_p), ("ldr", ctypes.c_int64), ("r_bo", ctypes.c_int64), ("r_bi", ctypes.c_int64),
        ("out_f32", ctypes.c_void_p), ("ldc", ctypes.c_int64), ("c_bo", ctypes.c_int64), ("c_bi", ctypes.c_int64),
        ("out_sb16", ctypes.c_void_p), ("ldo", ctypes.c_int64), ("o_plane", ctypes.c_int64), ("o_bo", ctypes.c_int64), ("o_bi", ctypes.c_int64),
        ("head_dim", ctypes.c_int32), ("head_stride", ctypes.c_int64),
        ("backend", ctypes.c_int32), ("a_is_f32", ctypes.c_int32), ("b_is_f32", ctypes.c_int32),
        ("row_mask", ctypes.c_void_p), ("b_const", ctypes.c_int32),
    ]


class DecodeCfg(ctypes.Structure):
    """Mirror of `WtsDecodeCfg`."""
    _fields_ = [("n_vocab", ctypes.c_int32), ("eot", ctypes.c_int32), ("timestamp_begin", ctypes.c_int32),
                ("no_timestamps", ctypes.c_int32), ("max_initial_ts", ctypes.c_int32), ("sample_len", ctypes.c_int32),
                ("n_ctx", ctypes.c_int32), ("tokens_ld", ctypes.c_int32)]


class DecLayer(ctypes.Structure):
    """Mirror of `WtsDecLayer`."""
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "ln1_g", "ln1_b", "b_qkv", "b_o", "ln2_g", "ln2_b", "b_cq", "b_co", "ln3_g", "ln3_b", "b_fc1", "b_fc2",
        "self_k", "self_v", "cross_k16", "cross_v16", "cross_k_align", "head_slot",
        "sb_qkv", "sb_o", "sb_cq", "sb_co", "sb_fc1", "sb_fc2")] + [(n, ctypes.c_int64) for n in (
        "pl_qkv", "pl_o", "pl_cq", "pl_co", "pl_fc1", "pl_fc2")] + [("align_s0", ctypes.c_int32), ("align_n", ctypes.c_int32)]


class DecodeSteps(ctypes.Structure):
    """Mirror of `WtsDecodeSteps`."""
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "layers", "emb", "pos", "ln_g", "ln_b", "tokens", "n_tokens", "n_prompt", "done",
        "logprobs", "full", "last_full", "qk_buf", "suppress", "blank",
        "x", "qkv", "att", "q", "mid", "logits", "emb_sb")] + [("emb_plane", ctypes.c_int64), ("cfg", DecodeCfg)] + [
        (n, ctypes.c_int32) for n in ("n_layer", "D", "H", "n_ctx", "n_audio_ctx", "n_slots", "cap", "lp_ld", "qk_rows",
                                      "max_rows")]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python whisper-timestamped_b200/build.py` "
            "(the product has no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.wts_version.restype = ctypes.c_int
    lib.wts_last_error.restype = ctypes.c_char_p
    lib.wts_dtw_dir_words.restype = ctypes.c_int64
    lib.wts_dtw_dir_words.argtypes = [ctypes.c_int32, ctypes.c_int32]
    lib.wts_dtw_bnd_doubles.restype = ctypes.c_int64
    lib.wts_dtw_bnd_doubles.argtypes = [ctypes.c_int32, ctypes.c_int32]
    vp, i32 = ctypes.c_void_p, ctypes.c_int32
    lib.wts_attn_prep_batch.restype = ctypes.c_int
    lib.wts_attn_prep_batch.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, vp, vp]
    lib.wts_attn_prep_batch_kernel.restype = ctypes.c_int
    lib.wts_attn_prep_batch_kernel.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, vp, i32, vp]
    lib.wts_dtw_batch.restype = ctypes.c_int
    lib.wts_dtw_batch.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.wts_dtw_batch_sized.restype = ctypes.c_int
    lib.wts_dtw_batch_sized.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, vp]
    lib.wts_disfluency_starts.restype = ctypes.c_int
    lib.wts_disfluency_starts.argtypes = [vp, vp, i32, vp, vp, vp]
    i64, f32p = ctypes.c_int64, vp
    lib.wts_gemm.restype = ctypes.c_int
    lib.wts_gemm.argtypes = [ctypes.POINTER(Gemm), vp]
    lib.wts_to_sb16.argtypes = [vp, i64, vp, vp, vp]
    lib.wts_layernorm.argtypes = [vp, i64, vp, vp, i32, i32, vp, i64, i64, vp, i64, vp]
    lib.wts_softmax_rows.argtypes = [vp, i64, i64, i32, vp, i64, i64, vp]
    lib.wts_frames.argtypes = [vp, i64, i64, i64, vp, i64, vp]
    lib.wts_power.argtypes = [vp, i64, i64, vp, i64, i64, vp]
    lib.wts_logmel_max.argtypes = [vp, i64, vp, vp]
    lib.wts_logmel_finish.argtypes = [vp, i64, i32, vp, vp, vp]
    lib.wts_window_gather.argtypes = [vp, i32, vp, vp, i32, vp, i64, vp]
    lib.wts_embed.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.wts_gather_rows.argtypes = [vp, i64, vp, i32, i32, vp, vp]
    lib.wts_decoder_attention.argtypes = [i32, vp, i64, vp, vp, i64, i32, vp, vp, i32, i32, vp, i64, i64, vp, vp, i32,
                                          i32, vp, vp, vp]
    lib.wts_cross_kv_pack.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.wts_cross_attention_f16.argtypes = [vp, i64, vp, vp, vp, vp, i32, i32, vp, i32, i32, vp, i64, i64, vp, i32, vp, vp, vp]
    lib.wts_cross_kv_pack_layer.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    lib.wts_cross_attention_f16_layer.argtypes = [vp, i64, vp, vp, vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, i64, i64,
                                                  vp, i32, vp, vp, vp]
    lib.wts_enc_attention.argtypes = [vp, i64, i64, vp, i64, i64, i32, i32, i32, i32, vp, i64, i64, vp]
    lib.wts_enc_attention.restype = ctypes.c_int
    lib.wts_kv_append.argtypes = [vp, vp, i64, vp, vp, i32, i32, i32, vp, vp, i64, vp]
    lib.wts_decode_select.argtypes = [vp, i64, ctypes.POINTER(DecodeCfg), vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, i32, vp]
    lib.wts_filtered_logprobs.argtypes = [vp, i64, ctypes.POINTER(DecodeCfg), vp, vp, vp, vp, vp, vp, i32, vp]
    lib.wts_filtered_logprobs.restype = ctypes.c_int
    lib.wts_decode_step_kernels.argtypes = [ctypes.POINTER(DecodeSteps), vp, vp]
    lib.wts_decode_step_kernels.restype = ctypes.c_int
    lib.wts_step_inputs.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp]
    lib.wts_softmax_pick.argtypes = [vp, i64, i32, i32, vp, i32, vp]
    lib.wts_logprob_gather.argtypes = [vp, i64, i32, vp, vp, vp, i32, vp]
    for name in ("wts_to_sb16", "wts_layernorm", "wts_softmax_rows", "wts_frames", "wts_power", "wts_logmel_max",
                 "wts_logmel_finish", "wts_window_gather", "wts_embed", "wts_gather_rows", "wts_decoder_attention",
                 "wts_kv_append", "wts_decode_select", "wts_step_inputs", "wts_softmax_pick", "wts_logprob_gather", "wts_cross_kv_pack",
                 "wts_cross_attention_f16", "wts_cross_kv_pack_layer", "wts_cross_attention_f16_layer"):
        getattr(lib, name).restype = ctypes.c_int
    return lib


lib = _load()

EXPORTED_SYMBOLS = [
    "wts_version", "wts_last_error", "wts_dtw_dir_words", "wts_dtw_bnd_doubles",
    "wts_attn_prep_batch", "wts_dtw_batch", "wts_dtw_batch_sized", "wts_disfluency_starts", "wts_gemm", "wts_to_sb16", "wts_layernorm", "wts_softmax_rows",
    "wts_frames", "wts_power", "wts_logmel_max", "wts_logmel_finish", "wts_window_gather", "wts_embed",
    "wts_gather_rows", "wts_decoder_attention", "wts_kv_append", "wts_decode_select", "wts_filtered_logprobs", "wts_decode_step_kernels", "wts_step_inputs",
    "wts_softmax_pick", "wts_logprob_gather", "wts_cross_kv_pack", "wts_cross_attention_f16", "wts_enc_attention",
    "wts_cross_kv_pack_layer", "wts_cross_attention_f16_layer", "wts_attn_prep_batch_kernel",
]


def check(rc: int, what: str):
    if rc != 0:
        raise WtsError(f"{what} failed ({rc}): {lib.wts_last_error().decode(errors='replace')}")


def ptr(t):
    """Device pointer of a tensor (or None)."""
    if t is None:
        return None
    assert t.is_contiguous(), "libwts needs contiguous buffers"
    return ctypes.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(t, name):
    if not t.is_cuda:
        raise WtsError(f"{name} must live on a CUDA device: libwts has no CPU path")
