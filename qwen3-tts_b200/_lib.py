"""ctypes binding of libqwen3tts_b200.so (C ABI declared in include/qwen3tts_b200.h).

The product path has NO CPU fallback: if the CUDA library is missing or fails to load, importing the engine
raises immediately.
"""
import ctypes as C
import os

from . import build as _build

MAXB = 32


class StackCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("hidden_size", "num_layers", "num_heads", "num_kv_heads", "head_dim",
                                          "intermediate_size", "vocab_size")] + [("rms_eps", C.c_float)]


class EngineCfg(C.Structure):
    _fields_ = [("talker", StackCfg), ("cp", StackCfg), ("num_code_groups", C.c_int32),
                ("has_cp_projection", C.c_int32), ("codec_eos_token_id", C.c_int32), ("max_batch", C.c_int32),
                ("max_ctx", C.c_int32), ("device", C.c_int32)]


class Sampling(C.Structure):
    _fields_ = [("do_sample", C.c_int32), ("top_k", C.c_int32), ("top_p", C.c_float), ("temperature", C.c_float),
                ("repetition_penalty", C.c_float), ("subtalker_dosample", C.c_int32), ("subtalker_top_k", C.c_int32),
                ("subtalker_top_p", C.c_float), ("subtalker_temperature", C.c_float), ("min_new_tokens", C.c_int32),
                ("suppress_eos", C.c_int32), ("seed", C.c_uint64)]


class CodecCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("codebook_size", "codebook_dim", "hidden_size", "latent_dim", "num_heads",
                                          "num_kv_heads", "head_dim", "sliding_window", "intermediate_size",
                                          "num_layers", "num_quantizers")] + \
               [("n_upsample_rates", C.c_int32), ("upsample_rates", C.c_int32 * 8),
                ("n_upsampling_ratios", C.c_int32), ("upsampling_ratios", C.c_int32 * 8),
                ("decoder_dim", C.c_int32), ("rms_eps", C.c_float), ("rope_theta", C.c_float),
                ("max_frames", C.c_int32), ("max_batch", C.c_int32), ("device", C.c_int32)]


class CodecEncCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("num_filters", "kernel_size", "last_kernel_size", "residual_kernel_size",
                                          "compress", "n_ratios")] + \
               [("ratios", C.c_int32 * 8)] + \
               [(n, C.c_int32) for n in ("hidden_size", "num_layers", "num_heads", "head_dim", "intermediate_size",
                                          "sliding_window")] + \
               [("norm_eps", C.c_float)] + \
               [(n, C.c_int32) for n in ("codebook_size", "codebook_dim", "num_semantic_quantizers", "num_quantizers",
                                          "downsample_stride", "max_frames", "device")]


class SpkCfg(C.Structure):
    _fields_ = [("mel_dim", C.c_int32), ("enc_dim", C.c_int32), ("n_blocks", C.c_int32), ("channels", C.c_int32 * 8),
                ("kernel_sizes", C.c_int32 * 8), ("dilations", C.c_int32 * 8), ("attention_channels", C.c_int32),
                ("res2net_scale", C.c_int32), ("se_channels", C.c_int32), ("n_fft", C.c_int32), ("hop", C.c_int32),
                ("win", C.c_int32), ("device", C.c_int32)]


# every symbol include/qwen3tts_b200.h declares (tests/test_abi.py checks the header against this list)
AR_SYMBOLS = ["q3_abi_version", "q3_last_error", "q3_engine_create", "q3_engine_destroy", "q3_engine_load_tensor",
              "q3_engine_finalize", "q3_prefill", "q3_decode", "q3_get_progress", "q3_set_debug",
              "q3_algorithmic_bytes", "q3_set_profile", "q3_describe_frame_program",
              "q3_session_begin", "q3_release_slots", "q3_append_trailing", "q3_set_hidden_capture",
              "q3_admit_with_sampling", "q3_sampling_check", "q3_set_trailing_open",
              "q3_prefix_create", "q3_prefix_free", "q3_prefix_length", "q3_admit_with_prefix",
              "q3_row_park", "q3_row_resume", "q3_row_discard"]
CODEC_SYMBOLS = ["q3_codec_create", "q3_codec_destroy", "q3_codec_load_tensor", "q3_codec_finalize",
                 "q3_codec_forward", "q3_codec_total_upsample", "q3_codec_last_launch_count", "q3_codec_debug_capture",
                 "q3_codec_stream_open", "q3_codec_stream_close",
                 "q3_codec_stream_step_rows", "q3_codec_stream_reset_rows", "q3_codec_stream_row_position",
                 "q3_codec_stream_copy_rows",
                 "q3_codec_enc_create", "q3_codec_enc_destroy", "q3_codec_enc_load_tensor", "q3_codec_enc_finalize",
                 "q3_codec_enc_encode", "q3_codec_enc_frames", "q3_codec_enc_hop", "q3_codec_enc_last_launch_count",
                 "q3_codec_enc_debug_capture",
                 "q3_codec_enc_stream_open", "q3_codec_enc_stream_step_rows", "q3_codec_enc_stream_finish_rows",
                 "q3_codec_enc_stream_reset_rows", "q3_codec_enc_stream_row_position", "q3_codec_enc_stream_close",
                 "q3_spk_create", "q3_spk_destroy", "q3_spk_load_tensor", "q3_spk_finalize", "q3_spk_frames", "q3_spk_mel",
                 "q3_spk_embed", "q3_spk_last_launch_count",
                 "q3_resample_open", "q3_resample_close", "q3_resample_add_filter", "q3_resample_reset_rows",
                 "q3_resample_step_rows", "q3_resample_save_rows", "q3_resample_load_rows",
                 "q3_resample_drop_filter", "q3_resample_release_rows",
                 "q3_stretch_open", "q3_stretch_close", "q3_stretch_set_window", "q3_stretch_reset_rows",
                 "q3_stretch_step_rows", "q3_stretch_save_rows", "q3_stretch_load_rows",
                 "q3_limit_open", "q3_limit_close", "q3_limit_reset_rows", "q3_limit_step_rows", "q3_limit_save_rows",
                 "q3_limit_load_rows",
                 "q3_loud_open", "q3_loud_close", "q3_loud_set_filter", "q3_loud_reset_rows", "q3_loud_step_rows",
                 "q3_loud_save_rows", "q3_loud_load_rows"]

_lib = None


def lib_path():
    return _build.LIB_PATH


def load():
    """Load (building first if the in-tree .so is stale/missing and nvcc is present)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    try:
        # no-op when lib/build.stamp matches the digest of csrc/ + include/ + flags; rebuilds a stale or missing .so
        path = _build.build(force=bool(os.environ.get("Q3_REBUILD")))
    except Exception as e:
        if not os.path.exists(path):
            raise
        import warnings
        warnings.warn(f"qwen3tts_b200: could not rebuild ({e!r}); loading the existing {path}", RuntimeWarning)
    try:
        import torch  # noqa: F401  (makes sure libcudart.so.12 is already mapped)
    except Exception:
        pass
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.q3_abi_version.restype = C.c_int
    lib.q3_last_error.restype = C.c_char_p
    lib.q3_engine_create.argtypes = [C.POINTER(EngineCfg), C.POINTER(vp)]
    lib.q3_engine_destroy.argtypes = [vp]
    lib.q3_engine_destroy.restype = None
    lib.q3_engine_load_tensor.argtypes = [vp, C.c_char_p, vp, i64, i64]
    lib.q3_engine_finalize.argtypes = [vp]
    lib.q3_prefill.argtypes = [vp, i32, vp, C.POINTER(i32), vp, C.POINTER(i32), i32, vp, C.POINTER(Sampling), vp]
    lib.q3_decode.argtypes = [vp, i32, vp, i32, vp]
    lib.q3_session_begin.argtypes = [vp, i32, i32, vp, C.POINTER(Sampling), vp]
    lib.q3_release_slots.argtypes = [vp, i32, C.POINTER(i32), vp]
    lib.q3_append_trailing.argtypes = [vp, i32, vp, i32, vp]
    lib.q3_set_hidden_capture.argtypes = [vp, vp, i32]
    lib.q3_set_trailing_open.argtypes = [vp, i32, i32]
    lib.q3_admit_with_sampling.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(C.c_uint32), C.POINTER(Sampling), vp,
                                           C.POINTER(i32), vp, C.POINTER(i32), i32, vp]
    lib.q3_admit_with_prefix.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(C.c_uint32), C.POINTER(Sampling), C.POINTER(i32),
                                         vp, C.POINTER(i32), vp, C.POINTER(i32), i32, vp]
    lib.q3_prefix_create.argtypes = [vp, vp, i32, vp, C.POINTER(i32)]
    lib.q3_prefix_free.argtypes = [vp, i32, vp]
    lib.q3_prefix_length.argtypes = [vp, i32]
    lib.q3_row_park.argtypes = [vp, i32, vp, C.POINTER(i32)]
    lib.q3_row_resume.argtypes = [vp, i32, i32, vp]
    lib.q3_row_discard.argtypes = [vp, i32, vp]
    lib.q3_sampling_check.argtypes = [C.POINTER(Sampling)]
    lib.q3_get_progress.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    lib.q3_set_debug.argtypes = [vp, vp, i32, vp, vp]
    lib.q3_set_profile.argtypes = [vp, vp]
    lib.q3_describe_frame_program.argtypes = [vp, C.POINTER(i32), i32]
    lib.q3_algorithmic_bytes.argtypes = [vp, i32, i32, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    if hasattr(lib, "q3_codec_create"):
        lib.q3_codec_create.argtypes = [C.POINTER(CodecCfg), C.POINTER(vp)]
        lib.q3_codec_destroy.argtypes = [vp]
        lib.q3_codec_destroy.restype = None
        lib.q3_codec_load_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32]
        lib.q3_codec_finalize.argtypes = [vp]
        lib.q3_codec_forward.argtypes = [vp, vp, i32, i32, vp, vp]
        lib.q3_codec_stream_open.argtypes = [vp, i32, i32, C.POINTER(vp)]
        lib.q3_codec_stream_step_rows.argtypes = [vp, vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_codec_stream_reset_rows.argtypes = [vp, i32, C.POINTER(i32), vp]
        lib.q3_codec_stream_row_position.argtypes = [vp, i32]
        lib.q3_codec_stream_copy_rows.argtypes = [vp, vp, i32, C.POINTER(i32), C.POINTER(i32), vp]
        lib.q3_codec_stream_close.argtypes = [vp]
        lib.q3_codec_stream_close.restype = None
        lib.q3_codec_total_upsample.argtypes = [vp]
        lib.q3_codec_last_launch_count.argtypes = [vp]
        lib.q3_codec_debug_capture.argtypes = [vp, i32, vp, i64]
        lib.q3_codec_enc_create.argtypes = [C.POINTER(CodecEncCfg), C.POINTER(vp)]
        lib.q3_codec_enc_destroy.argtypes = [vp]
        lib.q3_codec_enc_destroy.restype = None
        lib.q3_codec_enc_load_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32]
        lib.q3_codec_enc_finalize.argtypes = [vp]
        lib.q3_codec_enc_encode.argtypes = [vp, vp, i32, i32, vp, vp]
        lib.q3_codec_enc_frames.argtypes = [vp, i32]
        lib.q3_codec_enc_hop.argtypes = [vp]
        lib.q3_codec_enc_last_launch_count.argtypes = [vp]
        lib.q3_codec_enc_debug_capture.argtypes = [vp, i32, vp, i64]
        lib.q3_codec_enc_stream_open.argtypes = [vp, i32, i32, C.POINTER(vp)]
        lib.q3_codec_enc_stream_step_rows.argtypes = [vp, vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_codec_enc_stream_finish_rows.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), vp, vp, vp]
        lib.q3_codec_enc_stream_reset_rows.argtypes = [vp, i32, C.POINTER(i32), vp]
        lib.q3_codec_enc_stream_row_position.argtypes = [vp, i32]
        lib.q3_codec_enc_stream_close.argtypes = [vp]
        lib.q3_codec_enc_stream_close.restype = None
        lib.q3_spk_create.argtypes = [C.POINTER(SpkCfg), C.POINTER(vp)]
        lib.q3_spk_destroy.argtypes = [vp]
        lib.q3_spk_destroy.restype = None
        lib.q3_spk_load_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32]
        lib.q3_spk_finalize.argtypes = [vp]
        lib.q3_spk_frames.argtypes = [vp, i32]
        lib.q3_spk_mel.argtypes = [vp, vp, i32, i32, vp, vp]
        lib.q3_spk_embed.argtypes = [vp, vp, i32, i32, vp, i32, vp, vp]
        lib.q3_spk_last_launch_count.argtypes = [vp]
        lib.q3_resample_open.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
        lib.q3_resample_close.argtypes = [vp]
        lib.q3_resample_close.restype = None
        lib.q3_resample_add_filter.argtypes = [vp, i32, i32, vp, i32, C.POINTER(i32)]
        lib.q3_resample_reset_rows.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
        lib.q3_resample_step_rows.argtypes = [vp, vp, i64, C.POINTER(i32), C.POINTER(i32), vp, C.POINTER(i32), vp]
        lib.q3_resample_save_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_resample_load_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_resample_drop_filter.argtypes = [vp, i32]
        lib.q3_resample_release_rows.argtypes = [vp, i32, C.POINTER(i32)]
        lib.q3_stretch_open.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
        lib.q3_stretch_close.argtypes = [vp]
        lib.q3_stretch_close.restype = None
        lib.q3_stretch_set_window.argtypes = [vp, vp]
        lib.q3_stretch_reset_rows.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32)]
        lib.q3_stretch_step_rows.argtypes = [vp, vp, i64, C.POINTER(i32), C.POINTER(i32), vp, C.POINTER(i32), vp]
        lib.q3_stretch_save_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_stretch_load_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_limit_open.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
        lib.q3_limit_close.argtypes = [vp]
        lib.q3_limit_close.restype = None
        lib.q3_limit_reset_rows.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(C.c_float)]
        lib.q3_limit_step_rows.argtypes = [vp, vp, i64, C.POINTER(i32), C.POINTER(i32), vp, C.POINTER(i32), vp]
        lib.q3_limit_save_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_limit_load_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_loud_open.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
        lib.q3_loud_close.argtypes = [vp]
        lib.q3_loud_close.restype = None
        lib.q3_loud_set_filter.argtypes = [vp, C.POINTER(C.c_float)]
        lib.q3_loud_reset_rows.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(C.c_double)]
        lib.q3_loud_step_rows.argtypes = [vp, vp, i64, C.POINTER(i32), C.POINTER(i32), vp, C.POINTER(i32), vp]
        lib.q3_loud_save_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
        lib.q3_loud_load_rows.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise RuntimeError("qwen3tts_b200: " + load().q3_last_error().decode())
