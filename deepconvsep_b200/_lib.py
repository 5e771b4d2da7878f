"""ctypes binding of libdcs.so (include/dcs.h).  No torch types cross this boundary: plain
pointers and sizes only.  There is NO fallback: a missing library or a missing CUDA device
raises."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libdcs.so")

ARCH_IDS = {"dsd": 0, "ikala": 1, "ikala_nopool": 2, "bach10": 3, "bach10_score": 4, "dsd_ild": 5, "bach10_score_1x1": 6}
PATCHER_IDS = {"standalone": 0, "util": 1}
# frames per chunk of the Wiener post-filter's sums over time (DCS_WIENER_CHUNK_FRAMES, include/dcs.h)
WIENER_CHUNK_FRAMES = 128
# the largest polyphase bank a resampler takes (DCS_RESAMPLE_MAX_BANK_BYTES, include/dcs.h)
RESAMPLE_MAX_BANK_BYTES = 112 * 1024


class DcsError(RuntimeError):
    pass


_p = C.c_void_p
_i64 = C.c_int64
_SIGS = {
    "dcs_version": (C.c_int, []),
    "dcs_last_error": (C.c_char_p, []),
    "dcs_create": (C.c_int, [C.c_int, C.POINTER(_p)]),
    "dcs_destroy": (C.c_int, [_p]),
    "dcs_workspace_bytes": (_i64, [_p]),
    "dcs_launch_count": (_i64, [_p]),
    "dcs_set_spectrum_tap": (C.c_int, [_p, _p, _i64]),
    "dcs_set_pool_tap": (C.c_int, [_p, _p, _i64]),
    "dcs_set_wiener": (C.c_int, [_p, C.c_int]),
    "dcs_wiener_stereo": (C.c_int, [_p, _p, _i64, _p, _i64, C.c_int, _i64, _i64, C.c_int, C.c_int, _p]),
    "dcs_set_wiener_radius": (C.c_int, [_p, C.c_int]),
    "dcs_wiener_stereo_windowed": (C.c_int, [_p, _p, _i64, _p, _i64, C.c_int, _i64, _i64, C.c_int, C.c_int, C.c_int, _p]),
    "dcs_wiener_channels": (C.c_int, [_p, _p, C.c_int, _i64, _p, _i64, C.c_int, _i64, _i64, C.c_int, C.c_int, C.c_int, _p]),
    "dcs_profile": (C.c_int, [_p, C.c_int]),
    "dcs_profile_read": (C.c_int, [_p, C.c_char_p, C.c_int, _p, C.c_int]),
    "dcs_stft_plan": (C.c_int, [_p, C.c_int, C.c_int, _p, _p, C.POINTER(_p)]),
    "dcs_stft_plan_destroy": (C.c_int, [_p]),
    "dcs_num_frames": (_i64, [_i64, C.c_int]),
    "dcs_padded_bins": (_i64, [C.c_int]),
    "dcs_stft_forward": (C.c_int, [_p, _p, _i64, _p, _p, C.c_float, _i64, _p]),
    "dcs_stft_forward_polar": (C.c_int, [_p, _p, _i64, _p, _p, C.c_float, _i64, _p]),
    "dcs_istft": (C.c_int, [_p, _p, C.c_int, _i64, _i64, _i64, _p, _i64, _i64, _p]),
    "dcs_istft_polar": (C.c_int, [_p, _p, _p, _p, C.c_float, _i64, _i64, _p, _i64, _p]),
    "dcs_model_create": (C.c_int, [_p, C.c_int, C.c_int, C.c_int, C.c_int, _p, _p, _p, C.POINTER(_p)]),
    "dcs_model_destroy": (C.c_int, [_p]),
    "dcs_model_nsources": (C.c_int, [_p]),
    "dcs_num_patches": (_i64, [_i64, C.c_int, C.c_int, C.c_int]),
    "dcs_separate_spec": (C.c_int, [_p, _p, _p, _p, _i64, _i64, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_spec_channels": (C.c_int, [_p, _p, _p, _i64, _p, _i64, _i64, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_audio_score": (C.c_int, [_p, _p, _p, _p, _i64, _p, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_score_filters": (C.c_int, [_p, _p, C.c_int, C.c_int, C.c_int, _i64, _i64, C.c_int, _p, _i64, _p, _i64, _p]),
    "dcs_separate_audio_notes": (C.c_int, [_p, _p, _p, _p, _i64, _p, C.c_int, C.c_int, _i64, C.c_float, C.c_int, C.c_int,
                                           _p, _i64, _p]),
    "dcs_separate_audio_stereo": (C.c_int, [_p, _p, _p, _p, _i64, _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_masks": (C.c_int, [_p, _p, _p, _p, _i64, _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_masks_score": (C.c_int, [_p, _p, _p, _p, _i64, _p, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_masks_notes": (C.c_int, [_p, _p, _p, _p, _i64, _p, C.c_int, C.c_int, _i64, C.c_float, C.c_int, C.c_int,
                                           _p, _i64, _p]),
    "dcs_istft_masked": (C.c_int, [_p, _p, C.c_int, _i64, _p, C.c_int, _i64, _i64, _i64, _p, _i64, _i64, _p]),
    "dcs_apply_masks": (C.c_int, [_p, _p, _p, C.c_int, _i64, _i64, _p, C.c_int, _i64, _p, _i64, _p]),
    "dcs_separate_audio_channels": (C.c_int, [_p, _p, _p, _p, C.c_int, _i64, _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_audio_channels_wiener": (C.c_int, [_p, _p, _p, _p, C.c_int, _i64, _i64, C.c_float, C.c_int, C.c_int, C.c_int,
                                                     C.c_int, _p, _i64, _p]),
    "dcs_separate_batch_pcm16_channels_host": (C.c_int, [_p, _p, _p, C.c_int, _p, _p, C.c_int, C.c_int, C.c_int, C.c_float,
                                                         C.c_int, C.c_int, _p, _p, _p]),
    "dcs_xcorr_lags": (C.c_int, [_p, _p, _p, C.c_int, _i64, C.c_int, _p, _p]),
    "dcs_gemm_f32": (C.c_int, [_p, C.c_int, _p, _i64, _p, _i64, _p, _p, _i64, C.c_int, C.c_int, C.c_int, C.c_int, _p]),
    "dcs_gemm_view_f32": (C.c_int, [_p, C.c_int, C.c_int, _p, _p, _p]),
    "dcs_dsd_mask_f32": (C.c_int, [_p, C.c_int, _p, _p]),
    "dcs_dsd_convt2_f32": (C.c_int, [_p, _p, _p, _p]),
    "dcs_dsd_dense_f32": (C.c_int, [_p, _p, _p, C.c_int, C.c_int, _p]),
    "dcs_sconv_mask_f32": (C.c_int, [_p, C.c_int, _p, _p]),
    "dcs_separate_audio": (C.c_int, [_p, _p, _p, _p, _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_host": (C.c_int, [_p, _p, _p, _p, _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_batch_pcm16_host": (C.c_int, [_p, _p, _p, C.c_int, _p, _p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _p, _p, _p]),
    "dcs_separate_pcm16_host": (C.c_int, [_p, _p, _p, _p, _i64, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                           _p, _i64, _p]),
    "dcs_separate_audio_keep_channels": (C.c_int, [_p, _p, _p, _p, _i64, _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_separate_batch_pcm16_keep_channels_host": (C.c_int, [_p, _p, _p, C.c_int, _p, _p, C.c_float, C.c_int, C.c_int,
                                                              _p, _p, _p]),
    "dcs_resampler_create": (C.c_int, [_p, C.c_int, C.c_int, _p, C.c_int, C.POINTER(_p)]),
    "dcs_resampler_destroy": (C.c_int, [_p]),
    "dcs_resampled_length": (_i64, [_i64, C.c_int, C.c_int]),
    "dcs_resample": (C.c_int, [_p, _p, C.c_int, _i64, _i64, _p, _i64, _i64, _p]),
    "dcs_separate_batch_pcm16_channels_resampled_host": (C.c_int, [_p, _p, _p, _p, _p, C.c_int, _p, _p, C.c_int, C.c_int,
                                                                   C.c_int, C.c_float, C.c_int, C.c_int, _p, _p, _p]),
    "dcs_pcm16_decode": (C.c_int, [_p, _p, C.c_int, _p, _i64, C.c_int, _p, _i64, _p]),
    "dcs_pcm16_encode": (C.c_int, [_p, _p, C.c_int, _p, _i64, C.c_int, C.c_int, _i64, _p, _i64, _i64, _p]),
    "dcs_downmix_f32": (C.c_int, [_p, _p, C.c_int, _i64, _i64, _p, _p]),
    "dcs_separate_batch_channels_host": (C.c_int, [_p, _p, _p, _p, _p, C.c_int, C.c_int, C.c_int, _p, _p, C.c_int, C.c_int,
                                                   C.c_int, C.c_float, C.c_int, C.c_int, _p, _p, _p]),
    "dcs_channels_decode": (C.c_int, [_p, _p, C.c_int, _p, _i64, C.c_int, _p, _i64, _p]),
    "dcs_channels_encode": (C.c_int, [_p, _p, C.c_int, _p, _i64, C.c_int, C.c_int, _i64, _p, _i64, _i64, _p]),
    "dcs_long_segments": (_i64, [_i64, _i64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                 _p, _i64]),
    "dcs_separate_long_channels_host": (C.c_int, [_p, _p, _p, _p, _p, C.c_int, C.c_int, _p, _i64, C.c_int, C.c_int, C.c_int,
                                                  _i64, C.c_float, C.c_int, C.c_int, _p, _i64, _p]),
    "dcs_channels_decode_range": (C.c_int, [_p, _p, C.c_int, _p, _i64, _i64, _i64, C.c_int, _p, _i64, _i64, _p]),
    "dcs_channels_encode_range": (C.c_int, [_p, _p, C.c_int, _p, _i64, _i64, _i64, C.c_int, C.c_int, _p, _i64, _i64, _i64,
                                            _p]),
}
# modes of dcs_pcm16_decode / dcs_pcm16_encode beside the downmix 0..2 (include/dcs.h)
PCM16_MONO, PCM16_CHANNELS = 0, 3
# sample formats of dcs_separate_batch_channels_host (DCS_SAMPLE_*, include/dcs.h)
SAMPLE_I16, SAMPLE_I32, SAMPLE_F32 = 0, 1, 2
SAMPLE_I24 = 4   # packed 3-byte PCM; code 3 is not a format


class Segment(C.Structure):
    """dcs_segment (include/dcs.h): the in, model and kept ranges of one segment of a long recording."""
    _fields_ = [("in_start", _i64), ("in_stop", _i64), ("model_start", _i64), ("model_stop", _i64),
                ("out_start", _i64), ("out_stop", _i64)]



class GemmView(C.Structure):
    """dcs_gemm_view (include/dcs.h): the operand view of dcs_gemm_view_f32, field for field."""
    _fields_ = [("A", _p), ("B", _p), ("bias", _p), ("C", _p),
                ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
                ("a_valid_rows", C.c_int),
                ("m_inner", C.c_int), ("a_so", _i64), ("a_si", _i64),
                ("m_inner2", C.c_int), ("a_s2", _i64),
                ("k_seg", C.c_int), ("k_ss", _i64),
                ("ldb", _i64),
                ("cm_inner", C.c_int), ("c_so", _i64), ("c_si", _i64),
                ("cm_inner2", C.c_int), ("c_s2", _i64),
                ("n_seg", C.c_int), ("n_ss", _i64), ("c_col0", _i64),
                ("relu", C.c_int),
                ("kc_rows", C.c_int), ("kc_unit", C.c_int), ("kc_pad", C.c_int), ("kc_n", C.c_int), ("kc_taps", C.c_int),
                ("bias2", _p), ("code", _p),
                ("gate", _p), ("g_inner", C.c_int), ("g_inner2", C.c_int),
                ("g_so", _i64), ("g_si", _i64), ("g_s2", _i64), ("g_lim", _i64)]


class DsdMaskView(C.Structure):
    """dcs_dsd_mask_view (include/dcs.h): the arguments of dcs_dsd_mask_f32, field for field."""
    _fields_ = [("G", _p), ("ldg", C.c_int), ("W1t", _p), ("ldw", C.c_int), ("bout", _p), ("X", _p), ("S", _p),
                ("ldf", _i64), ("src_stride", _i64),
                ("T", C.c_int), ("P", C.c_int), ("tc", C.c_int), ("overlap", C.c_int), ("F", C.c_int),
                ("ndec", C.c_int)]


class DsdConvT2View(C.Structure):
    """dcs_dsd_convt2_view (include/dcs.h): the arguments of dcs_dsd_convt2_f32, field for field."""
    _fields_ = [("apad", _p), ("G", _p), ("ldg", C.c_int), ("npairs", C.c_int), ("tc", C.c_int)]


class DsdDenseView(C.Structure):
    """dcs_dsd_dense_view (include/dcs.h): the arguments of dcs_dsd_dense_f32, field for field."""
    _fields_ = [("z", _p), ("bias", _p), ("apad", _p), ("P", C.c_int), ("tc", C.c_int), ("ndec", C.c_int), ("nfc", C.c_int)]


class SconvMaskView(C.Structure):
    """dcs_sconv_mask_view (include/dcs.h): the arguments of dcs_sconv_mask_f32, field for field."""
    _fields_ = [("arch", C.c_int), ("G", _p), ("tie", _p), ("W", _p), ("bout", _p), ("X", _p), ("S", _p),
                ("ldf", _i64), ("src_stride", _i64),
                ("T", C.c_int), ("P", C.c_int), ("tc", C.c_int), ("overlap", C.c_int), ("F", C.c_int), ("J", C.c_int),
                ("WP", C.c_int), ("p_base", C.c_int), ("t0", C.c_int), ("t1", C.c_int)]


_lib = None


def exported_symbols():
    """Names include/dcs.h declares (kept in sync by tests/test_abi.py)."""
    return sorted(_SIGS)


def load():
    """dlopen libdcs.so and attach the signatures.  Raises DcsError if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DcsError("libdcs.so is missing (%s): build it with `python -m deepconvsep_b200.build` "
                       "-- there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise DcsError("libdcs error %d: %s" % (rc, load().dcs_last_error().decode("utf-8", "replace")))
