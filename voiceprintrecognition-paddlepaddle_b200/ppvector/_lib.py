"""ctypes binding of libppv_b200.so (C ABI: include/ppv_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``csrc/Makefile`` and lives next to this package
(``../lib/libppv_b200.so``).  Loading fails loudly: the product path has no CPU or eager-PyTorch fallback.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.normpath(os.path.join(_HERE, "..", "lib", "libppv_b200.so"))

PPV_PREC_BF16X3 = 0
PPV_PREC_BF16 = 1
PPV_MODEL_ECAPA_TDNN = 1
PPV_POOL_ASP, PPV_POOL_SAP, PPV_POOL_TAP, PPV_POOL_TSP = 0, 1, 2, 3


class PPVError(RuntimeError):
    pass


class FbankCfg(C.Structure):
    _fields_ = [("sample_rate", C.c_int), ("n_mels", C.c_int), ("frame_length_ms", C.c_float),
                ("frame_shift_ms", C.c_float), ("preemph", C.c_float), ("low_freq", C.c_float),
                ("high_freq", C.c_float), ("log_floor", C.c_float)]


class EcapaCfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("channels", C.c_int * 5),
                ("kernel_sizes", C.c_int * 5), ("dilations", C.c_int * 5), ("attention_channels", C.c_int),
                ("res2net_scale", C.c_int), ("se_channels", C.c_int), ("precision", C.c_int), ("pooling", C.c_int),
                ("global_context", C.c_int)]


class ResNetSECfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("layers", C.c_int * 4), ("num_filters", C.c_int * 4),
                ("attention_channels", C.c_int), ("reduction", C.c_int), ("precision", C.c_int)]


PPV_MODEL_RESNET_SE = 2
PPV_MODEL_ERES2NET = 3


class ERes2NetCfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("num_blocks", C.c_int * 4), ("m_channels", C.c_int),
                ("precision", C.c_int), ("version", C.c_int), ("base_width", C.c_int)]


PPV_MODEL_CAMPPLUS = 4
PPV_SPEC_SPECTROGRAM, PPV_SPEC_MEL, PPV_SPEC_LOGMEL, PPV_SPEC_MFCC = 1, 2, 3, 4
PPV_SPECAUG_NPARAM = 16
PPV_PREP_NI, PPV_PREP_NF = 8, 4
PPV_HEAD_AAM, PPV_HEAD_AAM_EASY, PPV_HEAD_AM, PPV_HEAD_ARM, PPV_HEAD_CE = 0, 1, 2, 3, 4
PPV_HEAD_SUBCENTER = 16  # | (K << 5) | easy_margin
PPV_HEAD_SPHEREFACE2 = 8  # | (t << 5) | (margin_type == 'A'); lanbuda in the label_smoothing slot


class SpectralCfg(C.Structure):
    _fields_ = [("method", C.c_int), ("sample_rate", C.c_int), ("n_fft", C.c_int), ("hop_length", C.c_int), ("win_length", C.c_int),
                ("power", C.c_float), ("center", C.c_int), ("n_mels", C.c_int), ("f_min", C.c_float), ("f_max", C.c_float),
                ("htk", C.c_int), ("norm_slaney", C.c_int), ("ref_value", C.c_float), ("amin", C.c_float), ("n_mfcc", C.c_int)]


class CamPPlusCfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("growth_rate", C.c_int), ("bn_size", C.c_int),
                ("init_channels", C.c_int), ("precision", C.c_int)]


_P = C.c_void_p
# name -> (restype, argtypes); this table is also what tests/test_abi.py checks against include/ppv_b200.h
SIGNATURES = {
    "ppv_version": (C.c_int, []),
    "ppv_last_error": (C.c_int, [C.c_char_p, C.c_size_t]),
    "ppv_device_sm_count": (C.c_int, []),
    "ppv_fbank_default_cfg": (None, [C.POINTER(FbankCfg)]),
    "ppv_fbank_create": (C.c_int, [C.POINTER(FbankCfg), C.POINTER(_P)]),
    "ppv_fbank_destroy": (C.c_int, [_P]),
    "ppv_fbank_num_frames": (C.c_int, [_P, C.c_int]),
    "ppv_fbank_feature_dim": (C.c_int, [_P]),
    "ppv_fbank_forward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ppv_spectral_default_cfg": (None, [C.POINTER(SpectralCfg), C.c_int]),
    "ppv_spectral_create": (C.c_int, [C.POINTER(SpectralCfg), C.POINTER(_P)]),
    "ppv_spectral_destroy": (C.c_int, [_P]),
    "ppv_spectral_num_frames": (C.c_int, [_P, C.c_int]),
    "ppv_spectral_feature_dim": (C.c_int, [_P]),
    "ppv_spectral_forward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ppv_spec_augment": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "ppv_ecapa_default_cfg": (None, [C.POINTER(EcapaCfg)]),
    "ppv_resnetse_default_cfg": (None, [C.POINTER(ResNetSECfg)]),
    "ppv_eres2net_default_cfg": (None, [C.POINTER(ERes2NetCfg)]),
    "ppv_campplus_default_cfg": (None, [C.POINTER(CamPPlusCfg)]),
    "ppv_model_create": (C.c_int, [C.c_int, _P, C.POINTER(_P)]),
    "ppv_model_destroy": (C.c_int, [_P]),
    "ppv_model_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int]),
    "ppv_model_finalize": (C.c_int, [_P]),
    "ppv_model_set_precision": (C.c_int, [_P, C.c_int]),
    "ppv_model_embd_dim": (C.c_int, [_P]),
    "ppv_model_workspace_bytes": (C.c_size_t, [_P, C.c_int, C.c_int]),
    "ppv_model_forward": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_model_forward_lengths": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_model_forward_wav": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_model_read_tap": (C.c_int, [_P, C.c_char_p, _P, C.c_size_t, _P]),
    "ppv_model_profile": (C.c_int, [_P, C.c_int]),
    "ppv_model_profile_read": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int64)]),
    "ppv_trainer_create": (C.c_int, [C.POINTER(EcapaCfg), C.c_int, C.POINTER(_P)]),
    "ppv_trainer_destroy": (C.c_int, [_P]),
    "ppv_trainer_param_count": (C.c_int64, [_P]),
    "ppv_trainer_stat_count": (C.c_int64, [_P]),
    "ppv_trainer_lookup": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "ppv_trainer_bind": (C.c_int, [_P, _P, _P, _P]),
    "ppv_trainer_set_precision": (C.c_int, [_P, C.c_int]),
    "ppv_set_pdl": (C.c_int, [C.c_int]),
    "ppv_trainer_workspace_bytes": (C.c_size_t, [_P, C.c_int, C.c_int]),
    "ppv_trainer_forward_backward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, _P, _P, _P,
                                               C.c_size_t, _P]),
    "ppv_trainer_read_tap": (C.c_int, [_P, C.c_char_p, _P, C.c_size_t, _P]),
    "ppv_adam_step": (C.c_int, [_P, _P, _P, _P, C.c_int64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int64, C.c_float, _P]),
    "ppv_cosine_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_cosine_matrix": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_cosine_pairlist": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, _P, _P]),
    "ppv_fbank_forward_ragged": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ppv_audio_prep_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "ppv_audio_prep": (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_audio_prep_reverb_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_audio_prep_reverb": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_int64, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                        _P, _P, C.c_size_t, _P]),
    "ppv_eer_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "ppv_eer_mindcf": (C.c_int, [_P, _P, C.c_int64, C.c_double, C.c_double, C.c_double, _P, _P, C.c_size_t, _P]),
    "ppv_eer_mindcf_matrix": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, _P, _P, C.c_size_t, _P]),
    "ppv_row_argmax": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P]),
    "ppv_cluster_prune": (C.c_int, [_P, C.c_int, C.c_double, _P]),
    "ppv_cluster_laplacian": (C.c_int, [_P, C.c_int, _P, _P]),
    "ppv_sym_eig_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "ppv_sym_eig_smallest": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, C.c_size_t, _P]),
    "ppv_kmeans_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "ppv_kmeans": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, C.c_size_t, _P]),
    "ppv_aam_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_aam_forward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float,
                                  _P, _P, _P, C.c_size_t, _P]),
    "ppv_aam_backward": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int,
                                   C.c_float, _P, _P, _P, C.c_size_t, _P]),
    "ppv_gemm_test_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_gemm_bench": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_size_t,
                                 C.POINTER(C.c_float), _P]),
    "ppv_gemm_test": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P,
                                C.c_size_t, _P]),
    "ppv_gemm_test_planes": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_conv2d_test_workspace_bytes": (C.c_size_t, [C.c_int] * 7),
    "ppv_conv2d_test": (C.c_int, [_P, _P, _P] + [C.c_int] * 13 + [_P, _P, C.c_size_t, _P]),
    "ppv_asp_fused_test_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "ppv_asp_fused_test": (C.c_int, [_P] * 6 + [C.c_int] * 8 + [_P, _P, _P, C.c_size_t, _P]),
}

_lib = None


def load(path: str = None):
    """dlopen the library and declare every prototype.  No compute, no GPU needed for this step."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise PPVError(f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       f"(there is no CPU fallback for the ppvector hot path)")
    lib = C.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def last_error(lib=None) -> str:
    lib = lib or load()
    buf = C.create_string_buffer(2048)
    lib.ppv_last_error(buf, 2048)
    return buf.value.decode("utf-8", "replace")


def check(rc: int, what: str = ""):
    if rc != 0:
        raise PPVError(f"{what} failed with status {rc}: {last_error()}")


def ptr(t):
    """Device pointer of a contiguous torch tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_contiguous(), "ppv: tensor must be contiguous"
    return C.c_void_p(t.data_ptr())


def require_cuda(t, name="tensor"):
    if not t.is_cuda:
        raise PPVError(f"ppv: {name} must be a CUDA tensor -- the ppvector hot path has no CPU fallback")


def current_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
