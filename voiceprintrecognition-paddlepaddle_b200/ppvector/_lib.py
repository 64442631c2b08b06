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
PPV_CLASSIFIER_COSINE, PPV_CLASSIFIER_LINEAR = 0, 1
PPV_RES2_CHAIN, PPV_RES2_CHAIN_PAIRED, PPV_RES2_PER_CONV = 0, 1, 2
PPV_OPT_ADAM, PPV_OPT_ADAMW, PPV_OPT_SGD, PPV_OPT_MOMENTUM, PPV_OPT_RMSPROP = 0, 1, 2, 3, 4


class PPVError(RuntimeError):
    pass


PPV_FBANK_WIN_POVEY, PPV_FBANK_WIN_HANNING, PPV_FBANK_WIN_HAMMING, PPV_FBANK_WIN_RECTANGULAR, PPV_FBANK_WIN_BLACKMAN = 0, 1, 2, 3, 4


class FbankCfg(C.Structure):
    _fields_ = [("sample_rate", C.c_int), ("n_mels", C.c_int), ("frame_length_ms", C.c_float),
                ("frame_shift_ms", C.c_float), ("preemph", C.c_float), ("low_freq", C.c_float),
                ("high_freq", C.c_float), ("log_floor", C.c_float), ("window_type", C.c_int), ("blackman_coeff", C.c_float),
                ("remove_dc_offset", C.c_int), ("snip_edges", C.c_int), ("use_power", C.c_int), ("use_log_fbank", C.c_int),
                ("vtln_warp", C.c_float), ("vtln_low", C.c_float), ("vtln_high", C.c_float)]


class EcapaCfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("channels", C.c_int * 5),
                ("kernel_sizes", C.c_int * 5), ("dilations", C.c_int * 5), ("attention_channels", C.c_int),
                ("res2net_scale", C.c_int), ("se_channels", C.c_int), ("precision", C.c_int), ("pooling", C.c_int),
                ("global_context", C.c_int)]


class OptimArgs(C.Structure):
    """ppv_optim_args: the hyper-parameters of one ppv_optimizer_step"""
    _fields_ = [("lr", C.c_float), ("weight_decay", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("epsilon", C.c_float),
                ("momentum", C.c_float), ("rho", C.c_float), ("rescale_grad", C.c_float), ("use_nesterov", C.c_int), ("centered", C.c_int)]


class ResNetSECfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("layers", C.c_int * 4), ("num_filters", C.c_int * 4),
                ("attention_channels", C.c_int), ("reduction", C.c_int), ("precision", C.c_int)]


PPV_MODEL_RESNET_SE = 2
PPV_MODEL_ERES2NET = 3


class ERes2NetCfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("num_blocks", C.c_int * 4), ("m_channels", C.c_int),
                ("precision", C.c_int), ("version", C.c_int), ("base_width", C.c_int)]


PPV_MODEL_CAMPPLUS = 4
PPV_MODEL_RES2NET = 5


class Res2NetCfg(C.Structure):
    _fields_ = [("input_size", C.c_int), ("embd_dim", C.c_int), ("layers", C.c_int * 4), ("m_channels", C.c_int), ("base_width", C.c_int),
                ("scale", C.c_int), ("attention_channels", C.c_int), ("precision", C.c_int)]


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


class VadCfg(C.Structure):
    _fields_ = [("window", C.c_int), ("shift", C.c_int), ("energy_threshold", C.c_float), ("energy_mean_scale", C.c_float),
                ("frames_context", C.c_int), ("proportion_threshold", C.c_float)]


TAPS_MAX_INPUTS, TAPS_MAX_SOURCES = 4, 16


class GemmTapsCase(C.Structure):
    """ppv_gemm_taps_case: one time-axis gather-GEMM case of ppv_gemm_test_taps"""
    _fields_ = [("x", C.c_void_p * TAPS_MAX_INPUTS), ("rows", C.c_int64 * TAPS_MAX_INPUTS), ("ld", C.c_int * TAPS_MAX_INPUTS),
                ("ninputs", C.c_int), ("nsrc", C.c_int),
                ("src_input", C.c_int * TAPS_MAX_SOURCES), ("src_col0", C.c_int * TAPS_MAX_SOURCES),
                ("src_ncols", C.c_int * TAPS_MAX_SOURCES), ("src_row_off", C.c_int * TAPS_MAX_SOURCES),
                ("W", C.c_void_p), ("bias", C.c_void_p), ("bn_scale", C.c_void_p), ("bn_shift", C.c_void_p), ("seg_scale", C.c_void_p),
                ("M", C.c_int), ("N", C.c_int), ("relu", C.c_int), ("seg_len", C.c_int), ("nseg", C.c_int), ("Tp", C.c_int), ("P", C.c_int),
                ("T", C.c_int), ("halo", C.c_int), ("zero_invalid", C.c_int), ("out_f32", C.c_int), ("out", C.c_void_p),
                ("out_rows", C.c_int64), ("out_ld", C.c_int), ("out_col0", C.c_int), ("block_n", C.c_int), ("block_k", C.c_int),
                ("precision", C.c_int)]


_P = C.c_void_p
# name ->(restype, argtypes); this table is also what tests/test_abi.py checks against include/ppv_b200.h
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
    "ppv_spectral_forward_ragged_samples": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ppv_spec_augment": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "ppv_ecapa_default_cfg": (None, [C.POINTER(EcapaCfg)]),
    "ppv_resnetse_default_cfg": (None, [C.POINTER(ResNetSECfg)]),
    "ppv_eres2net_default_cfg": (None, [C.POINTER(ERes2NetCfg)]),
    "ppv_campplus_default_cfg": (None, [C.POINTER(CamPPlusCfg)]),
    "ppv_res2net_default_cfg": (None, [C.POINTER(Res2NetCfg)]),
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
    "ppv_trainer_create_classifier": (C.c_int, [C.POINTER(EcapaCfg), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
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
    "ppv_optimizer_state_count": (C.c_int, [C.c_int, C.c_int]),
    "ppv_optimizer_step": (C.c_int, [C.c_int, _P, _P, _P, _P, _P, C.c_int64, C.POINTER(OptimArgs), C.c_int64, C.c_float, _P]),
    "ppv_cosine_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_cosine_matrix": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_cosine_pairlist": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, _P, _P]),
    "ppv_fbank_forward_ragged": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ppv_fbank_forward_ragged_samples": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ppv_audio_prep_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "ppv_audio_prep": (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_audio_prep_reverb_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_audio_prep_reverb": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_int64, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                        _P, _P, C.c_size_t, _P]),
    "ppv_eer_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "ppv_eer_mindcf": (C.c_int, [_P, _P, C.c_int64, C.c_double, C.c_double, C.c_double, _P, _P, C.c_size_t, _P]),
    "ppv_eer_mindcf_matrix": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, _P, _P, C.c_size_t, _P]),
    "ppv_row_argmax": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P]),
    "ppv_speaker_index_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "ppv_speaker_index_build": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_speaker_index_search_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "ppv_speaker_index_search": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_size_t, C.c_int, C.c_int, _P, _P, _P, C.c_size_t, _P]),
    "ppv_topn_row_stats": (C.c_int, [_P, C.c_int, C.c_int, C.c_int64, C.c_int, _P, _P, _P]),
    "ppv_as_norm_apply": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "ppv_vad_default_cfg": (None, [C.POINTER(VadCfg), C.c_int]),
    "ppv_vad_num_frames": (C.c_int64, [C.POINTER(VadCfg), C.c_int64]),
    "ppv_vad_workspace_bytes": (C.c_size_t, [C.POINTER(VadCfg), C.c_int, C.c_int64]),
    "ppv_vad_energy": (C.c_int, [C.POINTER(VadCfg), _P, C.POINTER(C.c_int64), C.c_int, _P, _P, _P, C.c_int64, _P, _P, C.c_size_t, _P]),
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
    "ppv_linear_head_forward": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float,
                                          _P, _P, _P, C.c_size_t, _P]),
    "ppv_linear_head_backward": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float,
                                           _P, _P, _P, _P, C.c_size_t, _P]),
    "ppv_gemm_test_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ppv_gemm_bench": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_size_t,
                                 C.POINTER(C.c_float), _P]),
    "ppv_gemm_test": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P,
                                C.c_size_t, _P]),
    "ppv_gemm_test_planes": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_conv2d_test_workspace_bytes": (C.c_size_t, [C.c_int] * 7),
    "ppv_conv2d_test": (C.c_int, [_P, _P, _P] + [C.c_int] * 13 + [_P, _P, C.c_size_t, _P]),
    "ppv_conv2d_test_clipped": (C.c_int, [_P, _P, _P, C.c_float] + [C.c_int] * 12 + [_P, _P, C.c_size_t, _P]),
    "ppv_stem_conv_test": (C.c_int, [_P, _P, _P] + [C.c_int] * 4 + [_P, _P]),
    "ppv_scale_res_test_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "ppv_scale_res_test": (C.c_int, [_P, _P, _P] + [C.c_int] * 6 + [C.c_float, _P, C.c_int, C.c_int, _P, C.c_size_t, _P]),
    "ppv_aff_combine_test_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "ppv_aff_combine_test": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_size_t, _P]),
    "ppv_res2net_stem_test": (C.c_int, [_P, _P, _P] + [C.c_int] * 3 + [_P, _P]),
    "ppv_res2net_avgpool_test_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "ppv_res2net_avgpool_test": (C.c_int, [_P] + [C.c_int] * 7 + [_P, _P, C.c_size_t, _P]),
    "ppv_asp_fused_test_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "ppv_asp_fused_test": (C.c_int, [_P] * 6 + [C.c_int] * 8 + [_P, _P, _P, C.c_size_t, _P]),
    "ppv_colstats_test_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "ppv_colstats_test": (C.c_int, [_P] + [C.c_int] * 8 + [C.c_float, C.c_float] + [_P, _P, _P, _P, C.c_size_t, _P]),
    "ppv_pool_stats_bwd_test_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "ppv_pool_stats_bwd_test": (C.c_int, [_P] * 3 + [C.c_int] * 6 + [_P, _P, C.c_size_t, _P]),
    "ppv_campplus_context_test_workspace_bytes": (C.c_size_t, [C.c_int] * 2),
    "ppv_campplus_context_test": (C.c_int, [_P] + [C.c_int] * 4 + [_P] * 6 + [C.c_size_t, _P]),
    "ppv_gemm_test_taps_workspace_bytes": (C.c_size_t, [C.POINTER(GemmTapsCase)]),
    "ppv_gemm_test_taps": (C.c_int, [C.POINTER(GemmTapsCase), _P, C.c_size_t, _P]),
    "ppv_res2net_test_workspace_bytes": (C.c_size_t, [C.c_int] * 5),
    "ppv_res2net_test": (C.c_int, [_P, C.c_int] + [_P] * 4 + [C.c_int] * 7 + [_P, C.c_int, _P, C.c_size_t, _P]),
    "ppv_skinny_linear_test_workspace_bytes": (C.c_size_t, [C.c_int] * 5),
    "ppv_skinny_linear_test": (C.c_int, [_P] + [C.c_int] * 3 + [_P] + [C.c_int] * 2 + [_P] + [C.c_int] * 2 + [_P] + [C.c_int] * 2
                               + [_P, C.c_size_t, _P]),
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
