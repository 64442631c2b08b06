"""The Fbank option grid shared by tests/test_fbank_options_cpu.py (fp64 oracle against torchaudio) and
tests/test_gpu_fbank_options.py (both CUDA kernels against the oracle).  Each case is a ``preprocess_conf.method_args``
dict under paddleaudio's keyword names, which are torchaudio's except ``sr`` and ``n_mels``."""

# FFT size of each case in the comment: next_pow2(int(sr * frame_length / 1000))
CASES = {
    "sr8000": dict(sr=8000, n_mels=80),                                        # 256
    "sr11025": dict(sr=11025, n_mels=64),                                      # 512, window 275: the specialised kernel
    "sr22050": dict(sr=22050, n_mels=80),                                      # 1024
    "sr44100": dict(sr=44100, n_mels=80),                                      # 2048
    "sr48000": dict(sr=48000, n_mels=80),                                      # 2048
    "fft128": dict(sr=16000, n_mels=23, frame_length=6.0, frame_shift=3.0),    # 128
    "fft256": dict(sr=16000, n_mels=40, frame_length=12.0, frame_shift=5.0),   # 256
    "fft1024": dict(sr=16000, n_mels=80, frame_length=50.0),                   # 1024
    "fft2048": dict(sr=16000, n_mels=128, frame_length=100.0, frame_shift=20.0),  # 2048
    "fft4096": dict(sr=48000, n_mels=80, frame_length=50.0),                   # 4096
    "hanning": dict(sr=16000, n_mels=80, window_type="hanning"),
    "hamming": dict(sr=16000, n_mels=80, window_type="hamming"),
    "rectangular": dict(sr=8000, n_mels=40, window_type="rectangular"),
    "blackman": dict(sr=16000, n_mels=80, window_type="blackman", blackman_coeff=0.40),
    "no_snip": dict(sr=16000, n_mels=80, snip_edges=False),
    "no_snip_8k": dict(sr=8000, n_mels=80, snip_edges=False),
    "no_dc": dict(sr=16000, n_mels=80, remove_dc_offset=False),
    "magnitude": dict(sr=16000, n_mels=80, use_power=False),
    "linear": dict(sr=16000, n_mels=80, use_log_fbank=False),
    "vtln09": dict(sr=16000, n_mels=80, vtln_warp=0.9),
    "vtln11": dict(sr=8000, n_mels=40, vtln_warp=1.1, vtln_low=200.0, vtln_high=-300.0),
    "subtract_mean": dict(sr=16000, n_mels=80, subtract_mean=True, htk_compat=True, raw_energy=False, energy_floor=0.5),
    "preemph_low_high": dict(sr=22050, n_mels=60, preemphasis_coefficient=0.5, low_freq=100.0, high_freq=-1000.0),
}

_ORACLE = {"frame_length": "frame_length_ms", "frame_shift": "frame_shift_ms", "preemphasis_coefficient": "preemph"}
_TORCHAUDIO = {"sr": "sample_frequency", "n_mels": "num_mel_bins"}
_NO_EFFECT = ("htk_compat", "raw_energy", "energy_floor")  # they only touch the energy column, which use_energy=False drops


def oracle_kwargs(args):
    """method_args -> keyword arguments of oracle.fbank.kaldi_fbank"""
    return {_ORACLE.get(k, k): v for k, v in args.items() if k not in _NO_EFFECT}


def torchaudio_kwargs(args):
    """method_args -> keyword arguments of torchaudio.compliance.kaldi.fbank"""
    return {_TORCHAUDIO.get(k, k): v for k, v in args.items()}


def frame_geometry(args):
    """(window, shift, snip_edges) in samples"""
    sr = args.get("sr", 16000)
    return (int(sr * args.get("frame_length", 25.0) * 0.001), int(sr * args.get("frame_shift", 10.0) * 0.001),
            args.get("snip_edges", True))
