"""Minimal audio preparation in front of the hot path (the reference delegates this to the un-vendored
``yeaudio.audio.AudioSegment``: ppvector/predict.py:189-216, ppvector/data_utils/reader.py:85-104).

Only what the drop-in entry points need: WAV decode (PCM 8/16/24/32-bit, IEEE float; `soundfile` for flac / mp3 when installed), float32 samples in
[-1,1), dB normalisation to ``target_db`` (gain = target - 10 log10(mean(x^2)); x *= 10^(gain/20)), resampling
by polyphase filtering.  GPU-side audio prep is SURVEY.md §8(f) rank 2 ("next")."""
import io
import struct

import numpy as np

_MAGIC = {b'fLaC': 'FLAC', b'OggS': 'Ogg', b'ID3': 'MP3', b'\xff\xfb': 'MP3', b'\xff\xf3': 'MP3', b'\xff\xf2': 'MP3'}


def _parse_riff_wave(buf):
    """RIFF/WAVE container -> (float32 [n, channels], sample_rate).  PCM 8 / 16 / 24 / 32 bit, IEEE float 32 / 64 bit, and
    WAVE_FORMAT_EXTENSIBLE wrappers of those (the stdlib `wave` module reads integer PCM only and rejects 24-bit packed / float)."""
    if len(buf) < 12 or buf[:4] not in (b'RIFF', b'RF64') or buf[8:12] != b'WAVE':
        kind = next((v for k, v in _MAGIC.items() if buf[:len(k)] == k), None)
        raise ValueError(f'unsupported audio container ({kind or "unknown"}): this build decodes WAV itself and everything else through '
                         f'`soundfile`, which is not installed')
    pos, fmt, data = 12, None, None
    while pos + 8 <= len(buf):
        cid, size = buf[pos:pos + 4], struct.unpack('<I', buf[pos + 4:pos + 8])[0]
        body = buf[pos + 8:pos + 8 + size]
        if cid == b'fmt ':
            fmt = body
        elif cid == b'data':
            data = body if size != 0xFFFFFFFF else buf[pos + 8:]
            if fmt is not None:
                break
        pos += 8 + size + (size & 1)
    if fmt is None or data is None or len(fmt) < 16:
        raise ValueError('malformed WAV file: missing fmt or data chunk')
    tag, ch, sr, _byte_rate, block, bits = struct.unpack('<HHIIHH', fmt[:16])
    if tag == 0xFFFE and len(fmt) >= 26:  # WAVE_FORMAT_EXTENSIBLE: the real format is the first two bytes of the sub-format GUID
        tag = struct.unpack('<H', fmt[24:26])[0]
    if tag not in (1, 3):
        raise ValueError(f'unsupported WAV encoding (format tag 0x{tag:04x}): PCM and IEEE float are implemented')
    if bits % 8 or bits == 0 or ch == 0:
        raise ValueError(f'unsupported WAV layout: {bits} bits x {ch} channels')
    nbytes = bits // 8
    n = (len(data) // (nbytes * ch)) * ch
    raw = data[:n * nbytes]
    if tag == 1:  # integer PCM
        if bits == 8:
            x = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
        elif bits == 16:
            x = np.frombuffer(raw, dtype='<i2').astype(np.float32) / 32768.0
        elif bits == 24:
            b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
            v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
            v = np.where(v >= 1 << 23, v - (1 << 24), v)
            x = v.astype(np.float32) / 8388608.0
        elif bits == 32:
            x = (np.frombuffer(raw, dtype='<i4').astype(np.float64) / 2147483648.0).astype(np.float32)
        else:
            raise ValueError(f'unsupported PCM sample width: {bits} bits')
    else:  # tag 3: IEEE float
        if bits not in (32, 64):
            raise ValueError(f'unsupported IEEE-float sample width: {bits} bits')
        x = np.frombuffer(raw, dtype='<f4' if bits == 32 else '<f8').astype(np.float32)
    return x.reshape(-1, ch), sr


def read_wav(source):
    """path | bytes | file object -> (float32 mono samples in [-1,1), sample_rate).  `soundfile` decodes when it is installed (the
    reference's yeaudio reads flac / mp3 / ogg through it: create_data.py lists CN-Celeb_flac); otherwise WAV is parsed here and any
    other container raises with the format named."""
    try:
        import soundfile
    except ImportError:
        soundfile = None
    if soundfile is not None:
        src = io.BytesIO(source) if isinstance(source, (bytes, bytearray)) else source
        x, sr = soundfile.read(src, dtype='float32', always_2d=True)
    else:
        if isinstance(source, (bytes, bytearray)):
            buf = bytes(source)
        elif hasattr(source, 'read'):
            buf = source.read()
        else:
            with open(source, 'rb') as f:
                buf = f.read()
        x, sr = _parse_riff_wave(buf)
    if x.shape[1] > 1:
        x = x.mean(axis=1)
    return np.ascontiguousarray(x.reshape(-1), dtype=np.float32), int(sr)


def resample(x, sr_from, sr_to):
    if sr_from == sr_to:
        return x
    from math import gcd
    from scipy.signal import resample_poly
    g = gcd(int(sr_from), int(sr_to))
    return resample_poly(x, int(sr_to) // g, int(sr_from) // g).astype(np.float32)


def normalize_db(x, target_db=-20.0, max_gain_db=300.0):
    mean_square = float(np.mean(x.astype(np.float64) ** 2))
    rms_db = 10.0 * np.log10(mean_square) if mean_square > 0.0 else -np.inf  # digital silence cannot be normalised (gain = +inf)
    gain = target_db - rms_db
    if gain > max_gain_db:
        raise ValueError(f'无法将音频归一化到 {target_db} dB: 增益 {gain} dB 超过 max_gain_db')
    return (x * np.float32(10.0 ** (gain / 20.0))).astype(np.float32)


class AudioSegment:
    """The slice of yeaudio.audio.AudioSegment the predictor uses: samples / sample_rate / duration /
    resample / normalize / vad / from_file / from_ndarray / from_bytes."""

    def __init__(self, samples, sample_rate):
        self.samples = np.ascontiguousarray(samples, dtype=np.float32)
        self.sample_rate = int(sample_rate)

    @classmethod
    def from_file(cls, f):
        return cls(*read_wav(f))

    @classmethod
    def from_bytes(cls, b):
        return cls(*read_wav(b))

    @classmethod
    def from_ndarray(cls, data, sample_rate=16000):
        data = np.asarray(data)
        if data.dtype == np.int16:
            data = data.astype(np.float32) / 32768.0
        return cls(data.astype(np.float32), sample_rate)

    @property
    def duration(self):
        return self.samples.shape[0] / float(self.sample_rate)

    def resample(self, target_sample_rate):
        self.samples = resample(self.samples, self.sample_rate, target_sample_rate)
        self.sample_rate = int(target_sample_rate)

    def normalize(self, target_db=-20.0, max_gain_db=300.0):
        self.samples = normalize_db(self.samples, target_db, max_gain_db)

    def vad(self, return_seconds=False, **opts):
        """The speech in the recording: [{'start', 'end'}, ...] in samples, or in seconds with return_seconds=True.  yeaudio runs silero-vad
        here; this build runs Kaldi's energy VAD on the GPU (infer_utils/vad.py, options as vad_options there)."""
        from ppvector.infer_utils import vad
        return vad.energy_vad([self.samples], self.sample_rate, return_seconds=return_seconds, **opts)[0]

    def to_wav_file(self, filepath):
        """Mono 32-bit IEEE-float WAV (format tag 3, yeaudio's default): read back by read_wav bit for bit."""
        data = np.ascontiguousarray(self.samples, dtype='<f4').tobytes()
        fmt = struct.pack('<HHIIHH', 3, 1, self.sample_rate, self.sample_rate * 4, 4, 32)
        with open(filepath, 'wb') as f:
            f.write(b'RIFF' + struct.pack('<I', 4 + 8 + len(fmt) + 8 + len(data)) + b'WAVE')
            f.write(b'fmt ' + struct.pack('<I', len(fmt)) + fmt)
            f.write(b'data' + struct.pack('<I', len(data)) + data)
