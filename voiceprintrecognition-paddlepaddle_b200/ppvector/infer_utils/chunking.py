"""Fixed-length chunk fan-out in front of the embedding path -- the part of the reference's speaker-diarization flow that feeds the hot path
(ppvector/predict.py:378-381: ``segments_audio`` -> ``predict_batch``; windowing rule ppvector/infer_utils/speaker_diarization.py:60-87,
defaults seg_duration 1.5 s, seg_shift 0.75 s).  SURVEY.md §8(f) rank 4.

Every voiced segment [start s, end s, samples] is covered by windows of ``seg_duration`` whose starts advance by ``seg_shift``; a window that
would run past the segment end is moved back so that it ends at the segment end (the last two windows overlap more); a segment shorter than one
window gives one zero-padded window.  All windows have the same length, so the whole recording becomes ONE [n_chunks, chunk_len] batch for the
embedding path -- no per-chunk padding ratios, no ragged batch.

Voice-activity detection (yeaudio's silero VAD) is not part of this package: callers pass the VAD segments (or none: the whole recording is
one segment).  The clustering and post-processing after the embeddings are infer_utils/speaker_diarization.py.
"""
import numpy as np

__all__ = ['chunk_windows', 'chunk_segments', 'fan_out_embeddings']


def chunk_windows(n_samples: int, chunk_len: int, chunk_shift: int) -> np.ndarray:
    """[n, 2] int64 (start, end) sample windows covering ``n_samples`` (end - start == chunk_len except for a segment shorter than a window)."""
    assert chunk_len > 0 and chunk_shift > 0
    if n_samples <= 0:
        return np.zeros((0, 2), dtype=np.int64)
    starts = np.arange(0, n_samples, chunk_shift, dtype=np.int64)
    ends = np.minimum(starts + chunk_len, n_samples)
    # windows are kept while their end still advances: the first window that reaches the segment end is the last one
    keep = np.ones(len(ends), dtype=bool)
    keep[1:] = ends[1:] > ends[:-1]
    ends = ends[keep]
    starts = np.maximum(ends - chunk_len, 0)  # a clipped window is moved back to end at the segment end
    return np.stack([starts, ends], axis=1)


def chunk_segments(vad_segments, seg_duration=1.5, seg_shift=0.75, sample_rate=16000):
    """vad_segments: iterable of (start_s, end_s, samples) -> (times [n, 2] float64 seconds, chunks [n, chunk_len] float32)."""
    chunk_len, chunk_shift = int(seg_duration * sample_rate), int(seg_shift * sample_rate)
    times, rows = [], []
    for seg_st, _seg_ed, data in vad_segments:
        data = np.asarray(data, dtype=np.float32)
        for st, ed in chunk_windows(data.shape[0], chunk_len, chunk_shift):
            row = np.zeros(chunk_len, dtype=np.float32)
            row[:ed - st] = data[st:ed]
            rows.append(row)
            times.append((st / sample_rate + seg_st, ed / sample_rate + seg_st))
    if not rows:
        return np.zeros((0, 2), dtype=np.float64), np.zeros((0, chunk_len), dtype=np.float32)
    return np.asarray(times, dtype=np.float64), np.stack(rows)


def fan_out_embeddings(vad_segments, embed_fn, seg_duration=1.5, seg_shift=0.75, sample_rate=16000, batch_size=256):
    """Chunk the segments and run ``embed_fn`` ([b, chunk_len] float32 -> [b, D]) over them ``batch_size`` rows at a time.
    Returns (times [n, 2] seconds, embeddings [n, D])."""
    times, chunks = chunk_segments(vad_segments, seg_duration, seg_shift, sample_rate)
    if len(chunks) == 0:
        return times, np.zeros((0, 0), dtype=np.float32)
    batch_size = max(1, int(batch_size))
    embs = [np.asarray(embed_fn(chunks[i:i + batch_size])) for i in range(0, len(chunks), batch_size)]
    return times, np.concatenate(embs, axis=0)
