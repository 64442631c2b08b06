"""Step 1 of the diarization evaluation: prepare a test corpus (for instance AIShell-4's test set) for infer_data.py and
compute_metrics.py.  Run from this directory; the default paths are the reference's.

  * concatenates the annotation directory's *.rttm files into the reference RTTM;
  * writes the data list, one `path<TAB>session` line per .wav / .flac recording (FLAC is decoded by `soundfile`, when installed);
  * cuts every reference turn of at least 0.3 s into <audio_db>/<session>/<label>/<turn>.wav, the per-session enrolment database
    that infer_data.py names the speakers from (samples [int(start * sr), int(end * sr)), as the reference cuts them).

    python create_test_rttm.py [--annotation_dir dataset/test/TextGrid] [--audio_dir dataset/test/wav] [--rttm_path dataset/references.rttm]
                               [--data_list_path dataset/data_list.txt] [--audio_db_path dataset/audio_db/]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'voiceprintrecognition-paddlepaddle_b200')]

from cli_common import parse_options  # noqa: E402

OPTIONS = [
    ('annotation_dir', str, 'dataset/test/TextGrid', 'directory of the per-session reference *.rttm files'),
    ('audio_dir', str, 'dataset/test/wav', 'directory of the recordings (.wav, .flac); the session is the file name up to its first dot'),
    ('rttm_path', str, 'dataset/references.rttm', 'reference RTTM written here'),
    ('data_list_path', str, 'dataset/data_list.txt', 'data list written here'),
    ('audio_db_path', str, 'dataset/audio_db/', 'per-session enrolment databases written here'),
]
MIN_TURN_S = 0.3


def create_rttm(annotation_dir, output_path):
    with open(output_path, 'w', encoding='utf-8') as f_w:
        for file in sorted(os.listdir(annotation_dir)):
            if not file.endswith('.rttm'):
                continue
            with open(os.path.join(annotation_dir, file), 'r', encoding='utf-8') as f_r:
                text = f_r.read()
            f_w.write(text if not text or text.endswith('\n') else text + '\n')


def create_audio_path_list(audio_dir, list_path):
    with open(list_path, 'w', encoding='utf-8') as f_w:
        for file in sorted(os.listdir(audio_dir)):
            if not file.endswith(('.wav', '.flac')):
                continue
            file_path = os.path.join(audio_dir, file).replace('\\', '/')
            f_w.write(f'{file_path}\t{file.split(".")[0]}\n')


def create_audio_db(data_list_path, rttm_path, output_dir):
    from ppvector.data_utils.audio import AudioSegment
    from ppvector.metric.der import load_rttm
    annotations = load_rttm(rttm_path)
    with open(data_list_path, 'r', encoding='utf-8') as f_r:
        lines = [line.strip() for line in f_r if line.strip()]
    for line in lines:
        audio_path, name = line.split('\t')
        if name not in annotations:
            raise KeyError(f'{rttm_path} has no SPEAKER turns for session {name!r} ({audio_path})')
        audio = AudioSegment.from_file(audio_path)
        sr, samples = audio.sample_rate, audio.samples
        for track, (start, end, label) in enumerate(annotations[name]):
            if end - start < MIN_TURN_S:
                continue
            save_path = os.path.join(output_dir, name, label, f'{track}.wav')
            os.makedirs(os.path.dirname(save_path), exist_ok=True)
            AudioSegment(samples[int(start * sr):int(end * sr)], sr).to_wav_file(save_path)
        print(f'{name}: enrolment turns written under {os.path.join(output_dir, name)}')


def main(opt):
    for path in (opt.rttm_path, opt.data_list_path):
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    create_rttm(opt.annotation_dir, opt.rttm_path)
    create_audio_path_list(opt.audio_dir, opt.data_list_path)
    create_audio_db(opt.data_list_path, opt.rttm_path, opt.audio_db_path)


if __name__ == '__main__':
    main(parse_options(__doc__, OPTIONS))
