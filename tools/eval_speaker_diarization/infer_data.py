"""Step 2 of the diarization evaluation: diarize every session of the data list (create_test_rttm.py) on the GPU and write the
hypothesis RTTM.  Each session gets its own predictor on its own enrolment database (<audio_db>/<session>/), so the speakers are
named from it (speaker_diarization(search_audio_db=True)); the session's audio_indexes.bin is deleted afterwards, as the reference
does.  Run from this directory; the default paths are the reference's.

    python infer_data.py [--configs ../../configs/cam++.yml] [--model_path ../../models/CAMPPlus_Fbank/best_model/]
                         [--data_list_path dataset/data_list.txt] [--result_path dataset/hypotheses.rttm] [--audio_db_path dataset/audio_db/]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'voiceprintrecognition-paddlepaddle_b200')]

from cli_common import parse_options  # noqa: E402

OPTIONS = [
    ('configs', str, '../../configs/cam++.yml', 'model / data configuration (YAML)'),
    ('use_gpu', bool, True, 'must stay True: this build has no CPU path'),
    ('data_list_path', str, 'dataset/data_list.txt', 'recordings to diarize: `path<TAB>session` lines'),
    ('result_path', str, 'dataset/hypotheses.rttm', 'hypothesis RTTM written here'),
    ('audio_db_path', str, 'dataset/audio_db/', 'per-session enrolment databases: <db>/<session>/<speaker>/*.wav'),
    ('threshold', float, 0.6, 'similarity at or above which a speaker is taken to be an enrolled one'),
    ('model_path', str, '../../models/CAMPPlus_Fbank/best_model/', 'directory or file holding the weights'),
]


def main(opt):
    from ppvector.metric.der import write_rttm
    from ppvector.predict import PPVectorPredictor
    with open(opt.data_list_path, 'r', encoding='utf-8') as f_r:
        lines = [line.strip() for line in f_r if line.strip()]
    with open(opt.result_path, 'w', encoding='utf-8') as f_w:
        for i, line in enumerate(lines):
            audio_path, name = line.split('\t')
            audio_db_path = os.path.join(opt.audio_db_path, name)
            predictor = PPVectorPredictor(configs=opt.configs, model_path=opt.model_path, threshold=opt.threshold,
                                          audio_db_path=audio_db_path, use_gpu=opt.use_gpu)
            results = predictor.speaker_diarization(audio_path, search_audio_db=True)
            write_rttm(f_w, name, [(r['start'], r['end'], str(r['speaker'])) for r in results])
            f_w.flush()
            os.remove(os.path.join(audio_db_path, 'audio_indexes.bin'))
            print(f'[{i + 1}/{len(lines)}] {name}: {len(results)} segments')


if __name__ == '__main__':
    main(parse_options(__doc__, OPTIONS))
