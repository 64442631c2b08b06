"""Speaker diarization of one recording: who speaks when, optionally named from an enrolment database
(counterpart of the reference's infer_speaker_diarization.py; same options).  Prints one {'speaker', 'start', 'end'} per segment and, with
--rttm_path, also writes them as RTTM (uri = the audio file's stem) for scoring by tools/eval_speaker_diarization/compute_metrics.py."""
import os

from cli_common import parse_options

OPTIONS = [
    ('configs', str, 'configs/cam++.yml', 'model / data configuration (YAML)'),
    ('audio_path', str, 'dataset/test_long.wav', 'recording to diarize (more than 5 s of speech)'),
    ('audio_db_path', str, 'audio_db/', 'enrolment database: <db>/<user>/*.wav'),
    ('speaker_num', int, None, 'number of speakers, if known (otherwise chosen by the eigengap)'),
    ('use_gpu', bool, True, 'must stay True: this build has no CPU path'),
    ('show_plot', bool, True, 'accepted for compatibility; the plot viewer is not part of this build'),
    ('search_audio_db', bool, True, 'name the speakers from the enrolment database'),
    ('threshold', float, 0.6, 'similarity at or above which a speaker is taken to be an enrolled user'),
    ('model_path', str, 'models/CAMPPlus_Fbank/best_model/', 'directory or file holding the weights'),
]
# options of this build beyond the reference's
EXTENSION_OPTIONS = [
    ('vad', bool, False, "find the speech first with Kaldi's energy VAD on the GPU (otherwise the whole recording is taken as speech)"),
    ('rttm_path', str, None, "also write the result to this RTTM file, uri = the audio file's stem"),
]


def main(opt):
    from loguru import logger

    from ppvector.metric.der import write_rttm
    from ppvector.predict import PPVectorPredictor
    if opt.search_audio_db:
        assert opt.audio_db_path is not None, '请指定音频库的路径'
    predictor = PPVectorPredictor(configs=opt.configs, model_path=opt.model_path, threshold=opt.threshold, audio_db_path=opt.audio_db_path,
                                  use_gpu=opt.use_gpu)
    results = predictor.speaker_diarization(opt.audio_path, speaker_num=opt.speaker_num, search_audio_db=opt.search_audio_db,
                                              vad=opt.vad)
    print('识别结果：')
    for result in results:
        print(result)
    if opt.rttm_path is not None:
        with open(opt.rttm_path, 'w', encoding='utf-8') as f:
            write_rttm(f, os.path.splitext(os.path.basename(opt.audio_path))[0], [(r['start'], r['end'], r['speaker']) for r in results])
    if opt.show_plot:
        logger.info('show_plot: the matplotlib viewer is not part of this build')


if __name__ == '__main__':
    main(parse_options(__doc__, OPTIONS + EXTENSION_OPTIONS))
