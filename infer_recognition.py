"""Speaker enrolment and identification against an enrolment database (counterpart of the reference's infer_recognition.py).

One action per call, on a recording given as a file (this build has no microphone capture, so the reference's record_seconds is
replaced by audio_path):
  --action register  --user_name NAME --audio_path x.wav   enrol the recording as NAME (stored under <audio_db_path>/NAME/)
  --action recognize --audio_path x.wav [--top_k K]        print the K best enrolled users at or above the threshold
  --action remove    --user_name NAME                      delete NAME and its recordings from the database"""
from cli_common import parse_options

OPTIONS = [
    ('configs', str, 'configs/cam++.yml', 'model / data configuration (YAML)'),
    ('use_gpu', bool, True, 'must stay True: this build has no CPU path'),
    ('audio_db_path', str, 'audio_db/', 'enrolment database: <db>/<user>/*.wav'),
    ('threshold', float, 0.6, 'similarity at or above which a speaker is taken to be an enrolled user'),
    ('model_path', str, 'models/CAMPPlus_Fbank/best_model/', 'directory or file holding the weights'),
    ('action', str, 'recognize', 'register | recognize | remove'),
    ('audio_path', str, None, 'recording to register or recognize'),
    ('user_name', str, None, 'user to register or remove'),
    ('top_k', int, 1, 'recognize: number of best users reported (1 to 8)'),
]
ACTIONS = ('register', 'recognize', 'remove')


def check_options(opt):
    if opt.action not in ACTIONS:
        raise SystemExit(f'--action must be one of {", ".join(ACTIONS)} (got {opt.action!r})')
    if opt.action in ('register', 'recognize') and not opt.audio_path:
        raise SystemExit(f'--action {opt.action} needs --audio_path')
    if opt.action in ('register', 'remove') and not opt.user_name:
        raise SystemExit(f'--action {opt.action} needs --user_name')
    if opt.audio_db_path is None:
        raise SystemExit('--audio_db_path is required')


def main(opt):
    check_options(opt)
    from ppvector.predict import PPVectorPredictor
    predictor = PPVectorPredictor(configs=opt.configs, threshold=opt.threshold, audio_db_path=opt.audio_db_path, model_path=opt.model_path,
                                  use_gpu=opt.use_gpu)
    if opt.action == 'register':
        predictor.register(user_name=opt.user_name, audio_data=opt.audio_path)
        print(f'已注册：{opt.user_name}')
    elif opt.action == 'remove':
        print(f'已删除：{opt.user_name}' if predictor.remove_user(user_name=opt.user_name) else f'没有该用户：{opt.user_name}')
    else:
        results = predictor.recognition_batch([opt.audio_path], top_k=opt.top_k)[0]
        if results:
            for name, score in results:
                print(f"识别说话的为：{name}，得分：{score}")
        else:
            print("没有识别到说话人，可能是没注册。")


if __name__ == '__main__':
    main(parse_options(__doc__, OPTIONS))
