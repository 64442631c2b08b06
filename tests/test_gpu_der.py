"""GPU: diarization results scored as RTTM.  infer_speaker_diarization.py --rttm_path writes what the predictor finds, and the three
tools of tools/eval_speaker_diarization (create_test_rttm.py -> infer_data.py -> compute_metrics.py) run end to end on a seeded
two-session corpus; their printed numbers are ppvector.metric.der's on the same files.  The tools run in this process (their main()
on their own option parsing), so the test opens no second CUDA context on the device."""
import importlib.util
import os
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, 'tools', 'eval_speaker_diarization')
CONFIG = os.path.join(ROOT, 'configs', 'ecapa_tdnn.yml')
SR = 16000


def save_weights(path):
    from oracle import ecapa as oe
    np.savez(path, **{k: v.float().numpy() for k, v in oe.make_ecapa_weights(seed=1000, dtype=torch.float64).items()})
    return str(path)


def tones(seed, freqs, seconds):
    """Consecutive noisy tones, one per turn (the recording of test_gpu_diarization.py for seed 7, (180, 420, 180), 4 s)."""
    rng = np.random.default_rng(seed)
    t = np.arange(int(SR * seconds)) / SR
    return np.concatenate([0.3 * np.sin(2 * np.pi * f * t) * (1 + 0.1 * rng.normal(size=t.size)) for f in freqs]).astype(np.float32)


def run_tool(name, args, capsys):
    """The tool's main() on `args`, from the current directory -> what it printed."""
    import cli_common
    spec = importlib.util.spec_from_file_location(name[:-3], os.path.join(TOOLS, name))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    capsys.readouterr()
    tool.main(cli_common.parse_options(tool.__doc__, tool.OPTIONS, args))
    return capsys.readouterr().out


def test_cli_rttm_path_writes_the_predictor_result(cuda, tmp_path):
    import cli_common
    import infer_speaker_diarization as cli
    from ppvector.data_utils.audio import AudioSegment
    from ppvector.metric.der import DiarizationErrorRate, load_rttm
    from ppvector.predict import PPVectorPredictor
    model = save_weights(tmp_path / 'model.npz')
    wav_path = str(tmp_path / 'meeting.take1.wav')
    AudioSegment(tones(7, (180, 420, 180), 4), SR).to_wav_file(wav_path)
    rttm = str(tmp_path / 'out.rttm')
    opt = cli_common.parse_options(cli.__doc__, cli.OPTIONS + cli.EXTENSION_OPTIONS,
                                   ['--configs', CONFIG, '--model_path', model, '--audio_path', wav_path, '--audio_db_path', 'None',
                                    '--search_audio_db', 'false', '--show_plot', 'false', '--rttm_path', rttm])
    np.random.seed(3)
    cli.main(opt)
    np.random.seed(3)
    out = PPVectorPredictor(CONFIG, model_path=model).speaker_diarization(wav_path)
    back = load_rttm(rttm)
    assert list(back) == ['meeting.take1']
    want = sorted(((o['start'], o['end'], str(o['speaker'])) for o in out), key=lambda s: (s[0], s[1]))
    got = back['meeting.take1']
    assert len(out) >= 1 and len(got) == len(want)
    assert [s[2] for s in got] == [s[2] for s in want]
    assert np.abs(np.array([s[:2] for s in got]) - np.array([s[:2] for s in want])).max() <= 1e-3 + 1e-9
    d = DiarizationErrorRate()(got, got, detailed=True)
    assert d['diarization error rate'] == 0.0 and d['total'] > 0


def test_eval_tools_end_to_end(cuda, tmp_path, monkeypatch, capsys):
    from ppvector.data_utils.audio import AudioSegment
    from ppvector.metric.der import DiarizationErrorRate, load_rttm, write_rttm
    model = save_weights(tmp_path / 'model.npz')
    wav_dir, ann_dir = tmp_path / 'dataset' / 'test' / 'wav', tmp_path / 'dataset' / 'test' / 'TextGrid'
    os.makedirs(wav_dir)
    os.makedirs(ann_dir)
    sessions = {'S01': (11, (180, 420, 180), ('spk_a', 'spk_b', 'spk_a'), 4.0),
                'S02': (12, (300, 650, 300, 650), ('p1', 'p2', 'p1', 'p2'), 3.5)}
    for name, (seed, freqs, labels, turn) in sessions.items():
        AudioSegment(tones(seed, freqs, turn), SR).to_wav_file(str(wav_dir / f'{name}.wav'))
        with open(ann_dir / f'{name}.rttm', 'w') as f:
            write_rttm(f, name, [(i * turn, (i + 1) * turn, lab) for i, lab in enumerate(labels)] + [(0.0, 0.2, labels[0])])

    monkeypatch.chdir(tmp_path)  # the tools' default paths are relative to where they run
    run_tool('create_test_rttm.py', [], capsys)
    refs = load_rttm(tmp_path / 'dataset' / 'references.rttm')
    assert sorted(refs) == ['S01', 'S02'] and len(refs['S01']) == 4 and len(refs['S02']) == 5
    with open(tmp_path / 'dataset' / 'data_list.txt') as f:
        assert [line.rstrip('\n').split('\t')[1] for line in f] == ['S01', 'S02']
    db = tmp_path / 'dataset' / 'audio_db'
    for name, (_, _, labels, turn) in sessions.items():
        assert sorted(os.listdir(db / name)) == sorted(set(labels))
        n_files = sum(len(os.listdir(db / name / lab)) for lab in set(labels))
        assert n_files == len(labels)  # the 0.2 s turn is too short to enrol
        x = AudioSegment.from_file(str(wav_dir / f'{name}.wav')).samples
        track = next(i for i, s in enumerate(refs[name]) if s[0] == turn)
        cut = AudioSegment.from_file(str(db / name / labels[1] / f'{track}.wav')).samples
        assert np.array_equal(cut, x[int(turn * SR):int(2 * turn * SR)])

    run_tool('infer_data.py', ['--configs', CONFIG, '--model_path', model, '--threshold', '0.5'], capsys)
    hyps = load_rttm(tmp_path / 'dataset' / 'hypotheses.rttm')
    assert sorted(hyps) == ['S01', 'S02'] and all(len(h) >= 1 for h in hyps.values())
    assert not any(os.path.exists(db / name / 'audio_indexes.bin') for name in sessions)

    text = run_tool('compute_metrics.py', [], capsys)
    printed = dict(re.findall(r'^([A-Za-z ]+): (\S+)$', text, flags=re.M))
    metric = DiarizationErrorRate()
    per_file = [metric(refs[u], hyps[u], detailed=True) for u in refs]
    for label, key in (('False alarm', 'false alarm'), ('Confusion', 'confusion'), ('Missed detection', 'missed detection'),
                       ('Diarization error rate', 'diarization error rate')):
        assert float(printed[label]) == round(sum(d[key] for d in per_file) / len(per_file), 5), label
    assert float(printed['Corpus diarization error rate']) == round(abs(metric), 5)
    assert all(re.search(rf'^{u} : \{{', text, flags=re.M) for u in refs)
