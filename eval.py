"""Equal error rate, minDCF and the EER threshold of a checkpoint on the enrolment / trials lists named in the config
(counterpart of the reference's eval.py; same options).  When the config sets dataset_conf.eval_conf.score_norm
({cohort_list, top_n, cohort}), the scores are AS-normalised against that cohort list first and the threshold is in normalised units."""
import time

from cli_common import parse_options

OPTIONS = [
    ('configs', str, 'configs/ecapa_tdnn.yml', 'model / data configuration (YAML)'),
    ('use_gpu', bool, True, 'must stay True: this build has no CPU path'),
    ('save_image_path', str, 'output/images/', 'accepted for compatibility; plots are not produced'),
    ('resume_model', str, 'models/EcapaTdnn_Fbank/best_model/', 'directory or file holding the weights'),
]


def main(opt):
    from ppvector.trainer import PPVectorTrainer
    trainer = PPVectorTrainer(configs=opt.configs, use_gpu=opt.use_gpu)
    began = time.time()
    eer, min_dcf, threshold = trainer.evaluate(resume_model=opt.resume_model, save_image_path=opt.save_image_path)
    print(f'evaluation took {int(time.time() - began)} s: threshold {threshold:.2f}, EER {eer:.5f}, MinDCF {min_dcf:.5f}')


if __name__ == '__main__':
    main(parse_options(__doc__, OPTIONS))
