"""PPVectorTrainer -- drop-in for ppvector/trainer.py:33-474 (feature extraction, training, evaluation).

``extract_features`` (trainer.py:134-157) and ``evaluate`` (trainer.py:367-447) keep their signatures, list-file formats and
return values; featurisation, the backbone, the trial x enrol cosine matrix and EER / minDCF (radix sort + sweep) run on the GPU
through libppv_b200; with the optional ``dataset_conf.eval_conf.score_norm`` key the matrix is AS-normalised against a cohort list first
(ppvector/metric/score_norm.py).  ``train`` (trainer.py:281-365 with the step of :206-229) runs the CUDA training step of
``ppvector.train_engine.TrainEngine`` (train-mode forward, AAM loss, backward, one gradient all-reduce over NCCL, the optimizer step)
with the reference's schedules; it is implemented for EcapaTdnn with any pooling head (ASP with or without the global context, SAP, TAP,
TSP), either classifier (Cosine or Linear, with any number of DenseLayer blocks) + AAMLoss + Adam, AdamW, SGD, Momentum or RMSProp +
WarmupCosineSchedulerLR (configs/ecapa_tdnn.yml) and raises for other combinations.  Checkpoints follow the
reference's directory layout (``<model>_<feature>/{epoch_N,last_model,best_model}`` with best-EER tracking, optimizer state and ``model.state``) and ``resume_model`` / an existing ``last_model`` restore the weights, the optimizer's
state, the step counters of both schedules and the epoch.  VisualDL logging is out of scope."""
import os

import numpy as np
import torch
import yaml
from loguru import logger
from tqdm import tqdm

from ppvector import _lib
from ppvector.data_utils.collate_fn import collate_fn
from ppvector.data_utils.featurizer import AudioFeaturizer
from ppvector.data_utils.reader import PPVectorDataset
from ppvector.metric.cosine import cosine_matrix
from ppvector.metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr, eer_mindcf_from_matrix_gpu  # noqa: F401
from ppvector.metric.score_norm import as_norm, cohort_stats, score_norm_config, speaker_cohort
from ppvector.models import build_model
from ppvector.utils.checkpoint import check_optimizer_state, find_resume_dir, load_checkpoint_dir, load_state_dict_file, save_checkpoint
from ppvector.utils.utils import dict_to_object, print_arguments


def init_classifier(shapes):
    """SpeakerIdentification's initial tensors (fc.py:25-38) with Paddle's default initialisers, in state_dict order: a block's Conv1D
    weight Normal(0, sqrt(2 / fan_in)) and bias 0; its BatchNorm1D weight 1, bias 0, running mean 0, running variance 1; the output
    weight Xavier uniform, a Linear bias 0.  Draws from torch's global generator."""
    out = {}
    for name, shape in shapes.items():
        if name.endswith('linear.weight'):
            out[name] = torch.randn(shape) * (2.0 / (shape[1] * shape[2])) ** 0.5
        elif name in ('classifier.weight', 'classifier.output.weight'):
            out[name] = torch.nn.init.xavier_uniform_(torch.empty(shape))  # fc.py:34-36 / nn.Linear
        elif name.endswith(('batchnorm.weight', '_variance')):
            out[name] = torch.ones(shape)
        else:
            out[name] = torch.zeros(shape)
    return out


def check_classifier_keys(loaded, shapes, path):
    """Refuses a checkpoint whose classifier tensors (``classifier.<name>``) are not exactly the configured classifier's; one with no
    classifier tensor (a backbone alone) passes."""
    if not loaded:
        return
    missing = sorted(set(shapes) - set(loaded))
    unexpected = sorted(set(loaded) - set(shapes))
    wrong = sorted(k for k in set(loaded) & set(shapes) if tuple(np.shape(np.asarray(loaded[k]))) != tuple(shapes[k]))
    if missing or unexpected or wrong:
        fmt = lambda ks: [('1.' + k[len('classifier.'):]) for k in ks]  # noqa: E731
        raise ValueError(f'{path}: the checkpoint\'s classifier does not match model_conf.classifier; missing keys {fmt(missing)}, '
                         f'unexpected keys {fmt(unexpected)}, keys of another shape {fmt(wrong)}')


class PPVectorTrainer(object):
    def __init__(self, configs, use_gpu=True, data_augment_configs=None, state_dict=None):
        """reference: trainer.py:34-81.  ``state_dict`` (extension): backbone weights given in memory."""
        if not use_gpu:
            raise _lib.PPVError('use_gpu=False: this build of ppvector has no CPU path')
        assert torch.cuda.is_available(), 'GPU不可用'
        self.use_gpu = use_gpu
        self.device = torch.device('cuda', torch.cuda.current_device())
        if isinstance(configs, str):
            with open(configs, 'r', encoding='utf-8') as f:
                configs = yaml.load(f.read(), Loader=yaml.FullLoader)
            print_arguments(configs=configs)
        self.configs = dict_to_object(configs)
        if isinstance(data_augment_configs, str):
            with open(data_augment_configs, 'r', encoding='utf-8') as f:
                data_augment_configs = yaml.load(f.read(), Loader=yaml.FullLoader)
        self.data_augment_configs = dict_to_object(data_augment_configs) if data_augment_configs else None
        self.model = None
        self.audio_featurizer = None
        self.enroll_dataset = self.trials_dataset = None
        self._state_dict = state_dict
        self.stop_train, self.stop_eval = False, False

    def _featurizer(self):
        if self.audio_featurizer is None:
            self.audio_featurizer = AudioFeaturizer(feature_method=self.configs.preprocess_conf.feature_method,
                                                    method_args=self.configs.preprocess_conf.get('method_args', {}))
        return self.audio_featurizer

    # ---- trainer.py:134-157 ------------------------------------------------------------------------------------
    def extract_features(self, save_dir='dataset/features', max_duration=100):
        fz = self._featurizer()
        for list_idx, data_list in enumerate([self.configs.dataset_conf.train_list, self.configs.dataset_conf.enroll_list,
                                              self.configs.dataset_conf.trials_list]):
            if not os.path.exists(data_list):
                logger.warning(f'{data_list} 不存在，跳过')
                continue
            dataset_args = dict(self.configs.dataset_conf.get('dataset', {}))
            dataset_args['max_duration'] = max_duration
            dataset = PPVectorDataset(data_list_path=data_list, audio_featurizer=fz, mode='extract_feature',
                                      device=self.device, **dataset_args)
            save_data_list = data_list.replace('.txt', '_features.txt')
            with open(save_data_list, 'w', encoding='utf-8') as f:
                for i in tqdm(range(len(dataset))):
                    feature, label = dataset[i]
                    # the reference names files by millisecond timestamps (collisions once extraction is fast): use counters
                    save_path = os.path.join(save_dir, str(label), f'{list_idx}_{i:08d}.npy').replace('\\', '/')
                    os.makedirs(os.path.dirname(save_path), exist_ok=True)
                    np.save(save_path, feature.cpu().numpy())
                    f.write(f'{save_path}\t{label}\n')
            logger.info(f'{data_list}列表中的数据已提取特征完成，新列表为：{save_data_list}')

    # ---- model -------------------------------------------------------------------------------------------------
    def _setup_model(self, resume_model=None):
        if self.model is None:
            self.model = build_model(input_size=self._featurizer().feature_dim, configs=self.configs)
        sd = self._state_dict
        if resume_model is not None:
            sd = load_state_dict_file(resume_model)
        if sd is not None:
            # Sequential(backbone, classifier) prefixes of the reference checkpoints: "0." backbone, "1." classifier
            sd = {(k[2:] if k.startswith('0.') else k): v for k, v in sd.items() if not k.startswith('1.')}
            self.model.load_state_dict({k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()})
        self.model.eval().to(self.device)
        return self.model

    def _embed_list(self, data_list, desc):
        dataset_args = dict(self.configs.dataset_conf.get('dataset', {}))
        dataset_args['max_duration'] = self.configs.dataset_conf.eval_conf.max_duration
        batch_size = self.configs.dataset_conf.eval_conf.batch_size
        dataset = PPVectorDataset(data_list_path=data_list, audio_featurizer=self._featurizer(), mode='eval',
                                  device=self.device, **dataset_args)
        feats, labels = [], []
        for i in tqdm(range(0, len(dataset), batch_size), desc=desc):
            if self.stop_eval:
                break
            # one launch sequence per batch (audio prep -> ragged front end); input_lens never reaches the model (trainer.py:392-395)
            features, label, _input_lens = dataset.load_batch(range(i, min(i + batch_size, len(dataset))))
            feats.append(self.model(features))
            labels.append(label)
        return torch.cat(feats, dim=0), torch.cat(labels).numpy().astype(np.int32)

    # ---- trainer.py:367-447 ------------------------------------------------------------------------------------
    def evaluate(self, resume_model=None, save_image_path=None):
        norm = score_norm_config(self.configs.dataset_conf.eval_conf.get('score_norm'))
        self._setup_model(resume_model)
        with torch.no_grad():
            enroll_features, enroll_labels = self._embed_list(self.configs.dataset_conf.enroll_list, '注册音频声纹特征')
            trials_features, trials_labels = self._embed_list(self.configs.dataset_conf.trials_list, '验证音频声纹特征')
            if norm is not None and not self.stop_eval:
                cohort_features, cohort_labels = self._embed_list(norm['cohort_list'], '归一化集合声纹特征')
        if self.stop_eval:
            return -1, -1, -1
        # the reference scores one trial against all enrolments per Python iteration (trainer.py:416-423): one GEMM here
        scores = cosine_matrix(trials_features, enroll_features)
        if norm is not None:  # extension: AS-norm against the cohort list (ppvector/metric/score_norm.py)
            cohort = speaker_cohort(cohort_features, cohort_labels) if norm['cohort'] == 'speaker' else cohort_features
            as_norm(scores, cohort_stats(trials_features, cohort, norm['top_n']), cohort_stats(enroll_features, cohort, norm['top_n']))
            logger.info(f"AS-norm against {cohort.shape[0]} cohort rows ({norm['cohort']}, top_n {norm['top_n']}): "
                        f"the threshold is in normalised score units")
        # EER / minDCF on the device too (metrics.py:4-37 definitions; csrc/metrics.cu): the M x N scores never visit the host
        eer, min_dcf, threshold = eer_mindcf_from_matrix_gpu(scores, trials_labels, enroll_labels)
        if save_image_path:
            logger.warning('save_image_path: plotting is out of scope of the CUDA hot path (ignored)')
        return float(eer), float(min_dcf), float(threshold)

    # ---- trainer.py:281-365, step :206-229 ---------------------------------------------------------------------
    def _train_batches(self, dataset, batch_size, epoch, rank, world, shuffle=True, drop_last=True):
        """paddle.io.DistributedBatchSampler: one permutation per epoch (seeded by the epoch), padded to a multiple of the
        world size, rank r takes every world-th index; batches of ``batch_size`` per rank."""
        from ppvector.parallel import train_sample_indices
        idx = train_sample_indices(len(dataset), epoch, rank, world, shuffle)
        for i in range(0, len(idx), batch_size):
            chunk = idx[i:i + batch_size]
            if len(chunk) < batch_size and (drop_last or len(chunk) < 2):
                break
            yield dataset.load_batch(chunk)  # one decode loop on the host, then ONE GPU launch sequence for the whole batch

    def train(self, save_model_path='models/', log_dir='log/', resume_model=None, pretrained_model=None, do_eval=True, max_steps=None):
        """reference: trainer.py:281-365.  ``max_steps`` (extension) stops early -- used by the tests and the bench tool.
        ``pretrained_model`` restores weights only (checkpoint.py:11-42); ``resume_model`` -- or ``<save_model_path>/<model>_<feature>/
        last_model`` when it exists -- restores weights, the optimizer's state and step count, both schedules and the epoch
        (checkpoint.py:45-101); a checkpoint written by another optimizer is refused."""
        import random as _random

        import torch.distributed as dist

        from ppvector.loss import build_loss
        from ppvector.optimizer import MarginScheduler, build_lr_scheduler, resolve_optimizer
        from ppvector.train_engine import TrainEngine
        cf = self.configs
        use_model = cf.model_conf.get('model', 'CAMPPlus')
        if use_model != 'EcapaTdnn':
            raise NotImplementedError(f'training on the H100 path is implemented for EcapaTdnn (got {use_model}); no fallback')
        if cf.loss_conf.get('loss', 'AAMLoss') not in ('AAMLoss', 'AMLoss', 'ARMLoss', 'CELoss', 'SubCenterLoss', 'SphereFace2'):
            raise NotImplementedError('training on the H100 path implements AAMLoss / AMLoss / ARMLoss / CELoss / SubCenterLoss / SphereFace2 (configs/ecapa_tdnn.yml)')
        # optimizer/__init__.py:12-18: paddle.optimizer.<optimizer>(**optimizer_args), checked here before any work
        opt_name = cf.optimizer_conf.get('optimizer', 'Adam')
        opt_args = resolve_optimizer(opt_name, cf.optimizer_conf.get('optimizer_args', {}))
        if cf.dataset_conf.get('is_use_pksampler', False):
            raise NotImplementedError('PKSampler is out of scope of the H100 path')
        model_args = dict(cf.model_conf.get('model_args', {}))
        pooling_type = model_args.get('pooling_type', 'ASP')
        if pooling_type not in ('ASP', 'SAP', 'TAP', 'TSP'):
            raise Exception(f'没有{pooling_type}池化层！')  # ecapa_tdnn.py:242-243
        if pooling_type == 'SAP' and int(model_args.get('attention_channels', 128)) != 128:  # the inference model refuses it too
            raise NotImplementedError('SAP pooling uses a 128-channel bottleneck (ecapa_tdnn.py:222): attention_channels must be 128')
        ch = list(model_args.get('channels', (512, 512, 512, 512, 1536)))
        if len(ch) != 5 or ch[1:4] != [ch[0]] * 3 or ch[4] != 3 * ch[0]:
            raise NotImplementedError(f'the CUDA training step implements channels [C, C, C, C, 3C] (got {ch})')
        torch.manual_seed(1000)  # trainer.py:290
        np.random.seed(1000)
        _random.seed(1000)
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank() if world > 1 else 0
        fz = self._featurizer()
        dataset_args = dict(cf.dataset_conf.get('dataset', {}))
        train_dataset = PPVectorDataset(data_list_path=cf.dataset_conf.train_list, audio_featurizer=fz, mode='train', device=self.device,
                                        aug_conf=self.data_augment_configs, num_speakers=int(cf.model_conf.classifier.num_speakers), **dataset_args)
        sampler = cf.dataset_conf.get('sampler', {})
        batch_size = int(sampler.get('batch_size', 64))
        num_speakers = int(cf.model_conf.classifier.num_speakers)
        backbone = build_model(input_size=fz.feature_dim, configs=cf)  # random init with the mirror's initialisers, names = state_dict
        cls_conf = dict(cf.model_conf.get('classifier', {}))
        cls_type = cls_conf.get('classifier_type', 'Cosine')
        if cls_type not in ('Cosine', 'Linear'):
            raise ValueError(f'不支持该输出层：{cls_type}')  # fc.py:39-40
        num_blocks, inter_dim = int(cls_conf.get('num_blocks', 0)), int(cls_conf.get('inter_dim', 512))
        loss_name = cf.loss_conf.get('loss', 'AAMLoss')
        loss_args = dict(cf.loss_conf.get('loss_args', {}) or {})
        if cls_type == 'Linear' and (loss_name in ('AAMLoss', 'SubCenterLoss') or
                                     (loss_name == 'SphereFace2' and loss_args.get('margin_type', 'C') == 'A')):
            # aamloss.py / subcenterloss.py / sphereface2.py (type A) take sqrt(1 - z^2) of the logits: NaN once a Linear logit leaves [-1, 1]
            raise NotImplementedError(f'{loss_name}{" (margin_type A)" if loss_name == "SphereFace2" else ""} reads the logits as cosines '
                                      f'(sqrt(1 - z^2)) and cannot train a Linear classifier; use classifier_type Cosine, or CELoss / AMLoss / '
                                      f'ARMLoss / SphereFace2 with margin_type C')
        # fc.py:33: K sub-centres per class (SubCenterLoss); the cosine classifier has num_speakers * K columns, a Linear one ignores K
        cls_K = int(cls_conf.get('K', 1)) if cls_type == 'Cosine' else 1
        loss_K = int(loss_args.get('K', 3)) if loss_name == 'SubCenterLoss' else 1
        if cls_K != loss_K:
            raise ValueError(f'classifier K={cls_K} and loss K={loss_K} differ (SubCenterLoss needs model_conf.classifier.K == loss_args.K)')
        num_classes = num_speakers
        num_speakers = num_speakers * cls_K  # columns of the classifier from here on
        engine_args = {k: model_args[k] for k in ('channels', 'kernel_sizes', 'dilations', 'attention_channels', 'res2net_scale', 'se_channels',
                                                  'pooling_type', 'global_context') if k in model_args}
        engine = TrainEngine(input_size=fz.feature_dim, num_speakers=num_speakers, embd_dim=model_args.get('embd_dim', 192), device=self.device,
                             classifier_type=cls_type, num_blocks=num_blocks, inter_dim=inter_dim, optimizer=opt_name, optimizer_args=opt_args,
                             **engine_args)
        if cf.train_conf.get('enable_amp', False):
            # reference trainer.py:167, 209-229: auto_cast(level='O1') + GradScaler(1024).  Here: single-pass bf16 GEMM operands, everything else
            # fp32; bf16 has fp32's exponent range, so no loss scaling (nothing to unscale, no skipped steps)
            engine.set_precision('bf16')
            logger.info('enable_amp: bf16 operands in every GEMM of the step, fp32 accumulation / BatchNorm / loss / master weights')
        shapes = {k: tuple(v.shape) for k, v in backbone.state_dict().items()}
        sd = {k: v for k, v in backbone.state_dict().items()}
        cls_shapes = engine.classifier_shapes
        sd.update(init_classifier(cls_shapes))
        resume_dir = find_resume_dir(cf, save_model_path, resume_model)
        opt_state, run_state = None, {}
        for path, is_resume in ((pretrained_model, False), (resume_dir, True)):
            if path is None:
                continue
            if is_resume:
                loaded, opt_state, run_state = load_checkpoint_dir(path)
            else:
                loaded = load_state_dict_file(path)
            # Sequential(backbone, classifier) keys: "1.<name>" is the classifier's "classifier.<name>" (checked whole before anything loads)
            cls_loaded = {'classifier.' + (k[2:] if k.startswith('1.') else k[len('classifier.'):]): v for k, v in loaded.items()
                          if k.startswith(('1.', 'classifier.'))}
            check_classifier_keys(cls_loaded, cls_shapes, path)
            if is_resume:
                check_optimizer_state(opt_state, opt_name, engine.optim_state, path)
            for k, v in loaded.items():
                if not k.startswith(('1.', 'classifier.')):
                    sd[k[2:] if k.startswith('0.') else k] = torch.as_tensor(np.asarray(v))
            sd.update({k: torch.as_tensor(np.asarray(v)) for k, v in cls_loaded.items()})
        engine.load_state_dict(sd)
        last_epoch, best_eer = 0, 1.0
        if opt_state is not None:  # checkpoint.py:64-85: optimizer state, epoch counter, best EER
            for k, t in engine.optim_state.items():
                t.copy_(opt_state[k])
            engine.step_count = int(opt_state['step_count'])
            last_epoch = int(run_state.get('last_epoch', opt_state.get('last_epoch', 0)))
            best_eer = float(run_state.get('eer', 1.0))
            logger.info(f'成功恢复模型参数和优化方法参数：{resume_dir}')
        if world > 1:  # every rank starts from rank 0's weights (fleet.distributed_model broadcasts them)
            dist.broadcast(engine.params, src=0)
            dist.broadcast(engine.stats, src=0)
        steps_per_epoch = max(1, (int(np.ceil(len(train_dataset) / world)) // batch_size))
        scheduler = build_lr_scheduler(step_per_epoch=steps_per_epoch, configs=cf)
        criterion = build_loss(cf)  # loss/__init__.py:16-22
        margin_scheduler = None
        if cf.loss_conf.get('use_margin_scheduler', False):  # trainer.py:182-190: defaults overridden with dict.update
            ms_args = dict(increase_start_epoch=int(cf.train_conf.max_epoch * 0.3), fix_epoch=int(cf.train_conf.max_epoch * 0.7))
            ms_args.update(dict(cf.loss_conf.get('margin_scheduler_args', {}) or {}))
            margin_scheduler = MarginScheduler(criterion=criterion, step_per_epoch=steps_per_epoch, **ms_args)
        if last_epoch > 0:  # checkpoint.py:80-84: replay the schedules up to the resumed epoch
            for _ in range(last_epoch * steps_per_epoch):
                scheduler.step()
            if margin_scheduler is not None:
                margin_scheduler.step(current_step=last_epoch * steps_per_epoch)
        logger.info(f'成功创建优化方法：{opt_name}，参数为：{opt_args}')
        logger.info('训练数据：{}'.format(len(train_dataset)))
        self.train_step, self.train_loss, self.train_acc = last_epoch * steps_per_epoch, None, None
        self.eval_eer = self.eval_min_dcf = self.eval_threshold = None
        history = []

        def checkpoint(epoch_no, best):
            self._state_dict = {k: v.cpu().numpy() for k, v in engine.state_dict(shapes).items()}
            # keys as in the reference's Sequential(backbone, classifier) checkpoint: "0.<backbone tensor>", "1.<classifier tensor>"
            ckpt = {'0.' + k: torch.from_numpy(v) for k, v in self._state_dict.items()}
            ckpt.update({'1.' + k[len('classifier.'):]: v.cpu() for k, v in engine.state_dict(cls_shapes).items()})
            opt = {'optimizer': opt_name, **{k: t.detach().cpu() for k, t in engine.optim_state.items()}, 'step_count': engine.step_count,
                   'last_epoch': epoch_no, 'scheduler_last_epoch': getattr(scheduler, 'last_epoch', None),
                   'margin_step': getattr(margin_scheduler, 'current_step', None)}
            return save_checkpoint(cf, ckpt, opt, save_model_path, epoch_no, eer=self.eval_eer, min_dcf=self.eval_min_dcf,
                                   threshold=self.eval_threshold, margin=margin_scheduler.get_margin() if margin_scheduler else None,
                                   best_model=best)

        for epoch_id in range(last_epoch, int(cf.train_conf.max_epoch)):
            losses, accs = [], []
            for features, label, _lens in self._train_batches(train_dataset, batch_size, epoch_id, rank, world, sampler.get('shuffle', True),
                                                              sampler.get('drop_last', True)):
                if self.stop_train or (max_steps is not None and self.train_step >= max_steps):
                    break
                loss, logits = engine.forward_backward(features, label, margin=criterion.margin, scale=criterion.scale,
                                                       easy_margin=criterion.easy_margin, label_smoothing=criterion.label_smoothing,
                                                       return_logits=True)
                engine.optimizer_step(lr=scheduler.get_lr(), grad_scale=engine.all_reduce_grads())
                if cls_K > 1:  # trainer.py:231-234: a class's logit is the max over its sub-centres
                    logits = logits.reshape(logits.shape[0], num_classes, cls_K).amax(2)
                accs.append((logits.argmax(1).cpu() == label.cpu()).float().mean().item())
                losses.append(float(loss))  # the reference syncs here too (trainer.py:237-238)
                self.train_step += 1
                if self.train_step % int(cf.train_conf.get('log_interval', 10)) == 0 and rank == 0:
                    self.train_loss, self.train_acc = float(np.mean(losses)), float(np.mean(accs))
                    logger.info(f'Train epoch: [{epoch_id}/{cf.train_conf.max_epoch}], step: {self.train_step}, loss: {self.train_loss:.5f}, '
                                f'accuracy: {self.train_acc:.5f}, learning rate: {scheduler.get_lr():.8f}, margin: {criterion.margin}')
                    losses, accs = [], []
                history.append(float(loss))
                scheduler.step()
                if margin_scheduler:
                    margin_scheduler.step()
            if self.stop_train or (max_steps is not None and self.train_step >= max_steps):
                break
            if world > 1:
                dist.barrier()  # the reference lets rank 0 evaluate while the others run ahead; keep the ranks together
            if rank == 0:  # trainer.py:336-365: evaluate, keep the best-EER model, save epoch_N / last_model
                epoch_no = epoch_id + 1
                self._state_dict = {k: v.cpu().numpy() for k, v in engine.state_dict(shapes).items()}
                if do_eval and os.path.exists(cf.dataset_conf.enroll_list):
                    self.model = None
                    self.eval_eer, self.eval_min_dcf, self.eval_threshold = self.evaluate()
                    logger.info(f'Test epoch: {epoch_no}, threshold: {self.eval_threshold:.2f}, EER: {self.eval_eer:.5f}, MinDCF: {self.eval_min_dcf:.5f}')
                    if self.eval_eer <= best_eer:
                        best_eer = self.eval_eer
                        checkpoint(epoch_no, best=True)
                checkpoint(epoch_no, best=False)
        self._state_dict = {k: v.cpu().numpy() for k, v in engine.state_dict(shapes).items()}
        self.engine = engine
        return history

    def export(self, *args, **kwargs):
        raise NotImplementedError('export is broken in the reference (trainer.py:467-469) and out of scope')
