"""Checkpoint I/O for the drop-in entry points.

The reference saves ``model.pdparams`` with ``paddle.save`` (ppvector/utils/checkpoint.py:104-159): a pickle of
{name: numpy array}.  Reading real ``.pdparams`` files (SURVEY.md §8(f) rank 1) needs no Paddle -- it is a plain
pickle of numpy arrays for the 2.x formats -- and is supported here on a best-effort basis; ``.npz`` and torch
``.pt/.pth`` state dicts are the native formats of this build."""
import json
import os
import pickle
import shutil

import numpy as np


def load_state_dict_file(path):
    if os.path.isdir(path):
        for name in ('model.pdparams', 'model.npz', 'model.pth', 'model.pt'):
            if os.path.exists(os.path.join(path, name)):
                path = os.path.join(path, name)
                break
        else:
            raise FileNotFoundError(f'{path} 模型不存在！')
    if path.endswith('.npz'):
        with np.load(path) as z:
            return {k: z[k] for k in z.files}
    if path.endswith(('.pt', '.pth')):
        import torch
        sd = torch.load(path, map_location='cpu')
        return {k: v.numpy() for k, v in sd.items()}
    with open(path, 'rb') as f:  # .pdparams: pickle of {name: ndarray} (paddle.save protocol 2-4)
        obj = pickle.load(f, encoding='latin1')
    out = {}
    for k, v in obj.items():
        if isinstance(v, np.ndarray):
            out[k] = v
        elif isinstance(v, (tuple, list)) and len(v) == 2 and isinstance(v[1], np.ndarray):
            out[k] = v[1]  # (name, ndarray) form used by some paddle versions
    return out


def save_state_dict_npz(state_dict, path):
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez(path, **{k: (v.detach().cpu().numpy() if hasattr(v, 'detach') else np.asarray(v)) for k, v in state_dict.items()})


# ---- training checkpoints: the reference's directory layout (ppvector/utils/checkpoint.py:104-159) ---------------------------------
#   <save_model_path>/<model>_<feature_method>/{epoch_N, last_model, best_model}/{model.pt, optimizer.pt, model.state}
# model.pt holds the reference's Sequential(backbone, classifier) keys ("0.<backbone tensor>", "1.weight"); optimizer.pt the optimizer's
# name ("optimizer"), its state tensors by name (Adam's "exp_avg" / "exp_avg_sq", ...), the step count and the LR / margin scheduler
# positions; model.state is the reference's json (last_epoch, eer, ...).
def checkpoint_root(configs, save_model_path):
    return os.path.join(save_model_path, f'{configs.model_conf.model}_{configs.preprocess_conf.feature_method}')


def save_checkpoint(configs, model_state, optimizer_state, save_model_path, epoch_id, eer=None, min_dcf=None, threshold=None,
                    margin=None, best_model=False, version='1.1.1'):
    import torch
    root = checkpoint_root(configs, save_model_path)
    model_path = os.path.join(root, 'best_model' if best_model else f'epoch_{epoch_id}')
    shutil.rmtree(model_path, ignore_errors=True)
    os.makedirs(model_path, exist_ok=True)
    torch.save(optimizer_state, os.path.join(model_path, 'optimizer.pt'))
    torch.save(model_state, os.path.join(model_path, 'model.pt'))
    data = {"last_epoch": epoch_id, "version": version, "model_conf.model": configs.model_conf.model,
            "feature_method": configs.preprocess_conf.feature_method, "loss": configs.loss_conf.get('use_loss', 'AAMLoss')}
    if eer is not None:
        data['threshold'], data['eer'], data['min_dcf'] = threshold, eer, min_dcf
    if margin is not None:
        data['margin'] = margin
    with open(os.path.join(model_path, 'model.state'), 'w', encoding='utf-8') as f:
        f.write(json.dumps(data, indent=4, ensure_ascii=False))
    if not best_model:
        last = os.path.join(root, 'last_model')
        shutil.rmtree(last, ignore_errors=True)
        shutil.copytree(model_path, last)
        shutil.rmtree(os.path.join(root, f'epoch_{epoch_id - 3}'), ignore_errors=True)  # keep the last three epochs
    return model_path


def find_resume_dir(configs, save_model_path, resume_model):
    """resume_model if given, else <root>/last_model when it holds a complete checkpoint (checkpoint.py:88-101), else None."""
    if resume_model is not None:
        return resume_model
    last = os.path.join(checkpoint_root(configs, save_model_path), 'last_model')
    if all(os.path.exists(os.path.join(last, n)) for n in ('model.pt', 'optimizer.pt', 'model.state')):
        return last
    return None


def check_optimizer_state(opt_state, name, state, path):
    """Refuses an optimizer.pt (``opt_state``; None passes) that another optimizer than ``name`` wrote, or whose state tensors are not
    exactly ``state``'s (name -> tensor) names and sizes.  An optimizer.pt without an ``optimizer`` entry was written by Adam."""
    if opt_state is None:
        return
    saved = opt_state.get('optimizer', 'Adam')
    if saved != name:
        raise ValueError(f'{path}: the checkpoint was trained with the {saved} optimizer and optimizer_conf.optimizer is {name}; resume it '
                         f'with {saved}, or start {name} from its weights with pretrained_model')
    have = {k: tuple(v.shape) for k, v in opt_state.items() if hasattr(v, 'shape')}
    want = {k: tuple(t.shape) for k, t in state.items()}
    if have != want:
        raise ValueError(f'{path}: optimizer.pt holds the {name} state {have}, the configured {name} needs {want}')


def load_checkpoint_dir(path):
    """-> (model state dict of numpy arrays, optimizer state or None, model.state json or {})"""
    import torch
    model = load_state_dict_file(path)
    opt, state = None, {}
    if os.path.isdir(path):
        if os.path.exists(os.path.join(path, 'optimizer.pt')):
            opt = torch.load(os.path.join(path, 'optimizer.pt'), map_location='cpu')
        if os.path.exists(os.path.join(path, 'model.state')):
            with open(os.path.join(path, 'model.state'), 'r', encoding='utf-8') as f:
                state = json.load(f)
    return model, opt, state
