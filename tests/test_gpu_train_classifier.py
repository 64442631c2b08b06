"""GPU: the ECAPA-TDNN training step with the classifiers of fc.py besides Cosine without blocks (tests/test_gpu_train.py covers that one):
DenseLayer blocks (1x1 conv + BatchNorm1D over the batch) in front of the output layer, and the Linear output layer.

  * one step against the reference's own step (tests/golden/ref_classifier.npz) and against torch autograd over the fp64 oracle
    (tests/classifier_oracle.py, pinned to that fixture in tests/test_train_classifier_cpu.py): loss, logits, block-output taps, every
    gradient, the blocks' running statistics -- with test_gpu_train.py's bounds for the head and fc, in bf16x3 and in bf16 (enable_amp);
  * the same at the config size (64 x 298, 2796 speakers, two 512-wide blocks), Cosine + AAMLoss and Linear + CELoss;
  * every variant bitwise reproducible; state_dict / load_state_dict through the new names;
  * the refusals: Linear with AAMLoss, SubCenterLoss or SphereFace2 type A, an unknown classifier_type, a checkpoint of another classifier;
  * PPVectorTrainer.train end to end: checkpoint keys, resume, evaluate and the predictor on the result."""
import copy
import json
import os
import wave

import numpy as np
import pytest
import torch
import yaml

from classifier_oracle import classifier_names, make_classifier_weights, train_step_grads
from oracle import ecapa as oe
from ppvector import _lib
from ppvector.train_engine import TrainEngine

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# tests/golden/make_classifier_fixture.py: tag -> (classifier_type, num_blocks, inter_dim, loss, output weight gain)
CASES = {"cos_b1_AAM": ("Cosine", 1, 512, "AAMLoss", 1.0), "cos_b2_AAM": ("Cosine", 2, 512, "AAMLoss", 1.0),
         "lin_b0_CE": ("Linear", 0, 512, "CELoss", 1.0), "lin_b2_CE": ("Linear", 2, 512, "CELoss", 1.0),
         "lin_b0_AM": ("Linear", 0, 512, "AMLoss", 1.0), "lin_b2_AM": ("Linear", 2, 512, "AMLoss", 1.0),
         "lin_b0_SF2C": ("Linear", 0, 512, "SphereFace2", 0.3), "lin_b2_SF2C": ("Linear", 2, 512, "SphereFace2", 0.3),
         "cos_b2_i96_AAM": ("Cosine", 2, 96, "AAMLoss", 1.0)}
B0, T0, S0, SEED, CLS_SEED = 4, 61, 37, 78, 79
# loss -> (head selector, margin, scale, label_smoothing slot) as the reference's default constructors (SphereFace2: t 3, lanbuda 0.7)
HEADS = {"AAMLoss": (_lib.PPV_HEAD_AAM, 0.2, 32.0, 0.0), "CELoss": (_lib.PPV_HEAD_CE, 0.0, 1.0, 0.0), "AMLoss": (_lib.PPV_HEAD_AM, 0.2, 30.0, 0.0),
         "SphereFace2": (_lib.PPV_HEAD_SPHEREFACE2 | (3 << 5), 0.2, 32.0, 0.7)}
HEAD = ("classifier", "fc.", "asp_bn.")


def zero_grads(nb):
    """Gradients that are exactly zero in exact arithmetic.  asp.conv.conv.bias: softmax over time is shift invariant.  With classifier
    blocks, a BatchNorm over the batch removes any per-channel constant added before it: every block's conv bias, every block's BatchNorm
    shift but the last one's, and the biases of fc and asp_bn (a constant shift of the embedding)."""
    z = {"asp.conv.conv.bias"}
    if nb:
        z |= {"fc.conv.bias", "asp_bn.norm.bias"} | {f"classifier.blocks.{i}.linear.bias" for i in range(nb)}
        z |= {f"classifier.blocks.{i}.nonlinear.batchnorm.bias" for i in range(nb - 1)}
    return z


def small_bounds(name, nb):
    """(relative L2, cosine) at the fixture's 4 x 61 in bf16x3: test_gpu_train.py::test_forward_taps_loss_and_all_gradients's head 5e-4 and
    backbone 5e-2 / 0.999, and two measured exceptions.  The 64-element conv and BatchNorm bias gradients of the Res2Net blocks are sums over
    244 frames that cancel: measured on an H100 up to 5.3e-2 / 0.99858 (blocks.3.res2net_block.blocks.2.conv.conv.bias), so they get
    test_gpu_train_pooling.py's 8e-2 / 0.998 for the same family.  Behind classifier blocks the head's tensors reach 6.0e-4
    (asp_bn.norm.weight): a BatchNorm over 4 embeddings subtracts a batch mean close to each value and magnifies the backbone's
    split-bf16 rounding of emb; they get 1e-3.  At 64 x 298 every tensor is within test_gpu_train.py's config-size bounds."""
    if name.startswith(HEAD):
        return (1e-3 if nb else 5e-4), 0.999
    if name.endswith(("conv.conv.bias", "norm.norm.bias")) and ".res2net_block." in name:
        return 8e-2, 0.998
    return 5e-2, 0.999


def problem(B, T, S, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    return f, torch.randint(0, S, (B,), generator=g)


_W = {}


def backbone():
    if not _W:
        _W.update(oe.make_ecapa_weights(seed=1000, dtype=torch.float64))
    return _W


def new_engine(cuda, ct, nb, inter, W, S, precision="bf16x3"):
    eng = TrainEngine(input_size=80, num_speakers=S, classifier_type=ct, num_blocks=nb, inter_dim=inter, device=cuda)
    eng.load_state_dict(W)
    eng.set_precision(precision)
    return eng


def step(eng, f, y, loss_name, cuda):
    sel, margin, scale, ls = HEADS[loss_name]
    return eng.forward_backward(f.float().to(cuda), y.to(cuda), margin=margin, scale=scale, easy_margin=sel, label_smoothing=ls, return_logits=True)


def rel_cos(gg, gw):
    rel = ((gg - gw).norm() / (gw.norm() + 1e-12)).item()
    cos = ((gg * gw).sum() / (gg.norm() * gw.norm() + 1e-30)).item()
    return rel, cos


def check_step(eng, f, y, W, ct, nb, loss_name, precision, cuda, big=False):
    """One step against the fp64 oracle; returns the oracle's (loss, logits, grads, stats) for the caller's further checks."""
    taps = {}
    loss, grads, stats, logits, emb = train_step_grads(f, y, W, ct, nb, loss=loss_name, taps=taps)
    got_loss, got_logits = step(eng, f, y, loss_name, cuda)
    torch.cuda.synchronize()
    amp = precision == "bf16"
    lscale = max(1.0, logits.abs().max().item())
    assert (got_logits.double().cpu() - logits).abs().max() < (5e-2 if amp else 1e-4) * lscale
    assert abs(got_loss.item() - loss.item()) < (5e-3 if amp else 1e-3) * max(1.0, abs(loss.item()))
    B = f.shape[0]
    for i in range(nb):
        name = f"classifier.blocks.{i}"
        got = eng.read_tap(name, (B, eng.inter_dim)).double().cpu()
        assert rel_cos(got, taps[name].detach())[0] < (5e-2 if amp else 1e-4), name
        got = eng.read_tap("g:" + name, (B, eng.inter_dim)).double().cpu()
        assert rel_cos(got, taps[name].grad)[0] < (5e-2 if amp else 5e-4), "g:" + name
    bad, worst = [], {}
    for name, gw in grads.items():
        if name == "emb":
            continue
        gg = eng.view(name, tuple(gw.shape), "grad").double().cpu()
        if name in zero_grads(nb):
            assert gw.abs().max() < 1e-10 and gg.abs().max() < 1e-4, name
            continue
        rel, cos = rel_cos(gg, gw)
        head = name.startswith(HEAD)
        if amp:  # test_gpu_train.py::test_amp_bf16_operands_track_the_fp64_oracle
            ok = rel < 5e-2 if head else (rel < 0.3 and cos > 0.96) if gw.dim() >= 2 else (rel < 0.6 and cos > 0.85)
        elif big:  # test_gpu_train.py::test_gradients_at_the_config_size; mfa.norm.norm.bias: see test_step_at_the_config_size
            tol = 3e-2 if name == "mfa.norm.norm.bias" else 2e-4 if head else 2.5e-2 if name.startswith(("asp.", "mfa.")) else 2e-2
            ok = rel < tol and cos > 0.999
        else:
            tol, min_cos = small_bounds(name, nb)
            ok = rel < tol and cos > min_cos
        key = "head" if head else "backbone"
        worst[key] = max(worst.get(key, 0.0), rel)
        if not ok:
            bad.append((name, rel, cos))
    print(f"{ct} {nb} blocks {loss_name} {precision} B={B}: worst relative gradient error", {k: f"{v:.2e}" for k, v in worst.items()})
    assert not bad, bad[:10]
    for name, sw in stats.items():
        gs = eng.view(name, tuple(sw.shape)).double().cpu()
        assert (gs - sw).abs().max() < (5e-2 if amp else 1e-4) * max(1.0, sw.abs().max().item()), name
    return loss, logits, grads, stats


# ------------------------------------------------------------------------------------------------ one step at the fixture's size
@pytest.fixture(scope="module")
def ref(golden_dir):
    return np.load(f"{golden_dir}/ref_classifier.npz")


# bf16 (enable_amp) at this size only without blocks: a BatchNorm over 4 embeddings magnifies their bf16 rounding (measured on an H100:
# Linear logits 6 % off with two blocks); test_step_at_the_config_size checks the blocks in bf16 at the config's batch of 64
@pytest.mark.parametrize("tag,precision", [(t, "bf16x3") for t in CASES] + [(t, "bf16") for t, c in CASES.items() if c[1] == 0])
def test_step_matches_reference_and_oracle(cuda, ref, tag, precision):
    ct, nb, inter, loss_name, gain = CASES[tag]
    f, y = problem(B0, T0, S0, SEED)
    Wc = make_classifier_weights(CLS_SEED, S0, ct, nb, inter, gain=gain)
    W = dict(backbone(), **Wc)
    eng = new_engine(cuda, ct, nb, inter, W, S0, precision)
    check_step(eng, f, y, W, ct, nb, loss_name, precision, cuda)
    # and straight against what the reference's own classes computed (the classifier tensors, fc, the running statistics)
    amp = precision == "bf16"
    got_loss = eng._loss[0].item()
    want = float(ref[f"{tag}_loss"])
    assert abs(got_loss - want) < (5e-3 if amp else 1e-3) * max(1.0, abs(want))
    for name in list(Wc) + ["fc.conv.weight", "fc.conv.bias"]:
        if name in zero_grads(nb):
            continue  # checked against the oracle above
        if name.endswith(("._mean", "._variance")):
            got = eng.view(name).double().cpu().numpy()
            assert np.abs(got - ref[f"{tag}_stat_{name}"]).max() < (5e-2 if amp else 1e-4), name
            continue
        shape = Wc[name].shape if name in Wc else backbone()[name].shape
        g = eng.view(name, tuple(shape), "grad").double().cpu()
        if g.dim() == 1:
            rel = np.linalg.norm(g.numpy() - ref[f"{tag}_grad_{name}"]) / np.linalg.norm(ref[f"{tag}_grad_{name}"])
        else:
            want = float(ref[f"{tag}_gradnorm_{name}"])
            rel = abs(float(g.norm()) - want) / want
        assert rel < (5e-2 if amp else 5e-4), (name, rel)


# ------------------------------------------------------------------------------------------------ the config size
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("ct,loss_name", [("Cosine", "AAMLoss"), ("Linear", "CELoss")])
def test_step_at_the_config_size(cuda, ct, loss_name, precision):
    """64 x 298 frames, 2796 speakers, two 512-wide blocks: test_gpu_train.py::test_gradients_at_the_config_size's bounds in bf16x3 (head
    2e-4), test_amp_bf16_operands_track_the_fp64_oracle's in bf16.  One exception: mfa.norm.norm.bias gets 3e-2 for 2.5e-2, measured at
    2.54e-2 / 0.99968 on an H100 with both classifiers -- most of that gradient cancels (a per-channel shift of mfa's output moves the
    pooled mean by a constant that asp_bn removes; only the attention path sees it)."""
    B, T, S = 64, 298, 2796
    f, y = problem(B, T, S, 64298)
    Wc = make_classifier_weights(CLS_SEED, S, ct, 2, 512)
    W = dict(backbone(), **Wc)
    eng = new_engine(cuda, ct, 2, 512, W, S, precision)
    check_step(eng, f, y, W, ct, 2, loss_name, precision, cuda, big=True)


# ------------------------------------------------------------------------------------------------ reproducibility, named views
@pytest.mark.parametrize("tag", list(CASES))
def test_step_is_bitwise_reproducible(cuda, tag):
    ct, nb, inter, loss_name, gain = CASES[tag]
    f, y = problem(4, 40, S0, 7)
    W = dict(backbone(), **make_classifier_weights(CLS_SEED, S0, ct, nb, inter, gain=gain))
    eng = new_engine(cuda, ct, nb, inter, W, S0)
    l1, z1 = step(eng, f, y, loss_name, cuda)
    g1, s1 = eng.grads.clone(), eng.stats.clone()
    eng.load_state_dict(W)  # running statistics back to the start
    l2, z2 = step(eng, f, y, loss_name, cuda)
    assert torch.equal(g1, eng.grads) and torch.equal(s1, eng.stats) and torch.equal(l1, l2) and torch.equal(z1, z2)


@pytest.mark.parametrize("ct,nb", [("Cosine", 2), ("Linear", 0), ("Linear", 3)])
def test_state_dict_round_trip_through_the_classifier_names(cuda, ct, nb):
    S, inter = 11, 64
    Wc = make_classifier_weights(5, S, ct, nb, inter)
    eng = TrainEngine(input_size=80, num_speakers=S, classifier_type=ct, num_blocks=nb, inter_dim=inter, device=cuda)
    assert list(eng.classifier_shapes) == classifier_names(ct, nb)
    eng.load_state_dict(dict(backbone(), **Wc))
    out = eng.state_dict(eng.classifier_shapes)
    assert list(out) == list(Wc)
    for k, v in Wc.items():
        assert torch.equal(out[k].cpu(), v.float()), k
    other = "classifier.weight" if ct == "Linear" else "classifier.output.weight"
    with pytest.raises(_lib.PPVError, match="unknown tensor"):
        eng.view(other)
    if nb:  # the blocks' running statistics live in the statistics buffer, beside the backbone's
        off, numel, is_stat = eng._lookup("classifier.blocks.0.nonlinear.batchnorm._variance")
        assert is_stat and numel == inter


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("sel", [_lib.PPV_HEAD_AAM, _lib.PPV_HEAD_AAM_EASY, _lib.PPV_HEAD_SUBCENTER | (1 << 5),
                                 _lib.PPV_HEAD_SPHEREFACE2 | (3 << 5) | 1], ids=["AAM", "AAM-easy", "SubCenter", "SphereFace2-A"])
def test_linear_classifier_refuses_cosine_only_heads(cuda, sel):
    W = dict(backbone(), **make_classifier_weights(CLS_SEED, S0, "Linear", 0))
    eng = new_engine(cuda, "Linear", 0, 512, W, S0)
    f, y = problem(4, 40, S0, 7)
    with pytest.raises(_lib.PPVError, match=r"sqrt\(1 - z\^2\)"):
        eng.forward_backward(f.float().to(cuda), y.to(cuda), easy_margin=sel)
    with pytest.raises(ValueError, match="不支持该输出层"):
        TrainEngine(input_size=80, num_speakers=S0, classifier_type="AMSoftmax", device=cuda)


def trainer_config(tmp_path, wav_paths, ct, nb, loss_name, loss_args=None):
    cfg = yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader)
    names = ["a_1", "a_2", "b_1", "b_2", "long3s"]
    spk = {"a_1": 0, "a_2": 0, "b_1": 1, "b_2": 1, "long3s": 2}
    for name, members in {"train": names + names, "enroll": ["a_1", "b_1", "long3s"], "trials": ["a_2", "b_2"]}.items():
        p = str(tmp_path / f"{name}_list.txt")
        with open(p, "w") as f:
            for n in members:
                f.write(f"{wav_paths[n]}\t{spk[n]}\n")
        cfg["dataset_conf"][f"{name}_list"] = p
    cfg["dataset_conf"]["sampler"]["batch_size"] = 4
    cfg["model_conf"]["classifier"].update({"num_speakers": 3, "classifier_type": ct, "num_blocks": nb})
    cfg["loss_conf"]["loss"] = loss_name
    if loss_args is not None:
        cfg["loss_conf"]["loss_args"] = loss_args
    cfg["train_conf"]["max_epoch"] = 2
    return cfg


@pytest.fixture(scope="module")
def wavs(tmp_path_factory, golden_dir):  # test_gpu_api.wavs
    d = tmp_path_factory.mktemp("wavs")
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    paths = {}
    for n in ["a_1", "a_2", "b_1", "b_2", "long3s"]:
        p = str(d / f"{n}.wav")
        with wave.open(p, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(16000)
            w.writeframes(g[n + "_pcm"].astype("<i2").tobytes())
        paths[n] = p
    return paths


def test_trainer_rejects_what_the_classifier_cannot_train(cuda, wavs, tmp_path):
    from ppvector.trainer import PPVectorTrainer
    for loss_name, loss_args in [("AAMLoss", None), ("SubCenterLoss", {"K": 3}), ("SphereFace2", {"margin_type": "A"})]:
        cfg = trainer_config(tmp_path, wavs, "Linear", 0, loss_name, loss_args)
        with pytest.raises(NotImplementedError, match=r"sqrt\(1 - z\^2\).*Linear classifier"):
            PPVectorTrainer(cfg, use_gpu=True).train(save_model_path=str(tmp_path / "m"))
    cfg = trainer_config(tmp_path, wavs, "Softmax", 0, "AAMLoss")
    with pytest.raises(ValueError, match="不支持该输出层"):
        PPVectorTrainer(cfg, use_gpu=True).train(save_model_path=str(tmp_path / "m"))


# ------------------------------------------------------------------------------------------------ PPVectorTrainer end to end
@pytest.mark.parametrize("ct,nb,loss_name", [("Linear", 0, "CELoss"), ("Cosine", 2, "AAMLoss"), ("Linear", 2, "CELoss")])
def test_trainer_train_checkpoint_resume_and_evaluate(cuda, wavs, tmp_path, ct, nb, loss_name):
    """Two epochs, checkpoint keys of the reference's Sequential(backbone, classifier), evaluate and the predictor on best_model, a resumed
    third epoch, and a checkpoint of another classifier refused before anything loads."""
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    from ppvector.predict import PPVectorPredictor
    from ppvector.trainer import PPVectorTrainer
    cfg = trainer_config(tmp_path, wavs, ct, nb, loss_name, {"label_smoothing": 0.0} if loss_name == "CELoss" else None)
    save = str(tmp_path / "models")
    tr = PPVectorTrainer(cfg, use_gpu=True)
    history = tr.train(save_model_path=save, do_eval=True)
    assert len(history) == 4 and all(np.isfinite(history))
    root = os.path.join(save, "EcapaTdnn_Fbank")
    assert sorted(os.listdir(root)) == ["best_model", "epoch_1", "epoch_2", "last_model"]
    ck = torch.load(os.path.join(root, "last_model", "model.pt"))
    sd = EcapaTdnn(input_size=80).state_dict()
    cls = {"1." + k[len("classifier."):]: s for k, s in tr.engine.classifier_shapes.items()}
    assert set(ck) == {"0." + k for k in sd} | set(cls)
    assert all(tuple(ck[k].shape) == tuple(s) for k, s in cls.items())
    if nb:  # the blocks' running statistics moved off their initial 0 / 1
        assert ck["1.blocks.1.nonlinear.batchnorm._mean"].abs().max() > 0
    eer, _, thr = PPVectorTrainer(cfg, use_gpu=True).evaluate(resume_model=os.path.join(root, "best_model"))
    assert 0.0 <= eer <= 1.0 and np.isfinite(thr)
    pred = PPVectorPredictor(cfg, model_path=os.path.join(root, "last_model"), use_gpu=True)
    assert np.isfinite(pred.contrast(wavs["a_1"], wavs["a_2"]))
    cfg3 = copy.deepcopy(cfg)
    cfg3["train_conf"]["max_epoch"] = 3
    tr3 = PPVectorTrainer(cfg3, use_gpu=True)
    h3 = tr3.train(save_model_path=save, do_eval=False)
    assert len(h3) == 2 and all(np.isfinite(h3)) and tr3.engine.step_count == 6 and tr3.train_step == 6
    assert json.load(open(os.path.join(root, "last_model", "model.state")))["last_epoch"] == 3
    # resuming with another classifier: refused, naming the keys
    other = copy.deepcopy(cfg3)
    other["train_conf"]["max_epoch"] = 4
    other["model_conf"]["classifier"].update({"classifier_type": "Cosine" if ct == "Linear" else "Linear", "num_blocks": 1})
    other["loss_conf"].update({"loss": "AMLoss", "loss_args": {}})
    with pytest.raises(ValueError, match=r"missing keys \['1\..*unexpected keys \['1\."):
        PPVectorTrainer(other, use_gpu=True).train(save_model_path=save, do_eval=False)
    # and as a pretrained model
    with pytest.raises(ValueError, match="does not match model_conf.classifier"):
        PPVectorTrainer(other, use_gpu=True).train(save_model_path=str(tmp_path / "fresh"), pretrained_model=os.path.join(root, "best_model"),
                                                   do_eval=False)
