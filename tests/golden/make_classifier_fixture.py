"""Mint tests/golden/ref_classifier.npz: one TRAIN-mode step of the reference's OWN EcapaTdnn, SpeakerIdentification and loss classes
(imported unmodified from /root/reference under tests/paddle_shim, with the helpers of make_ref_fixtures.py) for the classifiers the
reference builds besides Cosine without blocks (fc.py:6-90): Cosine + AAMLoss with one and two DenseLayer blocks, Linear + CELoss /
AMLoss / SphereFace2 (margin_type C) with none and two blocks, and one inter_dim other than 512.  Forward with batch statistics
(backbone and blocks), classifier, loss, backward through torch autograd, in fp64 (trainer.py:206-229).  Consumed by
tests/test_train_classifier_cpu.py on any machine; the file holds reference OUTPUTS only (loss, logits, the gradients of every
classifier tensor and of fc, and the blocks' updated running statistics); weights and inputs are re-derived from seeds by the consumer.

Runs only in the authoring container (needs /root/reference).
Usage:  python tests/golden/make_classifier_fixture.py            (rewrites ref_classifier.npz)
        python tests/golden/make_classifier_fixture.py --check    (recomputes and compares with the committed file)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_ref_fixtures import paddle, tap_slice  # noqa: E402  (sets up the shim and the reference's package path)

from ppvector.loss.aamloss import AAMLoss  # noqa: E402  (the REFERENCE's files)
from ppvector.loss.amloss import AMLoss  # noqa: E402
from ppvector.loss.celoss import CELoss  # noqa: E402
from ppvector.loss.sphereface2 import SphereFace2  # noqa: E402
from ppvector.models.ecapa_tdnn import EcapaTdnn  # noqa: E402
from ppvector.models.fc import SpeakerIdentification  # noqa: E402

from classifier_oracle import make_classifier_weights  # noqa: E402
from oracle import ecapa as o_ecapa  # noqa: E402

# tag -> (classifier_type, num_blocks, inter_dim, loss, output weight gain).  SphereFace2 runs its logits through a cubic and the
# reference's log(1 + exp(x)) overflows fp64 once x passes ~709, so its cases keep the Linear logits within a few units (the gain);
# some still fall below -1, where the cubic's base is negative.
CASES = {"cos_b1_AAM": ("Cosine", 1, 512, "AAMLoss", 1.0), "cos_b2_AAM": ("Cosine", 2, 512, "AAMLoss", 1.0),
         "lin_b0_CE": ("Linear", 0, 512, "CELoss", 1.0), "lin_b2_CE": ("Linear", 2, 512, "CELoss", 1.0),
         "lin_b0_AM": ("Linear", 0, 512, "AMLoss", 1.0), "lin_b2_AM": ("Linear", 2, 512, "AMLoss", 1.0),
         "lin_b0_SF2C": ("Linear", 0, 512, "SphereFace2", 0.3), "lin_b2_SF2C": ("Linear", 2, 512, "SphereFace2", 0.3),
         "cos_b2_i96_AAM": ("Cosine", 2, 96, "AAMLoss", 1.0)}
B, T, S, SEED, CLS_SEED = 4, 61, 37, 78, 79
LOSS_CLASSES = {"AAMLoss": AAMLoss, "CELoss": CELoss, "AMLoss": AMLoss, "SphereFace2": SphereFace2}


def problem():
    """Seeded, time-mean-subtracted features [B,T,80] and labels (the recipe of make_train_pooling_fixture.problem)."""
    g = torch.Generator().manual_seed(SEED)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    labels = torch.randint(0, S, (B,), generator=g)
    return f, labels


def classifier_fixture():
    d = {}
    f, labels = problem()
    W = o_ecapa.make_ecapa_weights(seed=1000, dtype=torch.float64)
    for tag, (ct, nb, inter, loss_name, gain) in CASES.items():
        Wc = make_classifier_weights(CLS_SEED, S, ct, nb, inter, gain=gain)
        model = EcapaTdnn(input_size=80)
        model.set_state_dict(W)
        clf = SpeakerIdentification(input_dim=192, num_speakers=S, classifier_type=ct, num_blocks=nb, inter_dim=inter)
        clf.set_state_dict({k[len("classifier."):]: v for k, v in Wc.items()})
        model.train()
        clf.train()
        out = clf(model(paddle.to_tensor(f)))
        loss = LOSS_CLASSES[loss_name]()(out, paddle.to_tensor(labels))
        loss.backward()
        d[f"{tag}_loss"] = np.array(float(loss))
        d[f"{tag}_logits"] = out["logits"].detach().numpy()
        params, sd = dict(clf.named_parameters()), clf.state_dict()
        for k in Wc:
            name = k[len("classifier."):]
            if k.endswith(("._mean", "._variance")):
                d[f"{tag}_stat_{k}"] = sd[name].numpy().copy()
                continue
            gr = params[name].grad
            # vectors whole; matrices as a slice plus their norm (keeps the file small)
            d[f"{tag}_grad_{k}"] = gr.numpy().copy() if gr.dim() == 1 else tap_slice(gr)
            d[f"{tag}_gradnorm_{k}"] = np.array(float(gr.norm()))
        mp = dict(model.named_parameters())
        d[f"{tag}_grad_fc.conv.bias"] = mp["fc.conv.bias"].grad.numpy().copy()
        d[f"{tag}_grad_fc.conv.weight"] = tap_slice(mp["fc.conv.weight"].grad)
        d[f"{tag}_gradnorm_fc.conv.weight"] = np.array(float(mp["fc.conv.weight"].grad.norm()))
    return d


def main():
    path = os.path.join(HERE, "ref_classifier.npz")
    d = classifier_fixture()
    if "--check" in sys.argv:
        old = np.load(path)
        assert sorted(old.files) == sorted(d), set(old.files) ^ set(d)
        assert all(np.isfinite(d[k]).all() for k in d)
        err = max(float(np.abs(old[k] - d[k]).max()) for k in d)
        print(f"ref_classifier.npz: {len(d)} arrays, max |committed - recomputed| = {err:.3e}")
        sys.exit(1 if err > 1e-12 else 0)
    assert all(np.isfinite(d[k]).all() for k in d), [k for k in d if not np.isfinite(d[k]).all()]
    np.savez_compressed(path, **d)
    print(f"wrote ref_classifier.npz: {len(d)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
