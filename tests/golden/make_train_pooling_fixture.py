"""Mint tests/golden/ref_train_pooling.npz: one TRAIN-mode step of the reference's OWN EcapaTdnn, SpeakerIdentification and AAMLoss
(imported unmodified from /root/reference under tests/paddle_shim, with the helpers of make_ref_fixtures.py) for each pooling head the
reference builds besides ASP with global context (ecapa_tdnn.py:212-241): ASP without global context, SAP, TAP and TSP.  Forward with
batch statistics, classifier, AAMLoss, backward through torch autograd, in fp64 (trainer.py:206-229).  Consumed by
tests/test_train_pooling_cpu.py on any machine; the file holds reference OUTPUTS only (loss, logits, the gradients of the head's own
parameters, of mfa and of the classifier, and the updated running statistics); weights and inputs are re-derived from seeds by the
consumer.

Runs only in the authoring container (needs /root/reference).
Usage:  python tests/golden/make_train_pooling_fixture.py            (rewrites ref_train_pooling.npz)
        python tests/golden/make_train_pooling_fixture.py --check    (recomputes and compares with the committed file)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_ref_fixtures import paddle, tap_slice  # noqa: E402  (sets up the shim and the reference's package path)

from ppvector.loss.aamloss import AAMLoss  # noqa: E402  (the REFERENCE's files)
from ppvector.models.ecapa_tdnn import EcapaTdnn  # noqa: E402
from ppvector.models.fc import SpeakerIdentification  # noqa: E402

from oracle import ecapa as o_ecapa  # noqa: E402

# tag -> (pooling_type, global_context)
HEADS = {"ASP_noctx": ("ASP", False), "SAP": ("SAP", True), "TAP": ("TAP", True), "TSP": ("TSP", True)}
B, T, S, SEED = 4, 61, 37, 78


def problem():
    """Seeded, time-mean-subtracted features [B,T,80], labels and classifier weight (the recipe of make_ref_fixtures.train_fixture)."""
    g = torch.Generator().manual_seed(SEED)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    labels = torch.randint(0, S, (B,), generator=g)
    Wc = (torch.rand(192, S, generator=g, dtype=torch.float64) * 2 - 1) * (6.0 / (192 + S)) ** 0.5
    return f, labels, Wc


def forward(model, x, pooling_type):
    """EcapaTdnn.forward (ecapa_tdnn.py:245-276) on the reference's own layers.  With SAP / TAP / TSP the reference's forward un-squeezes
    the pooled [N, C, 1] once more (ecapa_tdnn.py:272) and hands fc a 4-D tensor, which raises (make_ref_fixtures.models_fixture records
    it); here the pooled vector goes through asp_bn and fc as [N, C, 1], the one shape both accept."""
    if pooling_type == "ASP":
        return model(x)
    x = x.transpose([0, 2, 1])
    xl = []
    for layer in model.blocks:
        x = layer(x)
        xl.append(x)
    x = model.mfa(paddle.concat(xl[1:], axis=1))
    return model.fc(model.asp_bn(model.asp(x))).squeeze(-1)


def head_names(W):
    """The tensors of the pooling head, asp_bn, fc and mfa."""
    return [k for k in W if k.startswith(("mfa.", "asp.", "asp_bn.", "fc."))]


def train_pooling_fixture():
    d = {}
    f, labels, Wc = problem()
    for tag, (pt, gc) in HEADS.items():
        W = o_ecapa.make_ecapa_weights(seed=1000, dtype=torch.float64, pooling_type=pt, global_context=gc)
        model = EcapaTdnn(input_size=80, pooling_type=pt, global_context=gc)
        model.set_state_dict(W)
        clf = SpeakerIdentification(input_dim=192, num_speakers=S)
        clf.set_state_dict({"weight": Wc})
        model.train()
        out = clf(forward(model, paddle.to_tensor(f), pt))
        loss = AAMLoss(margin=0.2, scale=32, label_smoothing=0.0)(out, paddle.to_tensor(labels))
        loss.backward()
        d[f"{tag}_loss"] = np.array(float(loss))
        d[f"{tag}_logits"] = out["logits"].numpy()
        params, sd = dict(model.named_parameters()), model.state_dict()
        for k in head_names(W):
            if k.endswith(("._mean", "._variance")):
                d[f"{tag}_stat_{k}"] = sd[k].numpy().copy()
                continue
            gr = params[k].grad
            # vectors whole; matrices as a slice plus their norm (keeps the file small)
            d[f"{tag}_grad_{k}"] = gr.numpy().copy() if gr.dim() == 1 else tap_slice(gr)
            d[f"{tag}_gradnorm_{k}"] = np.array(float(gr.norm()))
        d[f"{tag}_grad_classifier.weight"] = clf.weight.grad.numpy().copy()
    return d


def main():
    path = os.path.join(HERE, "ref_train_pooling.npz")
    d = train_pooling_fixture()
    if "--check" in sys.argv:
        old = np.load(path)
        assert sorted(old.files) == sorted(d), set(old.files) ^ set(d)
        err = max(float(np.abs(old[k] - d[k]).max()) for k in d)
        print(f"ref_train_pooling.npz: {len(d)} arrays, max |committed - recomputed| = {err:.3e}")
        sys.exit(1 if err > 1e-12 else 0)
    np.savez_compressed(path, **d)
    print(f"wrote ref_train_pooling.npz: {len(d)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
