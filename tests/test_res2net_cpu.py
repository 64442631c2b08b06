"""CPU: Res2Net (reference ppvector/models/res2net.py) -- the fp64 oracle against the reference's own code, the backbone mirror's
state_dict, the settings build_model rejects, and the reference's configs/res2net.yml through build_model.

tests/golden/ref_res2net.npz was written by tests/golden/make_res2net_fixture.py, which runs the reference's res2net.py UNMODIFIED under
tests/paddle_shim (MaxPool2D pads with -inf; AvgPool2D is exclusive: each window divided by its in-bounds count).  T = 29 gives odd
grids and a last grid one frame wide."""

import numpy as np
import pytest
import torch

from oracle import res2net as orn

TOL = 1e-10


def feats(T, B=2):
    """make_res2net_fixture.feats(T)"""
    g = torch.Generator().manual_seed(5000 + T)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    return f - f.mean(1, keepdim=True)


def tap_slice(t):
    t = t.detach()
    idx = tuple(slice(0, min(n, 6)) for n in t.shape)
    return np.concatenate([t[idx].reshape(-1).numpy(), [float(t.abs().mean()), float(t.sum())]])


def close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() / max(1.0, np.abs(b).max())
    assert err <= tol, err


@pytest.fixture(scope="module")
def ref(golden_dir):
    return np.load(f"{golden_dir}/ref_res2net.npz")


def build(model_args):
    from ppvector.models import build_model
    from ppvector.utils.utils import dict_to_object
    return build_model(input_size=model_args.pop("input_size", 80),
                       configs=dict_to_object({"model_conf": {"model": "Res2Net", "model_args": model_args}}))


@pytest.mark.parametrize("T", [98, 298, 29])
def test_oracle_matches_reference_code(ref, T):
    W = orn.make_res2net_weights(seed=1000, dtype=torch.float64)
    taps = {}
    emb = orn.res2net_forward(feats(T), W, taps=taps)
    close(emb.numpy(), ref[f"res2net_T{T}_emb"])
    for mine, theirs in [("stem", "max_pool"), ("layer1", "layer1"), ("layer2", "layer2"), ("layer3", "layer3"), ("layer4", "layer4"),
                         ("asp", "pooling")]:
        close(tap_slice(taps[mine]), ref[f"res2net_T{T}_tap_{theirs}"])


def test_mirror_state_dict_matches_reference(ref):
    m = build({"embd_dim": 192, "pooling_type": "ASP", "m_channels": 32})
    sd = m.state_dict()
    names = [str(n) for n in ref["res2net_shape_names"]]
    assert sorted(sd) == names
    for n, dims, nd in zip(names, ref["res2net_shape_dims"], ref["res2net_shape_ndim"]):
        assert tuple(sd[n].shape) == tuple(int(d) for d in dims[:nd]), n
    assert sd["layer2.0.convs.0.weight"].shape == (32, 32, 3, 3) and sd["linear.weight"].shape == (4096, 192)
    assert "layer2.0.downsample.1._mean" in sd and "pooling.tdnn.conv.conv.weight" in sd and "bn2.norm.weight" in sd
    W = orn.make_res2net_weights(seed=1000, dtype=torch.float64)
    assert {k: tuple(v.shape) for k, v in W.items()} == {k: tuple(v.shape) for k, v in sd.items()}


def test_parameter_count():
    """5 624 176 parameters without the classifier (running statistics excluded), 5.10 M without the ASP's global-context columns
    (2 x 2048 x 128): the README's 5.0 M counts the head without them, as it does for ResNetSE (SURVEY.md §6)."""
    m = build({"embd_dim": 192})
    n = sum(p.numel() for p in m.parameters())
    assert n == orn.count_params(orn.make_res2net_weights(seed=0)) == 5624176
    print(f"\nRes2Net backbone parameters: {n} ({n / 1e6:.2f} M; README.md: 5.0 M)")
    assert abs((n - 2 * 2048 * 128) / 1e6 - 5.0) < 0.15


@pytest.mark.parametrize("pooling_type", ["SAP", "TAP", "TSP"])
def test_pooling_types_the_reference_cannot_run_are_refused(ref, pooling_type):
    assert int(ref[f"res2net_{pooling_type}_raises"]) == 1  # the reference raises on them (nn.Linear sees [N, C, 1])
    with pytest.raises(NotImplementedError, match=f"{pooling_type}.*reference Res2Net cannot run it"):
        build({"pooling_type": pooling_type})


def test_unsupported_settings_are_refused():
    with pytest.raises(NotImplementedError, match="scale 4"):
        build({"scale": 4})
    with pytest.raises(NotImplementedError, match="input_size 96 leaves a final grid of 2 rows.*= 3"):
        build({"input_size": 96})
    with pytest.raises(NotImplementedError, match="input_size 3"):
        build({"input_size": 3})
    build({"input_size": 80, "base_width": 32})  # the shipped setting builds


def test_reference_config_builds_res2net(ref):
    """The reference's configs/res2net.yml (recorded as the dictionary it parses to) drives build_model to this Res2Net; TDNN, the other
    reference-only backbone, still raises by name."""
    import json

    from ppvector.models import Res2Net, build_model
    from ppvector.utils.utils import dict_to_object
    cfg = json.loads(str(ref["res2net_config_json"]))
    assert cfg["model_conf"]["model"] == "Res2Net" and cfg["model_conf"]["model_args"] == {"embd_dim": 192, "pooling_type": "ASP", "m_channels": 32}
    assert cfg["preprocess_conf"] == {"feature_method": "Fbank", "method_args": {"sr": 16000, "n_mels": 80}}
    m = build_model(input_size=cfg["preprocess_conf"]["method_args"]["n_mels"], configs=dict_to_object(cfg))
    assert isinstance(m, Res2Net) and sum(p.numel() for p in m.parameters()) == 5624176
    with pytest.raises(NotImplementedError, match="TDNN is not implemented on the H100 path"):
        build_model(input_size=80, configs=dict_to_object({"model_conf": {"model": "TDNN", "model_args": {}}}))
