"""Mint tests/golden/ref_res2net.npz: run the reference's OWN ppvector/models/res2net.py (imported unmodified from /root/reference under
tests/paddle_shim, with the helpers of make_ref_fixtures.py) on the oracle's seeded weights and inputs, in fp64, and record what it
computes.  Consumed by tests/test_res2net_cpu.py on any machine; the file holds reference OUTPUTS (and the reference's
configs/res2net.yml as the dictionary it parses to), weights and inputs are re-derived from seeds by the consumer.

Runs only in the authoring container (needs /root/reference).
Usage:  python tests/golden/make_res2net_fixture.py            (rewrites ref_res2net.npz)
        python tests/golden/make_res2net_fixture.py --check    (recomputes and compares with the committed file)
"""
import json
import os
import sys

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_ref_fixtures import REF, paddle, run  # noqa: E402  (sets up the shim and the reference's package path)

from ppvector.models.res2net import Res2Net  # noqa: E402  (the REFERENCE's file)

from oracle import res2net as o_res2net  # noqa: E402

SEED = 5000


def feats(T, B=2):
    """Seeded, time-mean-subtracted features [B,T,80] (make_ref_fixtures.feats with seed 5000 + T)."""
    g = torch.Generator().manual_seed(SEED + T)
    f = torch.randn(B, T, 80, generator=g, dtype=torch.float64)
    return f - f.mean(1, keepdim=True)


def res2net_fixture():
    """Res2Net (res2net.py:90-167) at the settings of the reference's configs/res2net.yml: embeddings and layer taps at T = 98, 298 and
    29 (grids 9 x 9 conv, 13 x 5 pooled, then 7 x 3, 4 x 2 and 2 x 1: odd sizes and a last grid one frame wide), the state_dict shape
    table, the config, and the pooling types the reference cannot run."""
    d = {}
    W = o_res2net.make_res2net_weights(seed=1000, dtype=torch.float64)
    for T in (98, 298, 29):
        emb, taps = run(Res2Net(input_size=80), W, feats(T), ["max_pool", "layer1", "layer2", "layer3", "layer4", "pooling"])
        d[f"res2net_T{T}_emb"] = emb
        for k, v in taps.items():
            d[f"res2net_T{T}_tap_{k}"] = v
    sd = Res2Net(input_size=80).state_dict()
    names = sorted(sd)
    d["res2net_shape_names"] = np.array(names)
    d["res2net_shape_dims"] = np.array([list(sd[k].shape) + [0] * (4 - len(sd[k].shape)) for k in names], dtype=np.int64)
    d["res2net_shape_ndim"] = np.array([len(sd[k].shape) for k in names], dtype=np.int64)
    # the reference's configs/res2net.yml as the dictionary it parses to: build_model and the predictor are driven by it
    with open(os.path.join(REF, "configs", "res2net.yml")) as fh:
        d["res2net_config_json"] = np.array(json.dumps(yaml.load(fh, Loader=yaml.FullLoader), sort_keys=True))
    # SAP / TAP / TSP pool to [N, C, 1], which the head's nn.Linear(cat_channels, ...) then rejects (res2net.py:164-165)
    for pt in ("SAP", "TAP", "TSP"):
        try:
            with torch.no_grad():
                Res2Net(input_size=80, pooling_type=pt).eval()(paddle.to_tensor(feats(40)))
            d[f"res2net_{pt}_raises"] = np.array(0)
        except Exception as e:  # noqa: BLE001
            print(f"reference Res2Net(pooling_type={pt}) raises {type(e).__name__}: {str(e)[:80]}")
            d[f"res2net_{pt}_raises"] = np.array(1)
    return d


def main():
    path = os.path.join(HERE, "ref_res2net.npz")
    d = res2net_fixture()
    if "--check" in sys.argv:
        old = np.load(path)
        assert sorted(old.files) == sorted(d), set(old.files) ^ set(d)
        err = max(float(np.abs(old[k] - d[k]).max()) if d[k].dtype.kind != "U" else float((old[k] != d[k]).any()) for k in d)
        print(f"ref_res2net.npz: {len(d)} arrays, max |committed - recomputed| = {err:.3e}")
        sys.exit(1 if err > 1e-12 else 0)
    np.savez_compressed(path, **d)
    print(f"wrote ref_res2net.npz: {len(d)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
