"""GPU: ResNetSE forward (conv2d as wgmma gather-GEMMs over zero-bordered NHWC images) vs the fp64 oracle and golden
embeddings; SURVEY.md §8 row a6.  Tolerance: cosine scores within 1e-4 of the reference path."""
import numpy as np
import pytest
import torch

from oracle import head as oh
from oracle import resnet_se as orr
from ppvector.models.resnet_se import ResNetSE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def W64():
    return orr.make_resnet_se_weights(seed=1000, dtype=torch.float64)


@pytest.fixture(scope="module")
def model(cuda, W64):
    m = ResNetSE(input_size=80).eval()
    m.load_state_dict({k: v.float() for k, v in W64.items()}, strict=True)
    return m.to(cuda)


def test_param_count_and_names(W64):
    assert orr.count_params(W64) == 9132440  # SURVEY.md §6: 9.13 M with the ASP global-context head
    m = ResNetSE(input_size=80)
    assert sorted(m.state_dict().keys()) == sorted(W64.keys())


@pytest.mark.parametrize("T", [64, 149])
def test_stagewise_taps_and_embedding(cuda, model, W64, golden_dir, T):
    g = np.load(f"{golden_dir}/resnetse_seed1000.npz")
    gi = torch.Generator().manual_seed(2000 + T)
    f = torch.randn(2, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    taps = {}
    ref = orr.resnet_se_forward(f, W64, taps=taps)
    emb = model(f.float().to(cuda))
    torch.cuda.synchronize()
    for name in ["conv1", "layer1", "layer2", "layer3", "layer4", "flat", "asp"]:
        got = model.read_tap(name, 2, T).double().cpu()
        want = taps[name]
        if name.startswith("layer") or name == "conv1":
            want = want.permute(0, 2, 3, 1)  # oracle NCHW -> NHWC
        elif name == "flat":
            want = want.transpose(1, 2)      # oracle [B, C*H, T'] -> [B, T', C*H]
        assert got.shape == want.shape, (name, got.shape, want.shape)
        rel = (got - want).norm() / want.norm()
        assert rel < 3e-5, (name, rel.item())
    emb = emb.double().cpu()
    assert np.abs(emb.numpy() - g[f"emb_T{T}"]).max() < 5e-5
    cos = torch.nn.functional.cosine_similarity(emb, ref)
    assert (1 - cos).max() < 1e-8
    assert np.abs(oh.cosine_matrix(emb.numpy(), emb.numpy()) - oh.cosine_matrix(ref.numpy(), ref.numpy())).max() < 1e-4


@pytest.mark.parametrize("B,T", [(1, 8), (3, 33), (4, 298)])
def test_shapes(cuda, model, W64, B, T):
    gi = torch.Generator().manual_seed(B * 100 + T)
    f = torch.randn(B, T, 80, generator=gi)
    ref = orr.resnet_se_forward(f[:2].double(), W64)
    emb = model(f.to(cuda)).double().cpu()
    assert emb.shape == (B, 192)
    rel = (emb[:2][: ref.shape[0]] - ref).norm(dim=1) / ref.norm(dim=1)
    assert rel.max() < 1e-4, rel  # 50 stacked convolutions at ~2^-17 per product; T=8 leaves one pooled frame


def test_batch_independence(cuda, model):
    gi = torch.Generator().manual_seed(11)
    f = torch.randn(16, 298, 80, generator=gi).to(cuda)
    emb = model(f)
    assert torch.isfinite(emb).all()
    for b in (0, 7, 15):
        assert torch.equal(model(f[b:b + 1]), emb[b:b + 1])


def test_plans_no_pointwise_step(cuda, model):
    """ResNetSE runs every 1x1 conv on the wgmma gather-GEMM: its plan has no pointwise step (pointwise.cu), so PPV_POINTWISE does not
    apply to it.  The profiler's kernel names show which kernels a forward ran."""
    from torch.profiler import ProfilerActivity, profile
    f = torch.randn(3, 149, 80, generator=torch.Generator().manual_seed(77)).to(cuda)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(f)
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    assert any("gemm_wgmma_kernel" in n for n in names) and any("conv3x3_c32_kernel" in n for n in names), names
    assert not any("pw_conv_kernel" in n for n in names), names
