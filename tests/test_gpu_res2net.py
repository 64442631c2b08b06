"""GPU: Res2Net (csrc/res2net.cu) -- the fused 7x7 / 3 stem + max-pool and the exclusive 3x3 average pool against fp64 on their own
inputs, the whole forward against the fp64 oracle in both precisions, batch / workspace determinism at B = 256, the predictor and
the fused waveform path, and the launch profile.

Bounds: the CUDA-core kernels compute in fp32 and store split-bf16 planes: 2e-5 x max(|ref|, 1), as the conv2d kernel tests.  The
forward: bf16x3 as ResNetSE / ERes2Net (taps 5e-5 relative, 1 - cos of the embeddings 1e-8, cosine scores 1e-4); bf16 as the 2-D
models' bf16 test (1 - cos 2e-5; taps 1e-2 relative).  Run with -s to see the measured errors."""
import ctypes as C
import json
import wave

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import fbank as ofb
from oracle import head as oh
from oracle import res2net as orn
from ppvector import _lib
from ppvector.models.res2net import Res2Net

pytestmark = pytest.mark.gpu
KTOL = 2e-5
TAP_TOL = {"bf16x3": 5e-5, "bf16": 1e-2}
COS_TOL = {"bf16x3": 1e-8, "bf16": 2e-5}


def planes_to_f32(p):
    """split-bf16 planes [2][...] (int16 storage) -> hi + lo in fp64"""
    return p[0].view(torch.bfloat16).double() + p[1].view(torch.bfloat16).double()


# ------------------------------------------------------------------------------------------------ stem + max-pool kernel
def stem_ref(feat, w, bias):
    x = feat.double().transpose(1, 2).unsqueeze(1)
    y = F.relu(F.conv2d(x, w.double().view(32, 1, 7, 7), bias.double(), stride=3, padding=1))
    return F.max_pool2d(y, 3, 2, 1).permute(0, 2, 3, 1)  # [B, Hq, Wq, 32]


# (B, T, F): the default grid; F = 80 and T = 29 put the last conv row / column's 7x7 window on the padding row (3i + 5 = F);
# odd pooled grids; the smallest F and T; the full batch
@pytest.mark.parametrize("B,T,Fd", [(2, 298, 80), (3, 29, 80), (2, 31, 81), (1, 5, 5), (2, 17, 23), (256, 298, 80)])
def test_stem_kernel_against_fp64(cuda, B, T, Fd):
    g = torch.Generator().manual_seed(B * 1000 + T + Fd)
    feat = torch.randn(B, T, Fd, generator=g)
    w = torch.randn(32, 49, generator=g) / 7
    bias = torch.randn(32, generator=g) * 0.1
    H1, W1 = (Fd - 5) // 3 + 1, (T - 5) // 3 + 1
    Hq, Wq = (H1 - 1) // 2 + 1, (W1 - 1) // 2 + 1
    out = torch.full((2, B, Hq + 2, Wq + 2, 32), 0x7f7f, dtype=torch.int16, device=cuda)
    d = [t.to(cuda).contiguous() for t in (feat, w, bias)]
    _lib.check(_lib.load().ppv_res2net_stem_test(*[_lib.ptr(t) for t in d], B, T, Fd, _lib.ptr(out), _lib.current_stream()), "stem")
    got = planes_to_f32(out.cpu())
    assert (got[:, 0] == 0).all() and (got[:, -1] == 0).all() and (got[:, :, 0] == 0).all() and (got[:, :, -1] == 0).all()
    ref = stem_ref(feat, w, bias)
    err = float((got[:, 1:-1, 1:-1] - ref).abs().max()) / max(1.0, float(ref.abs().max()))
    print(f"\nstem B={B} T={T} F={Fd}: grid {Hq} x {Wq}, worst error {err:.2e} x max(|ref|, 1)")
    assert err < KTOL
    assert (ref[:, -1] > 0).any() and (ref[:, :, -1] > 0).any()  # the last row / column is not trivially zero


# ------------------------------------------------------------------------------------------------ exclusive average pool
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("B,H,W,ch,col0,ncols", [(2, 13, 49, 32, 16, 16), (3, 7, 25, 64, 32, 32), (2, 1, 1, 16, 8, 8), (1, 2, 3, 256, 128, 128),
                                                 (4, 4, 13, 128, 64, 64)])
def test_avgpool_against_fp64(cuda, stride, B, H, W, ch, col0, ncols):
    g = torch.Generator().manual_seed(B + 10 * H + 100 * W + stride)
    x = torch.zeros(B, H + 2, W + 2, ch)
    x[:, 1:-1, 1:-1] = torch.randn(B, H, W, ch, generator=g)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    lib = _lib.load()
    ws = torch.empty(lib.ppv_res2net_avgpool_test_workspace_bytes(B, H, W, ch), dtype=torch.uint8, device=cuda)

    def run(xin):
        out = torch.full((2, B, Ho + 2, Wo + 2, ch), 0x7f7f, dtype=torch.int16, device=cuda)
        xd = xin.to(cuda).contiguous()
        _lib.check(lib.ppv_res2net_avgpool_test(_lib.ptr(xd), B, H, W, ch, col0, ncols, stride, _lib.ptr(out), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                _lib.current_stream()), "avgpool")
        return planes_to_f32(out.cpu())

    got = run(x)
    xi = x[:, 1:-1, 1:-1, col0:col0 + ncols].permute(0, 3, 1, 2).double()
    ref = F.avg_pool2d(xi, 3, stride, 1, count_include_pad=False).permute(0, 2, 3, 1)
    err = float((got[:, 1:-1, 1:-1, col0:col0 + ncols] - ref).abs().max()) / max(1.0, float(ref.abs().max()))
    print(f"\navgpool {H} x {W} / {stride} cols [{col0}, {col0 + ncols}): worst error {err:.2e}")
    assert err < KTOL
    rest = got.clone()
    rest[:, 1:-1, 1:-1, col0:col0 + ncols] = 0
    assert (rest == 0).all()  # border and the other columns stay as zeroed
    # divisors: an all-ones image pools to exactly 1 everywhere (4 at a corner, 6 on an edge, 9 inside are all exclusive)
    ones = torch.zeros_like(x)
    ones[:, 1:-1, 1:-1] = 1.0
    assert (run(ones)[:, 1:-1, 1:-1, col0:col0 + ncols] == 1).all()
    if H >= 3 and W >= 3 and stride == 1:  # a corner window is the mean of its 4 in-bounds values, an edge window of its 6
        assert torch.allclose(got[0, 1, 1, col0], xi[0, 0, :2, :2].mean(), atol=1e-5)
        assert torch.allclose(got[0, 1, 2, col0], xi[0, 0, :2, :3].mean(), atol=1e-5)


# ------------------------------------------------------------------------------------------------ whole forward
@pytest.fixture(scope="module")
def W64():
    return orn.make_res2net_weights(seed=1000, dtype=torch.float64)


@pytest.fixture(scope="module")
def models(cuda, W64):
    out = {}
    for p in ("bf16x3", "bf16"):
        m = Res2Net(input_size=80, precision=p).eval()
        m.load_state_dict({k: v.float() for k, v in W64.items()}, strict=True)
        out[p] = m.to(cuda)
    return out


def feats(B, T, seed):
    f = torch.randn(B, T, 80, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    return f - f.mean(1, keepdim=True)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("T", [98, 298, 29])
def test_forward_and_taps_against_oracle(cuda, models, W64, precision, T):
    model = models[precision]
    f = feats(3, T, 5000 + T)
    taps = {}
    ref = orn.res2net_forward(f, W64, taps=taps)
    emb = model(f.float().to(cuda))
    torch.cuda.synchronize()
    for name in ["stem", "layer1", "layer2", "layer3", "layer4", "flat", "asp"]:
        got = model.read_tap(name, 3, T).double().cpu()
        want = taps[name]
        if name == "flat":
            want = want.transpose(1, 2)      # [B, C*H, T'] -> [B, T', C*H]
        elif name != "asp":
            want = want.permute(0, 2, 3, 1)  # NCHW -> NHWC
        assert got.shape == want.shape, (name, got.shape, want.shape)
        rel = float((got - want).norm() / want.norm())
        assert rel < TAP_TOL[precision], (name, rel)
    emb = emb.double().cpu()
    one_minus_cos = float((1 - F.cosine_similarity(emb, ref)).max())
    print(f"\nRes2Net {precision} T={T}: 1 - cos vs oracle {one_minus_cos:.1e}")
    assert one_minus_cos < COS_TOL[precision]
    assert np.abs(oh.cosine_matrix(emb.numpy(), emb.numpy()) - oh.cosine_matrix(ref.numpy(), ref.numpy())).max() < 1e-4


def test_full_batch_is_per_utterance_and_workspace_independent(cuda, models):
    model = models["bf16x3"]
    x = feats(256, 298, 7).float().to(cuda)
    emb = model(x)
    assert torch.isfinite(emb).all()
    for b in (0, 1, 128, 255):
        assert torch.equal(model(x[b:b + 1]), emb[b:b + 1]), b
    assert torch.equal(model(x), emb)  # the B = 256 plan rebuilt on the reused workspace


def test_precisions_differ_on_one_handle(cuda, W64):
    m = Res2Net(input_size=80).eval()
    m.load_state_dict({k: v.float() for k, v in W64.items()})
    m.to(cuda)
    x = feats(2, 98, 3).float().to(cuda)
    a = m(x)
    m.set_precision("bf16")
    b = m(x)
    m.set_precision("bf16x3")
    assert not torch.equal(a, b) and torch.equal(m(x), a)


def test_profile_splits_tensor_core_and_other_time(cuda, models):
    model = models["bf16x3"]
    x = feats(8, 298, 9).float().to(cuda)
    model(x)
    lib, h = _lib.load(), model._get_handle()
    _lib.check(lib.ppv_model_profile(h, 1), "ppv_model_profile")
    model(x)
    g_ms, o_ms, g_n, o_n = C.c_double(), C.c_double(), C.c_int64(), C.c_int64()
    _lib.check(lib.ppv_model_profile_read(h, C.byref(g_ms), C.byref(o_ms), C.byref(g_n), C.byref(o_n)), "ppv_model_profile_read")
    _lib.check(lib.ppv_model_profile(h, 0), "ppv_model_profile")
    assert g_ms.value > 0 and o_ms.value > 0 and g_n.value > 0 and o_n.value > 0


# ------------------------------------------------------------------------------------------------ waveform path and predictor
def test_forward_wav_matches_forward(cuda, models):
    from ppvector.data_utils.featurizer import AudioFeaturizer
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    g = torch.Generator().manual_seed(21)
    wav = (0.1 * torch.randn(3, 16000 * 3, generator=g)).clamp(-1, 1).to(cuda)
    ratio = torch.tensor([1.0, 0.7, 0.45], device=cuda)
    for p, m in models.items():
        assert torch.equal(m.forward_wav(fz, wav), m(fz(wav))), p
        assert torch.equal(m.forward_wav(fz, wav, ratio), m(fz(wav, ratio))), p


def test_predictor_with_res2net_config(cuda, tmp_path, golden_dir, W64):
    from ppvector.predict import PPVectorPredictor
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    paths = {}
    for n in ("a_2", "b_2"):
        paths[n] = str(tmp_path / f"{n}.wav")
        with wave.open(paths[n], "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(16000)
            w.writeframes(g[n + "_pcm"].astype("<i2").tobytes())
    cfg = json.loads(str(np.load(f"{golden_dir}/ref_res2net.npz")["res2net_config_json"]))  # the reference's configs/res2net.yml
    p = PPVectorPredictor(configs=cfg, state_dict={k: v.float().numpy() for k, v in W64.items()})

    def oracle(n):
        x = ofb.db_normalize(g[n + "_pcm"].astype(np.float32) / 32768.0, -20.0)
        return orn.res2net_forward(torch.from_numpy(ofb.audio_featurizer_fbank(x, None, dtype=np.float64, n_mels=80)), W64)[0].numpy()

    emb, ref = p.predict(paths["a_2"]), oracle("a_2")
    cos = float((emb * ref).sum() / np.linalg.norm(emb) / np.linalg.norm(ref))
    assert emb.shape == (192,) and 1 - cos < 1e-6, cos
    e2 = oracle("b_2")
    assert abs(p.contrast(paths["a_2"], paths["b_2"]) - float((ref * e2).sum() / np.linalg.norm(ref) / np.linalg.norm(e2))) < 1e-4
