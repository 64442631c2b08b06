"""GPU: the ECAPA-TDNN training step's plan bookkeeping -- the workspace size query, the tap table and its errors.

Asking for a workspace size must not disturb the plan of the last step: the taps stay readable and unchanged.  Every tap named in
the comment above ``trainer_read_tap`` (csrc/ecapa_train.cu) reads at its documented shape, misuse fails with the documented
status, and ``ppv_trainer_workspace_bytes`` returns the sizes recorded for the default configuration."""
import ctypes as C

import pytest
import torch

from oracle import ecapa as oe
from ppvector import _lib
from ppvector.train_engine import TrainEngine

pytestmark = pytest.mark.gpu

S = 37
PPV_EINVAL, PPV_ESTATE = -1, -4
P = 4  # reflect padding of the default config: max((5 - 1) / 2 * 1, dilations 2, 3, 4)
C1, C3, ATT, SE, D, F = 512, 1536, 128, 128, 192, 80

# (cols, per block) of every planes tap: fp32 [B, T, cols], or [B, T + 2P, cols] with "pad:"
PLANES = {"blocks.0": (C1, False), "blocks.1": (C1, False), "blocks.2": (C1, False), "blocks.3": (C1, False), "mfa": (C3, False),
          "X0": (F, False), "A0": (C1, False), "Y0": (C1, False), "OUTCAT": (C3, False), "Amfa": (C3, False), "M": (C3, False),
          "Aatt": (ATT, False), "A4": (ATT, False),
          **{n: (C1, True) for n in ("At1", "Yt1", "Ares", "RC", "IN", "At2", "Yt2")},
          "g:dZ0": (C1, False), "g:dOUTCAT": (C3, False), "g:dMd": (C3, False), "g:dMatt": (C3, False), "g:dZmfa": (C3, False),
          "g:dlogits": (C3, False), "g:dZatt": (ATT, False), "g:dA4": (ATT, False),
          **{"g:" + n: (C1, True) for n in ("D", "dZt2", "dRC", "dZres", "DIN", "dZt1", "dXt1")}}


def vec_taps(B, T):
    """(shape, per block) of every fp32 tap, read as stored."""
    Tp = T + 2 * P
    return {"asp": ((B, 2 * C3), False), "emb": ((B, D), False), "d_emb": ((B, D), False), "logits": ((B, Tp, C3), False),
            **{n: ((B, 2 * C3), False) for n in ("gstat", "dgs", "pn", "dpn", "dpooled")},
            "rs": ((B, C3), False), "rb": ((B, C3), False), "dg2": ((B, C1), False), "ds": ((B, C1), False), "dg1": ((B, SE), False),
            "se_s": ((B, C1), True), "se_g2": ((B, C1), True), "se_g1": ((B, SE), True)}


def stepped_engine(cuda, B, T, seed=7):
    eng = TrainEngine(input_size=F, num_speakers=S, device=cuda)
    g = torch.Generator().manual_seed(seed)
    eng.load_state_dict(oe.make_ecapa_weights(seed=1000, dtype=torch.float64),
                        (torch.rand(D, S, generator=g, dtype=torch.float64) * 2 - 1) * 0.15)
    f = torch.randn(B, T, F, generator=g)
    y = torch.randint(0, S, (B,), generator=g)
    eng.forward_backward(f.to(cuda), y.to(cuda))
    torch.cuda.synchronize()
    return eng


def read_status(eng, name, numel):
    """Status of ppv_trainer_read_tap into a buffer of `numel` floats."""
    out = torch.zeros(max(numel, 1), dtype=torch.float32, device=eng.device)
    rc = _lib.load().ppv_trainer_read_tap(eng._h, name.encode(), _lib.ptr(out), numel, _lib.current_stream())
    torch.cuda.synchronize()
    return rc


def test_size_query_leaves_the_plan_alone(cuda):
    B, T = 4, 40
    eng = stepped_engine(cuda, B, T)
    taps = {"emb": (B, D), "blocks.2": (B, T, C1), "pad:Yt1:1": (B, T + 2 * P, C1), "g:dZt2:2": (B, T, C1)}
    before = {n: eng.read_tap(n, s).cpu() for n, s in taps.items()}
    lib = _lib.load()
    assert lib.ppv_trainer_workspace_bytes(eng._h, 8, 100) > lib.ppv_trainer_workspace_bytes(eng._h, B, T) > 0
    for n, s in taps.items():
        assert torch.equal(eng.read_tap(n, s).cpu(), before[n]), n


def test_every_documented_tap_reads_at_its_shape(cuda):
    B, T = 3, 35
    Tp = T + 2 * P
    eng = stepped_engine(cuda, B, T)
    for name, (cols, per_block) in PLANES.items():
        for suffix in ([":0", ":1", ":2", ""] if per_block else [""]):
            n = name + suffix
            valid = eng.read_tap(n, (B, T, cols))
            padded = eng.read_tap("pad:" + n, (B, Tp, cols))
            assert torch.isfinite(padded).all(), n
            assert torch.equal(padded[:, P:P + T], valid), n
            assert read_status(eng, n, B * T * cols - 1) == PPV_EINVAL, n
            assert read_status(eng, "pad:" + n, B * Tp * cols - 1) == PPV_EINVAL, n
        if per_block:
            assert torch.equal(eng.read_tap(name, (B, T, cols)), eng.read_tap(name + ":0", (B, T, cols))), name
    for name, (shape, per_block) in vec_taps(B, T).items():
        numel = 1
        for s in shape:
            numel *= s
        for suffix in ([":0", ":1", ":2", ""] if per_block else [""]):
            got = eng.read_tap(name + suffix, shape)
            assert torch.isfinite(got).all(), name + suffix
            assert read_status(eng, name + suffix, numel - 1) == PPV_EINVAL, name + suffix
    # the block outputs are windows of OUTCAT; mfa is M
    outcat = eng.read_tap("OUTCAT", (B, T, C3))
    for b in (1, 2, 3):
        assert torch.equal(eng.read_tap(f"blocks.{b}", (B, T, C1)), outcat[..., C1 * (b - 1):C1 * b])
    assert torch.equal(eng.read_tap("mfa", (B, T, C3)), eng.read_tap("M", (B, T, C3)))
    assert torch.equal(eng.read_tap("blocks.0", (B, T, C1)), eng.read_tap("Y0", (B, T, C1)))


def test_bad_tap_names_fail_the_same_way(cuda):
    B, T = 2, 20
    eng = TrainEngine(input_size=F, num_speakers=S, device=cuda)
    assert read_status(eng, "emb", B * D) == PPV_ESTATE
    assert read_status(eng, "no_such_tap", B * D) == PPV_ESTATE
    eng = stepped_engine(cuda, B, T)
    big = B * (T + 2 * P) * C3
    for name in ["no_such_tap", "g:no_such_tap", "g:Y0", "dZ0", "blocks.4", "emb:1", "asp:0", "blocks.1:1", "M:0", "g:dZ0:0",
                 "pad:emb", "pad:logits", "pad:se_s:1", "pad:no_such_tap"]:
        assert read_status(eng, name, big) == PPV_EINVAL, name
    for name in ["Yt1:3", "g:D:5", "se_s:9", "pad:RC:3"]:
        assert read_status(eng, name, big) == PPV_EINVAL, name
    assert read_status(eng, "Yt1:2", big) == 0


# ppv_trainer_workspace_bytes of the default config with 37 classes on a 132-SM H100 (the weight-gradient split-K partials and the
# BatchNorm-backward frame splits scale with the SM count), recorded before the plan was moved onto the shared workspace helpers, less
# the 256 bytes of trailing slack the AAM block (the last buffer) stopped reserving when its size came from the AAM call's own carve.
WS_BYTES = {(2, 9): 87461888, (2, 298): 170561536, (3, 35): 108344832, (4, 40): 108453376, (8, 100): 212810240, (64, 9): 261409280,
            (64, 40): 573032960, (64, 298): 3252996608}


def test_workspace_sizes_are_unchanged(cuda):
    if torch.cuda.get_device_properties(cuda).multi_processor_count != 132:
        pytest.skip("sizes recorded on a 132-SM H100")
    eng = TrainEngine(input_size=F, num_speakers=S, device=cuda)
    lib = _lib.load()
    got = {bt: lib.ppv_trainer_workspace_bytes(eng._h, *bt) for bt in WS_BYTES}
    assert got == WS_BYTES
