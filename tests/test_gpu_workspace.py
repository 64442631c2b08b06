"""GPU: every call that takes a caller-owned workspace, run three ways on one small seeded case.
  - In a buffer of exactly the size its query returns, followed by a 4 KB sentinel tail: the tail is untouched and the outputs are
    bitwise those of a run in a generous workspace.
  - With one byte less than the query returns: PPV_EINVAL, and no output is written.
  - With the workspace 16 bytes past a 256-byte boundary: PPV_EINVAL, and no output is written.
Both rejections come from the host before any launch."""
import ctypes as C

import numpy as np
import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu

EINVAL = -1
FILL, TAIL = 0xA7, 0x5A
V = C.c_void_p


def out(shape, dtype):
    """an output buffer with every byte FILL"""
    t = torch.empty(shape, dtype=dtype, device="cuda")
    t.view(torch.uint8).fill_(FILL)
    return t


def randn(*shape, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64).to(dtype).cuda()


def stream():
    return _lib.current_stream()


# Each case returns (need, run), run(ws address, ws_bytes) -> (status, outputs).  run makes fresh outputs, every byte FILL (and a fresh
# copy of an input the call overwrites), on every call.
def case_aam():
    lib = _lib.load()
    B, D, S = 5, 80, 300
    emb, W = randn(B, D, seed=1), randn(D, S, seed=2)
    labels = torch.tensor([3, 0, 299, 17, 3], dtype=torch.int64, device="cuda")

    def run(ws, nb):
        logits, loss, d_emb, d_W = out((B, S), torch.float32), out((1,), torch.float32), out((B, D), torch.float32), out((D, S), torch.float32)
        rc = lib.ppv_aam_forward(_lib.ptr(emb), _lib.ptr(W), _lib.ptr(labels), B, D, S, 0.2, 32.0, 0, 0.1, _lib.ptr(logits), _lib.ptr(loss),
                                 V(ws), nb, stream())
        if rc == 0:  # the backward reads what the forward left in the same workspace
            rc = lib.ppv_aam_backward(_lib.ptr(emb), _lib.ptr(W), _lib.ptr(labels), _lib.ptr(logits), B, D, S, 0.2, 32.0, 0, 0.1,
                                      _lib.ptr(d_emb), _lib.ptr(d_W), V(ws), nb, stream())
        return rc, [logits, loss, d_emb, d_W]
    return lib.ppv_aam_workspace_bytes(B, D, S), run


def case_cosine():
    lib = _lib.load()
    M, N, D = 7, 130, 192
    A, Bm = randn(M, D, seed=3), randn(N, D, seed=4)

    def run(ws, nb):
        o = out((M, N), torch.float32)
        return lib.ppv_cosine_matrix(_lib.ptr(A), _lib.ptr(Bm), M, N, D, _lib.ptr(o), V(ws), nb, stream()), [o]
    return lib.ppv_cosine_workspace_bytes(M, N, D), run


def case_eer():
    lib = _lib.load()
    n = 5000
    s = randn(n, seed=5)
    lab = (randn(n, seed=6) > 1.0).to(torch.int32)
    s = s + lab.float()

    def run(ws, nb):
        o = out((4,), torch.float64)
        return lib.ppv_eer_mindcf(_lib.ptr(s), _lib.ptr(lab), n, 0.01, 1.0, 1.0, _lib.ptr(o), V(ws), nb, stream()), [o]
    return lib.ppv_eer_workspace_bytes(n), run


def laplacian(N, seed):
    X = randn(N, N, seed=seed, dtype=torch.float64)
    A = (X @ X.T).abs()
    return torch.diag(A.sum(1)) - A


def case_sym_eig():
    lib = _lib.load()
    N, m = 37, 5
    L0 = laplacian(N, 7)

    def run(ws, nb):
        L = L0.clone()
        ev, evec = out((m,), torch.float64), out((N, m), torch.float64)
        return lib.ppv_sym_eig_smallest(_lib.ptr(L), N, m, _lib.ptr(ev), _lib.ptr(evec), V(ws), nb, stream()), [ev, evec]
    return lib.ppv_sym_eig_workspace_bytes(N, m), run


def case_kmeans():
    lib = _lib.load()
    N, k, ld = 50, 3, 4
    X = randn(N, ld, seed=8, dtype=torch.float64)
    n_u = 1 + (k - 1) * (2 + int(np.log(k)))
    u = torch.rand(n_u, generator=torch.Generator().manual_seed(9), dtype=torch.float64).cuda()

    def run(ws, nb):
        labels, inertia = out((N,), torch.int32), out((1,), torch.float64)
        return lib.ppv_kmeans(_lib.ptr(X), ld, N, k, _lib.ptr(u), n_u, 30, _lib.ptr(labels), _lib.ptr(inertia), V(ws), nb, stream()), [labels, inertia]
    return lib.ppv_kmeans_workspace_bytes(N, k), run


def case_vad():
    lib = _lib.load()
    cfg = _lib.VadCfg()
    lib.ppv_vad_default_cfg(C.byref(cfg), 16000)
    lens = [16000, 400, 23456]
    g = np.random.default_rng(10)
    x = np.concatenate([g.standard_normal(n) * (0.3 if i % 2 else 0.01) for i, n in enumerate(lens)]).astype(np.float32)
    wav = torch.from_numpy(x).cuda()
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    T = sum(lib.ppv_vad_num_frames(C.byref(cfg), n) for n in lens)
    cap = sum((lib.ppv_vad_num_frames(C.byref(cfg), n) + 1) // 2 for n in lens)

    def run(ws, nb):
        energy, voiced, runs, n_runs = out((T,), torch.float64), out((T,), torch.uint8), out((cap, 3), torch.int32), out((1,), torch.int32)
        rc = lib.ppv_vad_energy(C.byref(cfg), _lib.ptr(wav), off.ctypes.data_as(C.POINTER(C.c_int64)), len(lens), _lib.ptr(energy),
                                _lib.ptr(voiced), _lib.ptr(runs), cap, _lib.ptr(n_runs), V(ws), nb, stream())
        return rc, [energy, voiced, runs, n_runs]
    return lib.ppv_vad_workspace_bytes(C.byref(cfg), len(lens), int(off[-1])), run


def prep_batch(B, raw):
    """B items of raw samples with crops and noise on every other item; speed 1 (new_len = raw)"""
    wav = randn(B, raw, seed=11) * 0.1
    noise = randn(5000, seed=12) * 0.05
    ip = np.zeros((B, _lib.PPV_PREP_NI), dtype=np.int32)
    fp = np.zeros((B, _lib.PPV_PREP_NF), dtype=np.float32)
    for b in range(B):
        n = raw - 37 * b
        ip[b, :4] = (n, n, 11 * b, n - 11 * b - 5)
        if b % 2:
            ip[b, 4:7] = (100 * b, 3000, 1)
        fp[b] = (1.0, 0.5 * b - 1.0, 5.0 + b, 0.0)
    return wav, noise, torch.from_numpy(ip).cuda(), torch.from_numpy(fp).cuda()


def case_audio_prep():
    lib = _lib.load()
    B, raw = 4, 20000
    wav, noise, ip, fp = prep_batch(B, raw)

    def run(ws, nb):
        o = out((B, raw), torch.float32)
        return lib.ppv_audio_prep(_lib.ptr(wav), raw, _lib.ptr(ip), _lib.ptr(fp), _lib.ptr(noise), B, raw, -20.0, 1, raw, _lib.ptr(o),
                                  V(ws), nb, stream()), [o]
    return lib.ppv_audio_prep_workspace_bytes(B, raw), run


def case_audio_prep_reverb():
    """items with and without a room response in one batch"""
    lib = _lib.load()
    B, raw, rmax = 4, 20000, 3000
    wav, noise, ip, fp = prep_batch(B, raw)
    rir = randn(8000, seed=13) * 0.2
    rp = torch.tensor([[0, 3000], [0, 0], [2500, 1234], [0, 0]], dtype=torch.int32, device="cuda")
    Lout = raw + rmax

    def run(ws, nb):
        o = out((B, Lout), torch.float32)
        return lib.ppv_audio_prep_reverb(_lib.ptr(wav), raw, _lib.ptr(ip), _lib.ptr(fp), _lib.ptr(noise), _lib.ptr(rir), rir.numel(),
                                         _lib.ptr(rp), B, raw, rmax, -20.0, 1, Lout, _lib.ptr(o), V(ws), nb, stream()), [o]
    return lib.ppv_audio_prep_reverb_workspace_bytes(B, raw, rmax), run


def case_speaker_index_search(k):
    lib = _lib.load()
    n, U, D, Q = 300, 100, 192, 70
    E = randn(n, D, seed=14)
    owner = torch.arange(n, device="cuda") % U
    order = torch.argsort(owner, stable=True).to(torch.int32)
    offsets = torch.arange(0, n + 1, n // U, dtype=torch.int32, device="cuda")
    means = torch.empty((U, D), device="cuda")
    ib = lib.ppv_speaker_index_bytes(U, D)
    index = torch.empty(ib, dtype=torch.uint8, device="cuda")
    _lib.check(lib.ppv_speaker_index_build(_lib.ptr(E), n, D, _lib.ptr(order), _lib.ptr(offsets), U, _lib.ptr(means), _lib.ptr(index), ib,
                                           stream()), "ppv_speaker_index_build")
    q = randn(Q, D, seed=15)

    def run(ws, nb):
        idx, sim = out((Q, k), torch.int32), out((Q, k), torch.float32)
        return lib.ppv_speaker_index_search(_lib.ptr(q), Q, D, _lib.ptr(index), ib, U, k, _lib.ptr(idx), _lib.ptr(sim), V(ws), nb,
                                            stream()), [idx, sim]
    return lib.ppv_speaker_index_search_workspace_bytes(Q, U, D, k), run


def case_gemm_test():
    lib = _lib.load()
    M, N, K = 130, 200, 192
    A, W, bias = randn(M, K, seed=16), randn(N, K, seed=17), randn(N, seed=18)

    def run(ws, nb):
        o = out((M, N), torch.float32)
        return lib.ppv_gemm_test(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), None, None, 1, M, N, K, 128, 64, _lib.PPV_PREC_BF16X3,
                                 _lib.ptr(o), V(ws), nb, stream()), [o]
    return lib.ppv_gemm_test_workspace_bytes(M, N, K), run


def case_gemm_test_planes():
    lib = _lib.load()
    Tp, P, M, N, K = 40, 2, 120, 64, 64
    A, W, bias = randn(M, K, seed=19), randn(N, K, seed=20), randn(N, seed=21)

    def run(ws, nb):
        o = out((2, M, N), torch.bfloat16)
        return lib.ppv_gemm_test_planes(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), None, None, None, 1, 0, Tp, P, M, N, K, 64,
                                        _lib.PPV_PREC_BF16X3, _lib.ptr(o), V(ws), nb, stream()), [o]
    return lib.ppv_gemm_test_workspace_bytes(M, N, K), run


def case_conv2d_test():
    lib = _lib.load()
    B, H, W, Cin, Cout, k = 2, 9, 13, 32, 32, 3
    x, w, bias = randn(B, H, W, Cin, seed=22), randn(Cout, Cin, k, k, seed=23) * 0.1, randn(Cout, seed=24)
    plane = B * (H + 2) * (W + 2) * Cout

    def run(ws, nb):
        o = out((2 * plane,), torch.int16)
        return lib.ppv_conv2d_test(_lib.ptr(x), _lib.ptr(w), _lib.ptr(bias), 1, B, H, W, Cin, Cout, k, 1, 1, 0, 0, 2,
                                   _lib.PPV_PREC_BF16X3, _lib.ptr(o), V(ws), nb, stream()), [o]
    return lib.ppv_conv2d_test_workspace_bytes(B, H, W, Cin, Cout, k, 0), run


def case_asp_fused_test():
    lib = _lib.load()
    B, T, P, Cc, K = 2, 50, 3, 128, 64
    Tp = T + 2 * P
    W, att, x = randn(Cc, K, seed=25) * 0.1, randn(B * Tp, K, seed=26), randn(B * Tp, Cc, seed=27)
    scale, shift = randn(2 * Cc, seed=28), randn(2 * Cc, seed=29)

    def run(ws, nb):
        raw, o = out((B, 2 * Cc), torch.float32), out((B, 2 * Cc), torch.float32)
        return lib.ppv_asp_fused_test(_lib.ptr(W), _lib.ptr(att), _lib.ptr(x), _lib.ptr(scale), _lib.ptr(shift), None, B, T, P, Tp, Cc, K,
                                      _lib.PPV_PREC_BF16X3, 0, _lib.ptr(raw), _lib.ptr(o), V(ws), nb, stream()), [raw, o]
    return lib.ppv_asp_fused_test_workspace_bytes(B, Tp, Cc, K), run


def case_colstats_test():
    lib = _lib.load()
    B, T, P, ld, col0, Cc = 3, 41, 2, 200, 64, 128
    Tp = T + 2 * P
    x = randn(B * Tp, ld, seed=30)

    def run(ws, nb):
        o = out((B, 2 * Cc), torch.float32)
        return lib.ppv_colstats_test(_lib.ptr(x), B, T, P, Tp, ld, col0, Cc, 1, 1e-5, 0.0, None, _lib.ptr(o), None, V(ws), nb,
                                     stream()), [o]
    return lib.ppv_colstats_test_workspace_bytes(B, Tp, ld, Cc), run


def case_campplus_context_test():
    lib = _lib.load()
    B, T, P = 2, 130, 1
    Tp = T + 2 * P
    h = randn(B * Tp, 128, seed=31)
    w1, b1, w2, b2 = randn(64, 128, seed=32) * 0.1, randn(64, seed=33), randn(32, 64, seed=34) * 0.1, randn(32, seed=35)
    nseg = (T + 99) // 100

    def run(ws, nb):
        o = out((B * nseg, 32), torch.float32)
        return lib.ppv_campplus_context_test(_lib.ptr(h), B, T, P, Tp, _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), _lib.ptr(b2), _lib.ptr(o),
                                             V(ws), nb, stream()), [o]
    return lib.ppv_campplus_context_test_workspace_bytes(B, Tp), run


def case_gemm_test_taps():
    lib = _lib.load()
    T, P, B, Cin, N = 30, 2, 2, 64, 128
    Tp = T + 2 * P
    x = randn(B * Tp, Cin, seed=36)
    W = randn(N, 3 * Cin, seed=37) * 0.1
    c = _lib.GemmTapsCase()
    c.ninputs, c.nsrc = 1, 3
    c.x[0], c.rows[0], c.ld[0] = x.data_ptr(), B * Tp, Cin
    for j in range(3):
        c.src_input[j], c.src_col0[j], c.src_ncols[j], c.src_row_off[j] = 0, 0, Cin, j - 1
    c.W, c.M, c.N, c.relu = W.data_ptr(), B * Tp, N, 1
    c.Tp, c.P, c.T = Tp, P, T
    c.out_f32, c.out_rows, c.out_ld, c.precision = 1, B * Tp, N, _lib.PPV_PREC_BF16X3

    def run(ws, nb):
        o = out((B * Tp, N), torch.float32)
        c.out = o.data_ptr()
        return lib.ppv_gemm_test_taps(C.byref(c), V(ws), nb, stream()), [o]
    return lib.ppv_gemm_test_taps_workspace_bytes(C.byref(c)), run


def case_res2net_test(variant):
    lib = _lib.load()
    nconv, B, T, dil, ld = 3, 3, 60, 2, 320
    Tp = T + 8
    w, bias = randn(nconv, 64, 64, 3, seed=39) * 0.07, randn(nconv, 64, seed=40)
    scale, shift = randn(nconv, 64, seed=41), randn(nconv, 64, seed=42)

    def run(ws, nb):  # x is read and written back: its FILL bytes are a small finite input
        xo, y = out((B * Tp, ld), torch.float32), out((B * Tp + 64, ld), torch.float32)
        return lib.ppv_res2net_test(_lib.ptr(xo), ld, _lib.ptr(w), _lib.ptr(bias), _lib.ptr(scale), _lib.ptr(shift), nconv, B, T, dil,
                                    variant, _lib.PPV_PREC_BF16X3, 0, _lib.ptr(y), ld, V(ws), nb, stream()), [xo, y]
    return lib.ppv_res2net_test_workspace_bytes(nconv, B, T, ld, ld), run


def case_skinny_linear_test():
    lib = _lib.load()
    M, ld, x_col0, N, K, out_ld = 37, 272, 8, 130, 256, 136
    x, W, bias = randn(M, ld, seed=43), randn(N, K, seed=44) * 0.1, randn(N, seed=45)

    def run(ws, nb):
        o = out((M, out_ld), torch.float32)
        return lib.ppv_skinny_linear_test(_lib.ptr(x), M, ld, x_col0, _lib.ptr(W), N, K, _lib.ptr(bias), 1, 1, _lib.ptr(o), out_ld, 3, V(ws),
                                          nb, stream()), [o]
    return lib.ppv_skinny_linear_test_workspace_bytes(M, ld, N, K, out_ld), run


def case_scale_res_test():
    lib = _lib.load()
    rows, rpg, Cc, res_ld, rc0, out_ld, oc0 = 3 * 45, 45, 64, 96, 32, 80, 16
    z, res, scale = randn(rows, Cc, seed=46), randn(rows, res_ld, seed=47), randn(3, Cc, seed=48)

    def run(ws, nb):
        o = out((2, rows, out_ld), torch.int16)
        return lib.ppv_scale_res_test(_lib.ptr(z), _lib.ptr(scale), _lib.ptr(res), res_ld, rc0, Cc, rpg, rows, 1, 20.0, _lib.ptr(o), out_ld,
                                      oc0, V(ws), nb, stream()), [o]
    return lib.ppv_scale_res_test_workspace_bytes(rows, Cc, res_ld), run


def case_aff_combine_test():
    lib = _lib.load()
    rows, Cc, x_ld, xc0, y_ld, yc0 = 150, 64, 96, 32, 128, 64
    x, y, t = randn(rows, x_ld, seed=49), randn(rows, y_ld, seed=50), torch.tanh(randn(rows, Cc, seed=51))

    def run(ws, nb):
        o = out((2, rows, Cc), torch.int16)
        return lib.ppv_aff_combine_test(_lib.ptr(x), x_ld, xc0, _lib.ptr(y), y_ld, yc0, _lib.ptr(t), Cc, rows, _lib.ptr(o), V(ws), nb,
                                        stream()), [o]
    return lib.ppv_aff_combine_test_workspace_bytes(rows, Cc, x_ld, y_ld), run


CASES = {
    "aam_forward_backward": case_aam, "cosine_matrix": case_cosine, "eer_mindcf": case_eer, "sym_eig_smallest": case_sym_eig,
    "kmeans": case_kmeans, "vad_energy": case_vad, "audio_prep": case_audio_prep, "audio_prep_reverb": case_audio_prep_reverb,
    "speaker_index_search_k1": lambda: case_speaker_index_search(1), "speaker_index_search_k5": lambda: case_speaker_index_search(5),
    "gemm_test": case_gemm_test, "gemm_test_planes": case_gemm_test_planes, "conv2d_test": case_conv2d_test,
    "asp_fused_test": case_asp_fused_test, "colstats_test": case_colstats_test, "campplus_context_test": case_campplus_context_test,
    "gemm_test_taps": case_gemm_test_taps, "res2net_test_chain": lambda: case_res2net_test(_lib.PPV_RES2_CHAIN),
    "res2net_test_chain_paired": lambda: case_res2net_test(_lib.PPV_RES2_CHAIN_PAIRED),
    "res2net_test_per_conv": lambda: case_res2net_test(_lib.PPV_RES2_PER_CONV), "skinny_linear_test": case_skinny_linear_test,
    "scale_res_test": case_scale_res_test, "aff_combine_test": case_aff_combine_test,
}


def bits(t):
    return t.contiguous().view(torch.uint8)


@pytest.mark.parametrize("name", sorted(CASES))
def test_workspace_exact_short_and_misaligned(cuda, name):
    need, run = CASES[name]()
    assert need > 0 and need % 256 == 0

    roomy = torch.zeros(need + (1 << 16), dtype=torch.uint8, device="cuda")
    rc, ref = run(roomy.data_ptr(), roomy.numel())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()

    buf = torch.zeros(need + 4096, dtype=torch.uint8, device="cuda")
    buf[need:] = TAIL
    rc, got = run(buf.data_ptr(), need)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    assert bool((buf[need:] == TAIL).all()), f"{name} wrote past the {need} bytes its size query returns"
    for r, g in zip(ref, got):
        assert torch.equal(bits(r), bits(g)), f"{name}: outputs differ between an exact and a generous workspace"

    for ws, nb, why in ((buf.data_ptr(), need - 1, "one byte short"), (buf.data_ptr() + 16, need, "16 bytes off alignment")):
        rc, outs = run(ws, nb)
        torch.cuda.synchronize()
        assert rc == EINVAL, f"{name}, workspace {why}: status {rc}"
        assert "workspace" in _lib.last_error()
        for o in outs:
            assert bool((bits(o) == FILL).all()), f"{name}, workspace {why}: an output was written"
