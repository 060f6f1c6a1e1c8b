"""Run-to-run reproducibility of the sums many blocks contribute to (DESIGN.md, "Run-to-run reproducibility"): every block
writes its partial into its own row of stream-ordered scratch memory and reduce_parts adds the rows in a fixed order, so two
runs on the same inputs must agree bit for bit.  Each kernel runs exactly twice on identical inputs, with its outputs reset
to identical contents; between the two runs a large block of the stream-ordered pool the scratch comes from is filled with
NaN and freed, so a kernel that reads scratch it did not write shows up as a difference (or as NaN).

The shapes are chosen so that the number of parts is > 1 on a 132-SM H100 (see each case).  The step-level check is
test_gpu_train_parity.py::test_captured_step_reproduces_the_eager_step."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200 import lib
    lib.lib()
    return lib


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).cuda()


def dirty_scratch(nbytes=256 << 20):
    """Allocates nbytes from the device's stream-ordered pool on the current stream (where the library's cudaMallocAsync
    scratch comes from), fills them with NaN and frees them, all in stream order."""
    cu = ctypes.CDLL('libcuda.so.1')
    p = ctypes.c_uint64(0)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert cu.cuMemAllocAsync(ctypes.byref(p), ctypes.c_size_t(nbytes), st) == 0
    assert cu.cuMemsetD32Async(ctypes.c_uint64(p.value), ctypes.c_uint(0x7FC00000), ctypes.c_size_t(nbytes // 4), st) == 0
    assert cu.cuMemFreeAsync(ctypes.c_uint64(p.value), st) == 0


def twice(fn, outs, what):
    """fn() twice; every output reset to its initial content before each run, scratch dirtied between the runs."""
    init = [o.clone() for o in outs]
    runs = []
    for run in range(2):
        for o, i in zip(outs, init):
            o.copy_(i)
        if run:
            dirty_scratch()
        fn()
        runs.append([o.clone() for o in outs])
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(zip(*runs)):
        assert bool(torch.isfinite(a).all()), '%s: output %d is not finite' % (what, k)
        assert torch.equal(a, b), '%s: output %d differs between two identical runs (max diff %g)' % (what, k, (a - b).abs().max().item())


@pytest.mark.parametrize('split', [0, 4])
def test_conv_wgrad(L, split):
    # 3x3x3 discriminator layer, 32 -> 64 channels: 1 x 1 tiles x 27 taps = 27 CTAs, so the automatic split is
    # 2 * 132 / 27 = 9 parts; 9 x 32 x 32 positions = 144 boxes of 64 allow it.  split 4 is an explicit split.
    x, dy = rnd(1, 9, 32, 32, 32), rnd(1, 9, 32, 32, 64, seed=1)
    g = L.geom((3, 3, 3), (1, 1, 1), (1, 1, 1))
    dwp = torch.zeros(27 * 64 * 32, device='cuda')
    twice(lambda: L.conv_wgrad(L.tensor_view(x, 32), L.tensor_view(dy, 64), g, dwp, 64, 1, split), [dwp], 'conv_wgrad')
    # 5x5 gate conv 72 -> 128 transposed (upsample) geometry with an explicit split
    x2, dy2 = rnd(2, 16, 16, 72, seed=2), rnd(2, 32, 32, 32, seed=3)
    g2 = L.geom((1, 6, 6), (1, 2, 2), (0, 2, 2), True)
    dwp2 = torch.zeros(36 * 32 * 96, device='cuda')
    twice(lambda: L.conv_wgrad(L.tensor_view(x2, 72), L.tensor_view(dy2, 32), g2, dwp2, 32, 3, split), [dwp2], 'conv_wgrad transposed')


def test_conv3d_c4_wgrad_tensor_cores(L):
    # first discriminator layer, the benchmark's clip shape per video: one CTA per line segment, partials added in CTA order
    N, D, H, W, C = 2, 10, 64, 64, 3
    x = torch.zeros(N, D, H, W, 4, device='cuda')
    x[..., :C] = rnd(N, D, H, W, C)
    dy = rnd(N, D, H, W, 32, seed=1)
    gw = torch.full((27 * C * 32,), 0.25, device='cuda')
    twice(lambda: L.check(L.lib().vp_conv3d_c4_wgrad_tc(L.ptr(x), L.ptr(dy), L.ptr(gw), N, D, H, W, C, L.stream_ptr())), [gw],
          'conv3d_c4_wgrad_tc')


@pytest.mark.parametrize('slab', ['1', '0'])
def test_inorm_act_bwd(L, monkeypatch, slab):
    # dgamma / dbeta: one part per sample (n = 6), slab (cluster) kernels and the fallback (VP_SLAB=0, read per call)
    monkeypatch.setenv('VP_SLAB', slab)
    N, P, C = 6, 1024, 64
    x, g, b, dy = rnd(N, P, C) * 2 + 1, rnd(C, seed=1), rnd(C, seed=2), rnd(N, P, C, seed=3)
    y, st = torch.zeros(N, P, C, device='cuda'), torch.zeros(N, C, 2, device='cuda')
    L.inorm_act(x.data_ptr(), C, y.data_ptr(), C, N, P, C, g, b, L.ACT_RELU, 0.0, st)
    dx, dg, db = torch.zeros_like(x), torch.full((C,), 0.5, device='cuda'), torch.full((C,), -0.5, device='cuda')
    twice(lambda: L.inorm_act_bwd(x.data_ptr(), C, [(dy.data_ptr(), C)], dx.data_ptr(), C, N, P, C, g, b, st, L.ACT_RELU, 0.0, dg, db),
          [dx, dg, db], 'inorm_act_bwd VP_SLAB=%s' % slab)


@pytest.mark.parametrize('slab', ['1', '0'])
def test_lstm_gates_bwd(L, monkeypatch, slab):
    # the four norm-parameter gradients: one part per sample (n = 6)
    monkeypatch.setenv('VP_SLAB', slab)
    N, P, Fl = 6, 256, 64
    pre, c0 = rnd(N, P, 4 * Fl) + 0.8, rnd(N, P, Fl, seed=1)
    g1, b1, g2, b2 = rnd(4 * Fl, seed=2) * 0.3 + 1, rnd(4 * Fl, seed=3) * 0.1, rnd(Fl, seed=4) * 0.3 + 1, rnd(Fl, seed=5) * 0.1
    c1, h = torch.zeros(N, P, Fl, device='cuda'), torch.zeros(N, P, Fl, device='cuda')
    s1, s2 = torch.zeros(N, 4 * Fl, 2, device='cuda'), torch.zeros(N, Fl, 2, device='cuda')
    L.lstm_gates_fwd(pre, N, P, Fl, c0, g1, b1, g2, b2, c1, [(h.data_ptr(), Fl)], s1, s2)
    dh, dc = rnd(N, P, Fl, seed=6), rnd(N, P, Fl, seed=7)
    outs = [torch.zeros_like(pre), torch.zeros_like(c0)] + [torch.full_like(t, 0.5) for t in (g1, b1, g2, b2)]
    twice(lambda: L.lstm_gates_bwd(pre, N, P, Fl, c0, g1, b1, g2, b2, s1, s2, [(dh.data_ptr(), Fl)], dc, *outs), outs,
          'lstm_gates_bwd VP_SLAB=%s' % slab)


def test_cdna_apply_bwd(L):
    # dkernels: one part per 256-pixel block of a 64x64 image (16 parts per sample)
    N, H, W, nk = 2, 64, 64, 4
    nl = nk + 3
    img = torch.zeros(N, H, W, 4, device='cuda')
    img[..., :3] = torch.rand(N, H, W, 3, device='cuda')
    kern = torch.softmax(rnd(N, 25, nk), dim=1).reshape(N, 25 * nk).contiguous()
    da, db = rnd(N, H, W, 4 * nl, seed=1), rnd(N, H, W, 4 * nl, seed=2)
    dimg, dk = torch.zeros(N, H, W, 4, device='cuda'), torch.full((N, 25 * nk), 0.5, device='cuda')
    twice(lambda: L.cdna_apply_bwd(img, kern, da.data_ptr(), 4 * nl, db.data_ptr(), 4 * nl, dimg, dk, N, H, W, 5, 5, nk),
          [dimg, dk], 'cdna_apply_bwd')


def test_dense(L):
    # the CDNA-kernel dense layer: K = 2048 in 64-wide parts (32 parts) for the forward; the tiled (K >= 1024) and the small
    # backward kernels
    for B, K, J in [(32, 2048, 100), (5, 300, 10)]:
        x, w, b, dy = rnd(B, K), rnd(K, J, seed=1, scale=0.05), rnd(J, seed=2), rnd(B, J, seed=3)
        sig = torch.tensor([1.7], device='cuda')
        y = torch.zeros(B, J, device='cuda')
        twice(lambda: L.dense_fwd(x, K, w, b, y, J, B, K, J, k_splits=32, inv_scale=sig), [y], 'dense_fwd %d %d %d' % (B, K, J))
        dx, dw, db = torch.zeros_like(x), torch.full_like(w, 0.5), torch.full_like(b, 0.5)
        twice(lambda: L.dense_bwd(x, K, w, dy, J, B, K, J, dx=dx, dx_stride=K, dw=dw, dbias=db, inv_scale=sig), [dx, dw, db],
              'dense_bwd %d %d %d' % (B, K, J))


def test_colsum(L):
    # bias gradients: positions in row blocks, one part per block (4096 positions -> several parts per sample)
    N, P, C = 4, 4096, 32
    x = rnd(N, P, C + 8)
    out = torch.full((N, C), 0.5, device='cuda')
    twice(lambda: L.colsum(x.data_ptr(), C + 8, out, N, P, C, 0.25), [out], 'colsum')


def test_spectral_norm(L):
    # 4x4x4 x 128 -> 256 discriminator kernel: rows = 8192 in 512-row parts (16 parts) for s = v W; the backward's
    # <g, W> dot in 592 block parts
    R, Cc = 64 * 128, 256
    W, u, G = rnd(R, Cc, scale=0.05), rnd(1, Cc, seed=1), rnd(R, Cc, seed=2)
    v, s, un, scal = [torch.zeros(n, device='cuda') for n in (R, Cc, Cc, 4)]
    twice(lambda: L.spectral_norm_fwd(W, u, R, Cc, v, s, un, scal), [v, s, un, scal], 'spectral_norm_fwd')
    gs, gt, dW = torch.zeros(Cc, device='cuda'), torch.zeros(R, device='cuda'), torch.full_like(W, 0.5)
    twice(lambda: L.spectral_norm_bwd(W, u, G, R, Cc, v, s, scal, gs, gt, dW), [gs, gt, dW, scal], 'spectral_norm_bwd')


@pytest.mark.parametrize('mode', [0, 1])
def test_pixel_loss(L, mode):
    # L1 (mode 0) / L2 (mode 1) over 16 x 64 x 64 pixels: one part per block (192 parts)
    rows = 16 * 64 * 64
    pred, tgt = torch.rand(rows, 4, device='cuda'), torch.rand(rows, 4, device='cuda')
    out, dp = torch.zeros(1, device='cuda'), torch.zeros(rows, 4, device='cuda')
    twice(lambda: L.pixel_loss(pred.data_ptr(), 4, tgt.data_ptr(), 4, dp.data_ptr(), 4, rows, 3, mode, rows * 3, 2.0, out), [out, dp],
          'pixel_loss mode %d' % mode)


def test_cosine_distance(L):
    # discriminator features, 64 channels: 16 lanes per row, 4096 rows -> 256 block parts
    a, b = rnd(4096, 64), rnd(4096, 64, seed=1)
    da, out = torch.full_like(a, 0.25), torch.zeros(1, device='cuda')
    twice(lambda: L.cosine_distance(a, b, da, 4096, 64, 3.0, out), [da, out], 'cosine_distance')
