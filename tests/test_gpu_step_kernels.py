"""GPU tests (-m gpu) of the kernels at both ends of the training step, each against an fp64 reference of the same operation
(torch autograd for the gradients): the losses that seed the backward pass (vp_gan_loss, vp_pixel_loss, vp_kl_loss), the z
sampler (vp_sample_z, vp_sample_z_bwd), the reductions and channel moves of the backward pass (vp_colsum, vp_avgpool,
vp_avgpool_bwd, vp_axpy_channels, vp_act_bwd, vp_select_rows, vp_broadcast_channels, vp_copy_channels), the spectral norm
of every discriminator weight and the Adam update; and a training step whose posterior log-variance is clipped in every row.

The inputs reach the branches a freshly initialised model never takes: saturated and overflowing logits, clipped log
variances, row counts where the loops over blocks engage, one-column spectral norms.  The library is built with
--use_fast_math (__expf, approximate division, flush to zero), so the tolerances are: bit-exact for copies and selects; 1e-6
of the reference for affine element-wise kernels; 1e-5 where exp / log / tanh enter; 1e-5 of the sum of absolute addends
for reductions.  Every loss adds into its slot, so every output starts at a non-zero value.  Each section also reruns its
calls through `twice` (bit-identical results with the scratch pool NaN-filled in between).  Outputs are written into
channel slices of wider buffers whose other channels hold NaN: they must come back untouched."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import savp_oracle as O
from test_gpu_engine import L  # noqa: F401  (fixture)
from test_gpu_reproducible import twice
from test_gpu_train_parity import (CASES, EXACT_GTOL, MODES, Model, _check_grads, _check_grads_tf32,  # noqa: F401  (fixture)
                                   _exempt, _gpu_step, _oracle_step, arithmetic, tf32_mode)

pytestmark = pytest.mark.gpu
NAN = float('nan')
WORST = {}          # '<section> (tol <t>)' -> worst measured error in units of the bound's scale


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\nworst error per section and tolerance (error / scale, against the tolerance):')
        for k in sorted(WORST):
            print('  %-48s %.3g' % (k, WORST[k]))


def _check(section, got, ref, tol, scale, what=''):
    """max |got - ref| / scale <= tol, element-wise when `scale` is a tensor; NaN in `got` fails."""
    got, ref = got.double(), ref.double()
    scale = scale.double() if torch.is_tensor(scale) else torch.tensor(float(scale), dtype=torch.float64, device=ref.device)
    r = ((got - ref).abs() / (scale + 1e-300)).max().item()
    key = '%s (tol %g)' % (section, tol)
    WORST[key] = max(WORST.get(key, 0.0), r) if r == r else float('nan')
    assert r <= tol, '%s %s: error %g of the scale, tolerance %g' % (section, what, r, tol)


def _randn(*shape, seed=0, scale=1.0, mean=0.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(*shape, generator=g, device='cuda') * scale + mean


def _rand(*shape, seed=0, lo=0.0, hi=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.rand(*shape, generator=g, device='cuda') * (hi - lo) + lo


def _slice(rows, c, cs, off, seed, mean=0.0):
    """[rows, cs] buffer: channels [off, off + c) N(mean, 1), every other channel NaN."""
    buf = torch.full((rows, cs), NAN, device='cuda')
    buf[:, off:off + c] = _randn(rows, c, seed=seed, mean=mean)
    return buf


def _untouched(buf, off, c):
    return bool(torch.isnan(buf[..., :off]).all()) and bool(torch.isnan(buf[..., off + c:]).all())


# ================================================================================================ A. losses
def _logits(regime, n, seed):
    if regime == 'normal':
        return _randn(n, seed=seed)
    sign = torch.where(torch.arange(n, device='cuda') % 2 == 0, 1.0, -1.0)      # n = 1: one positive logit
    return sign * (8.0 if regime == 'saturated' else 90.0)                         # 90: __expf(90) overflows to inf


def _ce_terms(x, label):
    """Per-element sigmoid cross-entropy max(x, 0) - x y + log(1 + exp(-|x|)) (the SNGAN softplus for y in {0, 1})."""
    return torch.clamp(x, min=0) - x * label + torch.log1p(torch.exp(-x.abs()))


@pytest.mark.parametrize('regime', ['normal', 'saturated', 'extreme'])
@pytest.mark.parametrize('label', [0.0, 1.0])
@pytest.mark.parametrize('kind', ['LSGAN', 'GAN', 'SNGAN'])
def test_gan_loss(L, kind, label, regime):  # noqa: F811
    """Value and gradient of losses.gan_loss for n = 1 ... 4096 logits (n > 256: several per thread); the gradient is
    within 1e-5 of grad_scale / n (the largest |gradient| of one sigmoid-CE element) of the fp64 one, and finite where
    exp(-x) overflows.  The value adds into a non-zero slot; dlogits = None leaves the value as it is."""
    for n in (1, 2, 16, 300, 4096):
        x = _logits(regime, n, seed=n)
        gs, out0 = 0.1 * (n % 7 + 1), 0.37
        out, dl = torch.full((1,), out0, device='cuda'), torch.full((n,), NAN, device='cuda')
        L.gan_loss(x, label, n, gs, kind, dl, out)
        xd = x.double().requires_grad_(True)
        ref = O.gan_loss(xd, label, kind)
        (g,) = torch.autograd.grad(gs * ref, xd)
        terms = (xd - label) ** 2 if kind == 'LSGAN' else _ce_terms(xd, label)
        torch.cuda.synchronize()
        what = '%s label %g %s n=%d' % (kind, label, regime, n)
        _check('A gan_loss value', out, out0 + ref.detach(), 1e-5, terms.detach().abs().mean() + out0, what)
        assert bool(torch.isfinite(dl).all()), what
        _check('A gan_loss dlogits', dl, g, 1e-5, max(g.abs().max().item(), gs / n), what)
        out2 = torch.full((1,), out0, device='cuda')
        L.gan_loss(x, label, n, gs, kind, None, out2)
        torch.cuda.synchronize()
        assert torch.equal(out2, out), what
    outs = [torch.full((1,), out0, device='cuda'), torch.zeros(n, device='cuda')]
    twice(lambda: L.gan_loss(x, label, n, gs, kind, outs[1], outs[0]), outs, 'gan_loss %s' % kind)


def test_gan_loss_rejects_bad_calls(L):  # noqa: F811
    """An unknown kind, and the sigmoid-CE kinds with a label outside {0, 1}, raise and write nothing; LSGAN takes any label."""
    n = 16
    x = _randn(n, seed=3)
    out, dl = torch.full((1,), 0.37, device='cuda'), torch.full((n,), 7.0, device='cuda')
    for kind, label in ((3, 1.0), (-1, 1.0), (1, 0.5), (2, 0.5)):
        with pytest.raises(L.VpError):
            L.check(L.lib().vp_gan_loss(L.ptr(x), ctypes.c_float(label), n, ctypes.c_float(1.0), kind, L.ptr(dl), L.ptr(out),
                                        L.stream_ptr()))
    torch.cuda.synchronize()
    assert bool((out == 0.37).all()) and bool((dl == 7.0).all())
    L.gan_loss(x, 0.5, n, 1.0, 'LSGAN', dl, out)
    xd = x.double().requires_grad_(True)
    ref = O.gan_loss(xd, 0.5, 'LSGAN')
    (g,) = torch.autograd.grad(ref, xd)
    torch.cuda.synchronize()
    _check('A gan_loss value', out, 0.37 + ref.detach(), 1e-5, ref.item() + 0.37, 'LSGAN label 0.5')
    _check('A gan_loss dlogits', dl, g, 1e-5, g.abs().max(), 'LSGAN label 0.5')


# (rows, C) of one call (one predicted frame): 64x64 batch 16 (below the 1184 x 256 elements of one grid-stride round) and
# 128x128 batch 8 (above), colour and grey (KTH)
PIXEL_SHAPES = [(16 * 4096, 3), (8 * 16384, 3), (16 * 4096, 1), (32 * 16384, 1)]


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
@pytest.mark.parametrize('rows,C', PIXEL_SHAPES)
def test_pixel_loss(L, rows, C, mode):  # noqa: F811
    """losses.l1_loss (mode 0) / l2_loss (mode 1), bit 1 accumulating the gradient into dpred, over C channels at stride 4
    with a mean over 11 frames' worth of elements (the step calls it once per frame).  pred == target in every fifth
    element: the L1 gradient there is exactly 0, as tf.sign gives."""
    count, gs, out0 = 11 * rows * C, 100.0, 0.37
    pred, tgt = torch.full((rows, 4), NAN, device='cuda'), torch.full((rows, 4), NAN, device='cuda')
    pred[:, :C], tgt[:, :C] = _rand(rows, C, seed=1), _rand(rows, C, seed=2)
    eq = (torch.arange(rows * C, device='cuda') % 5 == 0).view(rows, C)
    tgt[:, :C] = torch.where(eq, pred[:, :C], tgt[:, :C])
    dp0 = _randn(rows, C, seed=3, scale=gs / count)
    dp = torch.full((rows, 4), NAN, device='cuda')
    if mode & 2:
        dp[:, :C] = dp0
    out = torch.full((1,), out0, device='cuda')
    L.pixel_loss(pred.data_ptr(), 4, tgt.data_ptr(), 4, dp.data_ptr(), 4, rows, C, mode, count, gs, out)
    pd = pred[:, :C].double().requires_grad_(True)
    d = pd - tgt[:, :C].double()
    terms = d.abs() if mode & 1 == 0 else d ** 2
    ref = terms.sum() / count
    (g,) = torch.autograd.grad(gs * ref, pd)
    want = g + (dp0.double() if mode & 2 else 0.0)
    torch.cuda.synchronize()
    what = 'mode %d rows %d C %d' % (mode, rows, C)
    _check('A pixel_loss value', out, out0 + ref.detach(), 1e-5, ref.item() + out0, what)
    _check('A pixel_loss dpred', dp[:, :C], want, 1e-6, max(want.abs().max().item(), gs / count), what)
    if mode & 1 == 0:
        assert torch.equal(dp[:, :C][eq], dp0[eq] if mode & 2 else torch.zeros_like(dp0[eq])), what
    assert bool(torch.isnan(dp[:, C:]).all()), what
    out2 = torch.full((1,), out0, device='cuda')
    L.pixel_loss(pred.data_ptr(), 4, tgt.data_ptr(), 4, 0, 4, rows, C, mode, count, gs, out2)          # dpred = None
    torch.cuda.synchronize()
    assert torch.equal(out2, out), what
    dpr = torch.zeros(rows, 4, device='cuda')
    dpr[:, :C] = dp0
    outs = [torch.full((1,), out0, device='cuda'), dpr]
    twice(lambda: L.pixel_loss(pred.data_ptr(), 4, tgt.data_ptr(), 4, dpr.data_ptr(), 4, rows, C, mode, count, gs, outs[0]), outs,
          'pixel_loss ' + what)


@pytest.mark.parametrize('rows,nz', [(11 * 16, 8), (29 * 32, 8), (29 * 32, 32)])
def test_kl_loss(L, rows, nz):  # noqa: F811
    """losses.kl_loss with log sigma^2 spread over the whole clip range [-10, 10], at the (unroll steps x batch, nz) of the
    BASELINE configurations."""
    mu, lss = _randn(rows, nz, seed=1), _rand(rows, nz, seed=2, lo=-10.0, hi=10.0)
    out0 = 0.37
    out = torch.full((1,), out0, device='cuda')
    L.kl_loss(mu, lss, rows, nz, out)
    md, ld = mu.double(), lss.double()
    ref = O.kl_loss(md, ld)
    scale = 0.5 * (1 + ld - md ** 2 - torch.exp(ld)).abs().sum() / rows + out0
    torch.cuda.synchronize()
    _check('A kl_loss value', out, out0 + ref, 1e-5, scale, '%d x %d' % (rows, nz))
    outs = [torch.full((1,), out0, device='cuda')]
    twice(lambda: L.kl_loss(mu, lss, rows, nz, outs[0]), outs, 'kl_loss')


# ================================================================================================ B. z sampler
SPECIAL_LSS = [-30.0, -10.5, float(np.nextafter(np.float32(-10), np.float32(0))), 0.0,
               float(np.nextafter(np.float32(10), np.float32(0))), 10.5, 30.0]


def _pre_clip_lss(rows, nz, seed):
    """Pre-clip log sigma^2: the special values above in the first rows, U(-12, 12) elsewhere; never exactly +-10."""
    lss = _rand(rows, nz, seed=seed, lo=-12.0, hi=12.0)
    flat = lss.view(-1)
    k = 4 * len(SPECIAL_LSS)
    flat[:k] = torch.tensor(SPECIAL_LSS, device='cuda').repeat(4)
    assert not bool((lss.abs() == 10.0).any())
    return lss


def test_sample_z(L):  # noqa: F811
    """z = mu + sqrt(exp(clip(lss, -10, 10))) eps (savp_model.py:49, 712); the clip is written back bit-exactly."""
    rows, nz = 11 * 16, 8
    pre = _pre_clip_lss(rows, nz, seed=1)
    mu, eps = _randn(rows, nz, seed=2), _randn(rows, nz, seed=3)
    lss, z = pre.clone(), torch.full((rows, nz), NAN, device='cuda')
    L.sample_z(mu, lss, eps, z, rows * nz)
    torch.cuda.synchronize()
    assert torch.equal(lss, pre.clamp(-10.0, 10.0))
    assert bool((lss[pre >= 10] == 10.0).all()) and bool((lss[pre <= -10] == -10.0).all())
    sd = torch.sqrt(torch.exp(pre.double().clamp(-10, 10))) * eps.double()
    _check('B sample_z z', z, mu.double() + sd, 1e-5, mu.double().abs() + sd.abs())
    outs = [pre.clone(), torch.zeros(rows, nz, device='cuda')]
    twice(lambda: L.sample_z(mu, outs[0], eps, outs[1], rows * nz), outs, 'sample_z')


@pytest.mark.parametrize('dz_on,kl_on', [(True, True), (True, False), (False, True)])
def test_sample_z_bwd(L, dz_on, kl_on):  # noqa: F811
    """Gradients of mu and of the PRE-clip log sigma^2 through z and the KL term, against fp64 autograd through
    clamp(-10, 10), at the KL scale the step stages (kl_weight / (steps x batch)); kl_scale = None and dz = None drop the
    respective term.  Strictly outside (-10, 10) the log-variance gradient is exactly 0, strictly inside it is the full one.

    Exactly at +-10.0f the kernel deviates from the reference: sample_z clips in place, so the backward sees only the
    clipped value and gives 0 where |l| >= 10, while tf.clip_by_value (and torch.clamp) pass the gradient when the
    pre-clip value is exactly the bound.  The inputs never hold exactly +-10.0f, and that case is not compared."""
    rows, nz = 11 * 16, 8
    pre = _pre_clip_lss(rows, nz, seed=4)
    lss = pre.clamp(-10.0, 10.0)                      # what sample_z left in the buffer
    mu, eps, dz = _randn(rows, nz, seed=5), _randn(rows, nz, seed=6), _randn(rows, nz, seed=7)
    klw = 1e-3
    ks = torch.tensor([klw / rows], device='cuda')    # _stage_step_scalars: kl_weight / (S * B)
    dmu, dlss = torch.full((rows, nz), NAN, device='cuda'), torch.full((rows, nz), NAN, device='cuda')
    L.sample_z_bwd(mu, lss, eps, dz if dz_on else None, dmu, dlss, rows * nz, ks if kl_on else None)
    pd, md = pre.double().requires_grad_(True), mu.double().requires_grad_(True)
    lc = pd.clamp(-10, 10)
    sd = torch.sqrt(torch.exp(lc))
    loss = torch.zeros((), dtype=torch.float64, device='cuda')
    ks64 = ks.double().item()
    if dz_on:
        loss = loss + ((md + sd * eps.double()) * dz.double()).sum()
    if kl_on:
        loss = loss + ks64 * rows * O.kl_loss(md, lc)
    gmu, glss = torch.autograd.grad(loss, (md, pd))
    # the addends of each gradient (e and 1 for e - 1), for the error bound
    e = torch.exp(lss.double())
    a_mu = (dz.double().abs() if dz_on else 0.0) + (ks64 * md.detach().abs() if kl_on else 0.0)
    a_l = ((dz.double() * eps.double()).abs() * 0.5 * e.sqrt() if dz_on else 0.0) + (ks64 * 0.5 * (e + 1) if kl_on else 0.0)
    torch.cuda.synchronize()
    what = 'dz %s kl %s' % (dz_on, kl_on)
    _check('B sample_z_bwd dmu', dmu, gmu, 1e-6, a_mu, what)
    outside, inside = pre.abs() > 10, pre.abs() < 10
    assert bool(outside.any()) and bool((dlss[outside] == 0).all()), what
    assert bool((glss[outside] == 0).all())
    _check('B sample_z_bwd dlss', dlss[inside], glss[inside], 1e-5, a_l[inside], what)
    outs = [torch.zeros(rows, nz, device='cuda'), torch.zeros(rows, nz, device='cuda')]
    twice(lambda: L.sample_z_bwd(mu, lss, eps, dz if dz_on else None, outs[0], outs[1], rows * nz, ks if kl_on else None), outs,
          'sample_z_bwd')


# ================================================================================================ C. reductions, data movement
# (n, positions, c, channel stride, scale) -- n = 1: bias gradients over every unroll step and sample: 64x64 batch 16 x 11
# steps x 2 unrolls = 1,441,792 rows (colour / float4 slots, mask logits, 32 filters) and 29 steps of batch 32 = 7,602,176
# rows (29,696 block parts); the wider layers at their own resolutions with row counts that are not multiples of 256.
# n > 1: the tile-concat adjoint of the z slots (savp_train.py:513), 11 x 32 samples of a 32x32 plane into a strided output.
COLSUM_CASES = [(1, 1441792, 3, 4, 1.0), (1, 1441792, 7, 8, 1.0), (1, 1441792, 32, 32, 0.5),
                (1, 7602176, 3, 4, 1.0), (1, 7602176, 32, 32, 1.0),
                (1, 360448 + 77, 64, 64, 1.0), (1, 90112 + 13, 128, 128, 0.25), (1, 22528 + 5, 256, 256, 1.0),
                (1, 5632 + 200, 512, 512, 2.0), (352, 1024, 10, 48, 1.0)]


@pytest.mark.parametrize('n,P,c,cs,scale', COLSUM_CASES)
def test_colsum(L, n, P, c, cs, scale):  # noqa: F811
    """out[i][:c] += scale * sum over positions of x[i][p][:c], data with mean 0.5; error bound 1e-5 of scale * sum |x| (plus
    |out|) per column.  The channels around the slice in x are NaN (not read) and so are the out columns past c."""
    off = 4 if cs - c >= 4 else 0
    x = _slice(n * P, c, cs, off, seed=c + n, mean=0.5)
    os_ = c + 2 if n > 1 else c
    out0 = _randn(n, os_, seed=1)
    out = out0.clone()
    if n > 1:
        out[:, c:] = NAN
    L.colsum(x.data_ptr() + 4 * off, cs, out, n, P, c, scale, out_stride=os_)
    xs = x.view(n, P, cs)[..., off:off + c]
    ref = out0[:, :c].double() + scale * xs.double().sum(dim=1)
    bound = abs(scale) * xs.double().abs().sum(dim=1) + out0[:, :c].double().abs()
    torch.cuda.synchronize()
    _check('C colsum', out[:, :c], ref, 1e-5, bound, '%d x %d x %d' % (n, P, c))
    assert n == 1 or bool(torch.isnan(out[:, c:]).all())
    del ref, bound
    outs = [out0.clone()]
    twice(lambda: L.colsum(x.data_ptr() + 4 * off, cs, outs[0], n, P, c, scale, out_stride=os_), outs, 'colsum')


def test_colsum_rejects_too_many_rows(L):  # noqa: F811
    P = 65535 * 256 + 1                                     # one row past 65535 row blocks
    x = torch.zeros(P, device='cuda')
    out = torch.full((1,), 0.37, device='cuda')
    with pytest.raises(L.VpError):
        L.colsum(x.data_ptr(), 1, out, 1, P, 1)
    torch.cuda.synchronize()
    assert float(out) == np.float32(0.37)


@pytest.mark.parametrize('size', [64, 128])
def test_avgpool_fwd_bwd(L, size):  # noqa: F811
    """The posterior encoder's global average pool (networks.py:30-31) over its last layer (n_layers stride-2 convolutions:
    8x8 x 256 channels at 64x64, 16x16 x 256 at 128x128) for 11 steps x batch 16, from a channel slice, and its adjoint
    into a channel slice."""
    hp = O.make_hparams(context_frames=2, sequence_length=12, nz=8)
    P, C = (size >> hp.n_layers) ** 2, hp.nef * min(2 ** (hp.n_layers - 1), 4)
    N = 11 * 16
    x = _slice(N * P, C, C + 8, 4, seed=1, mean=0.3).view(N, P, C + 8)
    y = torch.full((N, C), NAN, device='cuda')
    L.avgpool(x[..., 4:], C + 8, y, N, P, C)
    xs = x[..., 4:4 + C].double()
    torch.cuda.synchronize()
    _check('C avgpool', y, xs.mean(dim=1), 1e-5, xs.abs().sum(dim=1) / P)
    dy = _randn(N, C, seed=2)
    dx = torch.full((N, P, C + 12), NAN, device='cuda')
    L.avgpool_bwd(dy, dx[..., 8:], C + 12, N, P, C)
    want = (dy.double() / P)[:, None, :].expand(N, P, C)
    torch.cuda.synchronize()
    _check('C avgpool_bwd', dx[..., 8:8 + C], want, 1e-6, want.abs().max())
    assert _untouched(dx, 8, C)
    outs = [torch.zeros(N, C, device='cuda'), torch.zeros(N, P, C, device='cuda')]

    def both():
        L.avgpool(x[..., 4:], C + 8, outs[0], N, P, C)
        L.avgpool_bwd(dy, outs[1], C, N, P, C)
    twice(both, outs, 'avgpool')


@pytest.mark.parametrize('accumulate', [0, 1])
def test_axpy_channels(L, accumulate):  # noqa: F811
    """dst = (dst if accumulate) + scale * src, rows of masked samples left alone (accumulate) or zeroed: the scheduled-
    sampling gate of the image gradient (savp_train.py:441), one mask entry per 64x64 image of 32 samples."""
    NB, HW, c = 32, 4096, 3
    rows = NB * HW
    src = _slice(rows, c, 4, 0, seed=1)
    mask = (torch.arange(NB, device='cuda', dtype=torch.int32) * 7 % 3 == 0).to(torch.int32)
    dst0 = _slice(rows, c, 8, 2, seed=2)
    for scale, row_mask in ((-0.7, mask), (1.0, None)):
        dst = dst0.clone()
        L.axpy_channels(src.data_ptr(), 4, dst.data_ptr() + 8, 8, rows, c, scale=scale, row_mask=row_mask, rows_per_mask=HW,
                        accumulate=accumulate)
        keep = torch.ones(rows, 1, device='cuda') if row_mask is None else (mask == 0).repeat_interleave(HW)[:, None].double()
        want = scale * src[:, :c].double() * keep + (dst0[:, 2:2 + c].double() if accumulate else 0.0)
        torch.cuda.synchronize()
        what = 'accumulate %d scale %g mask %s' % (accumulate, scale, row_mask is not None)
        _check('C axpy_channels', dst[:, 2:2 + c], want, 1e-6, want.abs().max(), what)
        if row_mask is not None:
            gated = (mask != 0).repeat_interleave(HW)
            assert torch.equal(dst[gated, 2:2 + c], dst0[gated, 2:2 + c] if accumulate else torch.zeros_like(dst0[gated, 2:2 + c]))
        assert _untouched(dst, 2, c), what
    outs = [torch.zeros(rows, c, device='cuda')]
    twice(lambda: L.axpy_channels(src.data_ptr(), 4, outs[0].data_ptr(), c, rows, c, scale=-0.7, row_mask=mask, rows_per_mask=HW,
                                  accumulate=accumulate), outs, 'axpy_channels')


def _act_fwd(L, act, x):  # noqa: F811
    return {L.ACT_NONE: lambda: x, L.ACT_RELU: lambda: torch.relu(x), L.ACT_LRELU: lambda: torch.maximum(0.2 * x, x),
            L.ACT_SIGMOID: lambda: torch.sigmoid(x), L.ACT_TANH: lambda: torch.tanh(x)}[act]()


def _act_grad(L, act, y):  # noqa: F811
    """act'(x) from the output y (fp64)."""
    return {L.ACT_NONE: lambda: torch.ones_like(y), L.ACT_RELU: lambda: (y > 0).double(),
            L.ACT_LRELU: lambda: torch.where(y > 0, 1.0, 0.2).double(), L.ACT_SIGMOID: lambda: y * (1 - y),
            L.ACT_TANH: lambda: 1 - y * y}[act]()


@pytest.mark.parametrize('two_sources', [False, True])
@pytest.mark.parametrize('act', ['none', 'relu', 'lrelu', 'sigmoid', 'tanh'])
def test_act_bwd(L, act, two_sources):  # noqa: F811
    """dx = (dy_a + dy_b) * act'(x) taken from the activation output y, every activation but ELU (its own test is in
    test_gpu_layer_choices.py), at 11 x 16 samples of a 16x16 x 128 plane with four different channel strides."""
    a = getattr(L, 'ACT_' + act.upper())
    rows, c = 11 * 16 * 256, 128
    y = torch.full((rows, c + 4), NAN, device='cuda')
    y[:, 4:] = _act_fwd(L, a, _randn(rows, c, seed=1, scale=2.0))
    dya, dyb = _slice(rows, c, c + 8, 0, seed=2), _slice(rows, c, c, 0, seed=3)
    dx = torch.full((rows, c + 12), NAN, device='cuda')
    L.act_bwd(y.data_ptr() + 16, c + 4, dya.data_ptr(), c + 8, dyb.data_ptr() if two_sources else 0, c, dx.data_ptr() + 32, c + 12,
              rows, c, a, 0.2)
    d = dya[:, :c].double() + (dyb.double() if two_sources else 0.0)
    want = d * _act_grad(L, a, y[:, 4:].double())
    torch.cuda.synchronize()
    _check('C act_bwd', dx[:, 8:8 + c], want, 1e-6, want.abs().max(), act)
    assert _untouched(dx, 8, c)
    outs = [torch.zeros(rows, c, device='cuda')]
    twice(lambda: L.act_bwd(y.data_ptr() + 16, c + 4, dya.data_ptr(), c + 8, dyb.data_ptr() if two_sources else 0, c,
                            outs[0].data_ptr(), c, rows, c, a, 0.2), outs, 'act_bwd ' + act)


def test_select_rows(L):  # noqa: F811
    """tf.where(ground_truth[t], images, gen_image) over 32 64x64 float4 images: bit-exact, the row past n untouched."""
    n, per = 32, 4096 * 4
    sel = (torch.arange(n, device='cuda', dtype=torch.int32) * 5 % 3 == 1).to(torch.int32)
    a, b = _randn(n, per, seed=1), _randn(n, per, seed=2)
    out = torch.full((n + 1, per), NAN, device='cuda')
    L.select_rows(sel, a, b, out, n, per)
    torch.cuda.synchronize()
    assert torch.equal(out[:n], torch.where(sel[:, None] != 0, a, b)) and bool(torch.isnan(out[n]).all())
    outs = [torch.zeros(n, per, device='cuda')]
    twice(lambda: L.select_rows(sel, a, b, outs[0], n, per), outs, 'select_rows')


def test_broadcast_channels(L):  # noqa: F811
    """The z / action tile-concat (savp_model.py:1222): vec [n][:c] (stride 12) into channels [20, 30) of every position."""
    n, P, c = 11 * 32, 1024, 10
    vec = _randn(n, 12, seed=1)
    dst = torch.full((n, P, 48), NAN, device='cuda')
    L.broadcast_channels(vec, 12, dst.data_ptr() + 4 * 20, 48, n, P, c)
    torch.cuda.synchronize()
    assert torch.equal(dst[..., 20:20 + c], vec[:, None, :c].expand(n, P, c)) and _untouched(dst, 20, c)
    outs = [torch.zeros(n, P, c, device='cuda')]
    twice(lambda: L.broadcast_channels(vec, 12, outs[0].data_ptr(), c, n, P, c), outs, 'broadcast_channels')


@pytest.mark.parametrize('rows,c', [(32 * 4096, 4), (16, 8), (11 * 32 * 1024 + 3, 3)])
def test_copy_channels(L, rows, c):  # noqa: F811
    """Channel-slice copies between concat buffers (images into the input concat, z into zcat): bit-exact."""
    src = _slice(rows, c, 12, 2, seed=c)
    dst = torch.full((rows, 20), NAN, device='cuda')
    L.copy_channels(src.data_ptr() + 8, 12, dst.data_ptr() + 32, 20, rows, c)
    torch.cuda.synchronize()
    assert torch.equal(dst[:, 8:8 + c], src[:, 2:2 + c]) and _untouched(dst, 8, c)
    outs = [torch.zeros(rows, c, device='cuda')]
    twice(lambda: L.copy_channels(src.data_ptr() + 8, 12, outs[0].data_ptr(), c, rows, c), outs, 'copy_channels')


# ================================================================================================ D. spectral norm, Adam
def _sn_shapes():
    """(rows, cols) of every spectrally-normalised weight of the video and image discriminators (ndf 32 / 64, 64x64 /
    128x128), read off the model's variable specs: conv kernels [k..., ci, co] -> (prod(k) ci, co), sn_fc4 -> (features, 1)."""
    from video_prediction_b200.models import get_model_class
    shapes = set()
    for size in (64, 128):
        for ndf in (32, 64):
            m = get_model_class('savp')(mode='train', hparams_dict=dict(context_frames=2, sequence_length=12, ndf=ndf,
                                                                        video_sn_gan_weight=0.1, image_sn_gan_weight=0.1))
            m.H = m.W = size
            m.C = 3
            for k, (s, _) in m._discriminator_param_specs().items():
                if k.endswith('/kernel'):
                    shapes.add((int(np.prod(s[:-1])), int(s[-1])))
    return sorted(shapes)


@pytest.mark.parametrize('rows,cols', _sn_shapes(), ids=lambda v: str(v))
def test_spectral_norm_fwd_bwd(L, rows, cols):  # noqa: F811
    """sigma, u' and dW (accumulated into a non-zero dW) against fp64 autograd of O.spectral_normed_weight (ops.py:1020-1049,
    one power iteration, differentiable through it)."""
    W, u, G = _randn(rows, cols, seed=rows + cols, scale=0.05), _randn(1, cols, seed=1), _randn(rows, cols, seed=2)
    v, s, un, scal = [torch.zeros(k, device='cuda') for k in (rows, cols, cols, 4)]
    L.spectral_norm_fwd(W, u, rows, cols, v, s, un, scal)
    Wd = W.double().requires_grad_(True)
    Wb, u1 = O.spectral_normed_weight(Wd, u.double())
    sigma = Wd.detach().norm() / Wb.detach().norm()
    (gW,) = torch.autograd.grad(Wb, Wd, G.double())
    gs, gt, dW = torch.zeros(cols, device='cuda'), torch.zeros(rows, device='cuda'), torch.full_like(W, 0.5)
    L.spectral_norm_bwd(W, u, G, rows, cols, v, s, scal, gs, gt, dW)
    want = 0.5 + gW
    torch.cuda.synchronize()
    what = '%d x %d' % (rows, cols)
    _check('D spectral_norm sigma', scal[2:3], sigma.reshape(1), 1e-5, sigma, what)
    _check('D spectral_norm u_new', un, u1.detach().reshape(-1), 1e-5, 1.0, what)
    _check('D spectral_norm dW', dW, want, 3e-5, want.abs().max(), what)
    outs = [v, s, un, scal]
    twice(lambda: L.spectral_norm_fwd(W, u, rows, cols, v, s, un, scal), outs, 'spectral_norm_fwd ' + what)
    outs = [gs, gt, torch.full_like(W, 0.5), scal]
    twice(lambda: L.spectral_norm_bwd(W, u, G, rows, cols, v, s, scal, gs, gt, outs[2]), outs, 'spectral_norm_bwd ' + what)


@pytest.mark.parametrize('grad_scale', [0.5, 0.125])
def test_adam(L, grad_scale):  # noqa: F811
    """Ten TF-Adam steps with grad_scale = 1 / world size.  Gradients of three magnitudes, the smallest (1e-8) where eps
    dominates sqrt(v) and the update is no longer invariant to the scale of g; every tenth element has g = 0 throughout
    and keeps p (and m = v = 0) exactly."""
    import math
    n, lr, b1 = 3001, 1e-3, 0.5
    b2 = float(np.float32(0.999))                      # the kernel's fp32 beta2: 1 - 0.999f is 1.3e-5 off 1e-3
    p0 = _randn(n, seed=1, scale=0.05)
    mag = torch.tensor([1.0, 1e-4, 1e-8], device='cuda').repeat_interleave(-(-n // 3))[:n]
    zero = torch.arange(n, device='cuda') % 10 == 0
    p, m, v = p0.clone(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    pr, mr, vr = p0.double(), torch.zeros(n, dtype=torch.float64, device='cuda'), torch.zeros(n, dtype=torch.float64, device='cuda')
    for t in range(1, 11):
        g = torch.where(zero, 0.0, _randn(n, seed=10 + t) * mag)
        lr_t = torch.tensor([lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)], device='cuda')
        L.adam(p, g, m, v, n, lr_t, b1, b2, grad_scale=grad_scale)
        pr, mr, vr = O.adam_tf(pr, g.double() * grad_scale, mr, vr, lr, b1, b2, t)
    torch.cuda.synchronize()
    _check('D adam p', p, pr, 1e-6, max(pr.abs().max().item(), 1.0), 'grad_scale %g' % grad_scale)
    _check('D adam m', m, mr, 1e-6, mr.abs().max(), 'grad_scale %g' % grad_scale)
    _check('D adam v', v, vr, 1e-6, vr.abs().max(), 'grad_scale %g' % grad_scale)
    assert torch.equal(p[zero], p0[zero]) and not bool(m[zero].any()) and not bool(v[zero].any())
    outs = [p0.clone(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')]
    twice(lambda: L.adam(outs[0], g, outs[1], outs[2], n, lr_t, b1, b2, grad_scale=grad_scale), outs, 'adam')


# ================================================================================================ E. clipped posterior
@pytest.mark.parametrize('mode', ['tf32', 'exact'])
def test_clipped_posterior_training_step(Model, mode):  # noqa: F811
    """The 'vae_l1' training step of test_gpu_train_parity.py with the z_log_sigma_sq bias at +12 for z unit 0 and -12 for
    unit 1, so that every row of those units is clipped (savp_model.py:49): the stored log-variances are exactly +-10, the
    KL loss (~1.1e4, dominated by exp(10) / 2) matches the oracle, the gradients of those units' bias entries and kernel
    columns are exactly 0 (as the oracle's are: no gradient passes a clip), and every other gradient is within the case's
    tolerance of the fp32 oracle."""
    case = 'vae_l1'
    hk = CASES[case]
    hp = O.make_hparams(**hk)
    B, step, shape = 2, 5, (64, 64, 3)
    params, _ = O.init_params(hp, shape, seed=0)
    kb, kk = 'generator/encoder/z_log_sigma_sq/dense/bias', 'generator/encoder/z_log_sigma_sq/dense/kernel'
    bias = params[kb].clone()
    bias[0], bias[1] = 12.0, -12.0
    params[kb] = bias
    inputs, noise = O.make_synthetic_inputs(hp, B, shape)
    sampling = torch.rand(hp.sequence_length - 1 - hp.context_frames, B, generator=torch.Generator().manual_seed(7)) < 0.5
    _, ltol, floor, otol = MODES[mode]
    with arithmetic(mode):
        model = _gpu_step(Model, hk, params, inputs, noise, step, sampling)
    res = _oracle_step(hp, params, inputs, noise, step, sampling, None, ())
    lss = model.outputs_time_major('zs_log_sigma_sq_enc').cpu()
    assert bool((lss[..., 0] == 10.0).all()) and bool((lss[..., 1] == -10.0).all())
    ref_lss = res['outputs']['zs_log_sigma_sq_enc']
    assert bool((ref_lss[..., 0] == 10.0).all()) and bool((ref_lss[..., 1] == -10.0).all())
    lv = model.losses()
    ref_l = {k: float(v) for k, v in res['g_losses'].items()}
    assert ref_l['gen_kl_loss'] > 1e4
    for k, v in ref_l.items():
        assert abs(lv[k] - v) <= ltol * abs(v) + 1e-6, (k, lv[k], v)
    for name, got, ref in ((kb, model.grads[kb][:2], res['g_grads'][kb][:2]), (kk, model.grads[kk][:, :2], res['g_grads'][kk][:, :2])):
        assert not bool(got.any()), (name, got)
        assert not bool(ref.any()), (name, ref)
    if mode == 'exact':
        _check_grads(model, res, EXACT_GTOL[case], floor, 'clipped posterior [exact] vs fp32 oracle')
    else:
        emu = _oracle_step(hp, params, inputs, noise, step, sampling, tf32_mode(), _exempt(model))
        _check_grads_tf32(model, res, emu, floor, 'clipped posterior')
    for k in ('gen_images', 'gen_images_enc'):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)
