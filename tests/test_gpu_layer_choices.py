"""GPU tests (-m gpu) of the generator's layer choices downsample_layer='conv2d', upsample_layer='deconv2d' (and the _v2
recipes) and activation_layer='elu': the engine at every new geometry of the 64x64 and 128x128 generators against fp64
(forward, dgrad, wgrad, DECONV packs), VP_ACT_ELU in every fused kernel against fp64, bit-identical reruns, rejected bad
calls, the generator and the training step against the fp32 reference (tests/savp_layers_oracle.py), the captured step,
and the restore of a TF bundle with conv2d / deconv2d names."""
import numpy as np
import pytest
import torch

import savp_layers_oracle as R
from oracle import savp_oracle as O
from test_gpu_engine import ALPHA, NAN, OFF, Checks, L, act_input, concat, mode, out_buf, ref_conv, ref_wgrad, rnd, tf32, unpack  # noqa: F401,E501
from test_gpu_engine import act_deriv as _act_deriv, act_ref as _act_ref
from test_gpu_reproducible import twice
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
SC = 'generator/rnn/savp_cell'
PLAIN, DECONV = 0, 3
LRELU, ELU = 2, 5
S2 = (1, 2, 2)
N_ODD = 3          # an odd batch: not a multiple of any box's batch depth


def _g(kind, k, ch, co, ext):
    ci_ref, ci_int, cmap = concat(*ch) if isinstance(ch, tuple) else (ch, ch, None)
    return (kind, k, ci_ref, ci_int, cmap, co, ext)


# (kind, k, ci_ref, ci_int, cmap, co, input extent) of the h{i} convolutions of the cfg2 64x64 and the 128x128 generator
# (ngf 32, nz 8) with downsample_layer='conv2d' (k x k, stride 2, pad (k - 2) // 2 before) and upsample_layer='deconv2d'
# (transposed 3x3, stride 2, pad 0 before)
GEOMS = [
    _g(PLAIN, 5, (3, 3, 8), 32, 64), _g(PLAIN, 3, 40, 64, 32), _g(PLAIN, 3, 72, 128, 16),                      # 64x64
    _g(DECONV, 3, 136, 64, 8), _g(DECONV, 3, 136, 32, 16), _g(DECONV, 3, 72, 32, 32),
    _g(PLAIN, 5, (3, 3, 8), 32, 128), _g(PLAIN, 3, 40, 64, 64), _g(PLAIN, 3, 72, 128, 32), _g(PLAIN, 3, 136, 256, 16),  # 128
    _g(DECONV, 3, 264, 256, 8), _g(DECONV, 3, 392, 128, 16), _g(DECONV, 3, 200, 64, 32), _g(DECONV, 3, 104, 32, 64),
]


def act_ref(v, act):
    """fp64 activation, VP_ACT_ELU included (tf.nn.elu)."""
    return torch.where(v > 0, v, torch.expm1(v.clamp(max=0))) if act == ELU else _act_ref(v, act)


def act_deriv(y, act):
    """act' from the activation output y in fp64; ELU: 1 above 0, y + 1 below."""
    return torch.where(y.double() > 0, 1.0, y.double() + 1.0) if act == ELU else _act_deriv(y, act)


def gid(c):
    return '%s%d_%d-%d_co%d_%d' % ('conv2d_k' if c[0] == PLAIN else 'deconv2d_k', c[1], c[2], c[3], c[5], c[6])


def _geometry(L, kind, k):  # noqa: F811
    """(forward geometry, dgrad geometry, out extent function) of a case, as savp_model's layer table builds them."""
    pad = (k - 2) // 2 if kind == PLAIN else 0
    t = kind == DECONV
    return L.geom((1, k, k), S2, (0, pad, pad), t), L.geom((1, k, k), S2, (0, pad, pad), not t), (0, pad, pad), t


def _eff(w, kind, cmap, ci_int):
    """Effective tap matrices [taps][ci_int][co] (fp64) of a reference-layout kernel: HWIO, or [3, 3, co, ci] for DECONV."""
    k = w.shape[0]
    w = w.double()
    if kind == DECONV:
        w = w.permute(0, 1, 3, 2)
    w = w.reshape(k * k, w.shape[2], w.shape[3])
    if cmap is None:
        return w
    out = w.new_zeros(k * k, ci_int, w.shape[2])
    for i, c in enumerate(cmap):
        if c >= 0:
            out[:, i] = w[:, c]
    return out


@pytest.mark.parametrize('case', GEOMS, ids=gid)
def test_new_geometries_match_fp64(L, mode, case):  # noqa: F811
    """Forward (bias + none / relu / lrelu / elu), dgrad, the fused activation-gradient dgrad (lrelu, elu) and the weight
    gradient (split_k 0, 1, 3) of each new geometry, with an odd batch, against ref_conv / ref_wgrad on the operands the
    tensor core reads, at test_gpu_engine.py's tolerances; the packs against the reference-layout kernel; unpack_wgrad
    back into that layout."""
    kind, k, ci_ref, ci_int, cmap, co, e = case
    g, gt, pad, transposed = _geometry(L, kind, k)
    ke, s, p = (1, k, k), S2, pad
    ext = (1, e, e)
    oext = (1, 2 * e, 2 * e) if transposed else (1, e // 2, e // 2)
    n = N_ODD
    taps = k * k
    ck = Checks(gid(case))
    kf = taps * ci_int / (4 if transposed else 1)
    kd = taps * co / (1 if transposed else 4)
    kw = n * (e * e if transposed else oext[1] * oext[2])
    cm = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device='cuda')
    wshape = (k, k, co, ci_ref) if kind == DECONV else (k, k, ci_ref, co)
    w = rnd(*wshape, seed=1, scale=(taps * ci_ref) ** -0.5)
    bias = rnd(co, seed=2, scale=0.3)
    wp, n_pad, kc = L.pack_weights(w, (1, k, k), ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm)
    wpd, n_pad_d, kc_d = L.pack_weights(w, (1, k, k), ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int, cmap=cm)
    wf, wd = unpack(wp, taps, n_pad, kc, co, ci_int), unpack(wpd, taps, n_pad_d, kc_d, ci_int, co)
    eff = _eff(w, kind, cmap, ci_int)
    tol = 2.0 ** -10 * eff.abs().max().item()           # TF32 rounding of the packed weights
    assert (wf - eff).abs().max().item() <= tol and (wd - eff.transpose(1, 2)).abs().max().item() <= tol

    x = act_input(n, ext, ci_int, cmap, seed=3)
    xv = L.tensor_view(x, ci_int)
    pre = ref_conv(tf32(x, mode)[..., :ci_int].double(), wf, ke, s, p, transposed, oext)
    for act in (L.ACT_NONE, L.ACT_RELU, L.ACT_LRELU, L.ACT_ELU):
        out = out_buf(n, oext, co)
        L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, co, OFF), bias, act, ALPHA)
        ck.close('fwd act %d' % act, 'fwd', out[..., OFF:OFF + co], act_ref(pre + bias.double(), act), kf)
        ck.untouched('fwd act %d' % act, out, co)

    dy = act_input(n, oext, (co + 3) // 4 * 4, None, seed=5)
    dy[..., co:] = NAN
    dyq = tf32(dy, mode)[..., :co].double()
    dyv = L.tensor_view(dy, co)
    dref = ref_conv(dyq, wd, ke, s, p, not transposed, ext)
    dx = out_buf(n, ext, ci_int)
    L.conv_igemm(dyv, gt, wpd, n_pad_d, kc_d, L.tensor_view(dx, ci_int, OFF))
    ck.close('dgrad', 'dgrad', dx[..., OFF:OFF + ci_int], dref, kd)
    ck.untouched('dgrad', dx, ci_int)
    add = rnd(n, *ext, ci_int, seed=6)
    for aux in (LRELU, ELU):
        y = act_ref(rnd(n, *ext, ci_int, seed=8).double(), aux).float()
        o = torch.full_like(add, NAN)
        L.conv_igemm_actgrad(dyv, gt, wpd, n_pad_d, kc_d, L.tensor_view(o, ci_int), y.data_ptr(), add.data_ptr(), aux, ALPHA, 0)
        ck.close('actgrad %d + addend' % aux, 'actgrad', o, (dref + add.double()) * act_deriv(y, aux), kd)

    wref = ref_wgrad(tf32(x, mode)[..., :ci_int].double(), dyq, ke, s, p, transposed).transpose(1, 2)    # [taps][co][ci]
    full = torch.zeros(taps, n_pad, kc * 32, device='cuda', dtype=torch.float64)
    full[:, :co, :ci_int] = wref
    for split in (0, 1, 3):
        dwp = torch.zeros(taps * n_pad * kc * 32, device='cuda')
        L.conv_wgrad(xv, dyv, g, dwp, n_pad, kc, split)
        ck.close('wgrad split_k %d' % split, 'wgrad', dwp.view(taps, n_pad, kc * 32), full, kw)
    # unpack_wgrad into the reference layout (accumulating): DECONV gradients come back as [3, 3, co, ci]
    dw0 = rnd(*wshape, seed=11)
    dw = dw0.clone()
    L.unpack_wgrad(dwp, (1, k, k), ci_ref, co, kind, dw, n_pad, kc, ci_int=ci_int, cmap=cm)
    want = torch.zeros(taps, ci_ref, co, dtype=torch.float64, device='cuda')
    for i, c in enumerate(cmap if cmap is not None else range(ci_int)):
        if c >= 0:
            want[:, c] += wref.transpose(1, 2)[:, i]
    want = want.reshape(k, k, ci_ref, co)
    if kind == DECONV:
        want = want.permute(0, 1, 3, 2)
    ck.close('unpack_wgrad', 'wgrad', dw - dw0, want, kw)
    ck.done()


@pytest.mark.parametrize('case', [GEOMS[1], GEOMS[3], GEOMS[10]], ids=gid)
def test_new_geometries_exact_mode(L, case):  # noqa: F811
    """The fp32-exact 3xTF32 mode (residual packs, conv3x) of a conv2d and two deconv2d geometries against fp64 on the raw
    operands, forward and dgrad."""
    from video_prediction_b200.models.savp_model import conv3x
    kind, k, ci_ref, ci_int, cmap, co, e = case
    assert cmap is None
    g, gt, p, transposed = _geometry(L, kind, k)
    ext = (1, e, e)
    oext = (1, 2 * e, 2 * e) if transposed else (1, e // 2, e // 2)
    n, taps = N_ODD, k * k
    ck = Checks(gid(case) + ' [exact]')
    wshape = (k, k, co, ci_ref) if kind == DECONV else (k, k, ci_ref, co)
    w = rnd(*wshape, seed=1, scale=(taps * ci_ref) ** -0.5)
    bias = rnd(co, seed=2, scale=0.3)
    pk = {lay: L.pack_weights(w, (1, k, k), ci_ref, co, kind, lay, ci_int=ci_int)
          for lay in (L.WLAYOUT_FWD, L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL, L.WLAYOUT_DGRAD, L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL)}
    eff = _eff(w, kind, None, ci_int)
    x = act_input(n, ext, ci_int, None, seed=3)
    pre = ref_conv(x[..., :ci_int].double(), eff, (1, k, k), S2, p, transposed, oext)
    out = out_buf(n, oext, co)
    (wp, n_pad, kc), (wlo, _, _) = pk[L.WLAYOUT_FWD], pk[L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL]
    conv3x(x, ci_int, g, wp, wlo, n_pad, kc, L.tensor_view(out, co, OFF), bias, L.ACT_ELU, 0.0)
    ck.close('conv3x forward + bias + elu', 'fwd', out[..., OFF:OFF + co], act_ref(pre + bias.double(), ELU), taps * ci_int,
             exact=True)
    dy = act_input(n, oext, co, None, seed=5)
    dref = ref_conv(dy[..., :co].double(), eff.transpose(1, 2), (1, k, k), S2, p, not transposed, ext)
    dx = out_buf(n, ext, ci_int)
    (wpd, n_pad_d, kc_d), (wdlo, _, _) = pk[L.WLAYOUT_DGRAD], pk[L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL]
    conv3x(dy, co, gt, wpd, wdlo, n_pad_d, kc_d, L.tensor_view(dx, ci_int, OFF), None, L.ACT_NONE, 0.0)
    ck.close('conv3x dgrad', 'dgrad', dx[..., OFF:OFF + ci_int], dref, taps * co, exact=True)
    ck.done()


def test_new_geometry_reruns_are_bit_identical(L):  # noqa: F811
    for case in (GEOMS[0], GEOMS[3]):
        kind, k, ci_ref, ci_int, cmap, co, e = case
        g, gt, _, transposed = _geometry(L, kind, k)
        cm = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device='cuda')
        wshape = (k, k, co, ci_ref) if kind == DECONV else (k, k, ci_ref, co)
        w = rnd(*wshape, seed=1, scale=0.1)
        wp, n_pad, kc = L.pack_weights(w, (1, k, k), ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm)
        x = act_input(N_ODD, (1, e, e), ci_int, cmap, seed=3)[..., :ci_int].contiguous()
        oe = 2 * e if transposed else e // 2
        out = torch.zeros(N_ODD, 1, oe, oe, co, device='cuda')
        dy = rnd(N_ODD, 1, oe, oe, co, seed=4)
        dwp = torch.zeros(k * k * n_pad * kc * 32, device='cuda')
        bias = rnd(co, seed=2)
        twice(lambda: L.conv_igemm(L.tensor_view(x, ci_int), g, wp, n_pad, kc, L.tensor_view(out, co), bias, L.ACT_RELU), [out],
              'conv ' + gid(case))
        twice(lambda: L.conv_wgrad(L.tensor_view(x, ci_int), L.tensor_view(dy, co), g, dwp, n_pad, kc, 0), [dwp], 'wgrad ' + gid(case))


def test_bad_weight_kinds_are_rejected_and_write_nothing(L):  # noqa: F811
    C = 32
    w = torch.randn(3, 3, C, C, device='cuda')
    wp, n_pad, kc = L.pack_weights(w, (1, 3, 3), C, C, DECONV, L.WLAYOUT_FWD)
    wbuf, dw = torch.full_like(wp, 7.0), torch.full((3, 3, C, C), 7.0, device='cuda')
    for kind in (-1, 4):
        with pytest.raises(L.VpError):
            L.pack_weights(w, (1, 3, 3), C, C, kind, L.WLAYOUT_FWD, out=wbuf)
        with pytest.raises(L.VpError):
            L.unpack_wgrad(wp, (1, 3, 3), C, C, kind, dw, n_pad, kc)
        with pytest.raises(L.VpError):
            L.PackPlan([(w, (1, 3, 3), C, C, kind, L.WLAYOUT_FWD, None, None, None, wbuf)])
    torch.cuda.synchronize()
    assert bool((wbuf == 7.0).all()) and bool((dw == 7.0).all())


# ------------------------------------------------------------------------------------------------ VP_ACT_ELU in the fused kernels
def _slab(N, P, C, cs, seed, off=0):
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((N, P, cs), NAN)
    buf[..., off:off + C] = torch.randn(N, P, C, generator=g) + 0.3 * torch.arange(C) / C
    return buf.cuda()


def _norm64(x, g, b, layer):
    dims = (1, 2) if layer else (1,)
    m = x.mean(dim=dims, keepdim=True)
    v = ((x - m) ** 2).mean(dim=dims, keepdim=True)
    return act_ref((x - m) * torch.rsqrt(v + (1e-12 if layer else 1e-6)) * g + b, ELU)


# (positions, channels): the cluster / slab kernels at the generator's extents (the 4096 x 32 backward is the loop kernel),
# and the fallback kernels of instance norm (channels not a multiple of 32, or a plane that is not a power of two)
NORM_EXTENTS = [(1024, 32), (256, 64), (64, 128), (4096, 32), (64, 256), (100, 12), (48, 36)]


@pytest.mark.parametrize('layer', [False, True], ids=['inorm', 'lnorm'])
@pytest.mark.parametrize('ext', NORM_EXTENTS, ids=lambda e: '%dx%d' % e)
def test_norm_act_elu_matches_fp64(L, ext, layer):  # noqa: F811
    """vp_inorm_act / vp_lnorm_act (forward) and their backward with VP_ACT_ELU against fp64 autograd, N = 5, strided
    slices; only the slice is written; bit-identical reruns."""
    P, C = ext
    N = 5
    fwd, bwd = (L.lnorm_act, L.lnorm_act_bwd) if layer else (L.inorm_act, L.inorm_act_bwd)
    x = _slab(N, P, C, C + 8, seed=P + C, off=4)
    gr = torch.Generator().manual_seed(1)
    g = (1.0 + 0.3 * torch.randn(C, generator=gr)).cuda()
    b = (0.2 * torch.randn(C, generator=gr)).cuda()
    y = torch.full((N, P, C + 4), NAN, device='cuda')
    st = torch.zeros(*((N, 2) if layer else (N, C, 2)), device='cuda')
    fwd(x.data_ptr() + 16, C + 8, y.data_ptr(), C + 4, N, P, C, g, b, L.ACT_ELU, 0.0, st)
    torch.cuda.synchronize()
    x64 = x[..., 4:4 + C].double()
    want = _norm64(x64, g.double(), b.double(), layer)
    assert (y[..., :C].double() - want).abs().max().item() <= 2e-5 * max(1.0, want.abs().max().item())
    assert torch.isnan(y[..., C:]).all()
    dys = _slab(N, P, C, C, seed=7)
    dx = torch.full((N, P, C + 4), NAN, device='cuda')
    dg0, db0 = torch.randn(C, generator=gr).cuda(), torch.randn(C, generator=gr).cuda()
    dg, db = dg0.clone(), db0.clone()
    bwd(x.data_ptr() + 16, C + 8, [(dys.data_ptr(), C)], dx.data_ptr(), C + 4, N, P, C, g, b, st, L.ACT_ELU, 0.0, dg, db)
    torch.cuda.synchronize()
    xg, g64, b64 = x64.clone().requires_grad_(True), g.double().requires_grad_(True), b.double().requires_grad_(True)
    (_norm64(xg, g64, b64, layer) * dys.double()).sum().backward()
    for got, ref, what in ((dx[..., :C], xg.grad, 'dx'), (dg - dg0, g64.grad, 'dgamma'), (db - db0, b64.grad, 'dbeta')):
        err = (got.double() - ref).abs().max().item() / max(1e-30, ref.abs().max().item())
        assert err <= 5e-5, (ext, layer, what, err)
    assert torch.isnan(dx[..., C:]).all()
    y2, dx2 = torch.zeros(N, P, C, device='cuda'), torch.zeros(N, P, C, device='cuda')
    st2 = torch.zeros_like(st)
    dg2, db2 = dg0.clone(), db0.clone()
    twice(lambda: fwd(x.data_ptr() + 16, C + 8, y2.data_ptr(), C, N, P, C, g, b, L.ACT_ELU, 0.0, st2), [y2, st2], 'norm elu')
    twice(lambda: bwd(x.data_ptr() + 16, C + 8, [(dys.data_ptr(), C)], dx2.data_ptr(), C, N, P, C, g, b, st2, L.ACT_ELU, 0.0,
                      dg2, db2), [dx2, dg2, db2], 'norm elu bwd')


def test_act_bwd_elu_matches_fp64(L):  # noqa: F811
    """vp_act_bwd (the norm_layer='none' sites' backward) with VP_ACT_ELU: (dy_a + dy_b) * elu'(y) from the output."""
    rows, C = 3000, 36
    y = act_ref(rnd(rows, C, seed=1, scale=3.0).double(), ELU).float()
    a, b2 = rnd(rows, C + 4, seed=2), rnd(rows, C, seed=3)
    dx = torch.full((rows, C + 8), NAN, device='cuda')
    L.act_bwd(y.data_ptr(), C, a.data_ptr(), C + 4, b2.data_ptr(), C, dx.data_ptr(), C + 8, rows, C, L.ACT_ELU)
    torch.cuda.synchronize()
    want = (a[:, :C].double() + b2.double()) * act_deriv(y, ELU)
    assert (dx[:, :C].double() - want).abs().max().item() <= 1e-6 * want.abs().max().item()
    assert torch.isnan(dx[:, C:]).all()
    out = torch.zeros(rows, C, device='cuda')
    twice(lambda: L.act_bwd(y.data_ptr(), C, a.data_ptr(), C + 4, 0, C, out.data_ptr(), C, rows, C, L.ACT_ELU), [out], 'act_bwd elu')


def test_bad_activations_are_rejected_and_write_nothing(L):  # noqa: F811
    C, N, P = 32, 2, 64
    x = torch.randn(N, 1, 8, 8, C, device='cuda')
    w = torch.randn(3, 3, C, C, device='cuda')
    wp, n_pad, kc = L.pack_weights(w, (1, 3, 3), C, C, PLAIN, L.WLAYOUT_FWD)
    out = torch.full((N, 1, 4, 4, C), 7.0, device='cuda')
    g = L.geom((1, 3, 3), S2, (0, 0, 0))
    y = torch.randn(N, 1, 8, 8, C, device='cuda')
    gm, be = torch.ones(C, device='cuda'), torch.zeros(C, device='cuda')
    st = torch.zeros(N, C, 2, device='cuda')
    dg, db = torch.full((C,), 7.0, device='cuda'), torch.full((C,), 7.0, device='cuda')
    dx = torch.full((N * P, C), 7.0, device='cuda')
    for bad in (-1, 6, 99):
        with pytest.raises(L.VpError):
            L.conv_igemm(L.tensor_view(x, C), g, wp, n_pad, kc, L.tensor_view(out, C), None, bad)
        with pytest.raises(L.VpError):
            L.conv_igemm_actgrad(L.tensor_view(x, C), g, wp, n_pad, kc, L.tensor_view(out, C), y.data_ptr(), 0, bad)
        with pytest.raises(L.VpError):
            L.act_bwd(y.data_ptr(), C, y.data_ptr(), C, 0, C, dx.data_ptr(), C, N * P, C, bad)
        for fwd, stats in ((L.inorm_act, st), (L.lnorm_act, torch.zeros(N, 2, device='cuda'))):
            with pytest.raises(L.VpError):
                fwd(y.data_ptr(), C, dx.data_ptr(), C, N, P, C, gm, be, bad, 0.0, stats)
        for bwd, stats in ((L.inorm_act_bwd, st), (L.lnorm_act_bwd, torch.zeros(N, 2, device='cuda'))):
            with pytest.raises(L.VpError):
                bwd(y.data_ptr(), C, [(y.data_ptr(), C)], dx.data_ptr(), C, N, P, C, gm, be, stats, bad, 0.0, dg, db)
    torch.cuda.synchronize()
    for t in (out, dx, dg, db):
        assert bool((t == 7.0).all())


# ------------------------------------------------------------------------------------------------ model level
@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def _params(hp, shape, seed=0):
    """Reference initial values with random norm parameters and cell biases (ones / zeros at init), and with
    norm_layer='none' random generator biases too: with zero biases and no normaliser a site's pre-activation sits at 0
    wherever its inputs do, where relu's branch is a rounding decision.  (Before a normaliser a bias cancels.)"""
    params, _ = R.init_params(hp, shape, seed=seed)
    g = torch.Generator().manual_seed(seed + 13)
    for k in list(params):
        if k.endswith(('/gamma', '/beta')) or k.endswith('basic_conv2dlstm_cell/bias') or \
                (hp.norm_layer == 'none' and k.startswith('generator/') and k.endswith('/bias')):
            params[k] = params[k] + torch.randn(params[k].shape, generator=g) * 0.2
    return params


BOTH = dict(downsample_layer='conv2d', upsample_layer='deconv2d')
ALL3 = dict(BOTH, activation_layer='elu')
GEN_CASES = {
    'vae_both': (dict(context_frames=2, sequence_length=12, nz=8, **BOTH), 4, (64, 64, 3)),
    'vae_conv2d': (dict(context_frames=2, sequence_length=8, nz=8, downsample_layer='conv2d'), 3, (64, 64, 3)),
    'det_deconv2d': (dict(context_frames=2, sequence_length=8, nz=0, upsample_layer='deconv2d'), 3, (64, 64, 3)),
    'vae_elu': (dict(context_frames=2, sequence_length=8, nz=8, activation_layer='elu'), 3, (64, 64, 3)),
    'v2': (dict(context_frames=2, sequence_length=8, nz=8, downsample_layer='conv_pool2d_v2',
                upsample_layer='upsample_conv2d_v2'), 3, (64, 64, 3)),
    'det_both_128': (dict(context_frames=2, sequence_length=6, nz=0, **BOTH), 2, (128, 128, 3)),
    'vae_all3_flow': (dict(context_frames=2, sequence_length=8, nz=8, transformation='flow', **ALL3), 3, (64, 64, 3)),
    'vae_all3_layer': (dict(context_frames=2, sequence_length=8, nz=8, norm_layer='layer', **ALL3), 3, (64, 64, 3)),
    'vae_all3_none': (dict(context_frames=2, sequence_length=8, nz=8, norm_layer='none', **ALL3), 3, (64, 64, 3)),
    'vae_all3_plain_cell': (dict(context_frames=2, sequence_length=8, nz=8, conv_rnn_norm_layer='none', **ALL3), 3, (64, 64, 3)),
    'det_all3_none_plain_cell': (dict(context_frames=2, sequence_length=8, nz=0, norm_layer='none', conv_rnn_norm_layer='none',
                                      **ALL3), 3, (64, 64, 3)),
}


# TF32 error fed back through the predicted frames: 1.09e-3 measured on an H100 for the 128x128 case (2 + 4 frames), whose
# frames pass through one more encoder / decoder level than the 64x64 ones
GEN_TOL = {'det_both_128': 2e-3}


@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_matches_oracle(Model, case):
    """gen_images (and gen_images_enc) within 1e-3 max-abs of the fp32 reference, as test_gpu_parity.py (GEN_TOL above)."""
    hk, B, shape = GEN_CASES[case]
    hp = O.make_hparams(**hk)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, seed=0)
    with torch.no_grad():
        ref = R.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B, None))
    model = Model(mode='test', hparams_dict=hk)
    model.set_params(params)
    binp = _batch_major(inputs)
    model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=False)
    model.generator_forward()
    torch.cuda.synchronize()
    report = {}
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - ref[k]).abs().max().item()
        report[k] = err
        assert err <= GEN_TOL.get(case, 1e-3), (case, k, err)
    print('layer choices generator %s: max-abs %s' % (case, {k: '%.2e' % v for k, v in report.items()}))


TRAIN_CASES = {
    'savp_both': dict(context_frames=2, sequence_length=8, clip_length=6, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
                      video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0,
                      kl_anneal_steps=(0, 10), **BOTH),
    'savp_all3': dict(context_frames=2, sequence_length=8, clip_length=6, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
                      video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0,
                      kl_anneal_steps=(0, 10), **ALL3),
    'vae_l1_both_none': dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3, kl_anneal_steps=(0, 10),
                             lr=1e-3, norm_layer='none', **BOTH),
    'vae_l1_all3_none': dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3, kl_anneal_steps=(0, 10),
                             lr=1e-3, norm_layer='none', **ALL3),
}
GTOL_OF = {'savp_both': 'savp', 'savp_all3': 'savp', 'vae_l1_both_none': 'vae_l1', 'vae_l1_all3_none': 'vae_l1'}


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return R.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_matches_fp32_oracle(Model, case, arith):
    """64x64, B = 2, random scheduled-sampling mask, the tolerances of test_gpu_norm_layer.py (the norm-free sites' bias
    gradients get the TF32 floor of 1e-1 there too)."""
    hk = TRAIN_CASES[case]
    hp = O.make_hparams(**hk)
    B, step, shape = 2, 5, (64, 64, 3)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape)
    sampling = torch.rand(hp.sequence_length - 1 - hp.context_frames, B, generator=torch.Generator().manual_seed(7)) < 0.5
    _, ltol, floor, otol = MODES[arith]
    with arithmetic(arith):
        model = Model(mode='train', hparams_dict=hk)
        model.set_params(params)
        model.build_graph(_batch_major(inputs))
    model.global_step = step
    model.train_step(_batch_major(inputs), noise, sampling=sampling)
    torch.cuda.synchronize()
    lv = model.losses()
    res = _oracle_step(hp, params, inputs, noise, step, sampling, None)
    emu = _oracle_step(hp, params, inputs, noise, step, sampling, tf32_mode()) if arith == 'tf32' else None
    ref_l = dict(res['g_losses'])
    ref_l.update(res.get('d_losses', {}))
    emu_l = {} if emu is None else dict(emu['g_losses'], **emu.get('d_losses', {}))
    for k, v in ref_l.items():
        tol = max(ltol * abs(v), 2.0 * abs(emu_l[k] - v) if emu_l else 0.0)
        assert abs(lv[k] - v) <= tol + 1e-6, (k, lv[k], v, emu_l.get(k))
    worst, bad = [], []
    none = hk.get('norm_layer') == 'none'
    for kind in ('g_grads', 'd_grads'):
        if kind not in res:
            continue
        items = [(k, g) for k, g in res[kind].items() if g is not None]
        gmax = max(g.double().norm().item() for _, g in items)
        for k, g in items:
            r, n = _rel(model.grads[k], g)
            if n < floor * gmax:
                continue
            floor_tf32 = 1e-1 if none and k.endswith('/bias') and k.startswith('generator/') else 5e-2
            tol = EXACT_GTOL[GTOL_OF[case]] if emu is None else max(floor_tf32, 2.0 * _rel(emu[kind][k], g)[0])
            worst.append((r, tol, k))
            if r > tol:
                bad.append((r, tol, k))
    worst.sort(reverse=True)
    print('layer choices %s [%s]: worst gradient errors %s' % (case, arith, ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    named = [k for k in res['g_grads'] if '/conv2d/kernel' in k and '/h' in k] + [k for k in res['g_grads'] if '/deconv2d/kernel' in k]
    assert named and all(float(model.grads[k].abs().max()) > 0 for k in named), named
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)


def test_captured_step_reproduces_the_eager_step(Model, tmp_path):
    """The eager step and two graph replays from the same checkpoint give bit-identical losses and gradients."""
    hk = TRAIN_CASES['savp_all3']
    hp = O.make_hparams(**hk)
    params = _params(hp, (64, 64, 3))
    inputs, _ = O.make_synthetic_inputs(hp, 2, (64, 64, 3))
    binp = _batch_major(inputs)
    runs = {}
    for how in ('eager', 'graph'):
        model = Model(mode='train', hparams_dict=hk)
        model.set_params(params)
        model.build_graph(binp)
        model.use_cuda_graph = how == 'graph'
        model.train_step(binp)
        ck = model.save(str(tmp_path / how))
        runs[how] = []
        for _ in range(2 if how == 'graph' else 1):
            model.restore(None, ck)
            model.train_step(binp)
            torch.cuda.synchronize()
            assert (model._graph is not None) == (how == 'graph')
            runs[how].append((model.loss_vals.clone(), model.g_grad.clone(), model.d_grad.clone()))
    ref = runs['eager'][0]
    for got in runs['graph']:
        for name, a, b in zip(('losses', 'g_grad', 'd_grad'), got, ref):
            assert torch.equal(a, b), (name, (a - b).abs().max().item())
    assert float(ref[1].abs().max()) > 0 and bool(torch.isfinite(ref[1]).all())


def test_tf_bundle_with_conv2d_deconv2d_names_restores_exactly(Model, tmp_path):
    """A reference checkpoint (TF tensor bundle) of a conv2d / deconv2d SAVP under the historical 'dna_cell' scope restores
    every variable bit for bit, deconv2d kernels in their [3, 3, oc, cin] layout, and the generator then matches the
    reference run on the same values."""
    from test_tf_checkpoint import write_bundle
    hk = dict(context_frames=2, sequence_length=4, nz=8, **BOTH)
    hp = O.make_hparams(**hk)
    params = _params(hp, (64, 64, 3), seed=3)
    assert SC + '/h0/conv2d/kernel' in params and params[SC + '/h3/deconv2d/kernel'].shape == (3, 3, 64, 136)
    inputs, noise = O.make_synthetic_inputs(hp, 1, (64, 64, 3))
    model = Model(mode='test', hparams_dict=hk)
    model.build_graph(_batch_major(inputs))
    tensors = {k.replace('savp_cell', 'dna_cell'): v.numpy().astype(np.float32) for k, v in params.items() if k.startswith('generator/')}
    tensors['global_step'] = np.array(77, np.int64)
    prefix = str(tmp_path / 'model-77')
    write_bundle(prefix, tensors)
    model.restore(None, prefix)
    assert model.global_step == 77
    for k, v in params.items():
        if k.startswith('generator/'):
            assert np.array_equal(model.params[k].cpu().numpy(), v.numpy().astype(np.float32)), k
    model.set_inputs(_batch_major(inputs), noise, sampling=False)
    model.generator_forward()
    with torch.no_grad():
        ref = R.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, 1, None))
    assert (model.outputs_time_major('gen_images').cpu() - ref['gen_images']).abs().max().item() <= 1e-3
