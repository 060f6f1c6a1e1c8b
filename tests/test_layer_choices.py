"""CPU tests of the generator's layer choices downsample_layer / upsample_layer / activation_layer: the reference (tests/savp_layers_oracle.py) against numpy loops, the v2 recipes restated in numpy against the v1 layers,
the model's parameter specs against the reference's variables, and which hparams the model accepts."""
import itertools

import numpy as np
import pytest
import torch

import savp_layers_oracle as R
from oracle import savp_oracle as O

SC = 'generator/rnn/savp_cell'
CFG2 = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, state_weight=0.0,
            context_frames=2, sequence_length=12)
TINY = dict(context_frames=2, sequence_length=4, nz=4, ngf=8, nef=8)
DOWN = ('conv_pool2d', 'conv_pool2d_v2', 'conv2d')
UP = ('upsample_conv2d', 'upsample_conv2d_v2', 'deconv2d')
ACT = ('relu', 'elu')
CHOICES = [dict(downsample_layer='conv2d'), dict(upsample_layer='deconv2d'), dict(activation_layer='elu'),
           dict(downsample_layer='conv_pool2d_v2', upsample_layer='upsample_conv2d_v2'),
           dict(downsample_layer='conv2d', upsample_layer='deconv2d', activation_layer='elu')]


# ---------------------------------------------------------------------------------- numpy restatements (float64)
def np_conv(x, k, stride, pad_before, out_hw):
    """Cross-correlation of x [N, H, W, Ci] with k [kh, kw, Ci, Co]: out[o] = sum_r x[stride o + r - pad_before] k[r],
    zero outside x."""
    N, H, W, _ = x.shape
    kh, kw = k.shape[:2]
    Ho, Wo = out_hw
    out = np.zeros((N, Ho, Wo, k.shape[3]))
    for oy in range(Ho):
        for ox in range(Wo):
            for r in range(kh):
                for s in range(kw):
                    iy, ix = stride * oy + r - pad_before, stride * ox + s - pad_before
                    if 0 <= iy < H and 0 <= ix < W:
                        out[:, oy, ox] += x[:, iy, ix] @ k[r, s]
    return out


def np_deconv2d(x, k_t):
    """tf.nn.conv2d_transpose(x, k_t [3, 3, Co, Ci], output 2H x 2W, stride 2, SAME) by scattering: input row i reaches
    output row 2 i + r (the 2H -> H SAME conv pads 0 before)."""
    N, H, W, _ = x.shape
    out = np.zeros((N, 2 * H + 2, 2 * W + 2, k_t.shape[2]))
    for iy in range(H):
        for ix in range(W):
            for r in range(3):
                for s in range(3):
                    out[:, 2 * iy + r, 2 * ix + s] += x[:, iy, ix] @ k_t[r, s].T
    return out[:, :2 * H, :2 * W]


def np_vec_conv(x, k, pad_before, pad_after):
    """Stride-1 correlation with explicit zero padding, vectorised over taps."""
    xp = np.pad(x, ((0, 0), (pad_before, pad_after), (pad_before, pad_after), (0, 0)))
    kh, kw = k.shape[:2]
    Ho, Wo = xp.shape[1] - kh + 1, xp.shape[2] - kw + 1
    out = np.zeros((x.shape[0], Ho, Wo, k.shape[3]))
    for r in range(kh):
        for s in range(kw):
            out += np.einsum('nhwc,cd->nhwd', xp[:, r:r + Ho, s:s + Wo], k[r, s])
    return out


def np_conv_pool2d_v2(x, k, b):
    """ops.conv_pool2d_v2 (ops.py:859): SAME stride-1 conv, 2x2 average pool with stride 2, bias."""
    kk = k.shape[0]
    y = np_vec_conv(x, k, (kk - 1) // 2, kk - 1 - (kk - 1) // 2)
    N, H, W, C = y.shape
    return y.reshape(N, H // 2, 2, W // 2, 2, C).mean(axis=(2, 4)) + b


def np_upsample_conv2d_v2(x, k, b):
    """ops.upsample_conv2d_v2 (ops.py:722): bilinear VALID 2x upsample (conv2d_transpose with the 4x4 kernel outer([.25,
    .75, .75, .25]), output 2H + 2), FULL 3x3 conv (pad 2 / 2, output 2H + 4), crop from (2 - 0) // 2 + 2 - 1 = 2, bias."""
    N, H, W, C = x.shape
    b1 = np.array([0.25, 0.75, 0.75, 0.25])
    up = np.zeros((N, 2 * H + 2, 2 * W + 2, C))
    for r in range(4):
        for s in range(4):
            up[:, r:r + 2 * H:2, s:s + 2 * W:2] += b1[r] * b1[s] * x
    y = np_vec_conv(up, k, 2, 2)
    return y[:, 2:2 + 2 * H, 2:2 + 2 * W] + b


def _t(a):
    return torch.tensor(a, dtype=torch.float64)


# ---------------------------------------------------------------------------------- the reference's layers
@pytest.mark.parametrize('ks', [5, 3])
def test_same_stride2_conv_matches_numpy_loops(ks):
    """ops.conv2d(strides=2, SAME) on an even extent: pads (k - 2) // 2 before, the rest after."""
    rng = np.random.default_rng(ks)
    for H, W in ((8, 6), (4, 4)):
        x, k, b = rng.standard_normal((2, H, W, 3)), rng.standard_normal((ks, ks, 3, 5)), rng.standard_normal(5)
        got = R.conv2d_s2(_t(x), _t(k), _t(b)).numpy()
        want = np_conv(x, k, 2, (ks - 2) // 2, (H // 2, W // 2)) + b
        assert got.shape == want.shape and np.abs(got - want).max() < 1e-12


def test_deconv2d_matches_numpy_loops():
    rng = np.random.default_rng(3)
    for H, W in ((4, 3), (1, 1), (5, 5)):
        x, k, b = rng.standard_normal((2, H, W, 4)), rng.standard_normal((3, 3, 6, 4)), rng.standard_normal(6)
        got = R.deconv2d(_t(x), _t(k), _t(b)).numpy()
        want = np_deconv2d(x, k) + b
        assert got.shape == (2, 2 * H, 2 * W, 6) and np.abs(got - want).max() < 1e-12


def test_deconv2d_is_the_adjoint_of_the_same_stride2_conv():
    """<deconv(x), y> = <x, conv(y)> with the same kernel read as the conv's [3, 3, 2H-channels, H-channels] filter."""
    rng = np.random.default_rng(4)
    x, y, k = rng.standard_normal((1, 4, 4, 3)), rng.standard_normal((1, 8, 8, 5)), rng.standard_normal((3, 3, 5, 3))
    lhs = (R.deconv2d(_t(x), _t(k), _t(np.zeros(5))).numpy() * y).sum()
    rhs = (x * R.conv2d_s2(_t(y), _t(k), _t(np.zeros(3))).numpy()).sum()
    assert abs(lhs - rhs) < 1e-10 * max(1.0, abs(lhs))


def test_elu_matches_numpy():
    x = np.concatenate([np.linspace(-30, 30, 601), [0.0, -0.0, 1e-30, -1e-30, -1e-8]])
    assert np.abs(R.elu(_t(x)).numpy() - np.where(x > 0, x, np.expm1(x))).max() < 1e-15
    y = np.where(x > 0, x, np.expm1(x))
    xs = _t(x).requires_grad_()
    R.elu(xs).sum().backward()
    assert np.abs(xs.grad.numpy() - np.where(y > 0, 1.0, y + 1.0)).max() < 1e-15      # the derivative from the output


def _shapes(size, nz=8):
    """(cin, oc, input extent) of every encoder and decoder layer of the size x size generator (cfg2 widths)."""
    m = _model(dict(CFG2, nz=nz), size, size)
    enc, dec = m.enc_specs, m.dec_specs
    out, cin, ext = [], 6, size
    outs = []
    for oc, _ in enc:
        out.append(('enc', 5 if not outs else 3, cin + nz, oc, ext))
        outs.append(oc)
        cin, ext = oc, ext // 2
    n = len(enc)
    for i, (oc, _) in enumerate(dec):
        cin = outs[-1] if i == 0 else outs[-1] + outs[n - i - 1]
        out.append(('dec', 3, cin + nz, oc, ext))
        outs.append(oc)
        ext *= 2
    return out


@pytest.mark.parametrize('size', [64, 128])
def test_v2_recipes_equal_the_v1_layers(size):
    """conv_pool2d_v2 / upsample_conv2d_v2, unfolded in numpy, equal the oracle's folded v1 layers to 1e-10 (float64) at
    every encoder / decoder shape: the model runs them on the v1 packs."""
    rng = np.random.default_rng(size)
    for kind, ks, cin, oc, ext in _shapes(size):
        x = rng.standard_normal((1, ext, ext, cin))
        k, b = 0.1 * rng.standard_normal((ks, ks, cin, oc)), rng.standard_normal(oc)
        if kind == 'enc':
            want, got = np_conv_pool2d_v2(x, k, b), O.conv_pool2d(_t(x), _t(k), _t(b)).numpy()
        else:
            want, got = np_upsample_conv2d_v2(x, k, b), O.upsample_conv2d(_t(x), _t(k), _t(b)).numpy()
        assert got.shape == want.shape, (kind, ext)
        assert np.abs(got - want).max() <= 1e-10 * max(1.0, np.abs(want).max()), (kind, ext, np.abs(got - want).max())


# ---------------------------------------------------------------------------------- the variant oracle
def test_defaults_leave_the_oracle_bit_identical():
    hp = O.make_hparams(**TINY)
    a, ta = O.init_params(hp, (32, 32, 3), seed=2)
    b, tb = R.init_params(hp, (32, 32, 3), seed=2)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a) and ta == tb
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3))
    gt = O.ground_truth_mask(hp, 2)
    with torch.no_grad():
        want = O.generator(O.Vars(a), hp, inputs, noise, gt)
        got = R.generator(O.Vars(a), hp, inputs, noise, gt)
    assert list(want) == list(got) and all(torch.equal(want[k], got[k]) for k in want)
    assert O.torch is torch and O.conv_pool2d.__module__ == O.__name__ and O.upsample_conv2d.__module__ == O.__name__


def test_variants_rename_the_h_layers_and_change_the_output():
    hp = O.make_hparams(**TINY)
    base, _ = R.init_params(hp, (32, 32, 3), seed=2)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3))
    gt = O.ground_truth_mask(hp, 2)
    with torch.no_grad():
        ref = R.generator(O.Vars(base), hp, inputs, noise, gt)['gen_images']
    v2 = O.make_hparams(**dict(TINY, downsample_layer='conv_pool2d_v2', upsample_layer='upsample_conv2d_v2'))
    with torch.no_grad():
        assert torch.equal(R.generator(O.Vars(base), v2, inputs, noise, gt)['gen_images'], ref)
    for ch in CHOICES[:3] + CHOICES[4:]:
        hpv = O.make_hparams(**dict(TINY, **ch))
        p, _ = R.init_params(hpv, (32, 32, 3), seed=2)
        assert list(p) == [R.model_name(k, hpv) for k in base]
        for k, v in base.items():
            if k.endswith('/upsample_conv2d/kernel') and hpv.upsample_layer == 'deconv2d':
                assert p[R.model_name(k, hpv)].shape == v.permute(0, 1, 3, 2).shape
            else:
                assert torch.equal(p[R.model_name(k, hpv)], v), k
        with torch.no_grad():
            out = R.generator(O.Vars(p), hpv, inputs, noise, gt)['gen_images']
        assert bool(torch.isfinite(out).all()) and (out - ref).abs().max() > 1e-5, ch


def test_elu_applies_at_the_sites_only():
    """With 'elu' the site normalisers' outputs go through elu; any other relu of the oracle (the CDNA kernels') stays."""
    x = torch.linspace(-2, 2, 9).view(1, 1, 9, 1).double()
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    with R.variant(O.make_hparams(activation_layer='elu')):
        y = O.instance_norm(x, one, zero)
        assert torch.equal(O.torch.relu(y), R.elu(y)) and torch.equal(O.torch.relu(x), torch.relu(x))
    with R.variant(O.make_hparams(activation_layer='elu', norm_layer='none')):
        assert torch.equal(O.torch.relu(O.instance_norm(x, R.NL.NO_NORM, None)), R.elu(x))
    assert O.torch is torch


# ---------------------------------------------------------------------------------- the model's specs and hparams
def _model(hk, H=64, W=64, mode='train'):
    from video_prediction_b200.models import SAVPVideoPredictionModel
    m = SAVPVideoPredictionModel(mode=mode, hparams_dict=hk)
    m.B, m.T, m.H, m.W, m.C, m.A, m.Sd = 1, hk['sequence_length'], H, W, 3, 0, 0
    m.S, m.Zc = m.T - 1, m.hparams.nz
    m.enc_specs, m.dec_specs = m.layer_specs(m.hparams.ngf, H, W)
    return m


@pytest.mark.parametrize('choice', CHOICES)
def test_param_counts_at_cfg2(choice):
    count = lambda specs: sum(int(np.prod(s)) for s, _ in specs.values())      # noqa: E731
    for nz, want in ((8, 7349993), (0, 6397177)):
        specs = _model(dict(CFG2, nz=nz, **choice))._generator_param_specs()
        assert count(specs) == want, (choice, nz, count(specs))
    specs = _model(dict(CFG2, **choice))._generator_param_specs()
    down, up = choice.get('downsample_layer', 'conv_pool2d'), choice.get('upsample_layer', 'upsample_conv2d')
    assert (SC + '/h0/conv2d/kernel' in specs) == (down == 'conv2d')
    assert (SC + '/h3/deconv2d/kernel' in specs) == (up == 'deconv2d')
    if up == 'deconv2d':
        assert specs[SC + '/h3/deconv2d/kernel'] == ((3, 3, 64, 136), 'kernel')      # [3, 3, oc, cin]


@pytest.mark.parametrize('choice', CHOICES)
def test_param_specs_match_the_reference(choice):
    for nz, size in ((8, 64), (0, 64), (8, 128), (0, 128)):
        hk = dict(CFG2, nz=nz, sequence_length=4, **choice)
        specs = _model(hk, size, size)._generator_param_specs()
        ref, _ = R.init_params(O.make_hparams(**dict(hk, video_sn_vae_gan_weight=0.0, video_sn_gan_weight=0.0)), (size, size, 3))
        gen_ref = {k: t for k, t in ref.items() if k.startswith('generator/')}
        assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
        for k, (shape, _) in specs.items():
            assert tuple(shape) == tuple(gen_ref[k].shape), k


def test_layer_hparams_accepted_and_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    base = dict(context_frames=2, sequence_length=12)
    cells = (dict(), dict(conv_rnn_norm_layer='none'), dict(ablation_conv_rnn_norm=True))
    for down, up, act, norm, cell in itertools.product(DOWN, UP, ACT, ('instance', 'layer', 'none'), cells):
        hk = dict(base, downsample_layer=down, upsample_layer=up, activation_layer=act, norm_layer=norm, **cell)
        SAVPVideoPredictionModel(mode='train', hparams_dict=hk)._check_supported()
    for key, bad in (('downsample_layer', 'max_pool2d'), ('downsample_layer', 'conv3d'), ('upsample_layer', 'upsample2d'),
                     ('upsample_layer', 'deconv3d'), ('activation_layer', 'lrelu'), ('activation_layer', 'tanh')):
        with pytest.raises(ValueError, match='Invalid'):
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, **{key: bad}))._check_supported()


def test_layer_geometry_table():
    """The engine geometry of each h{i} choice: stride 2 everywhere; conv2d pads (k - 2) // 2 before (1 at k = 5, 0 at
    k = 3); deconv2d is a transposed 3x3 with pad 0 and the DECONV kernel kind."""
    from video_prediction_b200 import lib as L
    m = _model(dict(CFG2, downsample_layer='conv2d', upsample_layer='deconv2d'))
    assert m._hconv_layer(0, 14, 32) == (SC + '/h0/conv2d', (5, 5, 14, 32), L.WKIND_PLAIN, 5, 1, False)
    assert m._hconv_layer(1, 40, 64) == (SC + '/h1/conv2d', (3, 3, 40, 64), L.WKIND_PLAIN, 3, 0, False)
    assert m._hconv_layer(3, 136, 64) == (SC + '/h3/deconv2d', (3, 3, 64, 136), L.WKIND_DECONV, 3, 0, True)
    d = _model(dict(CFG2))
    assert d._hconv_layer(0, 14, 32) == (SC + '/h0/conv_pool2d', (5, 5, 14, 32), L.WKIND_POOLED, 5, 2, False)
    assert d._hconv_layer(4, 72, 32) == (SC + '/h4/upsample_conv2d', (3, 3, 72, 32), L.WKIND_UPSAMPLED, 3, 2, True)
    assert m.site_act == L.ACT_RELU and _model(dict(CFG2, activation_layer='elu')).site_act == L.ACT_ELU
