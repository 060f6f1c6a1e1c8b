"""CPU tests of the generator's normaliser choice norm_layer = 'instance' | 'layer' | 'none': the reference
(tests/savp_norm_layer_oracle.py) against a numpy restatement of tf.contrib.layers.layer_norm, the unchanged default, the
model's parameter specs against the reference's variables, and which hparams the model accepts."""
import numpy as np
import pytest
import torch

import savp_norm_layer_oracle as R
from oracle import savp_oracle as O

SC = 'generator/rnn/savp_cell'
CFG2 = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, state_weight=0.0,
            context_frames=2, sequence_length=12)
TINY = dict(context_frames=2, sequence_length=4, nz=4, ngf=8, nef=8)


def _numpy_layer_norm_lrelu(x, g, b, alpha=0.2):
    """tf.contrib.layers.layer_norm(begin_norm_axis=1, begin_params_axis=-1), float32 epsilon 1e-12, then leaky relu."""
    n = x.shape[0]
    flat = x.reshape(n, -1)
    mean = flat.mean(axis=1).reshape((n,) + (1,) * (x.ndim - 1))
    var = ((x - mean) ** 2).reshape(n, -1).mean(axis=1).reshape(mean.shape)
    y = g * (x - mean) / np.sqrt(var + 1e-12) + b
    return np.maximum(alpha * y, y)


def test_layer_norm_site_matches_numpy():
    """An encoder site (layer_2) with norm_layer='layer' is layer norm over H, W, C; a ConvLSTM norm under the same
    variant stays instance norm; 'none' is the identity.  Inputs of variance ~1e-8 make eps = 1e-12 visible."""
    rng = np.random.default_rng(5)
    N, H, W, C = 3, 4, 5, 8
    g, b = rng.standard_normal(C), rng.standard_normal(C)
    for scale in (1.0, 1e-4):
        x = scale * rng.standard_normal((N, H, W, C)) + 0.3 * scale * np.arange(C)
        P = {'generator/encoder/layer_2/LayerNorm/gamma': torch.tensor(g), 'generator/encoder/layer_2/LayerNorm/beta': torch.tensor(b),
             SC + '/lstm_h0/InstanceNorm/gamma': torch.tensor(g), SC + '/lstm_h0/InstanceNorm/beta': torch.tensor(b)}
        V = O.Vars(P)
        with R.variant(O.make_hparams(norm_layer='layer')):
            gs = V.get('generator/encoder/layer_2/InstanceNorm/gamma', (C,), 'ones')
            bs = V.get('generator/encoder/layer_2/InstanceNorm/beta', (C,), 'zeros')
            y = O.lrelu(O.instance_norm(torch.tensor(x), gs, bs), 0.2).numpy()
            gl = V.get(SC + '/lstm_h0/InstanceNorm/gamma', (C,), 'ones')
            yi = O.instance_norm(torch.tensor(x), gl, V.get(SC + '/lstm_h0/InstanceNorm/beta', (C,), 'zeros')).numpy()
        want = _numpy_layer_norm_lrelu(x, g, b)
        assert np.abs(y - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), scale
        m, v = x.mean(axis=(1, 2), keepdims=True), x.var(axis=(1, 2), keepdims=True)
        assert np.abs(yi - (g * (x - m) / np.sqrt(v + 1e-6) + b)).max() < 1e-12
        with R.variant(O.make_hparams(norm_layer='none')):
            gs = V.get('generator/encoder/layer_2/InstanceNorm/gamma', (C,), 'ones')
            assert gs is R.NO_NORM
            assert np.array_equal(O.instance_norm(torch.tensor(x), gs, gs).numpy(), x)
    assert O.Vars.get is not None and O.instance_norm.__module__ == O.__name__     # restored after the calls


def test_instance_leaves_the_oracle_bit_identical():
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


def test_variants_change_only_the_site_norms():
    """'layer' renames every site norm (same values, same kernels), 'none' drops them; the ConvLSTM's norms stay; the
    variants compose with the norm-free cell; and the generator's output does depend on the choice."""
    hp = O.make_hparams(**TINY)
    base, _ = R.init_params(hp, (32, 32, 3), seed=2)
    sites = [k for k in base if R.SITE.search(k)]
    assert len(sites) == 2 * (4 + 2 + 2)       # 32x32: h0..h3, h4_scratch, h4_masks, encoder layer_2 and layer_3
    lay, _ = R.init_params(O.make_hparams(**dict(TINY, norm_layer='layer')), (32, 32, 3), seed=2)
    non, _ = R.init_params(O.make_hparams(**dict(TINY, norm_layer='none')), (32, 32, 3), seed=2)
    assert list(lay) == [R.site_name(k, 'layer') for k in base]
    assert all(torch.equal(lay[R.site_name(k, 'layer')], v) for k, v in base.items())
    assert list(non) == [k for k in base if k not in sites]
    assert any('/basic_conv2dlstm_cell/state/gamma' in k for k in lay)
    mixed, _ = R.init_params(O.make_hparams(**dict(TINY, norm_layer='layer', conv_rnn_norm_layer='none')), (32, 32, 3), seed=2)
    assert SC + '/h0/LayerNorm/gamma' in mixed and SC + '/lstm_h1/basic_conv2dlstm_cell/bias' in mixed
    abl, _ = R.init_params(O.make_hparams(**dict(TINY, norm_layer='none', ablation_conv_rnn_norm=True)), (32, 32, 3), seed=2)
    assert SC + '/lstm_h1/InstanceNorm/gamma' in abl and not any('/h1/InstanceNorm' in k or 'LayerNorm' in k for k in abl)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3))
    gt = O.ground_truth_mask(hp, 2)
    outs = {}
    with torch.no_grad():
        for norm, params in (('instance', base), ('layer', lay), ('none', non)):
            outs[norm] = R.generator(O.Vars(params), O.make_hparams(**dict(TINY, norm_layer=norm)), inputs, noise, gt)['gen_images']
    assert all(bool(torch.isfinite(v).all()) for v in outs.values())
    assert (outs['layer'] - outs['instance']).abs().max() > 1e-4 and (outs['none'] - outs['instance']).abs().max() > 1e-4


def _model(hk, H=64, W=64, mode='train'):
    from video_prediction_b200.models import SAVPVideoPredictionModel
    m = SAVPVideoPredictionModel(mode=mode, hparams_dict=hk)
    m.B, m.T, m.H, m.W, m.C, m.A, m.Sd = 1, hk['sequence_length'], H, W, 3, 0, 0
    m.S, m.Zc = m.T - 1, m.hparams.nz
    m.enc_specs, m.dec_specs = m.layer_specs(m.hparams.ngf, H, W)
    return m


def test_param_counts_at_cfg2():
    count = lambda specs: sum(int(np.prod(s)) for s, _ in specs.values())      # noqa: E731
    for norm, nz, want in (('instance', 8, 7349993), ('layer', 8, 7349993), ('none', 8, 7348393),
                           ('instance', 0, 6397177), ('layer', 0, 6397177), ('none', 0, 6396345)):
        specs = _model(dict(CFG2, norm_layer=norm, nz=nz))._generator_param_specs()
        assert count(specs) == want, (norm, nz, count(specs))
    specs = _model(dict(CFG2, norm_layer='layer'))._generator_param_specs()
    assert specs[SC + '/h0/LayerNorm/gamma'] == ((32,), 'ones') and specs['generator/encoder/layer_2/LayerNorm/beta'] == ((128,), 'zeros')
    assert not any('InstanceNorm' in k for k in specs)


@pytest.mark.parametrize('norm', ['layer', 'none'])
def test_param_specs_match_the_reference(norm):
    for nz, size in ((8, 64), (0, 64), (8, 128), (0, 128)):
        hk = dict(CFG2, nz=nz, norm_layer=norm, sequence_length=4)
        specs = _model(hk, size, size)._generator_param_specs()
        ref, _ = R.init_params(O.make_hparams(**dict(hk, video_sn_vae_gan_weight=0.0, video_sn_gan_weight=0.0)), (size, size, 3))
        gen_ref = {k: t for k, t in ref.items() if k.startswith('generator/')}
        assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
        for k, (shape, _) in specs.items():
            assert tuple(shape) == tuple(gen_ref[k].shape), k


def test_norm_layer_hparams_accepted_and_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    base = dict(context_frames=2, sequence_length=12)
    for norm in ('instance', 'layer', 'none'):
        for cell in (dict(), dict(conv_rnn_norm_layer='none'), dict(ablation_conv_rnn_norm=True)):
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, norm_layer=norm, **cell))._check_supported()
    for bad in ('batch', 'group'):
        with pytest.raises(NotImplementedError):
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, norm_layer=bad))._check_supported()
