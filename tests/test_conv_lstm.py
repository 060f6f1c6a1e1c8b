"""CPU tests of the norm-free ConvLSTM forms (conv_rnn_norm_layer='none', ablation_conv_rnn_norm): the reference
(tests/savp_conv_lstm_oracle.py) against numpy loops and the closed form of the cell, the model's parameter specs, and
which hparams the model accepts."""
import numpy as np
import pytest
import torch

import savp_conv_lstm_oracle as R
from oracle import savp_oracle as O

SC = 'generator/rnn/savp_cell'
CFG2 = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, state_weight=0.0,
            context_frames=2, sequence_length=12)
VARIANTS = (dict(conv_rnn_norm_layer='none'), dict(ablation_conv_rnn_norm=True))


def _sig(v):
    return 1.0 / (1.0 + np.exp(-v))


def _numpy_cell(x, c, h, K, b, ablation=None):
    """rnn_ops.py:137-171 without norms, with explicit loops over the 5x5 SAME convolution."""
    B, H, W, _ = x.shape
    F = c.shape[-1]
    a = np.concatenate([x, h], axis=-1)
    z = np.zeros((B, H, W, 4 * F))
    for n in range(B):
        for y in range(H):
            for xx in range(W):
                acc = b.copy()
                for dy in range(5):
                    for dx in range(5):
                        sy, sx = y + dy - 2, xx + dx - 2
                        if 0 <= sy < H and 0 <= sx < W:
                            acc = acc + a[n, sy, sx] @ K[dy, dx]
                z[n, y, xx] = acc
    i, j, f, o = np.split(z, 4, axis=-1)
    c2 = c * _sig(f + 1.0) + _sig(i) * np.tanh(j)
    h2 = np.tanh(c2) * _sig(o)
    out = h2
    if ablation is not None:
        g, be = ablation
        m = h2.mean(axis=(1, 2), keepdims=True)
        v = ((h2 - m) ** 2).mean(axis=(1, 2), keepdims=True)
        out = (h2 - m) / np.sqrt(v + 1e-6) * g + be
    return out, c2, h2


@pytest.mark.parametrize('ablation', [False, True])
def test_cell_step_matches_a_numpy_loop(ablation):
    rng = np.random.default_rng(3)
    B, H, W, Ci, F = 2, 6, 5, 3, 4
    x, c, h = rng.standard_normal((B, H, W, Ci)), rng.standard_normal((B, H, W, F)), rng.standard_normal((B, H, W, F))
    K, b = 0.2 * rng.standard_normal((5, 5, Ci + F, 4 * F)), rng.standard_normal(4 * F)
    g, be = rng.standard_normal(F), rng.standard_normal(F)
    scope = SC + '/lstm_h0/basic_conv2dlstm_cell'
    P = {scope + '/kernel': torch.tensor(K), scope + '/bias': torch.tensor(b),
         SC + '/lstm_h0/InstanceNorm/gamma': torch.tensor(g), SC + '/lstm_h0/InstanceNorm/beta': torch.tensor(be)}
    cell = R.ablation_conv_lstm_cell if ablation else R.plain_conv_lstm_cell
    with torch.no_grad():
        out, (c2, h2) = cell(O.Vars(P), scope, torch.tensor(x), (torch.tensor(c), torch.tensor(h)), F)
    w_out, w_c, w_h = _numpy_cell(x, c, h, K, b, (g, be) if ablation else None)
    for got, want in ((out, w_out), (c2, w_c), (h2, w_h)):
        assert np.abs(got.numpy() - want).max() < 1e-12
    if not ablation:
        assert out is h2


def test_zero_kernel_gives_the_closed_form_of_the_bias():
    rng = np.random.default_rng(7)
    B, H, W, F = 2, 4, 4, 8
    b = rng.standard_normal(4 * F)
    c = rng.standard_normal((B, H, W, F))
    scope = SC + '/lstm_h1/basic_conv2dlstm_cell'
    P = {scope + '/kernel': torch.zeros(5, 5, 3 + F, 4 * F, dtype=torch.float64), scope + '/bias': torch.tensor(b)}
    with torch.no_grad():
        h, (c2, _) = R.plain_conv_lstm_cell(O.Vars(P), scope, torch.tensor(rng.standard_normal((B, H, W, 3))),
                                            (torch.tensor(c), torch.tensor(rng.standard_normal((B, H, W, F)))), F)
    bi, bj, bf, bo = np.split(b, 4)
    want_c = c * _sig(bf + 1.0) + _sig(bi) * np.tanh(bj)
    assert np.abs(c2.numpy() - want_c).max() < 1e-12
    assert np.abs(h.numpy() - np.tanh(want_c) * _sig(bo)).max() < 1e-12


def _model(hk, H=64, W=64, mode='train'):
    from video_prediction_b200.models import SAVPVideoPredictionModel
    m = SAVPVideoPredictionModel(mode=mode, hparams_dict=hk)
    m.B, m.T, m.H, m.W, m.C, m.A, m.Sd = 1, hk['sequence_length'], H, W, 3, 0, 0
    m.S, m.Zc = m.T - 1, m.hparams.nz
    m.enc_specs, m.dec_specs = m.layer_specs(m.hparams.ngf, H, W)
    return m


def test_param_specs_follow_the_reference_scopes():
    """cfg2: 7,349,993 generator variables with the instance-norm cell; the norm-free cell drops 6F per ConvLSTM (10F of
    norms for a 4F bias), the ablation 4F (plus 2F for the output norm)."""
    count = lambda specs: sum(int(np.prod(s)) for s, _ in specs.values())      # noqa: E731
    assert count(_model(CFG2)._generator_param_specs()) == 7349993
    none = _model(dict(CFG2, conv_rnn_norm_layer='none'))._generator_param_specs()
    abl = _model(dict(CFG2, ablation_conv_rnn_norm=True))._generator_param_specs()
    assert count(none) == 7348073 and count(abl) == 7348713
    b = SC + '/lstm_h1/basic_conv2dlstm_cell'
    assert none[b + '/bias'] == ((256,), 'zeros') and b + '/state/gamma' not in none
    assert abl[SC + '/lstm_h1/InstanceNorm/gamma'] == ((64,), 'ones') and SC + '/lstm_h1/InstanceNorm/beta' in abl
    for v in VARIANTS:
        for nz, size in ((8, 64), (0, 64), (8, 128)):
            hk = dict(CFG2, nz=nz, **v)
            specs = _model(hk, size, size)._generator_param_specs()
            ref, _ = R.init_params(O.make_hparams(**hk), (size, size, 3))
            gen_ref = {k: t for k, t in ref.items() if k.startswith('generator/')}
            assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
            for k, (shape, _) in specs.items():
                assert tuple(shape) == tuple(gen_ref[k].shape), k


def test_variant_reference_restores_the_oracle_and_defaults_are_unchanged():
    hp = O.make_hparams(context_frames=2, sequence_length=4, nz=4, ngf=8, nef=8)
    a, _ = O.init_params(hp, (32, 32, 3), seed=2)
    b, _ = R.init_params(hp, (32, 32, 3), seed=2)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    for v in VARIANTS:
        R.init_params(O.make_hparams(**dict(hp, **v)), (32, 32, 3), seed=2)
        assert O.conv_lstm_cell is not R.plain_conv_lstm_cell and O.conv_lstm_cell is not R.ablation_conv_lstm_cell


def test_conv_rnn_norm_hparams_accepted_and_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    base = dict(context_frames=2, sequence_length=12)
    for ok in (dict(conv_rnn_norm_layer='instance'), dict(conv_rnn_norm_layer='none'),
               dict(conv_rnn_norm_layer='instance', ablation_conv_rnn_norm=True)):
        SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, **ok))._check_supported()
    for bad in (dict(conv_rnn_norm_layer='layer'), dict(conv_rnn_norm_layer='batch'),
                dict(conv_rnn_norm_layer='layer', ablation_conv_rnn_norm=True)):
        with pytest.raises(NotImplementedError):
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, **bad))._check_supported()
    with pytest.raises(ValueError):
        SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, conv_rnn_norm_layer='none',
                                                                 ablation_conv_rnn_norm=True))._check_supported()
