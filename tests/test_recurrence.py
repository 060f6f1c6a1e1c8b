"""CPU tests of the SAVP cell's recurrence choices (ablation_rnn, use_rnn_z=False, rnn='gru', learn_initial_state): which
hparams the model
accepts, its variable names, shapes and initialisers against the reference (tests/savp_recurrence_oracle.py), the GRU step
against a numpy loop of TF's equations, and the ablation's conv_h site against the closed form of its bias."""
import numpy as np
import pytest
import torch

import savp_recurrence_oracle as R
from oracle import savp_oracle as O
from test_conv_lstm import CFG2, _model

SC = 'generator/rnn/savp_cell'
GRID = [dict(ablation_rnn=True), dict(use_rnn_z=False), dict(rnn='gru'), dict(ablation_rnn=True, use_rnn_z=False),
        dict(ablation_rnn=True, norm_layer='layer'), dict(ablation_rnn=True, norm_layer='none'),
        dict(rnn='gru', conv_rnn_norm_layer='none'), dict(ablation_rnn=True, conv_rnn_norm_layer='none',
                                                           ablation_conv_rnn_norm=True),
        dict(learn_initial_state=True), dict(learn_initial_state=True, rnn='gru'),
        dict(learn_initial_state=True, use_rnn_z=False), dict(learn_initial_state=True, ablation_rnn=True)]


def _sig(v):
    return 1.0 / (1.0 + np.exp(-v))


def test_hparams_accepted_and_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    base = dict(context_frames=2, sequence_length=12)
    for ok in GRID + [dict(rnn='gru', nz=0), dict(use_rnn_z=False, nz=0), dict(ablation_rnn=True, nz=0)]:
        SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, **ok))._check_supported()
    for bad in (dict(rnn='rnn'), dict(conv_rnn='gru'), dict(conv_rnn='gru', ablation_rnn=True),
                dict(conv_rnn_norm_layer='layer', ablation_rnn=True), dict(use_e_rnn=True), dict(learn_prior=True)):
        with pytest.raises(NotImplementedError):
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, **bad))._check_supported()


@pytest.mark.parametrize('hk', GRID, ids=lambda d: ','.join('%s=%s' % kv for kv in sorted(d.items())))
@pytest.mark.parametrize('nz,size', [(8, 64), (0, 64), (8, 128)])
def test_param_specs_follow_the_reference_scopes(hk, nz, size):
    hk = dict(CFG2, nz=nz, **hk)
    specs = _model(hk, size, size)._generator_param_specs()
    ref, _ = R.init_params(O.make_hparams(**hk), (size, size, 3))
    gen_ref = {k: t for k, t in ref.items() if k.startswith('generator/')}
    assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
    for k, (shape, init) in specs.items():
        assert tuple(shape) == tuple(gen_ref[k].shape), k
        if init in ('ones', 'zeros'):
            assert torch.equal(gen_ref[k], torch.full(shape, 1.0 if init == 'ones' else 0.0)), k
    names = '\n'.join(specs)
    assert ('lstm_h' in names) == (not hk.get('ablation_rnn'))
    assert ('/conv_h' in names) == bool(hk.get('ablation_rnn'))
    zcell = None if not nz or not hk.get('use_rnn_z', True) else ('fc' if hk.get('ablation_rnn') else hk.get('rnn', 'lstm'))
    for cell, scope in (('lstm', '/lstm_z/'), ('gru', '/gru_z/'), ('fc', '/fc_z/')):
        assert (scope in names) == (zcell == cell), (cell, zcell)


def test_new_variable_shapes_and_initialisers():
    abl = _model(dict(CFG2, ablation_rnn=True))._generator_param_specs()
    # h1 is the first layer with a ConvLSTM at 64x64 (ngf 32): 64 channels, input h1 (64) + z (8)
    assert abl[SC + '/conv_h0/conv2d/kernel'] == ((5, 5, 40, 32), 'kernel')
    assert abl[SC + '/conv_h1/conv2d/kernel'] == ((5, 5, 72, 64), 'kernel')
    assert abl[SC + '/conv_h1/conv2d/bias'] == ((64,), 'zeros')
    assert abl[SC + '/conv_h1/InstanceNorm/gamma'] == ((64,), 'ones')
    assert abl[SC + '/fc_z/dense/kernel'] == ((8, 8), 'kernel') and abl[SC + '/fc_z/dense/bias'] == ((8,), 'zeros')
    gru = _model(dict(CFG2, rnn='gru'))._generator_param_specs()
    g = SC + '/gru_z/gru_cell'
    assert gru[g + '/gates/kernel'] == ((16, 16), 'kernel') and gru[g + '/gates/bias'] == ((16,), 'ones')
    assert gru[g + '/candidate/kernel'] == ((16, 8), 'kernel') and gru[g + '/candidate/bias'] == ((8,), 'zeros')
    nozc = _model(dict(CFG2, use_rnn_z=False))._generator_param_specs()
    assert not [k for k in nozc if '_z/' in k]


def test_default_configuration_keeps_its_variables():
    """The default model's variables, in order, are those of the oracle with the default cells."""
    m = _model(CFG2)
    specs = m._generator_param_specs()
    count = sum(int(np.prod(s)) for s, _ in specs.values())
    assert count == 7349993
    ref, _ = O.init_params(O.make_hparams(**CFG2), (64, 64, 3))
    assert set(specs) == {k for k in ref if k.startswith('generator/')}
    assert m.z_cell == 'lstm'


def test_variant_reference_restores_the_oracle_and_defaults_are_unchanged():
    hp = O.make_hparams(context_frames=2, sequence_length=4, nz=4, ngf=8, nef=8)
    a, _ = O.init_params(hp, (32, 32, 3), seed=2)
    b, _ = R.init_params(hp, (32, 32, 3), seed=2)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    saved = O.conv_lstm_cell, O.dense_lstm_cell
    for v in GRID:
        R.init_params(O.make_hparams(**dict(hp, **v)), (32, 32, 3), seed=2)
        assert (O.conv_lstm_cell, O.dense_lstm_cell) == saved


def test_gru_step_matches_a_numpy_loop():
    rng = np.random.default_rng(5)
    B, nz = 3, 6
    x, h = rng.standard_normal((B, nz)), rng.standard_normal((B, nz))
    wg, bg = 0.3 * rng.standard_normal((2 * nz, 2 * nz)), rng.standard_normal(2 * nz)
    wc, bc = 0.3 * rng.standard_normal((2 * nz, nz)), rng.standard_normal(nz)
    g = SC + '/gru_z/gru_cell'
    P = {g + '/gates/kernel': torch.tensor(wg), g + '/gates/bias': torch.tensor(bg),
         g + '/candidate/kernel': torch.tensor(wc), g + '/candidate/bias': torch.tensor(bc)}
    with torch.no_grad():
        out, (_, h2) = R.gru_z_cell(O.Vars(P), SC + '/lstm_z/basic_lstm_cell', torch.tensor(x), (None, torch.tensor(h)), nz)
    want = np.zeros((B, nz))
    for b in range(B):
        for i in range(nz):
            u_pre = sum(np.concatenate([x[b], h[b]])[k] * wg[k, nz + i] for k in range(2 * nz)) + bg[nz + i]
            u = _sig(u_pre)
            rh = np.array([_sig(sum(np.concatenate([x[b], h[b]])[k] * wg[k, j] for k in range(2 * nz)) + bg[j]) * h[b, j]
                           for j in range(nz)])
            c = np.tanh(sum(np.concatenate([x[b], rh])[k] * wc[k, i] for k in range(2 * nz)) + bc[i])
            want[b, i] = u * h[b, i] + (1 - u) * c
    assert np.abs(out.numpy() - want).max() < 1e-12 and out is h2


@pytest.mark.parametrize('norm_layer', ['instance', 'layer', 'none'])
def test_ablation_zero_kernel_gives_the_closed_form_of_the_bias(norm_layer):
    """conv_h with a zero kernel outputs act(norm(bias)): a per-channel constant, which instance and layer norm map to beta
    (instance: zero variance per channel; layer: the constant's spread over channels is normalised away only per sample,
    so layer norm gives gamma * (b - mean(b)) / std(b) + beta)."""
    rng = np.random.default_rng(9)
    B, H, W, F = 2, 4, 4, 8
    b, g, be = rng.standard_normal(F), rng.standard_normal(F), rng.standard_normal(F)
    s = SC + '/conv_h1'
    P = {s + '/conv2d/kernel': torch.zeros(5, 5, 3, F, dtype=torch.float64), s + '/conv2d/bias': torch.tensor(b)}
    if norm_layer != 'none':
        ns = s + ('/InstanceNorm' if norm_layer == 'instance' else '/LayerNorm')
        P[ns + '/gamma'], P[ns + '/beta'] = torch.tensor(g), torch.tensor(be)
    hp = O.make_hparams(norm_layer=norm_layer)
    state = (torch.ones(1), torch.ones(1))
    with torch.no_grad():
        out, st = R.conv_h_site(hp)(O.Vars(P), SC + '/lstm_h1/basic_conv2dlstm_cell',
                                    torch.tensor(rng.standard_normal((B, H, W, 3))), state, F)
    if norm_layer == 'instance':
        want = np.maximum(be, 0.0)
    elif norm_layer == 'layer':
        want = np.maximum(g * (b - b.mean()) / np.sqrt(b.var() + 1e-12) + be, 0.0)
    else:
        want = np.maximum(b, 0.0)
    assert np.abs(out.numpy() - want).max() < 1e-9 and st is state


def _initial_states(hk, size=64):
    m = _model(dict(CFG2, learn_initial_state=True, **hk), size, size)
    return [(n[len('generator/'):], tuple(sh), what, li) for n, sh, what, li in m._initial_state_specs()]


def test_initial_state_order_follows_nest_flatten():
    """nest.flatten({'conv_rnn_states': [...], 'rnn_z_state': ...}): the five ConvLSTMs' (c, h) in layer order, then the z
    cell's (c, h) or h; the 64x64 stack's ConvLSTMs are h0, h1, h2 (encoder) and h3, h4 (decoder)."""
    conv = [((32, 32, 32), 0), ((16, 16, 64), 1), ((8, 8, 128), 2), ((16, 16, 64), 3), ((32, 32, 32), 4)]
    want = [(s, w, li) for s, li in conv for w in ('c', 'h')]
    got = _initial_states({})
    assert [(sh, w, li) for _, sh, w, li in got] == want + [((8,), 'zc', -1), ((8,), 'zh', -1)]
    assert [n for n, _, _, _ in got] == ['initial_state_%d/initial_state' % k for k in range(12)]
    assert [(sh, w) for _, sh, w, _ in _initial_states(dict(rnn='gru'))][10:] == [((8,), 'zh')]
    assert len(_initial_states(dict(nz=0))) == len(_initial_states(dict(use_rnn_z=False))) == 10
    assert _initial_states(dict(ablation_rnn=True)) == []
    # the same order from the reference's construction (the oracle creates them in flatten order at t = 0)
    hp = O.make_hparams(**dict(CFG2, learn_initial_state=True))
    ref, _ = R.init_params(hp, (64, 64, 3))
    for k, (_, sh, _, _) in enumerate(got):
        assert tuple(ref['generator/initial_state_%d/initial_state' % k].shape) == sh
