"""CPU tests of where and how the SAVP cell takes its conditioning vector (where_add = 'input' | 'middle' | 'all',
use_tile_concat): which hparams the model accepts, its variable names and shapes against the reference
(tests/savp_conditioning_oracle.py), the reference restated unchanged at the defaults, and the float64 identity that an
instance norm removes the dense term of a site."""
import itertools
import re

import pytest
import torch

import savp_conditioning_oracle as CO
from oracle import savp_oracle as O
from test_conv_lstm import CFG2, _model

SC = 'generator/rnn/savp_cell'
COMBOS = list(itertools.product(('all', 'input', 'middle'), (True, False)))
CELLS = {
    'default': {},
    'norm_free': dict(norm_layer='none', conv_rnn_norm_layer='none'),
    'ablation_rnn': dict(ablation_rnn=True),
    'ablation_conv_rnn_norm': dict(ablation_conv_rnn_norm=True),
}
DENSE = re.compile(r'savp_cell/((conv_)?h\d+/dense/kernel|lstm_h\d+/basic_conv2dlstm_cell/weights)$')
INPUTS = {'vae': (8, 0, 0), 'actions_states': (8, 4, 3), 'deterministic': (0, 0, 0), 'deterministic_actions': (0, 4, 0)}


def _combo_id(c):
    return '%s-%s' % (c[0], 'tile' if c[1] else 'dense')


def _conditioned(hk, A=0, Sd=0, size=64):
    m = _model(hk, size, size)
    m.A, m.Sd = A, Sd
    m.Zc = A + Sd + m.hparams.nz
    return m


def test_every_combination_is_accepted_and_a_bogus_site_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    base = dict(context_frames=2, sequence_length=12)
    for where_add, tile in COMBOS:
        for extra in CELLS.values():
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, where_add=where_add, use_tile_concat=tile,
                                                                     **extra))._check_supported()
    with pytest.raises(ValueError):
        SAVPVideoPredictionModel(mode='train', hparams_dict=dict(base, where_add='bogus'))._check_supported()


@pytest.mark.parametrize('inputs', sorted(INPUTS))
@pytest.mark.parametrize('cell', sorted(CELLS))
@pytest.mark.parametrize('combo', COMBOS, ids=_combo_id)
def test_param_specs_follow_the_reference(combo, cell, inputs):
    nz, A, Sd = INPUTS[inputs]
    hk = dict(CFG2, nz=nz, where_add=combo[0], use_tile_concat=combo[1], **CELLS[cell])
    specs = _conditioned(hk, A, Sd)._generator_param_specs()
    ref, _ = CO.init_params(O.make_hparams(**hk), (64, 64, 3), action_dim=A, state_dim=Sd)
    gen_ref = {k: t for k, t in ref.items() if k.startswith('generator/')}
    assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
    for k, (shape, init) in specs.items():
        assert tuple(shape) == tuple(gen_ref[k].shape), k
    dense = [k for k in specs if DENSE.search(k)]
    assert bool(dense) != combo[1] and all(specs[k][0][0] == A + Sd + nz for k in dense)


def test_sites_per_where_add():
    """64x64 cfg2: h0..h2 encoder (ConvLSTMs at every layer), h3..h5 decoder; zc = 8 channels of rnn_z."""
    def kin(hk, li):
        return _conditioned(dict(CFG2, **hk))._generator_param_specs()['%s/h%d/%s/kernel' % (
            SC, li, 'conv_pool2d' if li < 3 else 'upsample_conv2d')][0][2]
    assert [kin({}, li) for li in range(6)] == [6 + 8, 32 + 8, 64 + 8, 128 + 8, 64 + 64 + 8, 32 + 32 + 8]
    assert [kin(dict(where_add='input'), li) for li in range(6)] == [6 + 8, 32, 64, 128, 64 + 64, 32 + 32]
    assert [kin(dict(where_add='middle'), li) for li in range(6)] == [6, 32, 64, 128 + 8, 64 + 64, 32 + 32]
    for where_add in ('input', 'middle'):
        specs = _conditioned(dict(CFG2, where_add=where_add))._generator_param_specs()
        assert specs[SC + '/lstm_h1/basic_conv2dlstm_cell/kernel'][0] == (5, 5, 64 + 64, 256)
        nt = _conditioned(dict(CFG2, where_add=where_add, use_tile_concat=False))._generator_param_specs()
        li = 0 if where_add == 'input' else 3
        assert [k for k in nt if DENSE.search(k)] == ['%s/h%d/dense/kernel' % (SC, li)]
    nt = _conditioned(dict(CFG2, use_tile_concat=False))._generator_param_specs()
    assert nt[SC + '/h0/conv_pool2d/kernel'][0] == (5, 5, 6, 32) and nt[SC + '/h0/dense/kernel'] == ((8, 32), 'kernel')
    assert nt[SC + '/lstm_h1/basic_conv2dlstm_cell/kernel'][0] == (5, 5, 128, 256)
    assert nt[SC + '/lstm_h1/basic_conv2dlstm_cell/weights'] == ((8, 256), 'kernel')
    abl = _conditioned(dict(CFG2, use_tile_concat=False, ablation_rnn=True))._generator_param_specs()
    assert abl[SC + '/conv_h1/dense/kernel'] == ((8, 64), 'kernel') and abl[SC + '/conv_h1/conv2d/kernel'][0] == (5, 5, 64, 64)


def test_deterministic_model_has_empty_dense_kernels():
    """nz = 0 without actions or states: the reference's concat([]) is a [B, 0] tensor, so every dense kernel is [0, oc],
    and the model's flat parameter buffer gives them empty views."""
    hk = dict(CFG2, nz=0, use_tile_concat=False)
    specs = _conditioned(hk)._generator_param_specs()
    dense = {k: s for k, (s, _) in specs.items() if DENSE.search(k)}
    assert len(dense) == 6 + 5 and all(s[0] == 0 for s in dense.values())
    assert dense[SC + '/h4/dense/kernel'] == (0, 32) and dense[SC + '/lstm_h2/basic_conv2dlstm_cell/weights'] == (0, 512)
    ref, _ = CO.init_params(O.make_hparams(**hk), (64, 64, 3))
    assert all(tuple(ref[k].shape) == s and ref[k].numel() == 0 for k, s in dense.items())


def test_oracle_is_the_reference_oracle_at_the_defaults():
    hp = O.make_hparams(context_frames=2, sequence_length=4, nz=4, ngf=8, nef=8)
    a, _ = O.init_params(hp, (32, 32, 3), batch=2, action_dim=3, seed=2)
    b, _ = CO.init_params(hp, (32, 32, 3), batch=2, action_dim=3, seed=2)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3), action_dim=3, seed=1)
    gt = O.ground_truth_mask(hp, 2)
    with torch.no_grad():
        want = O.generator(O.Vars(a), hp, inputs, noise, gt)
        got = CO.generator(O.Vars(b), hp, inputs, noise, gt)
    assert list(want) == list(got) and all(torch.equal(want[k], got[k]) for k in want)
    saved = O.savp_cell_step, O.tile_concat_z, O.conv_pool2d, O.upsample_conv2d, O.conv_lstm_cell, O.conv2d_tf
    for where_add, tile in COMBOS:
        CO.init_params(O.make_hparams(**dict(hp, where_add=where_add, use_tile_concat=tile)), (32, 32, 3), seed=2)
    assert (O.savp_cell_step, O.tile_concat_z, O.conv_pool2d, O.upsample_conv2d, O.conv_lstm_cell, O.conv2d_tf) == saved


def _gen64(hk, seed_noise):
    hp = O.make_hparams(**hk)
    params, _ = CO.init_params(hp, (32, 32, 3), batch=2, seed=3, dtype=torch.float64)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3), seed=1, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed_noise)
    noise = {k: torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in noise.items()}
    with torch.no_grad():
        return CO.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, 2))['gen_images']


@pytest.mark.parametrize('where_add', ['all', 'input', 'middle'])
def test_instance_norm_removes_the_dense_term(where_add):
    """use_tile_concat=False: dense(v) is constant per (sample, channel), and the instance norm after every site (h{i}, and
    the ConvLSTM's gate norm) removes it exactly -- gen_images do not depend on the zs.  With norm_layer='none' they do."""
    base = dict(context_frames=2, sequence_length=5, nz=4, ngf=8, nef=8, where_add=where_add, use_tile_concat=False)
    a, b = _gen64(base, 0), _gen64(base, 1)
    assert (a - b).abs().max().item() < 1e-12
    a, b = _gen64(dict(base, norm_layer='none'), 0), _gen64(dict(base, norm_layer='none'), 1)
    assert (a - b).abs().max().item() > 1e-6
    tile = dict(base, use_tile_concat=True)       # the tile-concat vector goes through the convolution's spatial taps
    assert (_gen64(tile, 0) - _gen64(tile, 1)).abs().max().item() > 1e-6
