"""GPU tests (-m gpu) of where and how the SAVP cell takes its conditioning vector (where_add, use_tile_concat): the generator
and the training step against the fp32 reference (tests/savp_conditioning_oracle.py) in the TF32 and fp32-exact modes, the
captured step, bit-identical reruns, and TF bundles with the new variable names."""
import re

import numpy as np
import pytest
import torch

import savp_conditioning_oracle as CO
import savp_state_oracle as ST
from oracle import savp_oracle as O
from test_gpu_conv_lstm import TRAIN_CASES
from test_gpu_engine import L  # noqa: F401  (fixture)
from test_gpu_reproducible import twice
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
DENSE = re.compile(r'savp_cell/((conv_)?h\d+/dense/kernel|lstm_h\d+/basic_conv2dlstm_cell/weights)$')
COMBOS = [(w, t) for w in ('all', 'input', 'middle') for t in (True, False)]
CELLS = {
    'default': {},
    'norm_free': dict(norm_layer='none', conv_rnn_norm_layer='none'),
    'ablation_rnn': dict(ablation_rnn=True),
}


def _combo_id(c):
    return '%s-%s' % (c[0], 'tile' if c[1] else 'dense')


@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def _hk(base, combo, cell):
    return dict(base, where_add=combo[0], use_tile_concat=combo[1], **CELLS[cell])


def _run_generator(Model, hk, A, Sd, arith, B=2, shape=(64, 64, 3)):
    hp = O.make_hparams(**hk)
    params, _ = CO.init_params(hp, shape, action_dim=A, state_dim=Sd)
    inputs, noise = ST.make_synthetic_inputs(hp, B, shape, action_dim=A, state_dim=Sd, seed=0)
    with torch.no_grad():
        ref = CO.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B, None))
    with arithmetic(arith):
        model = Model(mode='test', hparams_dict=hk)
        model.set_params(params)
        binp = _batch_major(inputs)
        model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=False)
    model.generator_forward()
    torch.cuda.synchronize()
    return model, ref


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('cell', sorted(CELLS))
@pytest.mark.parametrize('combo', COMBOS, ids=_combo_id)
def test_generator_matches_oracle(Model, combo, cell, arith):
    """gen_images and gen_images_enc within 1e-3 max-abs of the fp32 reference, with actions (vae, 4 action dims)."""
    hk = _hk(dict(context_frames=2, sequence_length=8, nz=8), combo, cell)
    model, ref = _run_generator(Model, hk, 4, 0, arith)
    errs = {k: (model.outputs_time_major(k).cpu() - ref[k]).abs().max().item() for k in ('gen_images', 'gen_images_enc')}
    print('conditioning %s %s [%s]: max-abs %s' % (_combo_id(combo), cell, arith, {k: '%.2e' % v for k, v in errs.items()}))
    assert all(v <= 1e-3 for v in errs.values()), errs


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('case', [('input', False, 'norm_free', 0), ('middle', False, 'default', 8), ('all', False, 'norm_free', 0),
                                  ('all', True, 'norm_free', 8)], ids=lambda c: '%s-%s-%s-nz%d' % (c[0], 'tile' if c[1] else 'dense',
                                                                                                   c[2], c[3]))
def test_generator_with_actions_and_states_matches_oracle(Model, case, arith):
    """Deterministic and stochastic models conditioned on actions (4) and robot states (3): gen_images and gen_states."""
    hk = _hk(dict(context_frames=2, sequence_length=8, nz=case[3]), case[:2], case[2])
    model, ref = _run_generator(Model, hk, 4, 3, arith)
    err = (model.outputs_time_major('gen_images').cpu() - ref['gen_images']).abs().max().item()
    B = model.B
    gst = model.Bf['gstates'][:, B:] if case[3] else model.Bf['gstates']
    serr = (gst.cpu() - ref['gen_states']).abs().max().item()
    print('conditioning states %s [%s]: gen_images %.2e gen_states %.2e' % (case, arith, err, serr))
    assert err <= 1e-3 and serr <= 1e-3, (err, serr)


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return CO.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


TRAIN = {
    'input-dense-norm_free': ('vae_l1', ('input', False), 'norm_free'),
    'middle-tile-default': ('vae_l1', ('middle', True), 'default'),
    'all-dense-default': ('vae_l1', ('all', False), 'default'),
    'all-dense-ablation_no_norm': ('vae_l1', ('all', False), 'ablation_rnn'),
    'all-dense-norm_free-savp': ('savp', ('all', False), 'norm_free'),
}
# Measured bounds where this file's grid is wider than test_gpu_train_parity.py's.  No norm at any site (the norm-free
# ablation): the h1 and conv_h1 bias gradients are 2.9e-3 / 2.5e-3 from the fp32 reference in the fp32-exact mode, with the
# reference within 1e-3 of fp64.  The TF32 mode of the default cells with dense sites: every gradient runs 7-9e-2 from the
# reference (the fp32-exact mode of the same case is within 2e-3), above twice the emulated operand rounding.
EXACT_TOL = {'all-dense-ablation_no_norm': 4e-3}
TF32_FLOOR = {'all-dense-default': 1.2e-1}


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('name', sorted(TRAIN))
def test_training_step_matches_fp32_oracle(Model, name, arith):
    """64x64, B = 2, random scheduled-sampling mask, the tolerances of test_gpu_train_parity.py.  The new dense kernels are
    compared too: where an instance norm follows (the default cell) their reference gradient is rounding noise, so they are
    held to an absolute bound of the gradient scale instead of a relative one."""
    case, combo, cell = TRAIN[name]
    hk = _hk(TRAIN_CASES[case], combo, cell)
    if name == 'all-dense-ablation_no_norm':
        hk['norm_layer'] = 'none'
    hp = O.make_hparams(**hk)
    B, step, shape = 2, 5, (64, 64, 3)
    params, _ = CO.init_params(hp, shape)
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
    ref_l = dict(res['g_losses'], **res.get('d_losses', {}))
    emu_l = {} if emu is None else dict(emu['g_losses'], **emu.get('d_losses', {}))
    for k, v in ref_l.items():
        tol = max(ltol * abs(v), 2.0 * abs(emu_l[k] - v) if emu_l else 0.0)
        assert abs(lv[k] - v) <= tol + 1e-6, (k, lv[k], v, emu_l.get(k))
    worst, bad = [], []
    dense = [k for k in res['g_grads'] if DENSE.search(k)]
    assert bool(dense) == (not combo[1]) and (len(dense) <= 1) == (combo[0] != 'all')
    cancelled = cell == 'default' and hk.get('norm_layer', 'instance') == 'instance'
    for kind in ('g_grads', 'd_grads'):
        if kind not in res:
            continue
        items = [(k, g) for k, g in res[kind].items() if g is not None]
        gmax = max(g.double().norm().item() for _, g in items)
        gabs = max(g.double().abs().max().item() for _, g in items)
        for k, g in items:
            if k in dense and cancelled:
                err = (model.grads[k].double().cpu() - g.double()).abs().max().item()
                worst.append((err / gabs, 1e-4, k + ' (absolute)'))
                if err > 1e-4 * gabs:
                    bad.append((err / gabs, 1e-4, k))
                continue
            r, n = _rel(model.grads[k], g)
            if n < floor * gmax:
                continue
            tol = EXACT_TOL.get(name, EXACT_GTOL[case]) if emu is None else \
                max(TF32_FLOOR.get(name, 5e-2), 2.0 * _rel(emu[kind][k], g)[0])
            worst.append((r, tol, k))
            if r > tol:
                bad.append((r, tol, k))
    if bad and emu is None:
        # fp32-exact mode: a gradient the fp32 reference itself cannot resolve to EXACT_GTOL gets twice its distance from an
        # fp64 run of the reference as its tolerance (as in test_gpu_recurrence.py)
        inp64, noise64 = O.make_synthetic_inputs(hp, B, shape, dtype=torch.float64)
        f64 = _oracle_step(hp, {k: v.double() for k, v in params.items()}, inp64, noise64, step, sampling, None)
        kinds = dict((k, kind) for kind in ('g_grads', 'd_grads') for k in res.get(kind, {}))
        bad = [(r, max(tol, 2.0 * _rel(res[kinds[k]][k], f64[kinds[k]][k])[0]), k) for r, tol, k in bad]
        limited = set(k for _, _, k in bad)
        worst = [w for w in worst if w[2] not in limited] + [(r, tol, k + ' (fp32 reference limited)') for r, tol, k in bad]
        bad = [x for x in bad if x[0] > x[1]]
    worst.sort(reverse=True)
    print('conditioning %s [%s]: worst gradient errors %s' % (name, arith, ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    if not cancelled:
        assert all(float(model.grads[k].abs().max()) > 0 for k in dense), dense
        for k in dense:
            r, n = _rel(model.grads[k], res['g_grads'][k])
            assert n > 0 and r <= (EXACT_TOL.get(name, EXACT_GTOL[case]) if emu is None else TF32_FLOOR.get(name, 5e-2)), (k, r)
    for k in ('gen_images', 'gen_images_enc'):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)


CAPTURE = {'all-dense-default': (('all', False), 'default'), 'input-dense-norm_free': (('input', False), 'norm_free'),
           'middle-dense-ablation_rnn': (('middle', False), 'ablation_rnn')}


def _model_at_checkpoint(Model, name, tmp_path, graph):
    combo, cell = CAPTURE[name]
    hk = _hk(TRAIN_CASES['savp'], combo, cell)
    hp = O.make_hparams(**hk)
    params, _ = CO.init_params(hp, (64, 64, 3), action_dim=4)
    inputs, _ = O.make_synthetic_inputs(hp, 2, (64, 64, 3), action_dim=4)
    binp = _batch_major(inputs)
    model = Model(mode='train', hparams_dict=hk)
    model.set_params(params)
    model.build_graph(binp)
    model.use_cuda_graph = graph
    model.train_step(binp)
    return model, model.save(str(tmp_path / ('graph' if graph else 'eager'))), binp


@pytest.mark.parametrize('name', sorted(CAPTURE))
def test_captured_step_reproduces_the_eager_step(Model, name, tmp_path):
    """With actions: the eager step and two graph replays from the same checkpoint give bit-identical losses and gradients."""
    runs = {}
    for how in ('eager', 'graph'):
        model, ck, binp = _model_at_checkpoint(Model, name, tmp_path, how == 'graph')
        runs[how] = []
        for _ in range(2 if how == 'graph' else 1):
            model.restore(None, ck)
            model.train_step(binp)
            torch.cuda.synchronize()
            assert (model._graph is not None) == (how == 'graph')
            runs[how].append((model.loss_vals.clone(), model.g_grad.clone(), model.d_grad.clone()))
    ref = runs['eager'][0]
    for got in runs['graph']:
        for nm, a, b in zip(('losses', 'g_grad', 'd_grad'), got, ref):
            assert torch.equal(a, b), (nm, (a - b).abs().max().item())
    dense = [k for k in model.grads if DENSE.search(k)]
    assert dense and all(bool(torch.isfinite(model.grads[k]).all()) for k in dense)


@pytest.mark.parametrize('name', sorted(CAPTURE))
def test_training_step_reruns_bit_identical(Model, name, tmp_path):
    """The eager step from the same checkpoint twice (scratch dirtied in between): identical losses and gradients."""
    model, ck, binp = _model_at_checkpoint(Model, name, tmp_path, False)

    def step():
        model.restore(None, ck)
        model.train_step(binp)
    twice(step, [model.loss_vals, model.g_grad, model.d_grad], 'conditioning step ' + name)


@pytest.mark.parametrize('combo', [('all', False), ('input', False)], ids=_combo_id)
def test_tf_bundle_with_the_new_names_restores_exactly(Model, combo, tmp_path):
    """A TensorFlow bundle under the historical 'dna_cell' scope with the dense kernels (h{i}/dense/kernel and the ConvLSTMs'
    weights) restores exactly."""
    from test_tf_checkpoint import write_bundle
    hk = dict(context_frames=2, sequence_length=6, nz=8, where_add=combo[0], use_tile_concat=combo[1])
    imgs = {'images': np.random.default_rng(0).uniform(size=(2, 6, 64, 64, 3)).astype(np.float32),
            'actions': np.random.default_rng(1).uniform(size=(2, 5, 4)).astype(np.float32)}
    src = Model(mode='test', hparams_dict=hk)
    src.build_graph(imgs)
    src.init_params(seed=9)
    want = src.get_params()
    dense = [k for k in want if DENSE.search(k)]
    assert dense and all(want[k].shape[0] == 12 for k in dense)
    tensors = {k.replace('savp_cell', 'dna_cell'): v for k, v in want.items()}
    tensors['global_step'] = np.array(31, np.int64)
    write_bundle(str(tmp_path / 'model-31'), tensors)
    (tmp_path / 'checkpoint').write_text('model_checkpoint_path: "model-31"\n')
    dst = Model(mode='test', hparams_dict=hk)
    dst.build_graph(imgs)
    dst.restore(None, str(tmp_path))
    got = dst.get_params()
    assert dst.global_step == 31 and set(got) == set(want)
    for k, v in want.items():
        assert np.array_equal(got[k], v), k
