"""GPU tests (-m gpu) of the SAVP cell's recurrence choices: vp_act_fwd and the GRU kernels against fp64, the engine at the
ablation's conv_h geometries, the generator and the training step against the fp32 reference
(tests/savp_recurrence_oracle.py) for ablation_rnn, use_rnn_z=False and rnn='gru', the captured step, TF bundles with the new
variable names, and the training / generation scripts."""
import os
import sys

import numpy as np
import pytest
import torch

import savp_recurrence_oracle as R
import test_gpu_engine as E
from oracle import savp_oracle as O
from test_gpu_conv_lstm import TRAIN_CASES
from test_gpu_engine import L, mode  # noqa: F401  (fixtures of the engine check)
from test_gpu_engine import PLAIN, S1, _case, _norm_cmap
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
SC = 'generator/rnn/savp_cell'
NAN = float('nan')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = {
    'ablation': dict(ablation_rnn=True),
    'ablation_layer_norm': dict(ablation_rnn=True, norm_layer='layer'),
    'ablation_no_norm': dict(ablation_rnn=True, norm_layer='none'),
    'ablation_no_rnn_z': dict(ablation_rnn=True, use_rnn_z=False),
    'no_rnn_z': dict(use_rnn_z=False),
    'gru': dict(rnn='gru'),
    'learned_state': dict(learn_initial_state=True),
    'learned_state_gru': dict(learn_initial_state=True, rnn='gru'),
}
NEW_SCOPES = ('/conv_h', '/fc_z/', '/gru_z/', '/initial_state_')


@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


# ------------------------------------------------------------------------------------------------ kernels
def _act64(x, act, alpha):
    return {L_ACT['none']: x, L_ACT['relu']: torch.relu(x), L_ACT['lrelu']: torch.where(x > 0, x, alpha * x),
            L_ACT['sigmoid']: torch.sigmoid(x), L_ACT['tanh']: torch.tanh(x), L_ACT['elu']: torch.nn.functional.elu(x)}[act]


L_ACT = dict(none=0, relu=1, lrelu=2, sigmoid=3, tanh=4, elu=5)


@pytest.mark.parametrize('act', sorted(L_ACT))
@pytest.mark.parametrize('rows,c', [(1, 1), (37, 5), (4096, 8)])
def test_act_fwd_matches_fp64(L, act, rows, c):  # noqa: F811
    g = torch.Generator().manual_seed(rows * 7 + c)
    xs, ys = c + 3, c + 9
    x = (torch.randn(rows, xs, generator=g) * 3).cuda()
    y = torch.full((rows, ys), NAN, device='cuda')
    L.act_fwd(x.data_ptr(), xs, y.data_ptr() + 4, ys, rows, c, L_ACT[act], 0.2)
    torch.cuda.synchronize()
    want = _act64(x[:, :c].double(), L_ACT[act], 0.2)
    assert (y[:, 1:1 + c].double() - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item())
    assert torch.isnan(y[:, 0]).all() and torch.isnan(y[:, 1 + c:]).all()      # nothing outside the slice is written


def test_act_fwd_rejects_bad_calls(L):  # noqa: F811
    x, y = torch.zeros(4, 8, device='cuda'), torch.zeros(4, 8, device='cuda')
    for args in ((x.data_ptr(), 8, y.data_ptr(), 8, 4, 8, 6),      # unknown activation
                 (x.data_ptr(), 4, y.data_ptr(), 8, 4, 8, 1),      # input stride narrower than c
                 (x.data_ptr(), 8, y.data_ptr(), 8, 4, 0, 1),      # no channels
                 (0, 8, y.data_ptr(), 8, 4, 8, 1)):                # null input
        with pytest.raises(L.VpError):
            L.act_fwd(*args)
    L.act_fwd(x.data_ptr(), 8, y.data_ptr(), 8, 0, 8, 1)          # zero rows: nothing to do


def _gru64(z, h, wg, bg, wc, bc):
    U = h.shape[-1]
    r, u = torch.split(torch.sigmoid(torch.cat([z, h], -1) @ wg + bg), U, -1)
    c = torch.tanh(torch.cat([z, r * h], -1) @ wc + bc)
    return u * h + (1 - u) * c


@pytest.mark.parametrize('b,units', [(1, 1), (37, 8), (512, 13)])
def test_gru_cell_matches_fp64(L, b, units):  # noqa: F811
    """One GRU step from the kernels and two dense layers (fp64 here) against autograd in fp64: h', dz, dh_prev and the
    two pre-activation gradients."""
    g = torch.Generator().manual_seed(b + units)
    d = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)      # noqa: E731
    z, h, dh = d(b, units), d(b, units), d(b, units)
    wg, bg, wc, bc = d(2 * units, 2 * units) * 0.5, d(2 * units), d(2 * units, units) * 0.5, d(units)
    zr, hr = z.clone().requires_grad_(True), h.clone().requires_grad_(True)
    out = _gru64(zr, hr, wg, bg, wc, bc)
    dz_ref, dh_ref = torch.autograd.grad(out, [zr, hr], dh)
    gates = (torch.cat([z, h], -1) @ wg + bg).float().cuda()
    hc, dhc = h.float().cuda(), dh.float().cuda()
    rh = torch.full((b, 2 * units + 3), NAN, device='cuda')
    L.gru_cell_fwd(0, gates, hc, None, rh.data_ptr() + 4 * units, 2 * units + 3, None, b, units)
    torch.cuda.synchronize()
    r = torch.sigmoid(gates.double().cpu()[:, :units])
    assert (rh[:, units:2 * units].double().cpu() - r * h).abs().max().item() <= 1e-6
    assert torch.isnan(rh[:, :units]).all() and torch.isnan(rh[:, 2 * units:]).all()
    cand_in = torch.cat([z, rh[:, units:2 * units].double().cpu()], -1)
    cand = (cand_in @ wc + bc).float().cuda()
    h_new = torch.full((b, units), NAN, device='cuda')
    L.gru_cell_fwd(1, gates, hc, cand, 0, 0, h_new, b, units)
    dgates = torch.full((b, 2 * units), NAN, device='cuda')
    dcand = torch.full((b, units), NAN, device='cuda')
    dh_prev = torch.full((b, units), NAN, device='cuda')
    L.gru_cell_bwd(0, gates, hc, cand, dhc, 0, 0, dgates, dcand, dh_prev, b, units)
    torch.cuda.synchronize()
    assert (h_new.double().cpu() - out.detach()).abs().max().item() <= 2e-5
    dcand_in = dcand.double().cpu() @ wc.t()                       # the candidate layer's dense backward
    drh = torch.full((b, 2 * units + 5), NAN, device='cuda')
    drh[:, 5:5 + units] = dcand_in[:, units:].float().cuda()
    L.gru_cell_bwd(1, gates, hc, None, None, drh.data_ptr() + 20, 2 * units + 5, dgates, None, dh_prev, b, units)
    torch.cuda.synchronize()
    dgates64 = dgates.double().cpu()
    dcat = dgates64 @ wg.t()                                        # the gates layer's dense backward
    dz = dcat[:, :units] + dcand_in[:, :units]
    dhp = dh_prev.double().cpu() + dcat[:, units:]
    # the pre-activation gradients against autograd through the same pre-activations
    gr, cr = gates.double().cpu().requires_grad_(True), cand.double().cpu().requires_grad_(True)
    rr, uu = torch.split(torch.sigmoid(gr), units, -1)
    hn = uu * h + (1 - uu) * torch.tanh(cr)
    dg_ref, dc_ref = torch.autograd.grad(hn, [gr, cr], dh, retain_graph=True)
    dg_ref = dg_ref + torch.autograd.grad(rr * h, gr, dcand_in[:, units:])[0]
    for got, want, nm in ((dgates64, dg_ref, 'dgates'), (dcand.double().cpu(), dc_ref, 'dcand'), (dz, dz_ref, 'dz'),
                          (dhp, dh_ref, 'dh_prev')):
        err = (got - want).abs().max().item() / max(1.0, want.abs().max().item())
        assert err <= 2e-5, (nm, err)


def test_gru_cell_rejects_bad_calls(L):  # noqa: F811
    t = torch.zeros(4, 16, device='cuda')
    with pytest.raises(L.VpError):
        L.gru_cell_fwd(2, t, t, t, t.data_ptr(), 16, t, 4, 8)         # no stage 2
    with pytest.raises(L.VpError):
        L.gru_cell_fwd(0, t, t, None, 0, 16, None, 4, 8)              # stage 0 needs rh
    with pytest.raises(L.VpError):
        L.gru_cell_fwd(1, t, t, None, 0, 0, t, 4, 8)                  # stage 1 needs cand
    with pytest.raises(L.VpError):
        L.gru_cell_fwd(0, t, t, None, t.data_ptr(), 4, None, 4, 8)    # rh stride narrower than units
    with pytest.raises(L.VpError):
        L.gru_cell_bwd(0, t, t, t, None, 0, 0, t, t, t, 4, 8)         # stage 0 needs dh
    with pytest.raises(L.VpError):
        L.gru_cell_bwd(1, t, t, None, None, 0, 16, t, None, t, 4, 8)  # stage 1 needs drh
    with pytest.raises(L.VpError):
        L.gru_cell_bwd(0, t, t, t, t, 0, 0, t, t, t, 0, 8)            # no rows


# ------------------------------------------------------------------------------------------------ engine at conv_h
# the conv_h{i} sites of the 64x64 (ngf 32) and 128x128 generators: (h{i} | z) -> oc, 5x5 stride 1, with nz 8 and nz 0
CONV_H_CASES = sorted(set(_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, oc + zc, oc, (1, hw, hw))
                          for zc in (8, 0) for hw, oc in ((32, 32), (16, 64), (8, 128), (32, 64), (16, 128), (8, 256))), key=str)


@pytest.mark.parametrize('case', CONV_H_CASES, ids=E.case_id)
def test_engine_at_conv_h_geometries(L, mode, case):  # noqa: F811
    E.test_engine_matches_fp64_reference(L, mode, case)


def test_conv_h_cases_cover_every_convolution(Model):
    """Every convolution of the cfg2 64x64 ablation model has an engine case: its conv_h sites in CONV_H_CASES, the others in
    MODEL_CASES."""
    import make_golden_b16 as G
    hk = dict(G.HK, ablation_rnn=True)
    hp = O.make_hparams(**hk)
    inputs, _ = O.make_synthetic_inputs(hp, 1, G.SHAPE)
    model = Model(mode='train', hparams_dict=hk)
    model.set_params(R.init_params(hp, G.SHAPE, seed=0)[0])
    model.build_graph(_batch_major(inputs))
    Bf, ext, conv_h = model.Bf, {}, set()
    for li, d in enumerate(model.gl):
        ext[id(d['conv'])] = (1,) + tuple(Bf['in%d' % li].shape[2:4])
        if 'rconv' in d:
            ext[id(d['rconv'])] = (1,) + tuple(Bf['rin%d' % li].shape[2:4])
            conv_h.add(id(d['rconv']))
    for c in (model.conv_scratch, model.conv_hmasks, model.conv_simg, model.conv_masks):
        ext[id(c)] = (1, model.H, model.W)
    for i, e in enumerate(getattr(model, 'enc_layers', [])):
        ext[id(e['conv'])] = (1,) + tuple((Bf['pairs'] if i == 0 else Bf['epre%d' % (i - 1)]).shape[1:3])
    missing = []
    for c in model.convs:
        t = (c.kind, tuple(c.k), tuple(c.stride), tuple(c.pad), bool(c.transposed), c.ci_ref, c.ci_int, _norm_cmap(c.cmap), c.co,
             ext[id(c)])
        if t not in (set(CONV_H_CASES) if id(c) in conv_h else set(E.MODEL_CASES)):
            missing.append('%s: %s' % (c.wname, t))
    assert len(conv_h) == 5 and not missing, missing


# ------------------------------------------------------------------------------------------------ model level
def _params(hp, shape, A=0, seed=0):
    """Reference initial values with the new variables' zero / one initialisers replaced by random values."""
    params, _ = R.init_params(hp, shape, action_dim=A, seed=seed)
    g = torch.Generator().manual_seed(seed + 11)
    for k in list(params):
        if any(s in k for s in NEW_SCOPES) and not k.endswith('/kernel'):
            params[k] = params[k] + torch.randn(params[k].shape, generator=g) * 0.3
    return params


GEN_CASES = {
    'deterministic': (dict(context_frames=2, sequence_length=8, nz=0), 0),
    'vae_actions': (dict(context_frames=2, sequence_length=8, nz=8), 4),
}


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('variant', sorted(VARIANTS))
@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_matches_oracle(Model, case, variant, arith):
    """gen_images (and gen_images_enc) within 1e-3 max-abs of the fp32 reference in TF32, 1e-4 in the fp32-exact mode."""
    hk, A = GEN_CASES[case]
    if not hk['nz'] and set(VARIANTS[variant]) <= {'use_rnn_z', 'rnn'}:
        pytest.skip('without z the z cell does not exist: the model is the default one')
    hk = dict(hk, **VARIANTS[variant])
    hp = O.make_hparams(**hk)
    B, shape = 2, (64, 64, 3)
    params = _params(hp, shape, A)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, action_dim=A, seed=0)
    with torch.no_grad():
        ref = R.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B, None))
    with arithmetic(arith):
        model = Model(mode='test', hparams_dict=hk)
        model.set_params(params)
        binp = _batch_major(inputs)
        model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=False)
    model.generator_forward()
    torch.cuda.synchronize()
    tol = 1e-3 if arith == 'tf32' else 1e-4
    report = {}
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - ref[k]).abs().max().item()
        report[k] = err
        assert err <= tol, (case, variant, arith, k, err)
    print('recurrence %s generator %s [%s]: max-abs %s' % (variant, case, arith, {k: '%.2e' % v for k, v in report.items()}))


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return R.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


TRAIN_VARIANTS = ('ablation', 'no_rnn_z', 'gru', 'learned_state')


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('variant', TRAIN_VARIANTS)
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_matches_fp32_oracle(Model, case, variant, arith):
    """64x64, B = 2, random scheduled-sampling mask, the tolerances of test_gpu_train_parity.py: exact mode EXACT_GTOL per
    gradient tensor, TF32 mode max(5e-2, 2 x the operand-rounding emulation).  Every new variable gets a nonzero gradient."""
    hk = dict(TRAIN_CASES[case], **VARIANTS[variant])
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
    for kind in ('g_grads', 'd_grads'):
        if kind not in res:
            continue
        items = [(k, g) for k, g in res[kind].items() if g is not None]
        gmax = max(g.double().norm().item() for _, g in items)
        for k, g in items:
            r, n = _rel(model.grads[k], g)
            if n < floor * gmax:
                continue
            tol = EXACT_GTOL[case] if emu is None else max(5e-2, 2.0 * _rel(emu[kind][k], g)[0])
            worst.append((r, tol, k))
            if r > tol:
                bad.append((r, tol, k))
    if bad and emu is None:
        # fp32-exact mode: a gradient the fp32 reference itself cannot resolve to EXACT_GTOL (its relative distance from an
        # fp64 run of the reference, measured on the CPU: 3.1e-3 for the h3 ConvLSTM's learned states in vae_l1) gets twice
        # that distance as its tolerance
        inp64, noise64 = O.make_synthetic_inputs(hp, B, shape, dtype=torch.float64)
        f64 = _oracle_step(hp, {k: v.double() for k, v in params.items()}, inp64, noise64, step, sampling, None)
        kinds = dict((k, kind) for kind in ('g_grads', 'd_grads') for k in res.get(kind, {}))
        bad = [(r, max(tol, 2.0 * _rel(res[kinds[k]][k], f64[kinds[k]][k])[0]), k) for r, tol, k in bad]
        limited = set(k for _, _, k in bad)
        worst = [w for w in worst if w[2] not in limited] + [(r, tol, k + ' (fp32 reference limited)') for r, tol, k in bad]
        bad = [b for b in bad if b[0] > b[1]]
    worst.sort(reverse=True)
    print('recurrence %s %s [%s]: worst gradient errors %s' % (variant, case, arith,
                                                                 ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    new = [k for k in res['g_grads'] if any(s in k for s in NEW_SCOPES)]
    assert bool(new) == (variant != 'no_rnn_z')
    assert all(float(model.grads[k].abs().max()) > 0 for k in new), new     # the new variables are trained
    for k in ('gen_images', 'gen_images_enc'):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)


@pytest.mark.parametrize('variant', TRAIN_VARIANTS)
def test_captured_step_reproduces_the_eager_step(Model, variant, tmp_path):
    """The eager step and two graph replays from the same checkpoint give bit-identical losses and gradients."""
    hk = dict(TRAIN_CASES['savp'], **VARIANTS[variant])
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


@pytest.mark.parametrize('variant', ['ablation', 'learned_state_gru'])
def test_tf_bundle_with_the_new_names_restores_exactly(Model, variant, tmp_path):
    """A TensorFlow bundle under the historical 'dna_cell' scope with conv_h / fc_z, or gru_z and the initial states (which
    are not under the cell's scope), restores exactly."""
    from test_tf_checkpoint import write_bundle
    hk = dict(context_frames=2, sequence_length=6, nz=8, **VARIANTS[variant])
    imgs = {'images': np.random.default_rng(0).uniform(size=(2, 6, 64, 64, 3)).astype(np.float32)}
    src = Model(mode='test', hparams_dict=hk)
    src.build_graph(imgs)
    src.init_params(seed=9)
    want = src.get_params()
    assert [k for k in want if any(s in k for s in NEW_SCOPES)]
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


def _scripts():
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    import generate
    import train
    return train, generate


@pytest.mark.parametrize('extra', ['ablation_rnn=True', 'use_rnn_z=False', 'rnn=gru', 'learn_initial_state=True'])
def test_scripts_train_save_restore_generate(Model, extra, tmp_path):
    train, generate = _scripts()
    out = str(tmp_path / 'run')
    model = train.main(['--input_dir', 'none', '--dataset', 'synthetic', '--dataset_hparams', 'sequence_length=6,num_examples=8',
                        '--model', 'savp', '--output_dir', out, '--progress_freq', '1', '--save_freq', '2', '--seed', '1',
                        '--model_hparams', 'batch_size=2,max_steps=2,clip_length=4,l1_weight=100.0,kl_weight=1.0,'
                        'video_sn_gan_weight=0.1,' + extra])
    assert model.global_step == 2 and np.isfinite(model.g_loss) and np.isfinite(model.d_loss)
    key, val = extra.split('=')
    assert str(getattr(model.hparams, key)) == val
    n = generate.main(['--input_dir', 'none', '--checkpoint', out, '--results_dir', str(tmp_path / 'results'), '--batch_size', '2',
                       '--num_samples', '2', '--num_stochastic_samples', '2', '--mode', 'test'])
    assert n == 2


@pytest.mark.parametrize('rnn', ['lstm', 'gru'])
def test_zero_learned_initial_states_are_the_zero_state(Model, rnn):
    """learn_initial_state=True with its zero initial values: outputs, losses and the gradients of every shared variable are
    bit-identical to learn_initial_state=False."""
    base = dict(TRAIN_CASES['savp'], rnn=rnn)
    hp = O.make_hparams(**base)
    params, _ = R.init_params(hp, (64, 64, 3))
    inputs, noise = O.make_synthetic_inputs(hp, 2, (64, 64, 3))
    binp = _batch_major(inputs)
    runs = []
    for learn in (False, True):
        model = Model(mode='train', hparams_dict=dict(base, learn_initial_state=learn))
        model.set_params(params)
        model.build_graph(binp)
        model.train_step(binp, noise)
        torch.cuda.synchronize()
        runs.append(model)
    a, b = runs
    init = [k for k in b.params if '/initial_state_' in k]
    assert len(init) == 10 + (2 if rnn == 'lstm' else 1) and all(float(b.params[k].abs().max()) > 0 for k in init)  # Adam moved them
    assert torch.equal(a.loss_vals, b.loss_vals)
    for k in ('gen_images', 'gen_images_enc'):
        assert torch.equal(a.outputs_time_major(k), b.outputs_time_major(k)), k
    for k in a.grads:
        assert torch.equal(a.grads[k], b.grads[k]), k
