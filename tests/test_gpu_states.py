"""GPU tests (-m gpu) of the robot-state path: vp_state_pred_fwd against fp64, the engine at the layer geometries of a states
model, the generator and the training step against the fp32 states reference (tests/savp_state_oracle.py), the captured
step, checkpoints and the scripts."""
import os
import sys

import numpy as np
import pytest
import torch

import savp_state_oracle as S
import test_gpu_engine as E
from oracle import savp_oracle as O
from test_gpu_engine import L, mode  # noqa: F401  (fixtures of the engine check)
from test_gpu_engine import PLAIN, POOLED, UPSAMPLED, S1, S2, _case, _norm_cmap
from test_gpu_train_parity import EXACT_GTOL, MODES, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
SC = 'generator/rnn/savp_cell'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def _batch_major(inputs):
    """The oracle's time-major inputs -> build_graph's batch-major dict."""
    return {k: (v.permute(1, 0, 2) if v.dim() == 3 else v.permute(1, 0, 2, 3, 4)) for k, v in inputs.items()}


# ------------------------------------------------------------------------------------------------ the kernel
def _sel(pattern, s, nb, ctx, g):
    if pattern == 'ground_truth':
        return torch.ones(s, nb, dtype=torch.int32)
    if pattern == 'context':
        sel = torch.zeros(s, nb, dtype=torch.int32)
        sel[:ctx] = 1
        return sel
    return (torch.rand(s, nb, generator=g) < 0.5).to(torch.int32)      # random per row, the first step included


def _reference(sel, states, actions, K, b):
    """fp64: state_t = sel ? states_t : gen_{t-1} (gen_{-1} = 0), gen_t = [a_t | state_t] @ K + b."""
    s, nb, sd = states.shape
    gen, zs, gens = torch.zeros(nb, sd, dtype=torch.float64), [], []
    for t in range(s):
        st = torch.where(sel[t].bool().view(-1, 1), states[t], gen)
        gen = torch.cat([actions[t], st], dim=1) @ K + b
        zs.append(st)
        gens.append(gen)
    return torch.stack(zs), torch.stack(gens)


KERNEL_CASES = [(a, sd, nb, s) for a in (0, 4) for sd in (1, 3, 7) for nb in (1, 37, 512) for s in (1, 11, 29)]


@pytest.mark.parametrize('A,Sd,NB,S', KERNEL_CASES)
def test_state_pred_kernel_matches_fp64(L, A, Sd, NB, S):  # noqa: F811
    """Relative L2 <= 1e-6 against fp64 for three `sel` patterns; zvec channels outside [A, A + Sd) keep their bits (NaN
    beyond the vector, the actions inside it); a rerun gives identical bits."""
    g = torch.Generator().manual_seed(A * 100000 + Sd * 10000 + NB * 10 + S)
    zs = (A + Sd + 3) // 4 * 4 + 4
    states = torch.randn(S, NB, Sd, generator=g).double()
    actions = torch.randn(S, NB, A, generator=g).double()
    K = (torch.randn(A + Sd, Sd, generator=g) * 0.3).double()
    b = (torch.randn(Sd, generator=g) * 0.1).double()
    st_buf = torch.full((S, NB, Sd + 2), float('nan'), device='cuda')      # states in a slice of a wider buffer
    st_buf[..., :Sd] = states.float().cuda()
    Kd, bd = K.float().cuda(), b.float().cuda()
    for pattern in ('ground_truth', 'context', 'random'):
        sel = _sel(pattern, S, NB, 2, g)
        runs = []
        for _ in range(2):
            z = torch.full((S, NB, zs), float('nan'), device='cuda')
            z[..., :A] = actions.float().cuda()
            before = z.clone()
            gen = torch.full((S, NB, Sd), float('nan'), device='cuda')
            L.state_pred_fwd(sel.cuda(), st_buf, Sd + 2, Kd, bd, z, zs, gen, S, NB, A, Sd)
            runs.append((z, gen, before))
        torch.cuda.synchronize()
        (z, gen, before), (z2, gen2, _) = runs
        keep = torch.ones(zs, dtype=torch.bool)
        keep[A:A + Sd] = False
        zb, bb = z[..., keep].cpu().view(torch.int32), before[..., keep].cpu().view(torch.int32)
        assert torch.equal(zb, bb), 'a channel outside the state slice was written'
        assert torch.equal(z.cpu().view(torch.int32), z2.cpu().view(torch.int32)) and torch.equal(gen.cpu(), gen2.cpu())
        ref_z, ref_gen = _reference(sel, states, actions, K, b)
        ez, eg = _rel(z[..., A:A + Sd], ref_z)[0], _rel(gen, ref_gen)[0]
        assert ez <= 1e-6 and eg <= 1e-6, (pattern, ez, eg)


def test_state_pred_kernel_rejects_bad_calls(L):  # noqa: F811
    S_, NB, A, Sd = 3, 5, 4, 3
    sel = torch.ones(S_, NB, dtype=torch.int32, device='cuda')
    st = torch.zeros(S_, NB, Sd, device='cuda')
    K, b = torch.zeros(A + Sd, Sd, device='cuda'), torch.zeros(Sd, device='cuda')
    z = torch.full((S_, NB, 8), float('nan'), device='cuda')
    gen = torch.full((S_, NB, Sd), float('nan'), device='cuda')
    bad = [
        (sel, st, Sd, K, b, z, 8, gen, S_, NB, A, 0),         # sd < 1
        (sel, st, Sd, K, b, z, 6, gen, S_, NB, A, Sd),        # zvec stride < a + sd
        (sel, st, 2, K, b, z, 8, gen, S_, NB, A, Sd),         # states stride < sd
        (sel, st, Sd, None, b, z, 8, gen, S_, NB, A, Sd),     # null kernel
        (None, st, Sd, K, b, z, 8, gen, S_, NB, A, Sd),       # null sel
        (sel, st, Sd, K, b, None, 8, gen, S_, NB, A, Sd),     # null zvec
        (sel, st, Sd, K, b, z, 8, gen, 0, NB, A, Sd),         # s < 1
        (sel, st, Sd, K, b, z, 8, gen, S_, 0, A, Sd),         # n < 1
        (sel, st, Sd, K, b, z, 8, gen, S_, NB, -1, Sd),       # a < 0
    ]
    for args in bad:
        with pytest.raises(L.VpError):
            L.state_pred_fwd(*args)
    torch.cuda.synchronize()
    assert torch.isnan(z).all() and torch.isnan(gen).all()


# ------------------------------------------------------------------------------------------------ engine geometries
def _state_model_cases(zc):
    """The tile-concat convolutions of the cfg2 generator (64x64x3, ngf 32) whose z segment holds zc = A + Sd (+ nz)."""
    return [
        _case(POOLED, (1, 5, 5), S2, (0, 2, 2), False, (3, 3, zc), 32, (1, 64, 64)),
        _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, (32, zc, 32), 128, (1, 32, 32)),
        _case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, (32, zc), 64, (1, 32, 32)),
        _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, (64, zc, 64), 256, (1, 16, 16)),
        _case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, (64, zc), 128, (1, 16, 16)),
        _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, (128, zc, 128), 512, (1, 8, 8)),
        _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, (128, zc), 64, (1, 8, 8)),
        _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, (64, 64, zc), 32, (1, 16, 16)),
        _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, (32, 32, zc), 32, (1, 32, 32)),
    ]


# cfg2 with A = 4, Sd = 3: z = [actions | state | rnn_z] (15 channels, nz 8) and its deterministic variant (7, nz 0); the
# action-conditioned posterior encoder reads (frame t | frame t+1 | actions)
STATE_CASES = sorted(set(_state_model_cases(4 + 3 + 8) + _state_model_cases(4 + 3) +
                         [_case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, (3, 3, 4), 64, (1, 64, 64))]) - set(E.MODEL_CASES), key=str)


@pytest.mark.parametrize('case', STATE_CASES, ids=E.case_id)
def test_engine_at_state_model_geometries(L, mode, case):  # noqa: F811
    E.test_engine_matches_fp64_reference(L, mode, case)


@pytest.mark.parametrize('nz', [8, 0])
def test_state_cases_cover_every_convolution_of_a_states_model(Model, nz):
    """Every generator / posterior convolution of the cfg2 states model (A = 4, Sd = 3) and of its nz = 0 variant has a case
    in MODEL_CASES or STATE_CASES."""
    import make_golden_b16 as G
    hk = dict(G.HK, nz=nz)
    hp = O.make_hparams(**hk)
    params, _ = S.init_params(hp, G.SHAPE, action_dim=4, state_dim=3, seed=0)
    inputs, _ = S.make_synthetic_inputs(hp, 1, G.SHAPE, action_dim=4, state_dim=3)
    model = Model(mode='train', hparams_dict=hk)
    model.set_params(params)
    model.build_graph(_batch_major(inputs))
    assert model.Sd == 3 and model.Zc == 4 + 3 + nz
    Bf, ext = model.Bf, {}
    for li, d in enumerate(model.gl):
        ext[id(d['conv'])] = (1,) + tuple(Bf['in%d' % li].shape[2:4])
        if 'rconv' in d:
            ext[id(d['rconv'])] = (1,) + tuple(Bf['rin%d' % li].shape[2:4])
    for c in (model.conv_scratch, model.conv_hmasks, model.conv_simg, model.conv_masks):
        ext[id(c)] = (1, model.H, model.W)
    for i, e in enumerate(getattr(model, 'enc_layers', [])):
        ext[id(e['conv'])] = (1,) + tuple((Bf['pairs'] if i == 0 else Bf['epre%d' % (i - 1)]).shape[1:3])
    table = set(E.MODEL_CASES) | set(STATE_CASES)
    missing = []
    for c in model.convs:
        t = (c.kind, tuple(c.k), tuple(c.stride), tuple(c.pad), bool(c.transposed), c.ci_ref, c.ci_int, _norm_cmap(c.cmap), c.co,
             ext[id(c)])
        if t not in table:
            missing.append('%s: %s' % (c.wname, t))
    assert not missing, missing


# ------------------------------------------------------------------------------------------------ generator vs oracle
GEN_CASES = {
    'deterministic_T12': (dict(context_frames=2, sequence_length=12, nz=0), False),
    'deterministic_T30': (dict(context_frames=2, sequence_length=30, nz=0), False),
    'savp_T12': (dict(context_frames=2, sequence_length=12, nz=8), False),
    'savp_T30': (dict(context_frames=2, sequence_length=30, nz=8), False),
    'savp_T12_train_mask': (dict(context_frames=2, sequence_length=12, nz=8), True),
}


@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_with_states_matches_oracle(Model, case):
    """64x64, B = 4, A = 4, Sd = 3 against the fp32 states reference: gen_images max-abs <= 1e-3 (as test_gpu_parity.py),
    gen_states / gen_states_enc <= 1e-5.  Test mode feeds the predicted state back over every future step; the train-mode
    case gives the posterior and the prior unroll different masks."""
    hk, train_mask = GEN_CASES[case]
    hp = O.make_hparams(**hk)
    B, shape, A, Sd = 4, (64, 64, 3), 4, 3
    params, _ = S.init_params(hp, shape, action_dim=A, state_dim=Sd, seed=0)
    params[SC + '/state_pred/dense/kernel'] = torch.randn(A + Sd, Sd, generator=torch.Generator().manual_seed(3)) * 0.3
    params[SC + '/state_pred/dense/bias'] = torch.tensor([0.1, -0.2, 0.05])
    inputs, noise = S.make_synthetic_inputs(hp, B, shape, action_dim=A, state_dim=Sd, seed=0)
    n_free = hp.sequence_length - 1 - hp.context_frames
    nb = 2 * B if hp.nz else B
    if train_mask:
        mask = torch.rand(n_free, nb, generator=torch.Generator().manual_seed(4)) < 0.5
        masks = {'enc': mask[:, :B], 'prior': mask[:, B:]}
        assert not torch.equal(masks['enc'], masks['prior'])
    else:
        mask = False
        masks = {'enc': None, 'prior': None}
    refs = {}
    with torch.no_grad():
        for which, m in masks.items():
            refs[which] = S.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B, m))
    model = Model(mode='train' if train_mask else 'test', hparams_dict=hk)
    model.set_params(params)
    binp = _batch_major(inputs)
    model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=mask)
    model.generator_forward()
    torch.cuda.synchronize()
    out = model.outputs
    keys = [('gen_images', 'prior', 'gen_images'), ('gen_states', 'prior', 'gen_states')]
    if hp.nz:
        keys += [('gen_images_enc', 'enc', 'gen_images_enc'), ('gen_states_enc', 'enc', 'gen_states_enc')]
    report = {}
    for k, which, rk in keys:
        ref = refs[which][rk]
        got = out[k].cpu().permute(1, 0, *range(2, ref.dim()))
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        err = (got - ref).abs().max().item()
        report[k] = err
        assert err <= (1e-3 if k.startswith('gen_images') else 1e-5), (case, k, err)
    print('states generator %s: max-abs %s' % (case, {k: '%.2e' % v for k, v in report.items()}))


def test_build_graph_validates_states(Model):
    hk = dict(context_frames=2, sequence_length=5, nz=0, ngf=8)
    imgs = torch.rand(1, 5, 32, 32, 3)
    for bad in (torch.rand(1, 4, 3), torch.rand(2, 5, 3), torch.rand(1, 5, 0), torch.rand(1, 5)):
        with pytest.raises(ValueError):
            Model(mode='test', hparams_dict=hk).build_graph({'images': imgs, 'states': bad})
    model = Model(mode='test', hparams_dict=hk)
    model.build_graph({'images': imgs})
    assert 'states' not in model.Bf and model.Sd == 0
    with pytest.raises(ValueError):          # a model built without states refuses them instead of ignoring them
        model.set_inputs({'images': imgs, 'states': torch.rand(1, 5, 3)})
    model = Model(mode='test', hparams_dict=hk)
    model.build_graph({'images': imgs, 'states': torch.rand(1, 5, 3)})
    with pytest.raises(ValueError):          # and the reverse
        model.set_inputs({'images': imgs})


# ------------------------------------------------------------------------------------------------ training step
TRAIN_CASES = {
    'vae_l1': dict(context_frames=2, sequence_length=12, nz=8, l1_weight=1.0, kl_weight=1e-3, kl_anneal_steps=(0, 10), lr=1e-3),
    'savp': dict(context_frames=2, sequence_length=12, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
                 video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, kl_anneal_steps=(0, 10)),
}


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return S.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_with_states_matches_fp32_oracle(Model, case, arith):
    """A = 4, Sd = 3, B = 2 with a random scheduled-sampling mask, with the tolerances of test_gpu_train_parity.py: exact
    mode 2e-3 (VAE-L1) and 1e-2 (GANs) per gradient tensor, TF32 mode max(5e-2, 2 x the operand-rounding emulation).  After
    the step the state_pred variables are bit-unchanged and their gradient is exactly 0."""
    hk = TRAIN_CASES[case]
    hp = O.make_hparams(**hk)
    B, step, shape, A, Sd = 2, 5, (64, 64, 3), 4, 3
    params, _ = S.init_params(hp, shape, action_dim=A, state_dim=Sd, seed=0)
    inputs, noise = S.make_synthetic_inputs(hp, B, shape, action_dim=A, state_dim=Sd)
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
        # TF32 mode: the GAN losses after the D update also move with operand rounding, bounded like the gradients by
        # 2 x the deviation of the operand-rounding emulation
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
    worst.sort(reverse=True)
    print('states %s [%s]: worst gradient errors %s' % (case, arith, ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    for k in ('gen_images', 'gen_images_enc'):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)
    for n in ('kernel', 'bias'):
        k = SC + '/state_pred/dense/' + n
        assert res['g_grads'][k] is None
        assert torch.equal(model.params[k].cpu(), params[k]), k
        assert float(model.grads[k].abs().max()) == 0.0, k


def test_captured_step_with_states_reproduces_the_eager_step(Model, tmp_path):
    """The eager step and two graph replays from the same checkpoint give bit-identical losses, gradients and gen_states
    (the captured graph replays the state recurrence with the step's redrawn mask)."""
    hk = dict(TRAIN_CASES['savp'], sequence_length=8, clip_length=6)
    hp = O.make_hparams(**hk)
    params, _ = S.init_params(hp, (64, 64, 3), action_dim=4, state_dim=3, seed=0)
    params[SC + '/state_pred/dense/kernel'] = torch.randn(7, 3, generator=torch.Generator().manual_seed(3)) * 0.3
    inputs, _ = S.make_synthetic_inputs(hp, 2, (64, 64, 3), action_dim=4, state_dim=3)
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
            runs[how].append((model.loss_vals.clone(), model.g_grad.clone(), model.d_grad.clone(), model.Bf['gstates'].clone()))
    ref = runs['eager'][0]
    for got in runs['graph']:
        for name, a, b in zip(('losses', 'g_grad', 'd_grad', 'gen_states'), got, ref):
            assert torch.equal(a, b), (name, (a - b).abs().max().item())
    assert torch.isfinite(ref[3]).all() and ref[3].abs().max() > 0


# ------------------------------------------------------------------------------------------------ checkpoints and scripts
def test_tf_checkpoint_of_a_states_model(Model, tmp_path):
    """A TensorFlow bundle of a states model's variables under the historical 'dna_cell' scope restores exactly; a model
    without states refuses it with the shape-mismatch ValueError."""
    from test_tf_checkpoint import write_bundle
    hk = dict(context_frames=2, sequence_length=6, nz=8)
    imgs = np.random.default_rng(0).uniform(size=(2, 6, 64, 64, 3)).astype(np.float32)
    acts = np.zeros((2, 5, 4), np.float32)
    src = Model(mode='test', hparams_dict=hk)
    src.build_graph({'images': imgs, 'actions': acts, 'states': np.zeros((2, 6, 3), np.float32)})
    src.init_params(seed=9)
    want = src.get_params()
    assert want[SC + '/state_pred/dense/kernel'].shape == (7, 3)
    tensors = {k.replace('savp_cell', 'dna_cell'): v for k, v in want.items()}
    tensors['global_step'] = np.array(77, np.int64)
    write_bundle(str(tmp_path / 'model-77'), tensors)
    (tmp_path / 'checkpoint').write_text('model_checkpoint_path: "model-77"\n')
    dst = Model(mode='test', hparams_dict=hk)
    dst.build_graph({'images': imgs, 'actions': acts, 'states': np.zeros((2, 6, 3), np.float32)})
    dst.restore(None, str(tmp_path))
    got = dst.get_params()
    assert dst.global_step == 77 and set(got) == set(want)
    for k, v in want.items():
        assert np.array_equal(got[k], v), k
    plain = Model(mode='test', hparams_dict=hk)
    plain.build_graph({'images': imgs, 'actions': acts})
    with pytest.raises(ValueError, match='shape mismatch'):
        plain.restore(None, str(tmp_path))


def _scripts():
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    import evaluate
    import generate
    import train
    return train, generate, evaluate


def _gen_states_shape(model):
    model._collect_outputs()
    return tuple(model.outputs['gen_states'].shape)


def test_train_on_bair_records_with_use_state_builds_a_states_model(Model, tmp_path):
    """The BAIR records of test_scripts.py (4-d actions, 3-d endeffector_pos) with use_state=True: the model gets Sd = 3."""
    train, _, _ = _scripts()
    from video_prediction_b200.datasets import tfrecord as R
    rng = np.random.default_rng(0)
    d = tmp_path / 'bair' / 'train'
    d.mkdir(parents=True)
    recs = []
    for _ in range(4):
        base = rng.integers(0, 255, (64, 64, 3), dtype=np.uint8)
        f = {}
        for t in range(30):
            f['%d/image_aux1/encoded' % t] = np.roll(base, (t, 2 * t), axis=(0, 1)).tobytes()
            f['%d/endeffector_pos' % t] = rng.standard_normal(3).astype(np.float32)
            if t < 29:
                f['%d/action' % t] = rng.standard_normal(4).astype(np.float32)
        recs.append(R.make_example(f))
    R.write_records(str(d / 'traj_0_to_3.tfrecords'), recs)
    model = train.main(['--input_dir', str(tmp_path / 'bair'), '--dataset', 'bair', '--dataset_hparams', 'use_state=True,sequence_length=6',
                        '--model', 'savp', '--output_dir', str(tmp_path / 'run'), '--progress_freq', '1', '--save_freq', '0',
                        '--seed', '2', '--model_hparams',
                        'batch_size=2,max_steps=2,clip_length=4,l1_weight=100.0,kl_weight=1.0,video_sn_gan_weight=0.1'])
    assert model.global_step == 2 and np.isfinite(model.g_loss) and np.isfinite(model.d_loss)
    assert model.A == 4 and model.Sd == 3 and _gen_states_shape(model) == (2, 5, 3)
    assert model.params[SC + '/h0/conv_pool2d/kernel'].shape[2] == 2 * 3 + 4 + 3 + 8


def test_synthetic_states_train_generate_evaluate(Model, tmp_path):
    train, generate, evaluate = _scripts()
    out = str(tmp_path / 'run')
    model = train.main(['--input_dir', 'none', '--dataset', 'synthetic', '--dataset_hparams',
                        'sequence_length=6,num_examples=8,action_dim=4,use_state=True', '--model', 'savp', '--output_dir', out,
                        '--progress_freq', '0', '--save_freq', '2', '--seed', '1', '--model_hparams',
                        'batch_size=2,max_steps=2,clip_length=4,l1_weight=100.0,kl_weight=1.0,video_sn_gan_weight=0.1'])
    assert model.Sd == 3 and model.A == 4 and _gen_states_shape(model) == (2, 5, 3)
    n = generate.main(['--input_dir', 'none', '--checkpoint', out, '--results_dir', str(tmp_path / 'results'), '--batch_size', '2',
                       '--num_samples', '2', '--num_stochastic_samples', '2', '--mode', 'test'])
    assert n == 2
    summary = evaluate.main(['--input_dir', 'none', '--checkpoint', out, '--mode', 'test', '--results_dir', str(tmp_path / 'eval'),
                             '--batch_size', '2', '--num_samples', '2', '--num_stochastic_samples', '2'])
    assert set(summary) == {'psnr', 'ssim', 'mse'} and all(np.isfinite(v) for v in summary.values())
