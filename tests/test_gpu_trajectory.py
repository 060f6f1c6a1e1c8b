"""Training over several steps (-m gpu): the state one step leaves for the next, CUDA-graph replays at steps other than the
capture step, and a resume in the middle of a run.  Every other parity test takes ONE step from a fresh optimizer state;
training (and the step bench.py times) is all later steps: non-zero Adam moments, two Adam counters, lr_t and the KL weight
moving with global_step, the spectral-norm u' of one step read by the next, and gradient buffers that have to be rewritten
(or zeroed) every step.

1. Teacher-forced parity: a K-step trajectory on the GPU, and before each step the oracle is run from a snapshot of the GPU's
   own state (parameters including u, Adam slots, counters, global_step), so that each step is a single-step comparison
   with test_gpu_train_parity.py's tolerances, and rounding cannot build up.  Adam is also checked on its own, in fp64
   from the snapshot and the GPU's gradient.
2. Bit identity of eager and replayed steps at every step of a run (B = 16 resident inputs, and explicit per-step inputs).
3. Resume: a model restored after step j (from this package's checkpoint and from a TF bundle) continues bit for bit as the
   run that never stopped, while every per-step buffer is filled with NaN before each step.

Worst errors per check and step are printed at the end of the module (pytest -s)."""
import os
import sys

import numpy as np
import pytest
import torch

import savp_compositor_oracle as C
import test_gpu_train_parity as TP
from oracle import savp_oracle as O
from test_gpu_reproducible import dirty_scratch
from test_tf_checkpoint import write_bundle

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'golden'))

K = 4                       # steps of a trajectory, from global_step = 0
B, SHAPE = 2, (64, 64, 3)
WORST = {}                  # '<check> <case> [<mode>] (tol <t>)' -> [worst error of step 0, 1, ...]


@pytest.fixture(scope='module')
def Model():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if WORST:
        print('\nworst error per check, case and tolerance, step by step:')
        for k in sorted(WORST):
            print('  %-70s %s' % (k, ' '.join('%.2e' % v for v in WORST[k])))


def _record(key, step, err):
    w = WORST.setdefault(key, [])
    while len(w) <= step:
        w.append(0.0)
    w[step] = max(w[step], err)


def _schedules(lr, kl='linear'):
    """lr decays linearly to lr / 4 over the K steps; the KL weight rises linearly from 0 (or along a sigmoid)."""
    s = dict(lr=lr, end_lr=0.25 * lr, decay_steps=(0, K))
    s.update(dict(kl_anneal='linear', kl_anneal_steps=(0, K)) if kl == 'linear' else dict(kl_anneal='sigmoid', kl_anneal_k=2.0))
    return s


# name -> (why the case is here, hparams, EXACT_GTOL key, a new batch every step).  The GAN cases keep
# test_gpu_train_parity.py's batch at every step: with B = 2 their discriminator gradients are a near-cancellation of the
# real and the fake clips, and how close depends on the batch (the tolerances there were set on that one).
CASES = {
    'savp': ('video towers on both unrolls, KL, CDNA: the shipped configuration',
             dict(TP.CASES['savp'], **_schedules(2e-4)), 'savp', False),
    'image_video_gan': ('image towers that share the video towers\' offsets, and both feature-cdist terms',
                        dict(TP.CASES['image_video_gan'], **_schedules(2e-4)), 'image_video_gan', False),
    'vae_flow': ('flow transforms (moved flow biases), sigmoid KL annealing',
                 dict(TP.CASES['vae_flow'], **_schedules(1e-3, kl='sigmoid')), 'vae_flow', True),
    'layers': ('layer norm, norm-free ConvLSTM, strided / transposed convolutions, and a frame history across time steps',
               dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3, norm_layer='layer',
                    conv_rnn_norm_layer='none', downsample_layer='conv2d', upsample_layer='deconv2d', last_frames=2,
                    **_schedules(1e-3)), 'vae_l1', True),
}
# fp32-exact mode, GAN cases: after a few discriminator updates the tower gradients near the logits are a sharper
# cancellation of real and fake clips than at the first step, and the exact mode's float atomics make each run's state a
# little different.  Measured on an H100 (relative L2, worst tensor): savp 7.5e-3 and 1.59e-2 at step 2 in two runs of the
# same trajectory (encoder/video sn_conv3_0 bias), image_video_gan 2.03e-2 at step 3 (image sn_conv3_0 kernel; 5.6e-3 at
# step 0).  EXACT_GTOL's 1e-2 holds at step 0 and 1.
TRAJ_EXACT_GTOL = {'savp': 3e-2, 'image_video_gan': 3e-2}
FLOW_BIAS = 'generator/rnn/savp_cell/flows/conv2d/bias'


def init_params(hp, hk):
    params, _ = C.init_params(hp, SHAPE, seed=0)
    if hk.get('transformation') == 'flow':     # off the floor() discontinuity of image_warp (test_gpu_train_parity.py)
        params[FLOW_BIAS] = torch.tensor([0.37, 1.27, -0.53, 2.17, 0.61, -1.43, 0.29, 1.71])
    return params


def step_data(hp, k, batch=B, new_clips=False):
    """Step k's inputs, noise (eps, z_prior, d_pre / d_post offsets) and scheduled-sampling mask [T-1-ctx, B].  The noise and
    the mask differ from step to step; the clips are test_gpu_train_parity.py's batch, or with new_clips a new batch every
    step."""
    inputs, _ = O.make_synthetic_inputs(hp, batch, SHAPE, seed=100 + k if new_clips else 0)
    _, noise = O.make_synthetic_inputs(hp, batch, SHAPE, seed=100 + k)
    g = torch.Generator().manual_seed(200 + k)
    sampling = torch.rand(hp.sequence_length - 1 - hp.context_frames, batch, generator=g) < 0.5
    return inputs, noise, sampling


def gpu_args(data):
    inputs, noise, sampling = data
    return {'images': inputs['images'].permute(1, 0, 2, 3, 4).contiguous()}, noise, sampling


def build(Model, hk, params, inputs, graph):
    model = Model(mode='train', hparams_dict=hk)
    model.set_params(params)
    model.build_graph({'images': inputs['images'].permute(1, 0, 2, 3, 4).contiguous()})
    model.global_step = 0
    model.use_cuda_graph = graph
    return model


def snapshot(model, names):
    """The state a step starts from: parameters (with u), Adam slots, both counters, global_step."""
    P = {k: model.params[k].detach().cpu().clone() for k in names}
    m, v = {}, {}
    for k in names:
        if k.endswith('/u'):
            continue
        flat, sm, sv = (model.g_flat, model.g_m, model.g_v) if k.startswith('generator/') else (model.d_flat, model.d_m, model.d_v)
        m[k] = model._view_of(sm, flat, k).detach().cpu().clone()
        v[k] = model._view_of(sv, flat, k).detach().cpu().clone()
    return dict(p=P, m=m, v=v, g_t=model.g_adam_t, d_t=model.d_adam_t, step=model.global_step)


def _oracle(case, hp, snap, data, quant):
    inputs, noise, sampling = data
    O.set_tf32_emulation(quant, ())
    try:
        params = {k: v.clone() for k, v in snap['p'].items()}
        opt = dict(m={k: v.clone() for k, v in snap['m'].items()}, v={k: v.clone() for k, v in snap['v'].items()}, t=snap['g_t'])
        step = C.train_step if case == 'layers' else O.train_step
        return step(params, opt, hp, inputs, noise, step=snap['step'], sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


def _check_step(case, mode, k, model, res, emu_fn):
    """One step against the oracle with test_gpu_train_parity.py's rules: losses, totals, per-tensor gradients (EXACT_GTOL,
    or max(5e-2, 2 x emulated) in TF32 mode), outputs, the stored u'."""
    hp_tag = '%s [%s]' % (case, mode)
    _, ltol, floor, otol = TP.MODES[mode]
    if 'd_grads' in res:
        us = [n for n in res['params'] if n.endswith('/u')]
        assert us
        e = max((model.params[n].cpu() - res['params'][n]).abs().max().item() for n in us)
        _record('1 stored u\' %s (max-abs, tol 1e-4)' % hp_tag, k, e)
        assert e <= 1e-4, (hp_tag, k, e)
    lv = model.losses()
    ref_l = dict(res['g_losses'])
    ref_l.update(res.get('d_losses', {}))
    worst_l, emu = 0.0, None
    for name, v in list(ref_l.items()) + [('g_loss', res['g_loss'])] + ([('d_loss', res['d_loss'])] if 'd_loss' in res else []):
        got = getattr(model, name) if name in ('g_loss', 'd_loss') else lv[name]
        tol = ltol * abs(v)
        if mode == 'tf32' and abs(got - v) > tol + 1e-6:
            # the post-update discriminator reads weights moved by +-lr Adam steps whose signs rounding can flip: as in
            # test_gpu_layer_choices.py, the bound is then 2 x the deviation of the oracle with the hardware's operand rounding
            emu = emu if emu is not None else emu_fn()
            ev = emu['g_loss'] if name == 'g_loss' else emu['d_loss'] if name == 'd_loss' else \
                dict(emu['g_losses'], **emu.get('d_losses', {}))[name]
            tol = max(tol, 2.0 * abs(ev - v))
        worst_l = max(worst_l, abs(got - v) / (tol + 1e-6))
        assert abs(got - v) <= tol + 1e-6, (hp_tag, k, name, got, v, tol)
    _record('1 losses %s (error / bound, tol 1)' % hp_tag, k, worst_l)
    worst, bad = 0.0, []
    for kind in ('g_grads', 'd_grads'):
        if kind not in res:
            continue
        items = [(n, g) for n, g in res[kind].items() if g is not None]
        gmax = max(g.double().norm().item() for _, g in items)
        for n, g in items:
            r, nrm = TP._rel(model.grads[n], g)
            if nrm < floor * gmax:
                continue
            if mode == 'exact':
                tol = TRAJ_EXACT_GTOL.get(case, TP.EXACT_GTOL[CASES[case][2]])
            else:
                tol = 5e-2
                if r > tol:             # only then does the emulated-rounding bound decide: run that oracle once
                    emu = emu if emu is not None else emu_fn()
                    tol = max(5e-2, 2.0 * TP._rel(emu[kind][n], g)[0])
            worst = max(worst, r / tol)
            if r > tol:
                bad.append((r, tol, n))
    _record('1 gradients %s (rel L2 / tol, tol 1)' % hp_tag, k, worst)
    assert not bad, (hp_tag, 'step', k, sorted(bad, reverse=True)[:5])
    outs = ('gen_images',) + (('gen_images_enc',) if model.hparams.nz else ())
    e = max((model.outputs_time_major(o).cpu() - res['outputs'][o]).abs().max().item() for o in outs)
    _record('1 gen_images %s (max-abs, tol %g)' % (hp_tag, otol), k, e)
    assert e <= otol, (hp_tag, k, e)


def _check_adam(case, mode, k, model, snap, hp):
    """p, m, v after the step against fp64 TF-Adam from the snapshot and the GPU's own gradient, with lr(global_step) and the
    snapshot's counter + 1 (test_gpu_step_kernels.py::test_adam's tolerances): pins lr_t, the counters and the slots apart
    from gradient rounding."""
    b2 = float(np.float32(hp.beta2))           # the kernel's fp32 beta2
    lr = O.learning_rate(hp, snap['step'])
    for prefix, t in (('generator/', snap['g_t']), ('discriminator/', snap['d_t'])):
        names = [n for n in snap['m'] if n.startswith(prefix)]
        if not names:
            continue
        cat = lambda d: torch.cat([d[n].reshape(-1).double() for n in names])      # noqa: E731
        flat = model.g_flat if prefix == 'generator/' else model.d_flat
        sm, sv = (model.g_m, model.g_v) if prefix == 'generator/' else (model.d_m, model.d_v)
        g = torch.cat([model.grads[n].detach().cpu().reshape(-1).double() for n in names])
        pr, mr, vr = O.adam_tf(cat(snap['p']), g, cat(snap['m']), cat(snap['v']), lr, hp.beta1, b2, t + 1)
        got = dict(p=torch.cat([model.params[n].detach().cpu().reshape(-1).double() for n in names]),
                   m=torch.cat([model._view_of(sm, flat, n).cpu().reshape(-1).double() for n in names]),
                   v=torch.cat([model._view_of(sv, flat, n).cpu().reshape(-1).double() for n in names]))
        for what, ref, scale in (('p', pr, max(pr.abs().max().item(), 1.0)), ('m', mr, mr.abs().max().item()),
                                 ('v', vr, vr.abs().max().item())):
            e = ((got[what] - ref).abs().max() / (scale + 1e-300)).item()
            _record('1 adam %s %s%s [%s] (max-abs / scale, tol 1e-6)' % (what, prefix, case, mode), k, e)
            assert e <= 1e-6, (case, mode, k, prefix, what, e)


@pytest.mark.parametrize('mode', ['tf32', 'exact'])
@pytest.mark.parametrize('case', sorted(CASES))
def test_trajectory_matches_oracle_step_by_step(Model, case, mode):
    """K steps from global_step 0 with a moving lr, KL weight, mask and noise; each compared with the oracle run from the
    GPU's own state before it.  The TF32 run captures the CUDA graph at step 1, so steps 2 .. K-1 are replays."""
    _, hk, _, new_clips = CASES[case]
    hp = O.make_hparams(**hk)
    params = init_params(hp, hk)
    data = [step_data(hp, k, new_clips=new_clips) for k in range(K)]
    with TP.arithmetic(mode):
        model = build(Model, hk, params, data[0][0], graph=(mode == 'tf32'))
        assert set(model.params) == set(params)
        for k in range(K):
            snap = snapshot(model, list(params))
            assert snap['step'] == k
            if model.dnets:
                assert snap['g_t'] == snap['d_t'] == k      # the oracle's single opt['t']
            model.train_step(*gpu_args(data[k]))
            torch.cuda.synchronize()
            assert model.global_step == k + 1
            assert (model._graph is not None) == (mode == 'tf32' and k >= 1)
            res = _oracle(case, hp, snap, data[k], None)
            _check_step(case, mode, k, model, res, lambda: _oracle(case, hp, snap, data[k], TP.tf32_mode()))
            _check_adam(case, mode, k, model, snap, hp)


# ---------------------------------------------------------------------------------------------- eager vs replay, every step
def state(model):
    """Everything a step writes that the next one reads, or that the caller sees."""
    out = dict(g_grad=model.g_grad, d_grad=model.d_grad, loss_vals=model.loss_vals, g_flat=model.g_flat, d_flat=model.d_flat,
               g_m=model.g_m, g_v=model.g_v, d_m=model.d_m, d_v=model.d_v, sel=model.Bf['sel'])
    if model.hparams.nz:
        out.update(eps=model.Bf['eps'], zprior=model.Bf['zprior'])
    for k in model.params:
        if k.endswith('/u'):
            out[k] = model.params[k]
    for scope, net in model.dnets.items():
        for key, t in net['ts'].items():
            out['%s/ts%s' % (scope, key)] = t
    return {k: v.detach().clone() for k, v in out.items()}


def _assert_identical(a, b, what):
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, (what, diff[:8])
    nonfinite = [k for k in a if a[k].is_floating_point() and not bool(torch.isfinite(a[k]).all())]
    assert not nonfinite, (what, nonfinite)


def test_replays_at_later_steps_are_the_eager_steps_b16_resident(Model):
    """The configuration and path bench.py times (cfg2, B = 16, resident inputs: the model draws its own eps, z_prior,
    mask and offsets from global_step), with schedule_sampling_k = 1 so that P(ground truth) falls 0.5, 0.27, 0.12, ...
    and the masks change from step to step.  Five steps eager and with the CUDA graph: bit-identical after every step.
    transformation='flow' and the fp32-exact mode still add with float atomics (DESIGN.md) and are not run-to-run exact,
    so they are not part of this check."""
    import make_golden_b16 as G
    hk = dict(G.HK, schedule_sampling_k=1.0)
    _, params, inputs, _ = G.case()
    binp = {'images': inputs['images'].permute(1, 0, 2, 3, 4).contiguous()}
    models = []
    with TP.arithmetic('tf32'):
        for graph in (False, True):
            m = Model(mode='train', hparams_dict=hk)
            m.set_params(params)
            m.build_graph(binp)
            m.set_inputs(binp)
            m.use_cuda_graph = graph
            models.append(m)
        sels = []
        for k in range(5):
            states = []
            for m in models:
                m.train_step()
                torch.cuda.synchronize()
                states.append(state(m))
            assert models[1]._graph is not None or k == 0
            _assert_identical(states[0], states[1], 'step %d' % k)
            sels.append(states[0])
    ctx = hk['context_frames']
    for k in range(1, len(sels)):
        prev, cur = sels[k - 1], sels[k]
        # fresh draws: the mask of a step is not the previous one thinned by the lower probability (the same uniforms)
        assert bool((cur['sel'][ctx:] > prev['sel'][ctx:]).any()), 'steps %d, %d: the mask was not redrawn' % (k - 1, k)
        same = [n for n in ('eps', 'zprior') + tuple(n for n in cur if '/ts' in n) if torch.equal(cur[n], prev[n])]
        assert not same, ('steps %d, %d draw the same values' % (k - 1, k), same)
    assert int(sels[0]['sel'][ctx:].sum()) > int(sels[-1]['sel'][ctx:].sum())


def test_replays_at_later_steps_are_the_eager_steps_explicit_inputs(Model):
    """The 'savp' trajectory with explicit per-step batches, noise and masks, eager and with the CUDA graph: set_inputs
    and stage_step have to copy every step's values into the buffers the graph reads."""
    hk = CASES['savp'][1]
    hp = O.make_hparams(**hk)
    params = init_params(hp, hk)
    data = [step_data(hp, k, new_clips=True) for k in range(K)]
    with TP.arithmetic('tf32'):
        models = [build(Model, hk, params, data[0][0], graph=g) for g in (False, True)]
        for k in range(K):
            states = []
            for m in models:
                m.train_step(*gpu_args(data[k]))
                torch.cuda.synchronize()
                states.append(state(m))
            _assert_identical(states[0], states[1], 'step %d' % k)


# ---------------------------------------------------------------------------------------------- resume, stale state poisoned
# Per-step buffers that must NOT be poisoned, because the step reads them without writing them: (see DESIGN.md (f))
PERSISTENT = ()


def poison_targets(model, persistent=PERSISTENT):
    """(name, buffer) of everything a step must rewrite before reading it: the flat gradients and the loss vector, the
    generator's gradient buffers, every discriminator tower's dlogits / dclip / dfeat / dcd rows, the spectral-norm
    gradient scratch, and every convolution's packed weight gradient."""
    out = [('g_grad', model.g_grad), ('d_grad', model.d_grad), ('loss_vals', model.loss_vals)]
    out += [('Gb/' + k, v) for k, v in model.Gb.items()]
    for scope, net in model.dnets.items():
        out += [(scope + '/dlogits', net['dlogits']), (scope + '/dclip', net['dclip'])]
        out += [('%s/dfeat%d' % (scope, i), t) for i, t in enumerate(net['dfeat'])]
        out += [('%s/dcd%d' % (scope, i), t) for i, t in enumerate(net['dcd'])]
        for lay in net['layers'] + [net['fc']]:
            out.append((lay.uname + ':gwbar', lay.gwbar))
            if not lay.is_fc:
                out.append((lay.wname + ':dwp', lay.conv.dwp))
    out += [(c.wname + ':dwp', c.dwp) for c in model.convs]
    return [(n, t) for n, t in out if n not in persistent]


def poison(model):
    for _, t in poison_targets(model):
        t.fill_(float('nan'))
    dirty_scratch()


def _bundle(model, prefix):
    """A TensorFlow checkpoint of the model's state as the reference writes it: variables, `<var>/Adam` and `<var>/Adam_1`
    slots, global_step and beta1_power = beta1^(t + 1)."""
    assert model.g_adam_t == model.d_adam_t
    tensors = {k: v.detach().cpu().numpy() for k, v in model.params.items()}
    for k in model.params:
        if k.endswith('/u'):
            continue
        flat, sm, sv = (model.g_flat, model.g_m, model.g_v) if k.startswith('generator/') else (model.d_flat, model.d_m, model.d_v)
        tensors[k + '/Adam'] = model._view_of(sm, flat, k).detach().cpu().numpy()
        tensors[k + '/Adam_1'] = model._view_of(sv, flat, k).detach().cpu().numpy()
    tensors['global_step'] = np.array(model.global_step, np.int64)
    tensors['beta1_power'] = np.array(model.hparams.beta1 ** (model.g_adam_t + 1), np.float32)
    write_bundle(prefix, tensors)
    with open(os.path.join(os.path.dirname(prefix), 'checkpoint'), 'w') as f:
        f.write('model_checkpoint_path: "%s"\n' % os.path.basename(prefix))


def test_resume_mid_trajectory_continues_bit_for_bit(Model, tmp_path):
    """Model A runs K steps with the CUDA graph, every per-step buffer NaN before each step, and is saved after step J.
    Models restored from that checkpoint (this package's .npz, and a TF bundle from which restore derives the Adam
    counter) run steps J .. K-1 on the same batches, noise and masks, poisoned the same way: their first step is eager,
    A's a replay, and every step must equal A's bit for bit.  A itself must equal an eager run that is never poisoned."""
    J = 2
    hk = CASES['savp'][1]
    hp = O.make_hparams(**hk)
    params = init_params(hp, hk)
    data = [step_data(hp, k, new_clips=True) for k in range(K)]
    with TP.arithmetic('tf32'):
        clean = build(Model, hk, params, data[0][0], graph=False)
        ref_clean = []
        for k in range(K):
            clean.train_step(*gpu_args(data[k]))
            torch.cuda.synchronize()
            ref_clean.append(state(clean))
        del clean
        a = build(Model, hk, params, data[0][0], graph=True)
        ref, ck = [], None
        for k in range(K):
            if k == J:
                ck = a.save(str(tmp_path / 'npz'))
                os.makedirs(str(tmp_path / 'tf'))
                _bundle(a, str(tmp_path / 'tf' / ('model-%d' % J)))
                adam_t = (a.g_adam_t, a.d_adam_t)
            poison(a)
            a.train_step(*gpu_args(data[k]))
            torch.cuda.synchronize()
            ref.append(state(a))
            _assert_identical(ref[k], ref_clean[k], 'poisoned run, step %d' % k)
        assert a._graph is not None
        for how, path in (('npz', ck), ('tf bundle', str(tmp_path / 'tf'))):
            b = build(Model, hk, init_params(hp, hk), data[0][0], graph=True)
            b.restore(None, path)
            assert b.global_step == J and (b.g_adam_t, b.d_adam_t) == adam_t, (how, b.global_step, b.g_adam_t, b.d_adam_t)
            for k in range(J, K):
                poison(b)
                b.train_step(*gpu_args(data[k]))
                torch.cuda.synchronize()
                assert (b._graph is not None) == (k > J)
                _assert_identical(state(b), ref[k], '%s resume, step %d' % (how, k))
