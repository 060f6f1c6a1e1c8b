"""GPU tests (-m gpu) of the per-frame image discriminator over the sampled clip (`images_sn_gan_weight`,
`images_sn_vae_gan_weight`): every convolution of the tower at the frame counts it runs (N = 2 B clip) against fp64, the
tower's forward and backward against the fp64 reference (tests/savp_images_d_oracle.py) with autograd, the training step
against the fp32 reference in both arithmetic modes, bit-identical reruns and graph replays, and checkpoints (.npz and a TF
bundle with the reference's names)."""
import numpy as np
import pytest
import torch

import savp_images_d_oracle as R
from oracle import savp_oracle as O
from test_gpu_engine import ACC_FLOOR, MAX_ABS, NAN, OFF, PLAIN, L, MODEL_CASES, _norm_cmap, act_input, mode, out_buf, ref_conv, ref_wgrad, rnd, tf32, unpack  # noqa: F401,E501
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, _check_grads, _check_grads_tf32, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
ALPHA = 0.1                 # the discriminator's leaky relu
IMAGE_CASES = MODEL_CASES[-7:]      # the image tower's seven geometries (one frame: extent (1, H, W))
# frames the engine sees per call: 2 B clip of cfg2 (B = 16, clip 10), and an odd 2 * 37 * 3
FRAMES = [320, 222]


def _gid(c):
    kind, k, s, p, t, ci_ref, ci_int, cmap, co, ext = c
    return 'k%d_s%d_%d-%d_co%d_%d' % (k[1], s[1], ci_ref, ci_int, co, ext[1])


def _close(errs, name, got, ref, K):
    """relative L2 within ACC_FLOOR accumulation floors (2^-24 sqrt(K)), max-abs within max(MAX_ABS, the same bound) of
    max|ref| (the weight gradient sums K = N H W products, 1.3 M at cfg2's first layer)"""
    d = got.double() - ref
    tol = ACC_FLOOR * 2.0 ** -24 * K ** 0.5
    rl2 = (d.norm() / ref.norm().clamp_min(1e-300)).item()
    mab = (d.abs().max() / ref.abs().max().clamp_min(1e-300)).item()
    errs.append((name, rl2, tol, mab, max(MAX_ABS, tol)))


@pytest.mark.parametrize('n', FRAMES)
@pytest.mark.parametrize('case', IMAGE_CASES, ids=_gid)
def test_tower_convolutions_match_fp64(L, mode, case, n):  # noqa: F811
    """Forward (bias + leaky relu), dgrad, the fused leaky-relu-gradient dgrad with addend, and the weight gradient (split_k
    auto) of each layer of the tower at N frames, against ref_conv / ref_wgrad on the operands the tensor core reads."""
    kind, k, s, p, transposed, ci_ref, ci_int, cmap, co, ext = case
    taps = k[1] * k[2]
    oext = tuple((i + 2 * pp - kk) // ss + 1 for i, ss, pp, kk in zip(ext, s, p, k))
    cm = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device='cuda')
    w = rnd(*k, ci_ref, co, seed=1, scale=(taps * ci_ref) ** -0.5)
    bias = rnd(co, seed=2, scale=0.3)
    wp, n_pad, kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm)
    wpd, n_pad_d, kc_d = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int, cmap=cm)
    wf, wd = unpack(wp, taps, n_pad, kc, co, ci_int), unpack(wpd, taps, n_pad_d, kc_d, ci_int, co)
    g, gt = L.geom(k, s, p, False), L.geom(k, s, p, True)
    errs = []
    x = act_input(n, ext, ci_int, cmap, seed=3)
    xv = L.tensor_view(x, ci_int)
    pre = ref_conv(tf32(x, mode)[..., :ci_int].double(), wf, k, s, p, False, oext)
    out = out_buf(n, oext, co)
    L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, co, OFF), bias, L.ACT_LRELU, ALPHA)
    _close(errs, 'fwd', out[..., OFF:OFF + co], torch.maximum(ALPHA * (pre + bias.double()), pre + bias.double()), taps * ci_int)
    del pre
    dy = act_input(n, oext, (co + 3) // 4 * 4, None, seed=5)
    dy[..., co:] = NAN
    dyq = tf32(dy, mode)[..., :co].double()
    dyv = L.tensor_view(dy, co)
    dref = ref_conv(dyq, wd, k, s, p, True, ext)
    kd = taps * co / (s[1] * s[2])
    dx = out_buf(n, ext, ci_int)
    L.conv_igemm(dyv, gt, wpd, n_pad_d, kc_d, L.tensor_view(dx, ci_int, OFF))
    _close(errs, 'dgrad', dx[..., OFF:OFF + ci_int], dref, kd)
    y = rnd(n, *ext, ci_int, seed=8)
    y = torch.where(y > 0, y, ALPHA * y)
    add = rnd(n, *ext, ci_int, seed=6)
    o = torch.full_like(add, NAN)
    L.conv_igemm_actgrad(dyv, gt, wpd, n_pad_d, kc_d, L.tensor_view(o, ci_int), y.data_ptr(), add.data_ptr(), L.ACT_LRELU, ALPHA, 0)
    _close(errs, 'actgrad', o, (dref + add.double()) * torch.where(y.double() > 0, 1.0, ALPHA), kd)
    del dref
    wref = ref_wgrad(tf32(x, mode)[..., :ci_int].double(), dyq, k, s, p, False).transpose(1, 2)
    full = torch.zeros(taps, n_pad, kc * 32, device='cuda', dtype=torch.float64)
    full[:, :co, :ci_int] = wref
    dwp = torch.zeros(taps * n_pad * kc * 32, device='cuda')
    L.conv_wgrad(xv, dyv, g, dwp, n_pad, kc, 0)
    _close(errs, 'wgrad', dwp.view(taps, n_pad, kc * 32), full, n * oext[1] * oext[2])
    untouched = bool(torch.isnan(out[..., :OFF]).all() and torch.isnan(out[..., OFF + co:]).all() and torch.isnan(dx[..., :OFF]).all())
    print('%s N=%d: %s' % (_gid(case), n, ' '.join('%s %.1e/%.1e' % (nm, r, t) for nm, r, t, _, _ in errs)))
    bad = [e for e in errs if not (e[1] <= e[2] and e[3] <= e[4])]
    assert not bad and untouched, (bad, untouched)


# ------------------------------------------------------------------------------------------------ model level
@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def test_cases_cover_every_tower_convolution(Model):
    """Every convolution of the images towers at cfg2 (and with an odd batch) runs a geometry of IMAGE_CASES on N frames of
    FRAMES: a new geometry or frame count fails here until it is tested above."""
    for B, want_n in ((16, 320), (37, 222)):
        hk = dict(context_frames=2, sequence_length=12, clip_length=10 if B == 16 else 3, nz=8, l1_weight=1.0,
                  images_sn_gan_weight=0.1, images_sn_vae_gan_weight=0.1)
        model = Model(mode='train', hparams_dict=hk)
        model.build_graph({'images': torch.zeros(B, 12, 64, 64, 3)})
        nets = [net for net in model.dnets.values() if net['kind'] == 'images']
        assert len(nets) == 2
        found = []
        for net in nets:
            for li, lay in enumerate(net['layers']):
                x = net['clip'] if li == 0 else net['feat'][li - 1]
                n = int(np.prod(x.shape[:2]))
                gm = lay.geom
                found.append(((PLAIN, tuple(lay.k3), tuple(lay.stride), (gm.pd, gm.ph, gm.pw), False, lay.cin_ref, lay.cin_int,
                               _norm_cmap(lay.cmap), lay.co, (1,) + tuple(x.shape[2:4])), n, lay.wname))
        missing = [(name, t, n) for t, n, name in found if t not in IMAGE_CASES or n != want_n]
        assert not missing, missing
        del model
        torch.cuda.empty_cache()


def test_tower_forward_and_backward_match_the_fp64_reference(Model):
    """One images tower (B = 3, clip 4: 24 frames) in the fp32-exact mode: logits and the 7 features (1e-4), then the
    backward of random logit gradients -- d clip and dW, db of every layer through the spectral norm -- against fp64
    autograd."""
    hk = dict(context_frames=2, sequence_length=6, clip_length=4, nz=0, ndf=32, l1_weight=1.0, images_sn_gan_weight=0.1)
    hp = O.make_hparams(**hk)
    B, shape = 3, (64, 64, 3)
    params, _ = R.init_params(hp, shape, seed=4)
    with arithmetic('exact'):
        model = Model(mode='train', hparams_dict=hk)
        model.set_params(params)
        model.build_graph({'images': torch.zeros(B, 6, 64, 64, 3)})
    net = model.dnets['discriminator/images']
    g = torch.Generator().manual_seed(11)
    clip = torch.rand(2 * B, 4, 64, 64, 3, generator=g)
    net['clip'].zero_()
    net['clip'][..., :3] = clip.cuda()
    model._d_sn_and_pack(net)
    model._d_forward(net, 0, 2 * B)
    dlog = torch.randn(2 * B * 4, generator=g)
    net['dlogits'].copy_(dlog.cuda())
    model.d_grad.zero_()
    net['dclip'].zero_()
    model._d_backward(net, 0, 2 * B, with_wgrad=True, to_clip=True)
    torch.cuda.synchronize()

    P = {k: v.double().requires_grad_(k.startswith('discriminator/') and not k.endswith('/u')) for k, v in params.items()}
    x = clip.double().permute(1, 0, 2, 3, 4).requires_grad_(True)          # time-major [clip, 2B, ...]
    feats, logits = R.images_sn_discriminator(O.Vars(P), 'discriminator/images', x, hp.ndf)
    lg = logits[..., 0].t().reshape(-1)                                   # the model's rows: sample-major, frame-minor
    assert (net['logits'].cpu().double() - lg).abs().max().item() <= 1e-4 * max(1.0, lg.abs().max().item())
    for l, f in enumerate(feats):
        got, ref = net['feat'][l].cpu().double(), f.permute(1, 0, 2, 3, 4)
        assert (got - ref).abs().max().item() <= 1e-4 * ref.abs().max().item(), l
    (lg * dlog.double()).sum().backward()
    dclip = net['dclip'][..., :3].cpu().double().permute(1, 0, 2, 3, 4)
    # the backward is held to the exact-mode gradient bound of test_gpu_train_parity.py's 'savp' case: the tensor core's fp32
    # accumulation through seven dgrads is less accurate than a CPU fp32 convolution (2.9e-3 measured on d clip, H100)
    assert _rel(dclip, x.grad)[0] <= EXACT_GTOL['savp']
    worst = []
    for k, v in P.items():
        if v.requires_grad:
            r, _ = _rel(model.grads[k], v.grad)
            worst.append((r, k))
    worst.sort(reverse=True)
    print('images tower backward: worst relative L2 %s' % ['%.2e %s' % w for w in worst[:3]])
    assert len(worst) == 16 and worst[0][0] <= EXACT_GTOL['savp'], worst[:3]


GAN = dict(context_frames=2, sequence_length=6, clip_length=4, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
           kl_anneal_steps=(0, 10))
TRAIN_CASES = {
    'images_gan_nz0': dict(GAN, nz=0, kl_weight=0.0, images_sn_gan_weight=0.1),
    'savp_video_images': dict(GAN, video_sn_gan_weight=0.1, video_sn_vae_gan_weight=0.1, images_sn_gan_weight=0.1,
                              images_sn_vae_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=1.0),
    'images_vae_gan': dict(GAN, images_sn_vae_gan_weight=0.1),
}


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return R.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


def _setup(case, B=2):
    hk = TRAIN_CASES[case]
    hp = O.make_hparams(**hk)
    params, _ = R.init_params(hp, (64, 64, 3), seed=0)
    inputs, noise = O.make_synthetic_inputs(hp, B, (64, 64, 3))
    return hk, hp, params, inputs, noise


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_matches_fp32_oracle(Model, case, arith):
    """B = 2, a random scheduled-sampling mask, test_gpu_train_parity.py's tolerances of its 'savp' case: losses, every
    gradient tensor, the generated frames and the stored u' of every tower."""
    hk, hp, params, inputs, noise = _setup(case)
    B, step = 2, 5
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
    ref_l = dict(res['g_losses'], **res['d_losses'])
    assert {k for k in ref_l if 'images_sn' in k}, ref_l
    for k, v in ref_l.items():
        assert abs(lv[k] - v) <= ltol * abs(v) + 1e-6, (k, lv[k], v)
    assert abs(model.g_loss - res['g_loss']) <= ltol * abs(res['g_loss']) + 1e-6, (model.g_loss, res['g_loss'])
    assert abs(model.d_loss - res['d_loss']) <= ltol * abs(res['d_loss']) + 1e-6, (model.d_loss, res['d_loss'])
    if arith == 'exact':
        _check_grads(model, res, EXACT_GTOL['savp'], floor, '%s [exact] vs fp32 oracle' % case)
    else:
        _check_grads_tf32(model, res, _oracle_step(hp, params, inputs, noise, step, sampling, tf32_mode()), floor, case)
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)
    us = [k for k in res['params'] if k.endswith('/u') and '/images/' in k]
    assert us
    for k in us:
        assert (model.params[k].cpu() - res['params'][k]).abs().max() <= 1e-4, k


def _step_state(model):
    torch.cuda.synchronize()
    return model.loss_vals.clone(), model.g_grad.clone(), model.d_grad.clone(), model.d_flat.clone()


def test_two_runs_are_bit_identical(Model):
    """Video and images towers on the same unroll add into the same rows of the frames' gradient: two runs of the step
    from the same state give the same bits."""
    hk, hp, params, inputs, noise = _setup('savp_video_images')
    runs = []
    for _ in range(2):
        model = Model(mode='train', hparams_dict=hk)
        model.set_params(params)
        model.build_graph(_batch_major(inputs))
        model.train_step(_batch_major(inputs), noise)
        runs.append(_step_state(model))
    for name, a, b in zip(('losses', 'g_grad', 'd_grad', 'd_flat'), *runs):
        assert torch.equal(a, b), (name, (a - b).abs().max().item())
    assert float(runs[0][2].abs().max()) > 0


def test_captured_step_reproduces_the_eager_step(Model, tmp_path):
    """The eager step and two graph replays from the same .npz checkpoint give bit-identical losses and gradients."""
    hk, hp, params, inputs, _ = _setup('savp_video_images')
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
            assert (model._graph is not None) == (how == 'graph')
            runs[how].append(_step_state(model))
    for got in runs['graph']:
        for name, a, b in zip(('losses', 'g_grad', 'd_grad', 'd_flat'), got, runs['eager'][0]):
            assert torch.equal(a, b), (name, (a - b).abs().max().item())


def test_checkpoints_round_trip(Model, tmp_path):
    """.npz save / restore returns every variable (images towers' kernels, biases and u included) and the Adam slots bit for
    bit; a TF bundle with the reference's variable names restores the images towers exactly."""
    from test_tf_checkpoint import write_bundle
    hk, hp, params, inputs, noise = _setup('savp_video_images')
    binp = _batch_major(inputs)
    model = Model(mode='train', hparams_dict=hk)
    model.set_params(params)
    model.build_graph(binp)
    model.train_step(binp, noise)
    path = model.save(str(tmp_path / 'npz'))
    other = Model(mode='train', hparams_dict=hk)
    other.build_graph(binp)
    other.restore(None, path)
    names = [k for k in model.params if '/images/' in k]
    assert len(names) == 48
    for k in model.params:
        assert torch.equal(other.params[k], model.params[k]), k
    for nm in ('d_m', 'd_v', 'g_m', 'g_v'):
        assert torch.equal(getattr(other, nm), getattr(model, nm)), nm
    tensors = {k: v.numpy().astype(np.float32) for k, v in params.items()}
    tensors['global_step'] = np.array(12, np.int64)
    write_bundle(str(tmp_path / 'model-12'), tensors)
    tf = Model(mode='train', hparams_dict=hk)
    tf.build_graph(binp)
    tf.restore(None, str(tmp_path / 'model-12'))
    assert tf.global_step == 12
    for k in names:
        assert np.array_equal(tf.params[k].cpu().numpy(), tensors[k]), k


def test_train_script_trains_and_resumes(Model, tmp_path):
    """scripts/train.py with both images weights: two steps on synthetic data, a checkpoint, then --resume continues from it
    with every images-tower variable restored."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'scripts'))
    import train
    out = str(tmp_path / 'run')
    hp = 'batch_size=2,max_steps=%d,clip_length=4,l1_weight=100.0,kl_weight=1.0,images_sn_gan_weight=0.1,images_sn_vae_gan_weight=0.1'
    args = ['--input_dir', 'none', '--dataset', 'synthetic', '--dataset_hparams', 'sequence_length=6,num_examples=8', '--model', 'savp',
            '--output_dir', out, '--progress_freq', '1', '--save_freq', '2', '--seed', '1']
    model = train.main(args + ['--model_hparams', hp % 2])
    assert model.global_step == 2 and np.isfinite(model.g_loss) and np.isfinite(model.d_loss)
    assert model.g_losses['gen_images_sn_vae_gan_loss'] > 0 and model.d_losses['discrim_images_sn_gan_loss'] > 0
    saved = {k: v.clone() for k, v in model.params.items() if '/images/' in k}
    assert len(saved) == 48
    resumed = train.main(args + ['--resume', '--model_hparams', hp % 3])
    assert resumed.global_step == 3
    changed = [k for k, v in saved.items() if not k.endswith('/u') and not torch.equal(resumed.params[k].cpu(), v.cpu())]
    assert changed          # one more step from the restored values
