"""GPU tests (-m gpu) of norm_layer = 'layer' | 'none': vp_lnorm_act / vp_lnorm_act_bwd against fp64 at every
(positions, channels, activation) extent of the 64x64 and 128x128 generators and the posterior encoder, bit-identical
reruns, rejected bad calls; the generator and the training step against the fp32 reference
(tests/savp_norm_layer_oracle.py); the captured step; and the restore of a TF bundle with LayerNorm names."""
import numpy as np
import pytest
import torch

import savp_norm_layer_oracle as R
from oracle import savp_oracle as O
from test_gpu_engine import L  # noqa: F401  (fixture)
from test_gpu_reproducible import twice
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
SC = 'generator/rnn/savp_cell'
NAN = float('nan')
NORMS = ('layer', 'none')

# (positions, channels, act) of every norm_layer site: 64x64 generator h0..h5 and heads, 128x128 generator, and the
# posterior encoder's layers 2 and 3 at 64x64 and 128x128 (leaky relu 0.2)
RELU, LRELU = 1, 2
EXTENTS = sorted(set([(1024, 32, RELU), (256, 64, RELU), (64, 128, RELU), (4096, 32, RELU),                        # 64x64
                      (4096, 32, RELU), (1024, 64, RELU), (256, 128, RELU), (64, 256, RELU), (256, 256, RELU),       # 128x128
                      (1024, 128, RELU), (4096, 64, RELU), (16384, 32, RELU),
                      (256, 128, LRELU), (64, 256, LRELU), (1024, 128, LRELU), (256, 256, LRELU)]))               # encoder


@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def _act(L, a):  # noqa: F811
    return {RELU: L.ACT_RELU, LRELU: L.ACT_LRELU}[a]


def _ref64(x, g, b, act):
    """fp64 layer norm + activation of x [N, P, C] (autograd-capable)."""
    m = x.mean(dim=(1, 2), keepdim=True)
    v = ((x - m) ** 2).mean(dim=(1, 2), keepdim=True)
    y = (x - m) * torch.rsqrt(v + 1e-12) * g + b
    return torch.relu(y) if act == RELU else torch.maximum(0.2 * y, y)


def _slab(N, P, C, cs, seed, off=0, fill=None):
    """[N, P, cs] buffer whose channels [off, off + C) hold data (N(0.5, 1) + a per-channel offset), the rest `fill`."""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((N, P, cs), NAN if fill is None else fill)
    buf[..., off:off + C] = torch.randn(N, P, C, generator=g) + 0.5 + 0.1 * torch.arange(C) / C
    return buf.cuda()


@pytest.mark.parametrize('ext', EXTENTS, ids=lambda e: '%dx%d_%s' % (e[0], e[1], 'relu' if e[2] == RELU else 'lrelu'))
def test_lnorm_act_matches_fp64(L, ext):  # noqa: F811
    P, C, act = ext
    N = 37
    x = _slab(N, P, C, C + 8, seed=P + C, off=4)
    gr = torch.Generator().manual_seed(1)
    g = (1.0 + 0.3 * torch.randn(C, generator=gr)).cuda()
    b = (0.2 * torch.randn(C, generator=gr)).cuda()
    ys = C + 12
    y = torch.full((N, P, ys), NAN, device='cuda')
    st = torch.full((N, 2), NAN, device='cuda')
    L.lnorm_act(x.data_ptr() + 16, C + 8, y.data_ptr() + 32, ys, N, P, C, g, b, _act(L, act), 0.2 if act == LRELU else 0.0, st)
    torch.cuda.synchronize()
    x64 = x[..., 4:4 + C].double()
    want = _ref64(x64, g.double(), b.double(), act)
    assert (y[..., 8:8 + C].double() - want).abs().max().item() <= 2e-5 * max(1.0, want.abs().max().item())
    assert torch.isnan(y[..., :8]).all() and torch.isnan(y[..., 8 + C:]).all()      # only the slice is written
    m = x64.mean(dim=(1, 2))
    r = torch.rsqrt(((x64 - m[:, None, None]) ** 2).mean(dim=(1, 2)) + 1e-12)
    assert (st[:, 0].double() - m).abs().max().item() <= 1e-5 and ((st[:, 1].double() - r) / r).abs().max().item() <= 1e-5

    # backward: 1 - 3 sources with their own strides, accumulation into non-zero dgamma / dbeta
    nsrc = 1 + (P + C) % 3
    srcs = [_slab(N, P, C, C + 4 * (k + 1), seed=100 + k, off=4 * k) for k in range(nsrc)]
    dy = sum(s[..., 4 * k:4 * k + C] for k, s in enumerate(srcs)).double()
    dx = torch.full((N, P, C + 4), NAN, device='cuda')
    dg0, db0 = torch.randn(C, generator=gr).cuda(), torch.randn(C, generator=gr).cuda()
    dg, db = dg0.clone(), db0.clone()
    L.lnorm_act_bwd(x.data_ptr() + 16, C + 8, [(s.data_ptr() + 16 * k, C + 4 * (k + 1)) for k, s in enumerate(srcs)], dx.data_ptr(), C + 4,
                    N, P, C, g, b, st, _act(L, act), 0.2 if act == LRELU else 0.0, dg, db)
    torch.cuda.synchronize()
    xg, g64, b64 = x64.clone().requires_grad_(True), g.double().requires_grad_(True), b.double().requires_grad_(True)
    (_ref64(xg, g64, b64, act) * dy).sum().backward()
    for got, want, what in ((dx[..., :C], xg.grad, 'dx'), (dg - dg0, g64.grad, 'dgamma'), (db - db0, b64.grad, 'dbeta')):
        err = (got.double() - want).abs().max().item() / max(1e-30, want.abs().max().item())
        assert err <= 5e-5, (ext, what, err)
    assert torch.isnan(dx[..., C:]).all()

    # the same calls again, the scratch pool NaN-filled in between: identical bits
    y2 = torch.zeros(N, P, C, device='cuda')
    st2 = torch.zeros(N, 2, device='cuda')
    dgr, dbr = dg0.clone(), db0.clone()
    dxr = torch.zeros(N, P, C, device='cuda')
    twice(lambda: L.lnorm_act(x.data_ptr() + 16, C + 8, y2.data_ptr(), C, N, P, C, g, b, _act(L, act), 0.2, st2), [y2, st2], 'lnorm_act')
    twice(lambda: L.lnorm_act_bwd(x.data_ptr() + 16, C + 8, [(s.data_ptr() + 16 * k, C + 4 * (k + 1)) for k, s in enumerate(srcs)],
                                  dxr.data_ptr(), C, N, P, C, g, b, st2, _act(L, act), 0.2, dgr, dbr), [dxr, dgr, dbr], 'lnorm_act_bwd')


def test_lnorm_rejects_bad_calls(L):  # noqa: F811
    N, P, C = 3, 64, 32
    x = torch.randn(N, P, C, device='cuda')
    y = torch.full((N, P, C), 7.0, device='cuda')
    g, b = torch.ones(C, device='cuda'), torch.zeros(C, device='cuda')
    st = torch.zeros(N, 2, device='cuda')
    dg, db = torch.full((C,), 7.0, device='cuda'), torch.full((C,), 7.0, device='cuda')
    fwd = dict(x=x.data_ptr(), xs=C, y=y.data_ptr(), ys=C, n=N, p=P, c=C)
    for bad in (dict(c=30, xs=30, ys=30), dict(x=0), dict(y=0), dict(n=0), dict(p=0), dict(c=0), dict(xs=34)):
        a = dict(fwd, **bad)
        with pytest.raises(L.VpError):
            L.lnorm_act(a['x'], a['xs'], a['y'], a['ys'], a['n'], a['p'], a['c'], g, b, L.ACT_RELU, 0.0, st)
    bwd = dict(x=x.data_ptr(), srcs=[(x.data_ptr(), C)], dx=y.data_ptr(), n=N, p=P, c=C, stats=st)
    for bad in (dict(c=30), dict(x=0), dict(dx=0), dict(srcs=[]), dict(srcs=[(0, C)]), dict(srcs=[(x.data_ptr(), 30)]),
                dict(n=0), dict(p=0), dict(stats=None), dict(srcs=[(x.data_ptr(), C)] * 5)):
        a = dict(bwd, **bad)
        with pytest.raises(L.VpError):
            L.lnorm_act_bwd(a['x'], C, a['srcs'], a['dx'], C, a['n'], a['p'], a['c'], g, b, a['stats'], L.ACT_RELU, 0.0, dg, db)
    with pytest.raises(L.VpError):
        L.lnorm_act_bwd(x.data_ptr(), C, [(x.data_ptr(), C)], y.data_ptr(), C, N, P, C, g, b, st, L.ACT_RELU, 0.0, None, db)
    torch.cuda.synchronize()
    assert bool((y == 7.0).all()) and bool((dg == 7.0).all()) and bool((db == 7.0).all())


# ------------------------------------------------------------------------------------------------ model level
def _params(hp, shape, seed=0):
    """Reference initial values with random site and ConvLSTM norm parameters (ones / zeros at init)."""
    params, _ = R.init_params(hp, shape, seed=seed)
    g = torch.Generator().manual_seed(seed + 13)
    for k in list(params):
        if k.endswith(('/gamma', '/beta')) or k.endswith('basic_conv2dlstm_cell/bias'):
            params[k] = params[k] + torch.randn(params[k].shape, generator=g) * 0.2
    return params


GEN_CASES = {
    'deterministic': (dict(context_frames=2, sequence_length=12, nz=0), 4, (64, 64, 3)),
    'vae': (dict(context_frames=2, sequence_length=12, nz=8), 4, (64, 64, 3)),
    'deterministic_128': (dict(context_frames=2, sequence_length=6, nz=0), 2, (128, 128, 3)),
    'vae_flow': (dict(context_frames=2, sequence_length=8, nz=8, transformation='flow'), 3, (64, 64, 3)),
    'vae_plain_cell': (dict(context_frames=2, sequence_length=8, nz=8, conv_rnn_norm_layer='none'), 3, (64, 64, 3)),
}


@pytest.mark.parametrize('norm', NORMS)
@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_matches_oracle(Model, case, norm):
    """gen_images (and gen_images_enc) within 1e-3 max-abs of the fp32 reference, as test_gpu_parity.py."""
    hk, B, shape = GEN_CASES[case]
    hk = dict(hk, norm_layer=norm)
    hp = O.make_hparams(**hk)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, seed=0)
    with torch.no_grad():
        ref = R.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B, None))
    model = Model(mode='test', hparams_dict=hk)
    model.set_params(params)
    binp = _batch_major(inputs)
    model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=False)
    model.generator_forward()
    torch.cuda.synchronize()
    report = {}
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - ref[k]).abs().max().item()
        report[k] = err
        assert err <= 1e-3, (case, norm, k, err)
    print('norm_layer=%s generator %s: max-abs %s' % (norm, case, {k: '%.2e' % v for k, v in report.items()}))


TRAIN_CASES = {
    'deterministic_l1': dict(context_frames=2, sequence_length=8, nz=0, l1_weight=1.0, lr=1e-3),
    'vae_l1': dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3, kl_anneal_steps=(0, 10), lr=1e-3),
    'savp': dict(context_frames=2, sequence_length=8, clip_length=6, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
                 video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, kl_anneal_steps=(0, 10)),
}


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return R.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('norm', NORMS)
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_matches_fp32_oracle(Model, case, norm, arith):
    """64x64, B = 2, random scheduled-sampling mask, the tolerances of test_gpu_train_parity.py: exact mode EXACT_GTOL per
    gradient tensor, TF32 mode max(5e-2, 2 x the operand-rounding emulation).  One exception, TF32 with norm_layer='none':
    the bias gradients of the site convolutions get a floor of 1e-1.  Without a normaliser a site's bias gradient is the
    sum of its dpre over every position and sample, whose terms largely cancel, so the TF32 rounding of the dgrad
    operands is a larger share of it than of any kernel gradient (with a norm that gradient is about zero and falls below
    the floor).  Measured on an H100: 5.2e-2 for h2/conv_pool2d/bias (VAE-L1)."""
    hk = dict(TRAIN_CASES[case], norm_layer=norm)
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
            floor_tf32 = 1e-1 if norm == 'none' and k.endswith('/bias') and k.startswith('generator/') else 5e-2
            tol = EXACT_GTOL[case] if emu is None else max(floor_tf32, 2.0 * _rel(emu[kind][k], g)[0])
            worst.append((r, tol, k))
            if r > tol:
                bad.append((r, tol, k))
    worst.sort(reverse=True)
    print('norm_layer=%s %s [%s]: worst gradient errors %s' % (norm, case, arith, ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    if norm == 'layer':
        ln = [k for k in res['g_grads'] if '/LayerNorm/' in k]
        assert ln and all(float(model.grads[k].abs().max()) > 0 for k in ln), ln
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)


@pytest.mark.parametrize('norm', NORMS)
def test_captured_step_reproduces_the_eager_step(Model, norm, tmp_path):
    """The eager step and two graph replays from the same checkpoint give bit-identical losses and gradients."""
    hk = dict(TRAIN_CASES['savp'], norm_layer=norm)
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


def test_tf_bundle_with_layer_norm_names_restores_exactly(Model, tmp_path):
    """A reference checkpoint of a layer-norm SAVP (TF tensor bundle, .../LayerNorm/gamma names) restores every variable
    bit for bit, and the model's own .npz round-trips."""
    from test_tf_checkpoint import write_bundle
    hk = dict(context_frames=2, sequence_length=4, nz=8, norm_layer='layer')
    hp = O.make_hparams(**hk)
    params = _params(hp, (64, 64, 3), seed=3)
    assert SC + '/h0/LayerNorm/gamma' in params and 'generator/encoder/layer_2/LayerNorm/beta' in params
    inputs, _ = O.make_synthetic_inputs(hp, 1, (64, 64, 3))
    model = Model(mode='test', hparams_dict=hk)
    model.build_graph(_batch_major(inputs))
    tensors = {k: v.numpy().astype(np.float32) for k, v in params.items() if k.startswith('generator/')}
    tensors['global_step'] = np.array(1234, np.int64)
    prefix = str(tmp_path / 'model-1234')
    write_bundle(prefix, tensors)
    model.restore(None, prefix)
    assert model.global_step == 1234
    for k, v in tensors.items():
        if k != 'global_step':
            assert np.array_equal(model.params[k].cpu().numpy(), v), k
    ck = model.save(str(tmp_path / 'npz'))
    other = Model(mode='test', hparams_dict=hk)
    other.build_graph(_batch_major(inputs))
    other.restore(None, ck)
    assert all(torch.equal(other.params[k], model.params[k]) for k in model.params)
