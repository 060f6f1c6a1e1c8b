"""GPU tests (-m gpu) of the pixel-distribution path: vp_pix_distrib_fwd against an fp64 torch reference and across reruns,
generator outputs against the oracle in both arithmetic modes, and a training step that must not change when the inputs
carry pix_distribs."""
import os

import numpy as np
import pytest
import torch

import savp_pix_oracle as P
from oracle import savp_oracle as O
from test_pix_distribs import make_pix

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200 import lib
    lib.lib()
    return lib


@pytest.fixture(scope='module')
def Model(L):
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def _rel(a, b):
    a, b = a.detach().double().reshape(-1).cpu(), b.detach().double().reshape(-1).cpu()
    return ((a - b).norm() / b.norm()).item()


# ------------------------------------------------------------------------------------------------ the kernel
class Case(object):
    """Inputs of one vp_pix_distrib_fwd call, every map in a channel slice of a wider buffer whose other channels hold NaN."""
    NK, KH, KW = 4, 5, 5

    def __init__(self, transformation, D, H, NB, t, seed=0):
        g = torch.Generator(device='cpu').manual_seed(seed)
        W, NK, L_ = H, self.NK, self.NK + 3
        self.transformation, self.D, self.H, self.W, self.NB, self.t = transformation, D, H, W, NB, t
        self.Dp = (D + 3) // 4 * 4
        self.pcs, self.poff = self.Dp + 4, 2              # ground truth: stride Dp + 4, channels [2, 2 + D)
        self.gcs, self.goff = self.Dp + 4, 1              # generated maps
        self.tcs, self.toff = L_ * self.Dp + 4, 1         # transformed: slot l at toff + l * Dp

        def f32(x):                                       # inputs exactly representable in fp32: both sides see the same
            return x.float().double()

        def planes(n):
            x = torch.rand(n, NB, H, W, D, generator=g, dtype=torch.float64) ** 4
            return f32(x / x.sum(dim=(2, 3), keepdim=True))
        self.gt, self.first, self.prev = planes(1)[0], planes(1)[0], planes(1)[0]
        self.sel = (torch.rand(NB, generator=g) < 0.5).to(torch.int32)
        self.masks = f32(torch.softmax(torch.randn(NB, H, W, L_, generator=g, dtype=torch.float64) * 2, dim=-1))
        k = torch.rand(NB, self.KH, self.KW, NK, generator=g, dtype=torch.float64) + 1e-3
        self.kern = f32(k / k.sum(dim=(1, 2), keepdim=True))
        self.flows = f32(torch.randn(NB, H, W, 2 * NK, generator=g, dtype=torch.float64) * 3)

    def device_inputs(self):
        def slab(x, cs, off):
            buf = torch.full(x.shape[:-1] + (cs,), float('nan'), device='cuda')
            buf[..., off:off + self.D] = x.float().cuda()
            return buf
        m = torch.full((self.NB, self.H, self.W, 8), float('nan'), device='cuda')
        m[..., :self.NK + 3] = self.masks.float().cuda()
        return dict(gt=slab(self.gt, self.pcs, self.poff), first=slab(self.first, self.pcs, self.poff),
                    prev=slab(self.prev, self.gcs, self.goff), masks=m, sel=self.sel.cuda(),
                    kern=self.kern.reshape(self.NB, -1, self.NK).float().cuda().contiguous(), flows=self.flows.float().cuda())

    def outputs(self):
        return (torch.full((self.NB, self.H, self.W, self.gcs), float('nan'), device='cuda'),
                torch.full((self.NB, self.H, self.W, self.tcs), float('nan'), device='cuda'))

    def launch(self, L, x, gen, tr):
        cdna = self.transformation == 'cdna'
        L.pix_distrib_fwd(x['sel'], x['gt'].data_ptr() + 4 * self.poff, x['first'].data_ptr() + 4 * self.poff, self.pcs,
                          x['prev'].data_ptr() + 4 * self.goff if self.t else 0, x['kern'] if cdna else None,
                          None if cdna else x['flows'], 0 if cdna else 2 * self.NK, x['masks'], 8,
                          gen.data_ptr() + 4 * self.goff, self.gcs, tr.data_ptr() + 4 * self.toff, self.tcs, self.Dp,
                          self.NB, self.H, self.W, self.D, self.KH, self.KW, self.NK)

    def reference(self):
        """fp64, from the oracle's transformation functions (savp_model.py:598-653)."""
        dev = 'cuda'
        use_gt = torch.ones(self.NB, dtype=torch.bool) if self.t == 0 else self.sel.bool()
        p = torch.where(use_gt.view(-1, 1, 1, 1), self.gt, self.prev).to(dev)
        if self.transformation == 'cdna':
            slots = O.apply_cdna_kernels(p, self.kern.to(dev))
        else:
            fl = self.flows.to(dev).reshape(self.NB, self.H, self.W, 2, self.NK)
            slots = [O.image_warp(p, fl[..., k]) for k in range(self.NK)]
        slots = slots + [p, self.first.to(dev), p]
        m = self.masks.to(dev)
        g = sum(s * m[..., l:l + 1] for l, s in enumerate(slots))
        return g / g.sum(dim=(1, 2), keepdim=True), torch.stack(slots, dim=-1)


def _check_slices(case, gen, tr):
    """Values of the written slices, and every channel outside them still NaN."""
    D, Dp = case.D, case.Dp
    gmask = torch.zeros(case.gcs, dtype=torch.bool)
    gmask[case.goff:case.goff + D] = True
    tmask = torch.zeros(case.tcs, dtype=torch.bool)
    for l in range(case.NK + 3):
        tmask[case.toff + l * Dp:case.toff + l * Dp + D] = True
    gmask, tmask = gmask.cuda(), tmask.cuda()
    assert torch.isnan(gen[..., ~gmask]).all() and torch.isnan(tr[..., ~tmask]).all(), 'a channel outside the slice was written'
    g = gen[..., case.goff:case.goff + D]
    t = torch.stack([tr[..., case.toff + l * Dp:case.toff + l * Dp + D] for l in range(case.NK + 3)], dim=-1)
    assert torch.isfinite(g).all() and torch.isfinite(t).all()
    return g, t


KERNEL_CASES = [(tr, D, H, NB, t) for tr in ('cdna', 'flow') for D in (1, 2, 3, 5) for H in (64, 128)
                for NB, t in ((37, 3),)] + [('cdna', 1, 128, 512, 0), ('flow', 2, 64, 512, 5)]


@pytest.mark.parametrize('transformation,D,H,NB,t', KERNEL_CASES)
def test_pix_distrib_kernel_matches_fp64(L, transformation, D, H, NB, t):
    """Relative L2 against fp64 within 10 * 2^-24 * sqrt(H*W): the accumulation floor of the plane sum, derived, not
    measured.  Measured on an H100 80GB HBM3 (700 W): worst gen 8.8e-8 (0.0023 floors at 64x64), transformed 4.6e-8."""
    case = Case(transformation, D, H, NB, t, seed=D * 1000 + H + NB)
    x = case.device_inputs()
    gen, tr = case.outputs()
    case.launch(L, x, gen, tr)
    torch.cuda.synchronize()
    g, tt = _check_slices(case, gen, tr)
    rg, rt = case.reference()
    floor = 10 * 2.0 ** -24 * np.sqrt(H * case.W)
    eg, et = _rel(g, rg), _rel(tt, rt)
    print('pix kernel %s D=%d %dx%d NB=%d t=%d: rel L2 gen %.2e (%.2f floors), transformed %.2e (%.2f floors)'
          % (transformation, D, H, H, NB, t, eg, eg / floor, et, et / floor))
    assert eg <= floor and et <= floor, (eg, et, floor)


def test_pix_distrib_kernel_is_reproducible(L):
    from test_gpu_reproducible import dirty_scratch
    for transformation in ('cdna', 'flow'):
        case = Case(transformation, 3, 128, 40, 2, seed=11)
        x = case.device_inputs()
        runs = []
        for run in range(2):
            gen, tr = case.outputs()
            if run:
                dirty_scratch()
            case.launch(L, x, gen, tr)
            runs.append((gen, tr))
        torch.cuda.synchronize()
        for a, b in zip(*runs):
            assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0)), transformation


def test_pix_distrib_kernel_rejects_bad_calls(L):
    case = Case('cdna', 2, 64, 3, 1)
    x = case.device_inputs()
    gen, tr = case.outputs()
    with pytest.raises(L.VpError):       # both transformations given
        L.pix_distrib_fwd(x['sel'], x['gt'].data_ptr(), x['first'].data_ptr(), case.pcs, 0, x['kern'], x['flows'], 8, x['masks'], 8,
                          gen.data_ptr(), case.gcs, tr.data_ptr(), case.tcs, case.Dp, 3, 64, 64, 2, 5, 5, 4)
    with pytest.raises(L.VpError):       # channel stride not a multiple of 4
        L.pix_distrib_fwd(x['sel'], x['gt'].data_ptr(), x['first'].data_ptr(), 6, 0, x['kern'], None, 0, x['masks'], 8,
                          gen.data_ptr(), case.gcs, tr.data_ptr(), case.tcs, case.Dp, 3, 64, 64, 2, 5, 5, 4)
    with pytest.raises(L.VpError):       # more slots than the masks buffer holds
        L.pix_distrib_fwd(x['sel'], x['gt'].data_ptr(), x['first'].data_ptr(), case.pcs, 0, x['kern'], None, 0, x['masks'], 8,
                          gen.data_ptr(), case.gcs, tr.data_ptr(), case.tcs, case.Dp, 3, 64, 64, 2, 5, 5, 6)
    torch.cuda.synchronize()
    assert torch.isnan(gen).all() and torch.isnan(tr).all()


# ------------------------------------------------------------------------------------------------ generator vs oracle
FLOW_BIAS = [0.37, 1.27, -0.53, 2.17, 0.61, -1.41, 0.23, 1.79]
GEN_CASES = {
    'cfg1_deterministic': (dict(context_frames=2, sequence_length=8, nz=0), 2, 64, 0, 2, False),
    'cfg2_savp': (dict(context_frames=2, sequence_length=8, nz=8), 2, 64, 0, 1, False),
    'flow': (dict(context_frames=2, sequence_length=8, nz=8, transformation='flow'), 2, 64, 0, 3, False),
    'actions': (dict(context_frames=2, sequence_length=8, nz=8), 2, 64, 4, 2, False),
    'cfg4_128': (dict(context_frames=2, sequence_length=5, nz=8), 1, 128, 0, 2, False),
    'scheduled_sampling': (dict(context_frames=2, sequence_length=8, nz=8), 2, 64, 0, 5, True),
}
EXACT_TOL = 1e-4
TF32_FLOOR = 1e-3


class arithmetic(object):
    def __init__(self, exact):
        self.v = '1' if exact else '0'

    def __enter__(self):
        self.old = os.environ.get('VP_EXACT')
        os.environ['VP_EXACT'] = self.v

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop('VP_EXACT', None)
        else:
            os.environ['VP_EXACT'] = self.old


def _model_forward(Model, hk, params, binp, noise, sampling, exact):
    with arithmetic(exact):
        model = Model(mode='test', hparams_dict=hk)
        model.set_params(params)
        model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=sampling if sampling is not None else False)
    model.generator_forward()
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in model.outputs.items()}


@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_pix_distribs_match_oracle(Model, case):
    """Exact mode: relative L2 <= EXACT_TOL.  TF32 mode: err <= max(TF32_FLOOR, 2 x the deviation of the TF32-emulating
    oracle from fp64), as DESIGN.md (c) does for gradients: the masks come from TF32 convolutions.  gen_images are
    bit-identical with and without pix_distribs in the inputs.  Measured on an H100 80GB HBM3 (700 W): exact mode at most
    7.1e-6 (cfg4_128, transformed); TF32 mode within 1.27 x the emulating oracle's own deviation (cfg4_128, gen, 3.6e-4)."""
    hk, B, S, A, D, ss = GEN_CASES[case]
    hp = O.make_hparams(**hk)
    shape = (S, S, 3)
    params, _ = O.init_params(hp, shape, action_dim=A, seed=0)
    if hk.get('transformation') == 'flow':
        params['generator/rnn/savp_cell/flows/conv2d/bias'] = torch.tensor(FLOW_BIAS)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, action_dim=A, seed=0)
    inputs['pix_distribs'] = make_pix(hp, B, S, S, D, seed=3, dtype=torch.float32)
    n_free = hp.sequence_length - 1 - hp.context_frames
    sampling = (torch.rand(n_free, B, generator=torch.Generator().manual_seed(4)) < 0.5) if ss else None
    if ss:
        sampling[0] = True                       # ground truth right after the context frames in every sample
    gt = O.ground_truth_mask(hp, B, sampling)
    refs = {}
    with torch.no_grad():
        p64 = {k: v.double() for k, v in params.items()}
        i64 = {k: v.double() for k, v in inputs.items()}
        n64 = {k: v.double() for k, v in noise.items() if torch.is_tensor(v)}
        refs['fp64'] = P.generator(O.Vars(p64), hp, i64, n64, gt)
        O.set_tf32_emulation('trunc')
        try:
            refs['tf32'] = P.generator(O.Vars(params), hp, inputs, noise, gt)
        finally:
            O.set_tf32_emulation(None)
    binp = {'images': inputs['images'].permute(1, 0, 2, 3, 4), 'pix_distribs': inputs['pix_distribs'].permute(1, 0, 2, 3, 4)}
    if A:
        binp['actions'] = inputs['actions'].permute(1, 0, 2)
    nz = hp.nz
    keys = ['gen_pix_distribs', 'transformed_pix_distribs'] + (['gen_pix_distribs_enc', 'transformed_pix_distribs_enc'] if nz else [])
    report = {}
    for exact in (True, False):
        out = _model_forward(Model, hk, params, binp, noise, sampling, exact)
        for k in keys:
            ref = refs['fp64'][k]
            got = out[k].permute(1, 0, *range(2, ref.dim()))
            assert got.shape == ref.shape, (k, got.shape, ref.shape)
            err = _rel(got, ref)
            if exact:
                report[(k, 'exact')] = err
                assert err <= EXACT_TOL, (case, k, err)
            else:
                dev = _rel(refs['tf32'][k], ref)
                report[(k, 'tf32')] = (err, dev)
                assert err <= max(TF32_FLOOR, 2 * dev), (case, k, err, dev)
        sums = out['gen_pix_distribs'].double().sum(dim=(2, 3))
        assert (sums - 1).abs().max().item() < 1e-4
        if not exact:
            plain = {k: v for k, v in binp.items() if k != 'pix_distribs'}
            base = _model_forward(Model, hk, params, plain, noise, sampling, exact)
            assert set(out) - set(base) == set(keys)
            for k, v in base.items():
                assert torch.equal(out[k], v), k
    print('pix generator %s: %s' % (case, {'%s/%s' % k: v for k, v in report.items()}))


def test_build_graph_validates_pix_distribs(Model):
    hk = dict(context_frames=2, sequence_length=5, nz=0, ngf=8)
    imgs = torch.rand(1, 5, 32, 32, 3)
    for bad in (torch.rand(1, 5, 32, 16, 1), torch.rand(1, 4, 32, 32, 1), torch.rand(1, 5, 32, 32, 0), torch.rand(1, 5, 32, 32)):
        with pytest.raises(ValueError):
            Model(mode='test', hparams_dict=hk).build_graph({'images': imgs, 'pix_distribs': bad})
    model = Model(mode='test', hparams_dict=hk)
    model.build_graph({'images': imgs})
    assert 'pix' not in model.Bf
    with pytest.raises(ValueError):          # a model built without the maps refuses them instead of ignoring them
        model.set_inputs({'images': imgs, 'pix_distribs': torch.rand(1, 5, 32, 32, 1)})


# ------------------------------------------------------------------------------------------------ training step
def test_training_step_unchanged_by_pix_distribs(Model):
    """Same losses, gradients and updated variables with and without pix_distribs, on the eager step and on graph replays
    (the captured step also computes the maps)."""
    hk = dict(context_frames=2, sequence_length=8, clip_length=6, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
              video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, kl_anneal_steps=(0, 10))
    hp = O.make_hparams(**hk)
    B = 2
    params, _ = O.init_params(hp, (64, 64, 3), seed=0)
    inputs, _ = O.make_synthetic_inputs(hp, B, (64, 64, 3))
    binp = {'images': inputs['images'].permute(1, 0, 2, 3, 4)}
    pinp = dict(binp, pix_distribs=make_pix(hp, B, 64, 64, 2, dtype=torch.float32).permute(1, 0, 2, 3, 4))
    models = []
    for inp in (binp, pinp):
        m = Model(mode='train', hparams_dict=hk)
        m.set_params(params)
        m.build_graph(inp)
        m.use_cuda_graph = True
        models.append((m, inp))
    for step in range(3):                         # eager, capture + replay, replay
        snap = []
        for m, inp in models:
            m.train_step(inp)
            torch.cuda.synchronize()
            snap.append([m.loss_vals.clone(), m.g_grad.clone(), m.d_grad.clone(), m.g_flat.clone(), m.d_flat.clone()])
        assert (models[0][0]._graph is not None) == (step > 0) and (models[1][0]._graph is not None) == (step > 0)
        for name, a, b in zip(('losses', 'g_grad', 'd_grad', 'g_vars', 'd_vars'), *snap):
            assert torch.equal(a, b), (step, name, (a - b).abs().max().item())
        m = models[1][0]
        m._collect_outputs()
        s = m.outputs['gen_pix_distribs'].double().sum(dim=(2, 3))
        assert (s - 1).abs().max().item() < 1e-4
