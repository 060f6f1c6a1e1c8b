"""GPU tests (-m gpu) of the compositing hparams: the slot writers (vp_cdna_slots / vp_flow_slots and their backward) at
F = 1..3 history frames and vp_composite(_bwd) at 1..32 layers against fp64 torch, rejected bad calls, bit-identical
reruns, the generator and the training step against the fp32 reference (tests/savp_compositor_oracle.py), the captured
step, and the restore of a TF bundle of a model without scratch or masks heads."""
import numpy as np
import pytest
import torch

import savp_compositor_oracle as CO
from oracle import savp_oracle as O
from test_gpu_reproducible import twice
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, Model, _rel, arithmetic, tf32_mode  # noqa: F401

pytestmark = pytest.mark.gpu
NAN = float('nan')
SC = 'generator/rnn/savp_cell'


@pytest.fixture(scope='module')
def L():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200 import lib
    lib.lib()
    return lib


def _rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).cuda()


def _image(n, h, w, seed):
    """A float4-padded image [n, h, w, 4] (pad lane 0, as the model stores it)."""
    x = torch.zeros(n, h, w, 4, device='cuda')
    x[..., :3] = _rnd(n, h, w, 3, seed=seed)
    return x


def _slots_buf(n, h, w, nslots, off=4, extra=8):
    """A concat buffer whose slot region starts `off` channels in; every channel holds NaN until written."""
    return torch.full((n, h, w, off + 4 * nslots + extra), NAN, device='cuda'), off


def _cdna_ref(img, k):
    """apply_cdna_kernels in fp64: img [n, h, w, 4], k [n, kh, kw, g] -> g images [n, h, w, 4]."""
    return O.apply_cdna_kernels(img.double().cpu(), k.double().cpu())


def _norm_kernels(n, kh, kw, nk, seed):
    k = torch.rand(n, kh * kw, nk, generator=torch.Generator().manual_seed(seed)) + 0.05
    return (k / k.sum(1, keepdim=True)).cuda()


def _check_nan_outside(buf, lo, hi, what):
    mask = torch.ones(buf.shape[-1], dtype=torch.bool)
    mask[lo:hi] = False
    assert bool(torch.isnan(buf[..., mask.cuda()]).all()), '%s wrote outside its slots' % what


# ---------------------------------------------------------------------------------- slot writers vs fp64
@pytest.mark.parametrize('nf', [1, 2, 3])
def test_cdna_slots_fwd_bwd(L, nf):
    n, h, w, kh, kw, g = 3, 16, 20, 5, 5, 2
    nk = nf * g
    frames = [_image(n, h, w, seed=10 + f) for f in range(nf)]
    bgs = [frames[-1], _image(n, h, w, seed=30), _image(n, h, w, seed=31)]
    kern = _norm_kernels(n, kh, kw, nk, seed=nf)
    nsl = nk + len(bgs)
    buf, off = _slots_buf(n, h, w, nsl)
    L.slots([f.data_ptr() for f in frames], nk, [b.data_ptr() for b in bgs], buf.data_ptr() + 4 * off, buf.shape[-1], n, h, w,
            kernels=kern, kh=kh, kw=kw)
    torch.cuda.synchronize()
    kr = kern.view(n, kh, kw, nk)
    for f in range(nf):
        ref = _cdna_ref(frames[f], kr[..., f * g:(f + 1) * g])
        for j in range(g):
            s = off + 4 * (f * g + j)
            assert (buf[..., s:s + 4].double().cpu() - ref[j]).abs().max().item() <= 1e-5, (f, j)
    for b, img in enumerate(bgs):
        s = off + 4 * (nk + b)
        assert torch.equal(buf[..., s:s + 4], img)
    _check_nan_outside(buf, off, off + 4 * nsl, 'cdna_slots')
    # backward: dT = dA + dB; frame 0 without a gradient when nf > 1; the previous image is background 0 (slot nk)
    cs = 4 * nsl + 4
    dA, dB = _rnd(n, h, w, cs, seed=40), _rnd(n, h, w, cs, seed=41)
    dfr = [_rnd(n, h, w, 4, seed=50 + f) for f in range(nf)]
    init = [d.clone() for d in dfr]
    dk = torch.zeros(n, kh * kw, nk, device='cuda')
    dptr = [0 if (f == 0 and nf > 1) else d.data_ptr() for f, d in enumerate(dfr)]
    L.slots_bwd([f.data_ptr() for f in frames], nk, nk, dA.data_ptr(), cs, dB.data_ptr(), cs, dptr, n, h, w, kernels=kern, dkernels=dk,
                kh=kh, kw=kw)
    torch.cuda.synchronize()
    fr = [f.double().cpu().requires_grad_() for f in frames]
    kk = kr.double().cpu().requires_grad_()
    dT = (dA + dB).double().cpu()
    loss = (fr[-1] * dT[..., 4 * nk:4 * nk + 4]).sum()
    for f in range(nf):
        for j, y in enumerate(O.apply_cdna_kernels(fr[f], kk[..., f * g:(f + 1) * g])):
            k = f * g + j
            loss = loss + (y * dT[..., 4 * k:4 * k + 4]).sum()
    loss.backward()
    assert (dk.view(n, kh, kw, nk).double().cpu() - kk.grad).abs().max().item() <= 1e-4 * max(1.0, kk.grad.abs().max().item())
    for f in range(nf):
        if dptr[f]:
            want = init[f].double().cpu()[..., :3] + fr[f].grad[..., :3]
            assert (dfr[f][..., :3].double().cpu() - want).abs().max().item() <= 1e-4, f
            assert torch.equal(dfr[f][..., 3], init[f][..., 3])
        else:
            assert torch.equal(dfr[f], init[f])
    twice(lambda: L.slots_bwd([f.data_ptr() for f in frames], nk, nk, dA.data_ptr(), cs, dB.data_ptr(), cs, dptr, n, h, w,
                              kernels=kern, dkernels=dk, kh=kh, kw=kw), dfr + [dk], 'cdna_slots_bwd nf=%d' % nf)


@pytest.mark.parametrize('nf', [1, 2])
def test_flow_slots_fwd_bwd(L, nf):
    n, h, w, g = 2, 16, 12, 3
    nk = nf * g
    frames = [_image(n, h, w, seed=60 + f) for f in range(nf)]
    bgs = [_image(n, h, w, seed=70), frames[-1]]
    fcs = 2 * nk + 2
    flows = _rnd(n, h, w, fcs, seed=80, scale=3.0)
    nsl = nk + len(bgs)
    buf, off = _slots_buf(n, h, w, nsl)
    L.slots([f.data_ptr() for f in frames], nk, [b.data_ptr() for b in bgs], buf.data_ptr() + 4 * off, buf.shape[-1], n, h, w,
            flows=flows, flows_cs=fcs)
    torch.cuda.synchronize()
    fl = flows.double().cpu()
    for k in range(nk):
        ref = O.image_warp(frames[k // g].double().cpu(), torch.stack([fl[..., k], fl[..., nk + k]], -1))
        s = off + 4 * k
        assert (buf[..., s:s + 4].double().cpu() - ref).abs().max().item() <= 1e-5, k
    for b, img in enumerate(bgs):
        assert torch.equal(buf[..., off + 4 * (nk + b):off + 4 * (nk + b + 1)], img)
    _check_nan_outside(buf, off, off + 4 * nsl, 'flow_slots')
    cs = 4 * nsl
    dA, dB = _rnd(n, h, w, cs, seed=90), _rnd(n, h, w, cs, seed=91)
    dfr = [torch.zeros(n, h, w, 4, device='cuda') for _ in range(nf)]
    dfl = torch.full((n, h, w, fcs), NAN, device='cuda')
    prev = nk + 1
    L.slots_bwd([f.data_ptr() for f in frames], nk, prev, dA.data_ptr(), cs, dB.data_ptr(), cs, [d.data_ptr() for d in dfr], n, h, w,
                flows=flows, flows_cs=fcs, dflows=dfl)
    torch.cuda.synchronize()
    fr = [f.double().cpu().requires_grad_() for f in frames]
    flr = fl.clone().requires_grad_()
    dT = (dA + dB).double().cpu()
    loss = (fr[-1][..., :3] * dT[..., 4 * prev:4 * prev + 3]).sum()
    for k in range(nk):
        y = O.image_warp(fr[k // g], torch.stack([flr[..., k], flr[..., nk + k]], -1))
        loss = loss + (y[..., :3] * dT[..., 4 * k:4 * k + 3]).sum()
    loss.backward()
    assert (dfl[..., :2 * nk].double().cpu() - flr.grad[..., :2 * nk]).abs().max().item() <= 1e-4
    assert bool(torch.isnan(dfl[..., 2 * nk:]).all())
    for f in range(nf):
        assert (dfr[f][..., :3].double().cpu() - fr[f].grad[..., :3]).abs().max().item() <= 1e-4, f


@pytest.mark.parametrize('nl', [1, 2, 7, 8, 9, 16, 20, 32])
def test_composite_fwd_bwd(L, nl):
    n, h, w = 2, 8, 12
    P = n * h * w
    lcs = nl + 3
    logits = torch.full((n, h, w, lcs), NAN, device='cuda')
    logits[..., :nl] = _rnd(n, h, w, nl, seed=nl, scale=2.0)
    buf, off = _slots_buf(n, h, w, nl)
    layers = _rnd(n, h, w, nl, 4, seed=100)
    buf[..., off:off + 4 * nl] = layers.view(n, h, w, 4 * nl)
    masks = torch.full((n, h, w, lcs), NAN, device='cuda')
    gen = torch.zeros(n, h, w, 4, device='cuda')
    L.composite(logits, lcs, buf.data_ptr() + 4 * off, buf.shape[-1], masks, lcs, gen, P, nl)
    torch.cuda.synchronize()
    m = torch.softmax(logits[..., :nl].double().cpu(), -1)
    lay = layers.double().cpu()
    assert (masks[..., :nl].double().cpu() - m).abs().max().item() <= 1e-6
    assert bool(torch.isnan(masks[..., nl:]).all())
    assert (gen.double().cpu() - (lay * m[..., None, :].transpose(-1, -2)).sum(-2)).abs().max().item() <= 1e-5
    dgen = _rnd(n, h, w, 4, seed=101)
    dlog = torch.full((n, h, w, lcs), NAN, device='cuda')
    dlay = torch.full((n, h, w, 4 * nl + 4), NAN, device='cuda')
    L.composite_bwd(dgen, masks, lcs, buf.data_ptr() + 4 * off, buf.shape[-1], dlog, lcs, dlay, 4 * nl + 4, P, nl)
    torch.cuda.synchronize()
    lg = logits[..., :nl].double().cpu().requires_grad_()
    lr = lay.clone().requires_grad_()
    mm = torch.softmax(lg, -1)
    ((lr * mm[..., None, :].transpose(-1, -2)).sum(-2) * dgen.double().cpu()).sum().backward()
    assert (dlog[..., :nl].double().cpu() - lg.grad).abs().max().item() <= 1e-5
    assert (dlay[..., :4 * nl].double().cpu().view(n, h, w, nl, 4) - lr.grad).abs().max().item() <= 1e-6
    assert bool(torch.isnan(dlay[..., 4 * nl:]).all())
    if nl > 8:
        twice(lambda: (L.composite(logits, lcs, buf.data_ptr() + 4 * off, buf.shape[-1], masks, lcs, gen, P, nl),
                       L.composite_bwd(dgen, masks, lcs, buf.data_ptr() + 4 * off, buf.shape[-1], dlog, lcs, dlay, 4 * nl + 4, P, nl)),
              [masks[..., :nl], gen, dlog[..., :nl], dlay[..., :4 * nl]], 'composite L=%d' % nl)


def test_bad_calls_are_rejected(L):
    n, h, w = 1, 8, 8
    img = _image(n, h, w, 0)
    buf = torch.zeros(n, h, w, 4 * 40, device='cuda')
    kern = _norm_kernels(n, 3, 3, 17, 0)
    p, b = img.data_ptr(), buf.data_ptr()
    bad = [
        lambda: L.slots([p] * 17, 17, [], b, 160, n, h, w, kernels=kern, kh=3, kw=3),           # nk > 16
        lambda: L.slots([p, p], 3, [], b, 160, n, h, w, kernels=kern, kh=3, kw=3),              # nk % frames
        lambda: L.slots([p, 0], 4, [], b, 160, n, h, w, kernels=kern, kh=3, kw=3),              # null frame
        lambda: L.slots([p], 4, [p] * 29, b, 160, n, h, w, kernels=kern, kh=3, kw=3),           # 33 layers
        lambda: L.slots([p], 4, [p, 0], b, 160, n, h, w, kernels=kern, kh=3, kw=3),             # null background
        lambda: L.slots([p], 4, [p, p], b, 20, n, h, w, kernels=kern, kh=3, kw=3),              # stride < 4 * slots
        lambda: L.slots([p], 4, [p], b, 160, n, h, w, kernels=None, kh=3, kw=3),                # no kernels
        lambda: L.slots([p], 4, [p], b, 160, n, h, w, flows=buf, flows_cs=6),                   # flows stride < 2 nk
        lambda: L.slots_bwd([p], 4, 2, b, 160, b, 160, [p], n, h, w, kernels=kern, dkernels=kern, kh=3, kw=3),   # prev in transforms
        lambda: L.slots_bwd([p], 4, 32, b, 160, b, 160, [p], n, h, w, kernels=kern, dkernels=kern, kh=3, kw=3),
        lambda: L.slots_bwd([p], 4, 4, b, 160, b, 160, [p], n, h, w, kernels=kern, dkernels=None, kh=3, kw=3),
        lambda: L.slots_bwd([p], 2, 2, b, 160, b, 160, [p], n, h, w, flows=buf, flows_cs=8, dflows=None),
        lambda: L.composite(buf, 40, b, 160, buf, 40, img, n * h * w, 0),
        lambda: L.composite(buf, 40, b, 160, buf, 40, img, n * h * w, 33),
        lambda: L.composite(buf, 8, b, 160, buf, 40, img, n * h * w, 9),                         # logits stride < L
        lambda: L.composite(buf, 40, b, 160, buf, 8, img, n * h * w, 9),                         # masks stride < L
        lambda: L.composite_bwd(img, buf, 8, b, 160, buf, 40, buf, 160, n * h * w, 9),
        lambda: L.composite_bwd(img, buf, 40, b, 160, buf, 8, buf, 160, n * h * w, 9),
        lambda: L.cdna_apply(img, img, kern, b, 160, n, h, w, 3, 3, 5),                          # the old entry points keep
        lambda: L.flow_apply(img, img, buf, 20, b, 160, n, h, w, 7),                              # their limits
    ]
    before = buf.clone()
    for i, fn in enumerate(bad):
        with pytest.raises(L.VpError):
            fn()
        torch.cuda.synchronize()
        assert torch.equal(buf, before), i


# ---------------------------------------------------------------------------------- the generator and the training step
GEN_CASES = {
    'lf2_cdna': dict(context_frames=2, sequence_length=8, nz=8, last_frames=2),
    'lf2_flow': dict(context_frames=2, sequence_length=8, nz=8, last_frames=2, transformation='flow', num_transformed_images=3),
    'noscratch_independent': dict(context_frames=2, sequence_length=8, nz=8, generate_scratch_image=False, dependent_mask=False),
    'last_and_last_context': dict(context_frames=3, sequence_length=8, nz=0, last_image_background=True,
                                  last_context_image_background=True),
    'context_images': dict(context_frames=3, sequence_length=8, nz=8, context_images_background=True, last_frames=2),
    'single_layer': dict(context_frames=2, sequence_length=6, nz=8, num_transformed_images=0, generate_scratch_image=False,
                         first_image_background=False),
    'no_transforms_flow': dict(context_frames=2, sequence_length=6, nz=0, num_transformed_images=0, transformation='flow',
                               norm_layer='layer'),
}


def _params(hp, shape, seed=0):
    params, _ = CO.init_params(hp, shape, seed=seed)
    g = torch.Generator().manual_seed(seed + 13)
    for k in list(params):
        if k.endswith(('/gamma', '/beta')):
            params[k] = params[k] + torch.randn(params[k].shape, generator=g) * 0.2
    return params


# max-abs tolerance of the outputs against the fp32 reference per arithmetic mode.  In TF32 the transformed images (the
# scratch image straight from a TF32 convolution, transforms of generated frames) and the masks differ by up to 1.42e-3,
# measured on an H100 (the lf2_cdna case); gen_images stay within 1e-3 as in test_gpu_parity.py.  The fp32-exact mode
# holds every output to 1e-4, which checks the slot layout and the masks exactly.
GEN_TOL = {'tf32': dict(gen_images=1e-3, transformed_images=2e-3, masks=2e-3),
           'exact': dict(gen_images=1e-4, transformed_images=1e-4, masks=1e-4)}


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_matches_oracle(Model, case, arith):
    hk = GEN_CASES[case]
    hp = O.make_hparams(**hk)
    B, shape = 3, (64, 64, 3)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, seed=0)
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
    report = {}
    for k in ('gen_images', 'transformed_images', 'masks'):
        got = model.outputs[k].cpu()
        want = ref[k].transpose(0, 1)
        assert got.shape == want.shape, (k, got.shape, want.shape)
        report[k] = err = (got - want).abs().max().item()
        assert err <= GEN_TOL[arith][k], (case, arith, k, err)
    print('compositor generator %s [%s]: max-abs %s' % (case, arith, {k: '%.2e' % v for k, v in report.items()}))


PIX_CASES = {
    'lf2_cdna': dict(context_frames=2, sequence_length=7, nz=8, last_frames=2),
    'lf2_flow_context_images': dict(context_frames=3, sequence_length=7, nz=0, last_frames=2, transformation='flow',
                                    num_transformed_images=2, context_images_background=True, dependent_mask=False),
}


@pytest.mark.parametrize('case', sorted(PIX_CASES))
def test_pix_distribs_with_history_match_fp64_oracle(Model, case):
    """pix_distribs with last_frames = 2 (the transforms act on the selected maps of two steps) and more than 8 slots, in
    the fp32-exact mode against the fp64 reference, with the relative L2 tolerance of test_gpu_pix_distribs.py."""
    from test_gpu_pix_distribs import EXACT_TOL
    from test_pix_distribs import make_pix
    hk = PIX_CASES[case]
    hp = O.make_hparams(**hk)
    B, shape = 2, (64, 64, 3)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, seed=0)
    inputs['pix_distribs'] = make_pix(hp, B, 64, 64, 2, seed=3, dtype=torch.float32)
    sampling = torch.rand(hp.sequence_length - 1 - hp.context_frames, B, generator=torch.Generator().manual_seed(4)) < 0.5
    gt = O.ground_truth_mask(hp, B, sampling)
    with torch.no_grad():
        ref = CO.pix_generator(O.Vars({k: v.double() for k, v in params.items()}), hp,
                               {k: v.double() for k, v in inputs.items()}, {k: v.double() for k, v in noise.items() if torch.is_tensor(v)}, gt)
    with arithmetic('exact'):
        model = Model(mode='test', hparams_dict=hk)
        model.set_params(params)
        binp = {'images': inputs['images'].transpose(0, 1), 'pix_distribs': inputs['pix_distribs'].transpose(0, 1)}
        model.build_graph(binp)
    assert model.nlayers > 8
    model.set_inputs(binp, noise, sampling=sampling)
    model.generator_forward()
    torch.cuda.synchronize()
    report = {}
    for k in ('gen_pix_distribs', 'transformed_pix_distribs'):
        got = model.outputs[k].transpose(0, 1).cpu()
        assert got.shape == ref[k].shape, (k, got.shape, ref[k].shape)
        report[k] = err = _rel(got, ref[k])[0]
        assert err <= EXACT_TOL, (case, k, err)
    print('compositor pix %s: relative L2 %s' % (case, {k: '%.2e' % v for k, v in report.items()}))


def test_pix_slots_reject_bad_calls(L):
    n, h, w = 1, 8, 8
    m = torch.full((n, h, w, 4), 0.5, device='cuda')
    masks = torch.full((n, h, w, 40), NAN, device='cuda')
    gen, tr = torch.full_like(m, NAN), torch.full((n, h, w, 4 * 40), NAN, device='cuda')
    sel = torch.ones(n, dtype=torch.int32, device='cuda')
    kern = _norm_kernels(n, 3, 3, 17, 0)
    p, g, t = m.data_ptr(), gen.data_ptr(), tr.data_ptr()
    bad = [
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [], 17, [0], 1, masks, 40, g, 4, t, 160, 4, 0, n, h, w, 1, kernels=kern, kh=3, kw=3),
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [], 0, [0] * 33, 0, masks, 40, g, 4, t, 160, 4, 0, n, h, w, 1),      # 33 slots
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [], 0, [], 0, masks, 40, g, 4, t, 160, 4, 0, n, h, w, 1),            # no slot
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [p], 3, [0], 1, masks, 40, g, 4, t, 160, 4, 0, n, h, w, 1, kernels=kern, kh=3, kw=3),
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [], 2, [0], 1, masks, 3, g, 4, t, 160, 4, 0, n, h, w, 1, kernels=kern, kh=3, kw=3),
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [0], 2, [0], 1, masks, 40, g, 4, t, 160, 4, 0, n, h, w, 1, kernels=kern, kh=3, kw=3),
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [], 0, [0], 1, masks, 40, g, 4, t, 160, 4, 0, n, h, w, 1, kernels=kern, kh=3, kw=3),
        lambda: L.pix_slots_fwd(sel, p, 4, 0, [], 0, [0] * 20, 1, masks, 40, g, 4, t, 40, 4, 0, n, h, w, 1),       # transformed
    ]
    for i, fn in enumerate(bad):
        with pytest.raises(L.VpError):
            fn()
        torch.cuda.synchronize()
        assert torch.isnan(gen).all() and torch.isnan(tr).all(), i


TRAIN_CASES = {
    'vae_l1_lf2_cdna': (dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3, kl_anneal_steps=(0, 10),
                             lr=1e-3, last_frames=2), 'vae_l1'),
    'vae_l1_lf2_flow_independent': (dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3,
                                         kl_anneal_steps=(0, 10), lr=1e-3, last_frames=2, transformation='flow',
                                         num_transformed_images=2, generate_scratch_image=False, dependent_mask=False),
                                    'vae_l1'),
    'savp_context_images': (dict(context_frames=3, sequence_length=8, clip_length=5, lr=2e-4, beta1=0.5, l1_weight=100.,
                                 kl_weight=1.0, video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1,
                                 vae_gan_feature_cdist_weight=10.0, kl_anneal_steps=(0, 10), context_images_background=True,
                                 last_context_image_background=True), 'savp'),
}


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return CO.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_matches_fp32_oracle(Model, case, arith):
    """64x64, B = 2, a random scheduled-sampling mask (so the history carries gradient into earlier generated frames), the
    tolerances of test_gpu_layer_choices.py."""
    hk, gtol = TRAIN_CASES[case]
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
            tol = EXACT_GTOL[gtol] if emu is None else max(5e-2, 2.0 * _rel(emu[kind][k], g)[0])
            worst.append((r, tol, k))
            if r > tol:
                bad.append((r, tol, k))
    worst.sort(reverse=True)
    print('compositor %s [%s]: worst gradient errors %s' % (case, arith, ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)


def test_captured_step_reproduces_the_eager_step(Model, tmp_path):
    """The eager step and two graph replays from the same checkpoint give bit-identical losses and gradients."""
    hk = TRAIN_CASES['vae_l1_lf2_flow_independent'][0]
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
            runs[how].append((model.loss_vals.clone(), model.g_grad.clone()))
    ref = runs['eager'][0]
    for got in runs['graph']:
        for name, a, b in zip(('losses', 'g_grad'), got, ref):
            assert torch.equal(a, b), (name, (a - b).abs().max().item())
    assert float(ref[1].abs().max()) > 0 and bool(torch.isfinite(ref[1]).all())


def test_tf_bundle_without_scratch_or_masks_heads_restores(Model, tmp_path):
    """One CDNA transform as the only layer (no backgrounds, no scratch image): the reference has no h_scratch,
    scratch_image, h_masks or masks variables; its bundle restores bit for bit and the generator matches the reference."""
    from test_tf_checkpoint import write_bundle
    hk = dict(context_frames=2, sequence_length=4, nz=8, num_transformed_images=1, prev_image_background=False,
              first_image_background=False, generate_scratch_image=False)
    hp = O.make_hparams(**hk)
    params = _params(hp, (64, 64, 3), seed=3)
    assert not any(('scratch' in k or 'masks' in k) for k in params) and SC + '/cdna_kernels/dense/kernel' in params
    inputs, noise = O.make_synthetic_inputs(hp, 1, (64, 64, 3))
    model = Model(mode='test', hparams_dict=hk)
    model.build_graph(_batch_major(inputs))
    assert set(model.params) == {k for k in params if k.startswith('generator/')}
    tensors = {k: v.numpy().astype(np.float32) for k, v in params.items() if k.startswith('generator/')}
    tensors['global_step'] = np.array(11, np.int64)
    prefix = str(tmp_path / 'model-11')
    write_bundle(prefix, tensors)
    model.restore(None, prefix)
    assert model.global_step == 11
    for k, v in tensors.items():
        if k != 'global_step':
            assert np.array_equal(model.params[k].cpu().numpy(), v), k
    model.set_inputs(_batch_major(inputs), noise, sampling=False)
    model.generator_forward()
    with torch.no_grad():
        ref = CO.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, 1, None))
    assert (model.outputs_time_major('gen_images').cpu() - ref['gen_images']).abs().max().item() <= 1e-3
    assert torch.equal(model.outputs['masks'].cpu(), torch.ones_like(model.outputs['masks'].cpu()))
