"""CPU tests of the compositing hparams (last_frames, num_transformed_images, the five background flags,
generate_scratch_image, dependent_mask): accepted and refused values, the generator's variables against the reference's
(tests/savp_compositor_oracle.py), and float64 identities of the reference itself."""
import itertools

import pytest
import torch

import savp_compositor_oracle as CO
import savp_pix_oracle as P
from oracle import savp_oracle as O

SC = 'generator/rnn/savp_cell'
CFG2 = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, state_weight=0.0,
            nz=8, context_frames=2, sequence_length=12, clip_length=10)
TINY = dict(context_frames=2, sequence_length=5, nz=4, ngf=8, nef=8)
# the defaults turned off, one at a time, and the new options on
CASES = [
    dict(),
    dict(last_frames=2), dict(last_frames=3, num_transformed_images=2), dict(last_frames=2, transformation='flow'),
    dict(num_transformed_images=0), dict(last_frames=0), dict(generate_scratch_image=False), dict(dependent_mask=False),
    dict(prev_image_background=False), dict(first_image_background=False),
    dict(last_image_background=True, last_context_image_background=True),
    dict(context_images_background=True), dict(context_images_background=True, context_frames=10, sequence_length=11),
    dict(num_transformed_images=0, generate_scratch_image=False, first_image_background=False),          # L == 1
    dict(num_transformed_images=0, generate_scratch_image=False, prev_image_background=False),           # L == 1
    dict(generate_scratch_image=False, dependent_mask=False, transformation='flow', num_transformed_images=6),
]


def _model(hk, H=64, W=64):
    from video_prediction_b200.models import SAVPVideoPredictionModel
    m = SAVPVideoPredictionModel(mode='train', hparams_dict=hk)
    m.B, m.T, m.H, m.W, m.C, m.A, m.Sd = 1, hk['sequence_length'], H, W, 3, 0, 0
    m.S, m.Zc = m.T - 1, m.hparams.nz
    m.enc_specs, m.dec_specs = m.layer_specs(m.hparams.ngf, H, W)
    return m


def _layers(hk):
    return len(CO.sources(O.make_hparams(**hk)))


@pytest.mark.parametrize('case', CASES, ids=lambda c: ','.join('%s=%s' % kv for kv in sorted(c.items())) or 'default')
def test_param_specs_match_the_reference(case):
    hk = dict(CFG2, sequence_length=4)
    hk.update(case)
    for nz in (8, 0):
        hk['nz'] = nz
        specs = _model(hk, 32, 32)._generator_param_specs()
        ref, _ = CO.init_params(O.make_hparams(**dict(hk, video_sn_vae_gan_weight=0.0, video_sn_gan_weight=0.0)), (32, 32, 3))
        gen_ref = {k: t for k, t in ref.items() if k.startswith('generator/')}
        assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
        for k, (shape, _) in specs.items():
            assert tuple(shape) == tuple(gen_ref[k].shape), k


def test_heads_follow_the_slots():
    specs = _model(dict(CFG2, num_transformed_images=0, generate_scratch_image=False, first_image_background=False))
    specs = specs._generator_param_specs()
    assert not any(('masks' in k or 'scratch' in k or 'cdna' in k or 'flow' in k) for k in specs if k.startswith(SC + '/h'))
    assert not any(k.startswith((SC + '/masks', SC + '/scratch_image', SC + '/cdna_kernels')) for k in specs)
    m = _model(dict(CFG2, dependent_mask=False, context_images_background=True))._generator_param_specs()
    assert m[SC + '/masks/conv2d/kernel'][0] == (3, 3, 32, 4 + 1 + 2 + 1)
    d = _model(dict(CFG2, last_frames=2, transformation='flow'))._generator_param_specs()
    assert d[SC + '/flows/conv2d/kernel'][0] == (3, 3, 32, 16)
    assert d[SC + '/masks/conv2d/kernel'][0] == (3, 3, 32 + 11 * 3, 11)


def test_compositing_layout():
    from video_prediction_b200.models import SAVPVideoPredictionModel as M
    c = M.compositing(O.make_hparams())
    assert (c['nk'], c['F'], c['bgs'], c['scratch'], c['L'], c['prev_slot']) == (4, 1, ['prev', 'first'], True, 7, 4)
    c = M.compositing(O.make_hparams(last_frames=3, num_transformed_images=2, prev_image_background=False,
                                     last_image_background=True, last_context_image_background=True))
    assert (c['nk'], c['F'], c['bgs'], c['L'], c['prev_slot']) == (6, 3, ['first', 'last', 'last_context'], 10, -1)
    c = M.compositing(O.make_hparams(context_images_background=True, context_frames=3, last_image_background=True))
    assert c['bgs'] == ['prev', ('context', 0), ('context', 1), ('context', 2)] and c['L'] == 9
    for case in CASES:
        hk = dict(TINY, **case)
        assert M.compositing(O.make_hparams(**hk))['L'] == _layers(hk), case


def test_compositing_hparams_accepted_and_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel as M
    base = dict(context_frames=2, sequence_length=12)
    for case in CASES:
        M(mode='train', hparams_dict=dict(base, **case))._check_supported()
    for flags in itertools.product((False, True), repeat=5):
        hk = dict(base, prev_image_background=flags[0], first_image_background=flags[1], last_image_background=flags[2],
                  last_context_image_background=flags[3], context_images_background=flags[4], num_transformed_images=0,
                  generate_scratch_image=False)
        if _layers(hk) == 0:
            with pytest.raises(ValueError, match='Either one of the following should be true'):
                M(mode='train', hparams_dict=hk)._check_supported()
        else:
            M(mode='train', hparams_dict=hk)._check_supported()
    for norm, cell in itertools.product(('instance', 'layer', 'none'), (dict(), dict(conv_rnn_norm_layer='none'))):
        M(mode='train', hparams_dict=dict(base, last_frames=2, dependent_mask=False, norm_layer=norm, **cell))._check_supported()
    # KTH: 10 context frames as backgrounds and 4 frames of 4 transforms = 16 + 1 + 10 + 1 = 28 layers
    kth = dict(context_frames=10, sequence_length=20, context_images_background=True, last_frames=4)
    M(mode='train', hparams_dict=kth)._check_supported()
    for bad in (dict(last_frames=17, num_transformed_images=1), dict(last_frames=5, num_transformed_images=4),
                dict(context_frames=31, sequence_length=40, context_images_background=True, num_transformed_images=1),
                dict(num_transformed_images=-1)):
        with pytest.raises(NotImplementedError):
            M(mode='train', hparams_dict=dict(base, **bad))._check_supported()


# ---------------------------------------------------------------------------------- float64 identities of the reference
def _run(case, seed=3, sampling=None):
    hp = O.make_hparams(**dict(TINY, **case))
    params, _ = CO.init_params(hp, (32, 32, 3), seed=seed, dtype=torch.float64)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3), seed=seed, dtype=torch.float64)
    with torch.no_grad():
        out = CO.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, 2, sampling))
    return hp, inputs, out


def test_prev_image_alone_copies_the_input():
    hp, inputs, out = _run(dict(num_transformed_images=0, generate_scratch_image=False, first_image_background=False))
    assert out['transformed_images'].shape[-1] == 1 and torch.equal(out['masks'], torch.ones_like(out['masks']))
    gen = out['gen_images']
    images = inputs['images']
    for t in range(hp.sequence_length - 1):     # ground truth in the context, then the previous generated frame
        want = images[t] if t < hp.context_frames else gen[t - 1]
        assert torch.equal(gen[t], want), t
    assert torch.equal(gen[-1], images[hp.context_frames - 1])


def test_first_image_alone_repeats_the_first_frame():
    hp, inputs, out = _run(dict(num_transformed_images=0, generate_scratch_image=False, prev_image_background=False))
    assert torch.equal(out['gen_images'], inputs['images'][0].expand_as(out['gen_images']))


def test_slot_order_follows_the_reference():
    case = dict(last_frames=2, num_transformed_images=1, last_image_background=True, last_context_image_background=True,
                context_frames=3, sequence_length=6)
    hp, inputs, out = _run(case)
    tr, gen, images = out['transformed_images'], out['gen_images'], inputs['images']
    assert [s[0] for s in CO.sources(hp)] == ['transform', 'transform', 'prev', 'first', 'last', 'last_context', 'scratch']
    for t in range(hp.sequence_length - 1):
        image = images[t] if t < hp.context_frames else gen[t - 1]
        assert torch.equal(tr[t, ..., 2], image)
        assert torch.equal(tr[t, ..., 3], images[0])
        assert torch.equal(tr[t, ..., 4], images[hp.context_frames - 1])
        assert torch.equal(tr[t, ..., 5], images[min(t, hp.context_frames - 1)])
    ctx = _run(dict(context_images_background=True, context_frames=3, sequence_length=6, first_image_background=True))
    hp, inputs, out = ctx
    for i in range(3):
        assert torch.equal(out['transformed_images'][..., 5 + i], inputs['images'][i].expand_as(out['gen_images']))
    # the history: with identity-like kernels the older frame's transform differs from the current frame's
    hp, inputs, out = _run(dict(last_frames=2, num_transformed_images=1))
    tr = out['transformed_images']
    assert not torch.equal(tr[1, ..., 0], tr[1, ..., 1])


def test_defaults_leave_the_oracles_bit_identical():
    hp = O.make_hparams(**TINY)
    params, _ = O.init_params(hp, (32, 32, 3), seed=2)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3))
    inputs['pix_distribs'] = torch.rand(hp.sequence_length, 2, 32, 32, 2, generator=torch.Generator().manual_seed(1))
    gt = O.ground_truth_mask(hp, 2, torch.tensor([[True, False], [False, True]]))
    with torch.no_grad():
        want = P.generator(O.Vars(params), hp, inputs, noise, gt)
        got = CO.pix_generator(O.Vars(params), hp, inputs, noise, gt)
    assert list(want) == list(got) and all(torch.equal(want[k], got[k]) for k in want)
    assert O.savp_cell_step.__module__ == O.__name__ and P.generator_given_z.__module__ == P.__name__


def test_pix_maps_take_the_image_slots():
    """With last_frames = 2 and context backgrounds, the maps' slots follow the images' slot list: the backgrounds are the
    ground-truth maps, the previous-image and scratch slots the selected map."""
    case = dict(last_frames=2, num_transformed_images=1, context_images_background=True, context_frames=2)
    hp = O.make_hparams(**dict(TINY, **case))
    params, _ = CO.init_params(hp, (32, 32, 3), seed=3, dtype=torch.float64)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3), seed=3, dtype=torch.float64)
    pix = torch.rand(hp.sequence_length, 2, 32, 32, 1, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    inputs['pix_distribs'] = pix / pix.sum(dim=(2, 3), keepdim=True)
    with torch.no_grad():
        out = CO.pix_generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, 2))
    tr, gen = out['transformed_pix_distribs'], out['gen_pix_distribs']
    assert tr.shape[-1] == len(CO.sources(hp)) == 6 and out['transformed_images'].shape[-1] == 6
    for t in range(hp.sequence_length - 1):
        p = inputs['pix_distribs'][t] if t < hp.context_frames else gen[t - 1]
        assert torch.equal(tr[t, ..., 2], p) and torch.equal(tr[t, ..., 5], p)
        assert torch.equal(tr[t, ..., 3], inputs['pix_distribs'][0]) and torch.equal(tr[t, ..., 4], inputs['pix_distribs'][1])
    assert torch.allclose(gen.sum(dim=(2, 3)), torch.ones_like(gen.sum(dim=(2, 3))))
