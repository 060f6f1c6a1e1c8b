"""CPU tests of the per-frame image discriminator over the sampled clip (`images_sn_gan_weight`,
`images_sn_vae_gan_weight`): the reference (tests/savp_images_d_oracle.py) against the oracle's image tower frame by frame,
the model's variables against the reference's, the loss names and weights, and the clip offsets the towers draw."""
from collections import OrderedDict

import numpy as np
import pytest
import torch

import savp_images_d_oracle as R
from oracle import savp_oracle as O

BASE = dict(context_frames=2, sequence_length=12, lr=2e-4, beta1=0.5, l1_weight=100.0, kl_weight=1.0)
CASES = {
    'images_only': dict(BASE, images_sn_gan_weight=0.1, images_sn_vae_gan_weight=0.1),
    'images_video': dict(BASE, video_sn_gan_weight=0.1, video_sn_vae_gan_weight=0.1, images_sn_gan_weight=0.1,
                         images_sn_vae_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=1.0),
    'images_nz0': dict(BASE, nz=0, kl_weight=0.0, images_sn_gan_weight=0.1),
}


def _model(hk, H=64, W=64):
    from video_prediction_b200.models import SAVPVideoPredictionModel
    m = SAVPVideoPredictionModel(mode='train', hparams_dict=hk)
    m.B, m.T, m.H, m.W, m.C, m.A, m.Sd = 4, hk['sequence_length'], H, W, 3, 0, 0
    m.S, m.Zc = m.T - 1, m.hparams.nz
    m.enc_specs, m.dec_specs = m.layer_specs(m.hparams.ngf, H, W)
    return m


def _with_towers(m):
    """The fields of m.dnets that _set_tstarts reads, on the CPU."""
    m.device = torch.device('cpu')
    m.dnets = OrderedDict((tw['scope'], dict(tw, clip_len=m._d_clip_len(tw['kind']))) for tw in m._d_towers())
    return m


def test_tower_on_a_clip_is_the_image_tower_frame_by_frame():
    """with_flat_batch(image_sn_discriminator) on [clip, B, ...] = the image tower on each frame, in fp64."""
    hp = O.make_hparams(**dict(CASES['images_nz0'], ndf=8, clip_length=3))
    g = torch.Generator().manual_seed(3)
    clip = torch.rand(3, 2, 32, 32, 3, generator=g, dtype=torch.float64)
    V = O.Vars(None, np.random.default_rng(5), torch.float64)
    feats, logits = R.images_sn_discriminator(V, 'discriminator/images', clip, hp.ndf)
    assert logits.shape == (3, 2, 1) and len(feats) == 7
    for t in range(3):
        f_t, l_t = O.image_sn_discriminator(V, 'discriminator/images', clip[t], hp.ndf)
        assert (logits[t] - l_t).abs().max().item() <= 1e-12
        for a, b in zip(feats, f_t):
            assert a[t].shape == b.shape and (a[t] - b).abs().max().item() <= 1e-12
    # the loss terms are means over every frame: the order of the frames does not enter
    perm = torch.randperm(6, generator=g)
    flat = logits.reshape(6, 1)
    assert abs(O.gan_loss(flat, 1.0, 'LSGAN') - O.gan_loss(flat[perm], 1.0, 'LSGAN')).item() <= 1e-15
    fake = [f.flip(0) for f in feats]
    a = sum(O.cosine_distance(x, y) for x, y in zip(fake, feats))
    b = sum(O.cosine_distance(x.reshape((6,) + x.shape[2:])[perm], y.reshape((6,) + y.shape[2:])[perm]) for x, y in zip(fake, feats))
    assert abs(a - b).item() <= 1e-12


@pytest.mark.parametrize('case', sorted(CASES))
def test_variables_match_the_reference(case):
    hk = CASES[case]
    m = _model(hk)
    specs = m._discriminator_param_specs()
    ref, trainable = R.init_params(O.make_hparams(**hk), (64, 64, 3))
    dref = {k: v for k, v in ref.items() if k.startswith('discriminator/')}
    assert set(specs) == set(dref), sorted(set(specs) ^ set(dref))[:5]
    for k, (shape, init) in specs.items():
        assert tuple(shape) == tuple(dref[k].shape), k
        assert (init == 'u') == (not trainable[k]), k
    scopes = ['discriminator/encoder/images', 'discriminator/images'] if m.hparams.nz else ['discriminator/images']
    for sc in scopes:
        names = sorted(k for k in specs if k.startswith(sc + '/'))
        assert names == sorted('%s/%s/%s/%s' % (sc, lay, sub, v) for lay, sub in
                               [('sn_conv%d_%d' % (i // 2, i % 2), 'conv2d') for i in range(7)] + [('sn_fc4', 'dense')]
                               for v in ('kernel', 'u', 'bias'))
        # the image tower's shapes (networks.py:35-69): 64x64 -> 8x8x256, the dense reads one frame
        assert specs[sc + '/sn_conv0_0/conv2d/kernel'][0] == (3, 3, 3, 32)
        assert specs[sc + '/sn_conv3_0/conv2d/kernel'][0] == (3, 3, 256, 256)
        assert specs[sc + '/sn_fc4/dense/kernel'][0] == (8 * 8 * 256, 1)
        # 1,463,136 kernel + 2 x 928 bias and u entries in the convolutions, 16,384 + 2 in the dense
        assert sum(int(np.prod(specs[k][0])) for k in names) == 1481378
    # the images towers come after the existing ones, so the existing variables keep their positions
    first = next(i for i, k in enumerate(specs) if '/images/' in k)
    assert all('/images/' in k for k in list(specs)[first:])


def test_reference_is_the_oracle_without_the_images_weights():
    hk = dict(BASE, video_sn_gan_weight=0.1, video_sn_vae_gan_weight=0.1, ngf=8, nef=8, ndf=8, sequence_length=6, clip_length=4)
    a, _ = O.init_params(O.make_hparams(**hk), (32, 32, 3), seed=2)
    b, _ = R.init_params(O.make_hparams(**hk), (32, 32, 3), seed=2)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    c, _ = R.init_params(O.make_hparams(**dict(hk, images_sn_gan_weight=0.1)), (32, 32, 3), seed=2)
    assert all(torch.equal(a[k], c[k]) for k in a)      # the images variables come from their own generator
    assert sorted(set(c) - set(a))[0].startswith('discriminator/encoder/images/')


def test_images_weights_are_accepted_and_feature_l2_stays_refused():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    for hk in CASES.values():
        SAVPVideoPredictionModel(mode='train', hparams_dict=hk)._check_supported()
    for bad in (dict(gan_feature_l2_weight=1.0), dict(vae_gan_feature_l2_weight=1.0)):
        with pytest.raises(NotImplementedError):
            SAVPVideoPredictionModel(mode='train', hparams_dict=dict(CASES['images_video'], **bad))._check_supported()


def test_loss_names_and_weights_follow_the_reference():
    """loss_weights / split_losses carry the reference's term names (base_model.py:771-852) at the reference's weights."""
    from video_prediction_b200.models import savp_train
    assert savp_train.IMAGES_LOSS_SLOTS == ['gen_images_sn_gan_loss', 'gen_images_sn_vae_gan_loss',
                                            'gen_images_sn_vae_gan_feature_cdist_loss', 'gen_images_sn_gan_feature_cdist_loss',
                                            'discrim_images_sn_gan_loss', 'discrim_images_sn_vae_gan_loss']
    # a model without the images towers reports the same terms as before they existed; with them, their six come last
    base = _model(dict(BASE, video_sn_gan_weight=0.1))
    assert base.loss_slots() == savp_train.LOSS_SLOTS and len(savp_train.LOSS_SLOTS) == 15
    assert list(base.loss_weights(step=3)) == savp_train.LOSS_SLOTS
    assert not any('images' in k for k in savp_train.LOSS_SLOTS)
    for hk in CASES.values():
        m = _model(hk)
        assert m.loss_slots() == savp_train.LOSS_SLOTS + savp_train.IMAGES_LOSS_SLOTS
        assert list(m.loss_weights(step=3)) == m.loss_slots()
    hk = dict(CASES['images_video'], ngf=8, nef=8, ndf=8, sequence_length=6, clip_length=4, kl_anneal='none')
    hp = O.make_hparams(**hk)
    params, _ = R.init_params(hp, (32, 32, 3), seed=1)
    inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3))
    opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
    res = R.train_step(params, opt, hp, inputs, noise, step=3)
    m = _model(hk, 32, 32)
    w = m.loss_weights(step=3)
    assert {k for k, v in w.items() if v} == set(res['g_losses']) | set(res['d_losses'])
    for k in ('gen_images_sn_gan_loss', 'gen_images_sn_vae_gan_loss', 'discrim_images_sn_gan_loss', 'discrim_images_sn_vae_gan_loss'):
        assert w[k] == 0.1, k
    assert w['gen_images_sn_gan_feature_cdist_loss'] == 1.0 and w['gen_images_sn_vae_gan_feature_cdist_loss'] == 10.0
    vals = OrderedDict((k, 0.0) for k in savp_train.LOSS_SLOTS)
    vals.update(res['g_losses'])
    vals.update(res['d_losses'])
    g, d, g_loss, d_loss = m.split_losses(vals, w)
    assert set(g) == set(res['g_losses']) and set(d) == set(res['d_losses'])
    assert {'gen_images_sn_gan_loss', 'gen_images_sn_vae_gan_loss', 'gen_images_sn_gan_feature_cdist_loss',
            'gen_images_sn_vae_gan_feature_cdist_loss'} <= set(g)
    assert {'discrim_images_sn_gan_loss', 'discrim_images_sn_vae_gan_loss'} <= set(d)
    assert g_loss == pytest.approx(res['g_loss'], rel=1e-6) and d_loss == pytest.approx(res['d_loss'], rel=1e-6)


def test_images_towers_share_the_video_towers_offsets():
    m = _with_towers(_model(CASES['images_video']))
    for noise in (None, O.make_synthetic_inputs(O.make_hparams(**CASES['images_video']), 4, (8, 8, 3))[1]):
        m.global_step += 1
        m._set_tstarts(noise)
        for enc in ('encoder/', ''):
            v, i = m.dnets['discriminator/%svideo' % enc], m.dnets['discriminator/%simages' % enc]
            for key in [(w, r) for w in ('d_pre', 'd_post') for r in (0, 1)]:
                assert torch.equal(i['ts'][key], v['ts'][key]), (enc, key)
            if noise is not None:
                for r, k in enumerate(v['keys']):
                    assert torch.equal(i['ts'][('d_post', r)], noise['d_post'][k].to(torch.int32))
    # without a video tower the images towers draw their own offsets from the video tower's range, per (call, role)
    m = _with_towers(_model(CASES['images_only']))
    m._set_tstarts(None)
    hi = m.S - m.hparams.clip_length
    draws = [t for net in m.dnets.values() for t in net['ts'].values()]
    assert len(draws) == 8 and all(int(t.min()) >= 0 and int(t.max()) <= hi for t in draws)
    assert len({tuple(t.tolist()) for t in draws}) > 1


def test_adding_the_images_towers_leaves_the_other_draws_unchanged():
    base = dict(BASE, image_sn_gan_weight=0.1, image_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, video_sn_vae_gan_weight=0.1)
    a = _with_towers(_model(base))
    b = _with_towers(_model(dict(base, images_sn_gan_weight=0.1, images_sn_vae_gan_weight=0.1)))
    assert list(b.dnets)[:4] == list(a.dnets)
    for step in (0, 7):
        a.global_step = b.global_step = step
        a._set_tstarts(None)
        b._set_tstarts(None)
        for scope, net in a.dnets.items():
            for key, t in net['ts'].items():
                assert torch.equal(b.dnets[scope]['ts'][key], t), (scope, key)
