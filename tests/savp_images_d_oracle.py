"""CPU reference of the per-frame image discriminator over the sampled clip (`images_sn_gan_weight`,
`images_sn_vae_gan_weight`; savp_model.py:120-126), built on the SAVP oracle (oracle/savp_oracle.py) without changing it.

Inside one discriminator_given_video_fn call the `images` tower reads the same clip_sample as the video tower, so it takes
the video tower's clip offsets (`t_starts['real']`, ... -- the same keys).  The tower is the oracle's
`image_sn_discriminator` under `tf_utils.with_flat_batch`: the clip [clip, B, H, W, C] is flattened to clip * B frames, and
features and logits are reshaped back to [clip, B, ...].  Its loss terms follow base_model.py:771-852 with the infix
`_images_sn`: the GAN losses are means over the clip * B logits, the feature distances sums over the 7 features of the
mean over frames and positions.

With both images weights at zero every function returns the oracle's result."""
from collections import OrderedDict

import numpy as np
import torch

from oracle import savp_oracle as O


def has_images(hp):
    return bool(hp.images_sn_gan_weight or hp.images_sn_vae_gan_weight)


def has_d(hp):
    return bool(hp.video_sn_gan_weight or hp.video_sn_vae_gan_weight or hp.image_sn_gan_weight or hp.image_sn_vae_gan_weight
                or has_images(hp))


def images_sn_discriminator(V, scope, clip, ndf, u_out=None):
    """tf_utils.with_flat_batch(networks.image_sn_discriminator) on a time-major clip [clip, B, H, W, C]: 7 feature maps
    [clip, B, H', W', C'] and logits [clip, B, 1]."""
    T, B = clip.shape[:2]
    feats, logits = O.image_sn_discriminator(V, scope, clip.reshape((T * B,) + tuple(clip.shape[2:])), ndf, u_out)
    return [f.reshape((T, B) + tuple(f.shape[1:])) for f in feats], logits.reshape(T, B, 1)


def discriminator(V, hp, inputs, gen_outputs, t_starts, u_out=None):
    """O.discriminator (image / video towers) followed by the images towers, on the clips of the same offsets."""
    out = O.discriminator(V, hp, inputs, gen_outputs, t_starts, u_out)
    if not has_images(hp):
        return out
    real = inputs['images'][1:]

    def run(prefix, video, key, suffix):
        clip = O.gather_clip(video, t_starts[key], hp.clip_length)
        feats, logits = images_sn_discriminator(V, prefix + '/images', clip, hp.ndf, u_out)
        out['discrim_images_sn_logits' + suffix] = logits
        for i, f in enumerate(feats):
            out['discrim_images_sn_feature%d%s' % (i, suffix)] = f
    if hp.nz:
        run('discriminator/encoder', real, 'enc_real', '_enc_real')
        run('discriminator/encoder', gen_outputs['gen_images_enc'], 'enc_fake', '_enc_fake')
    run('discriminator', real, 'real', '_real')
    run('discriminator', gen_outputs['gen_images'], 'fake', '_fake')
    return out


def generator_losses(hp, inputs, outputs, step):
    L = O.generator_losses(hp, inputs, outputs, step)
    infix, w_gan, w_vae = '_images_sn', hp.images_sn_gan_weight, hp.images_sn_vae_gan_weight
    if w_gan:
        L['gen%s_gan_loss' % infix] = (O.gan_loss(outputs['discrim%s_logits_fake' % infix], 1.0, hp.gan_loss_type), w_gan)
        if hp.gan_feature_cdist_weight:
            sm = sum(O.cosine_distance(outputs['discrim%s_feature%d_fake' % (infix, i)],
                                       outputs['discrim%s_feature%d_real' % (infix, i)]) for i in range(7))
            L['gen%s_gan_feature_cdist_loss' % infix] = (sm, hp.gan_feature_cdist_weight)
    if w_vae and hp.nz:
        L['gen%s_vae_gan_loss' % infix] = (O.gan_loss(outputs['discrim%s_logits_enc_fake' % infix], 1.0, hp.gan_loss_type), w_vae)
        if hp.vae_gan_feature_cdist_weight:
            sm = sum(O.cosine_distance(outputs['discrim%s_feature%d_enc_fake' % (infix, i)],
                                       outputs['discrim%s_feature%d_enc_real' % (infix, i)]) for i in range(7))
            L['gen%s_vae_gan_feature_cdist_loss' % infix] = (sm, hp.vae_gan_feature_cdist_weight)
    return L


def discriminator_losses(hp, outputs):
    L = O.discriminator_losses(hp, outputs)
    t, infix = hp.gan_loss_type, '_images_sn'
    if hp.images_sn_gan_weight:
        L['discrim%s_gan_loss' % infix] = (O.gan_loss(outputs['discrim%s_logits_real' % infix], 1.0, t) +
                                           O.gan_loss(outputs['discrim%s_logits_fake' % infix], 0.0, t), hp.images_sn_gan_weight)
    if hp.images_sn_vae_gan_weight and hp.nz:
        L['discrim%s_vae_gan_loss' % infix] = (O.gan_loss(outputs['discrim%s_logits_enc_real' % infix], 1.0, t) +
                                               O.gan_loss(outputs['discrim%s_logits_enc_fake' % infix], 0.0, t),
                                               hp.images_sn_vae_gan_weight)
    return L


def train_step(params, opt, hp, inputs, noise, step, sampling=None):
    """O.train_step with the images towers in both discriminator forwards and their terms in both losses: the same order
    (u <- u'; D loss -> Adam(D); D forward with the updated weights -> G loss -> Adam(G); u' stored at the end)."""
    dt = next(iter(params.values())).dtype
    P = OrderedDict((k, v.clone().requires_grad_(True)) for k, v in params.items())
    V = O.Vars(P, None, dt)
    B = inputs['images'].shape[1]
    gen_out = O.generator(V, hp, inputs, noise, O.ground_truth_mask(hp, B, sampling))
    g_names = [k for k in P if k.startswith('generator/')]
    d_names = [k for k in P if k.startswith('discriminator/') and not k.endswith('/u')]
    res = dict(outputs=gen_out)
    lr = O.learning_rate(hp, step)
    t = opt['t'] + 1
    newp = OrderedDict((k, v.detach()) for k, v in P.items())
    u_new = {}
    allout = gen_out
    if has_d(hp):
        d_out = discriminator(V, hp, inputs, {k: v.detach() for k, v in gen_out.items()}, noise['d_pre'], u_new)
        d_losses = discriminator_losses(hp, d_out)
        d_loss = O.total_loss(d_losses)
        d_grads = torch.autograd.grad(d_loss, [P[k] for k in d_names], allow_unused=True)
        res.update(d_losses={k: float(l.detach()) for k, (l, w) in d_losses.items()}, d_loss=float(d_loss.detach()),
                   d_grads=OrderedDict(zip(d_names, d_grads)), d_outputs=d_out)
        for k, g in zip(d_names, d_grads):
            if g is not None:
                newp[k], opt['m'][k], opt['v'][k] = O.adam_tf(newp[k], g, opt['m'][k], opt['v'][k], lr, hp.beta1, hp.beta2, t)
        P2 = OrderedDict(P)
        for k in d_names:
            P2[k] = newp[k]
        allout = OrderedDict(gen_out)
        allout.update(discriminator(O.Vars(P2, None, dt), hp, inputs, gen_out, noise['d_post']))
    g_losses = generator_losses(hp, inputs, allout, step)
    g_loss = O.total_loss(g_losses)
    g_grads = torch.autograd.grad(g_loss, [P[k] for k in g_names], allow_unused=True)
    for k, g in zip(g_names, g_grads):
        if g is not None:
            newp[k], opt['m'][k], opt['v'][k] = O.adam_tf(newp[k], g, opt['m'][k], opt['v'][k], lr, hp.beta1, hp.beta2, t)
    newp.update(u_new)
    opt['t'] = t
    res.update(g_losses={k: float(l.detach()) for k, (l, w) in g_losses.items()}, g_loss=float(g_loss.detach()),
               g_grads=OrderedDict(zip(g_names, g_grads)), params=newp, lr=lr)
    return res


def init_params(hp, image_shape, batch=1, action_dim=0, seed=0, dtype=torch.float32):
    """O.init_params, then the images towers' variables from a second generator (seed, 1), so that every other variable
    keeps the oracle's value."""
    params, trainable = O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
    if not has_images(hp):
        return params, trainable
    V = O.Vars(params, np.random.default_rng([seed, 1]), dtype)
    V.trainable = trainable
    clip = torch.zeros((hp.clip_length, batch) + tuple(image_shape), dtype=dtype)
    with torch.no_grad():
        for prefix in (('discriminator/encoder', 'discriminator') if hp.nz else ('discriminator',)):
            images_sn_discriminator(V, prefix + '/images', clip, hp.ndf)
    return V.params, V.trainable
