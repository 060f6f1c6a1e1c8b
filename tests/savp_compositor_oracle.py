"""CPU reference of the compositing stage's hparams (savp_model.py:239-246, 349-351, 407-410, 519-653), built on the SAVP
oracle (oracle/savp_oracle.py) without changing it:

- last_frames = F: the transforms read the F most recent images oldest first, [img_{t-F+1} .. img_t], with img_s =
  images[0] for s < 0 (zero_state, :349-351); the nk = F * num_transformed_images kernels (or flows) are split along the
  last axis into F consecutive groups, group j for image j (apply_kernels / apply_flows, :926-965).  No transforms, and no
  cdna_kernels / h{n}_flow / flows variables, unless last_frames and num_transformed_images.
- backgrounds, in this order (:581-594): the step's input image (prev_image_background), images[0]
  (first_image_background), images[context_frames-1] (last_image_background), images[min(t, context_frames-1)]
  (last_context_image_background) -- the last three only without context_images_background --, and all
  images[:context_frames] (context_images_background);
- the scratch image last (generate_scratch_image), with its h{n}_scratch / scratch_image variables only then;
- masks (:623-644): for L > 1 layers h{n}_masks and a 3x3 conv to L channels over [h_masks] + layers (dependent_mask) or
  h_masks alone, then softmax; a single layer has the mask 1 and no mask variables; L == 0 is a ValueError.

For the duration of a call the oracle's `savp_cell_step` and `generator_given_z` are replaced by the general forms below
(the encoder / decoder stack is the oracle's, step for step), inside the norm_layer / ConvLSTM / layer-choice variants of
savp_layers_oracle.  With the default hparams every function returns exactly the oracle's result."""
from contextlib import contextmanager

import torch

import savp_layers_oracle as R
import savp_pix_oracle as P
from oracle import savp_oracle as O

L0_MESSAGE = ('Either one of the following should be true: last_frames and num_transformed_images, first_image_background, '
              'prev_image_background, generate_scratch_image')


def sources(hp):
    """The slot list of one step as the reference builds it (:576-596): ('transform', frame j, k) for each of the nk
    transforms, then the backgrounds ('prev',), ('first',), ('last',), ('last_context',), ('context', i), then
    ('scratch',)."""
    out = []
    if hp.last_frames and hp.num_transformed_images:
        for j in range(hp.last_frames):
            out += [('transform', j, j * hp.num_transformed_images + k) for k in range(hp.num_transformed_images)]
    ctx = hp.context_images_background
    if hp.prev_image_background:
        out.append(('prev',))
    if hp.first_image_background and not ctx:
        out.append(('first',))
    if hp.last_image_background and not ctx:
        out.append(('last',))
    if hp.last_context_image_background and not ctx:
        out.append(('last_context',))
    if ctx:
        out += [('context', i) for i in range(hp.context_frames)]
    if hp.generate_scratch_image:
        out.append(('scratch',))
    return out


def _stack(V, hp, scope, inp, image, first_image, states, saz, new_rnn):
    """The encoder / decoder stack of O.savp_cell_step (:448-519), step for step."""
    enc_specs, dec_specs = O.layer_specs(hp, image.shape[1], image.shape[2])
    layers = []
    rnn_states = states['conv_rnn_states']
    for i, (oc, use_rnn) in enumerate(enc_specs):
        h = torch.cat([image, first_image], dim=-1) if i == 0 else layers[-1][-1]
        ks = 5 if i == 0 else 3
        h = O.tile_concat_z(h, saz)
        k = V.get('%s/h%d/conv_pool2d/kernel' % (scope, i), (ks, ks, h.shape[-1], oc))
        b = V.get('%s/h%d/conv_pool2d/bias' % (scope, i), (oc,), 'zeros')
        h = O.conv_pool2d(h, k, b)
        g = V.get('%s/h%d/InstanceNorm/gamma' % (scope, i), (oc,), 'ones')
        be = V.get('%s/h%d/InstanceNorm/beta' % (scope, i), (oc,), 'zeros')
        h = O.torch.relu(O.instance_norm(h, g, be))
        if use_rnn:
            rh, st = O.conv_lstm_cell(V, '%s/lstm_h%d/basic_conv2dlstm_cell' % (scope, i), O.tile_concat_z(h, saz),
                                      rnn_states[len(new_rnn)], oc)
            new_rnn.append(st)
            layers.append((h, rh))
        else:
            layers.append((h,))
    n_enc = len(layers)
    for i, (oc, use_rnn) in enumerate(dec_specs):
        li = len(layers)
        h = layers[-1][-1] if i == 0 else torch.cat([layers[-1][-1], layers[n_enc - i - 1][-1]], dim=-1)
        h = O.tile_concat_z(h, saz)
        k = V.get('%s/h%d/upsample_conv2d/kernel' % (scope, li), (3, 3, h.shape[-1], oc))
        b = V.get('%s/h%d/upsample_conv2d/bias' % (scope, li), (oc,), 'zeros')
        h = O.upsample_conv2d(h, k, b)
        g = V.get('%s/h%d/InstanceNorm/gamma' % (scope, li), (oc,), 'ones')
        be = V.get('%s/h%d/InstanceNorm/beta' % (scope, li), (oc,), 'zeros')
        h = O.torch.relu(O.instance_norm(h, g, be))
        if use_rnn:
            rh, st = O.conv_lstm_cell(V, '%s/lstm_h%d/basic_conv2dlstm_cell' % (scope, li), O.tile_concat_z(h, saz),
                                      rnn_states[len(new_rnn)], oc)
            new_rnn.append(st)
            layers.append((h, rh))
        else:
            layers.append((h,))
    assert len(new_rnn) == len(rnn_states)
    return layers, n_enc


def savp_cell_step(V, hp, scope, t, inp, first_image, states, ground_truth_t, tap=None):
    """O.savp_cell_step with the general compositing stage; states carry 'last_images' and 'all_images'."""
    B, H, W, C = inp['images'].shape
    images = states['all_images']
    gt = ground_truth_t.view(B, 1, 1, 1)
    image = torch.where(gt, inp['images'], states['gen_image'])
    last_images = states['last_images'][1:] + [image]                                   # :407
    saz = []
    if 'actions' in inp:
        saz.append(inp['actions'])
    new_states = dict(states)
    if 'zs' in inp:
        if hp.use_rnn_z:
            rnn_z, rz_state = O.dense_lstm_cell(V, scope + '/lstm_z/basic_lstm_cell', inp['zs'], states['rnn_z_state'], hp.nz)
            new_states['rnn_z_state'] = rz_state
            saz.append(rnn_z)
        else:
            saz.append(inp['zs'])
    saz = torch.cat(saz, dim=-1) if saz else None
    new_rnn = []
    layers, n_enc = _stack(V, hp, scope, inp, image, first_image, states, saz, new_rnn)
    nl = len(layers)
    top = layers[-1][-1]

    def conv3x3(name, x, oc):
        k = V.get('%s/%s/conv2d/kernel' % (scope, name), (3, 3, x.shape[-1], oc))
        b = V.get('%s/%s/conv2d/bias' % (scope, name), (oc,), 'zeros')
        return O.conv2d_tf(x, k, padding='SAME', bias=b)

    def norm_relu(name, x):
        g = V.get('%s/%s/InstanceNorm/gamma' % (scope, name), (x.shape[-1],), 'ones')
        be = V.get('%s/%s/InstanceNorm/beta' % (scope, name), (x.shape[-1],), 'zeros')
        return O.torch.relu(O.instance_norm(x, g, be))

    kh, kw = hp.kernel_size
    nk = hp.last_frames * hp.num_transformed_images
    kernels = flows = None
    if hp.last_frames and hp.num_transformed_images:
        if hp.transformation == 'flow':
            h_flow = norm_relu('h%d_flow' % nl, conv3x3('h%d_flow' % nl, top, hp.ngf))
            flows = conv3x3('flows', h_flow, 2 * nk).reshape(B, H, W, 2, nk)
        else:
            flat = layers[n_enc - 1][-1].reshape(B, -1)
            dk = V.get(scope + '/cdna_kernels/dense/kernel', (flat.shape[1], kh * kw * nk))
            db = V.get(scope + '/cdna_kernels/dense/bias', (kh * kw * nk,), 'zeros')
            kernels = O.dense(flat, dk, db).reshape(B, kh, kw, nk)
            kernels = kernels + torch.tensor(O.identity_kernel((kh, kw)), dtype=kernels.dtype)[None, :, :, None]
            kernels = torch.relu(kernels - O.RELU_SHIFT) + O.RELU_SHIFT
            kernels = kernels / kernels.sum(dim=(1, 2), keepdim=True)
    scratch = None
    if hp.generate_scratch_image:
        h_scratch = norm_relu('h%d_scratch' % nl, conv3x3('h%d_scratch' % nl, top, hp.ngf))
        scratch = torch.sigmoid(conv3x3('scratch_image', h_scratch, C))
    ctx = hp.context_frames
    transformed = []
    for src in sources(hp):
        if src[0] == 'transform':
            j, k = src[1], src[2]
            if flows is not None:
                transformed.append(O.image_warp(last_images[j], flows[..., k]))
            else:                   # one call per group, as apply_kernels splits them (:939-943)
                G = hp.num_transformed_images
                transformed.append(O.apply_cdna_kernels(last_images[j], kernels[..., j * G:(j + 1) * G])[k - j * G])
        elif src[0] == 'prev':
            transformed.append(image)
        elif src[0] == 'first':
            transformed.append(images[0])
        elif src[0] == 'last':
            transformed.append(images[ctx - 1])
        elif src[0] == 'last_context':
            transformed.append(images[t] if t < ctx else images[ctx - 1])
        elif src[0] == 'context':
            transformed.append(images[src[1]])
        else:
            transformed.append(scratch)
    if len(transformed) > 1:
        h_masks = norm_relu('h%d_masks' % nl, conv3x3('h%d_masks' % nl, top, hp.ngf))
        if hp.dependent_mask:
            h_masks = torch.cat([h_masks] + transformed, dim=-1)
        mask_logits = conv3x3('masks', h_masks, len(transformed))
        masks = torch.softmax(mask_logits, dim=-1)
    elif len(transformed) == 1:
        mask_logits, masks = None, torch.ones(B, H, W, 1, dtype=image.dtype)
    else:
        raise ValueError(L0_MESSAGE)
    gen_image = sum(tr * masks[..., k:k + 1] for k, tr in enumerate(transformed))
    if tap is not None:
        tap.update(dict(image=image, kernels=kernels, flows=flows, scratch=scratch, mask_logits=mask_logits, layers=layers,
                        rnn_z=saz))
    new_states.update(gen_image=gen_image, conv_rnn_states=new_rnn, last_images=last_images)
    outputs = dict(gen_images=gen_image, transformed_images=torch.stack(transformed, dim=-1),
                   masks=torch.stack([masks[..., k:k + 1] for k in range(masks.shape[-1])], dim=-1))
    return outputs, new_states


def generator_given_z(V, hp, inputs, ground_truth, scope='generator/rnn/savp_cell', taps=None):
    """O.generator_given_z with the history state last_images = [images[0]] * last_frames (:349-351)."""
    images = inputs['images']
    T = hp.sequence_length
    B, H, W, C = images.shape[1:]
    enc_specs, dec_specs = O.layer_specs(hp, H, W)
    dt = images.dtype
    rnn_states = []
    hh, ww = H, W
    for oc, use in enc_specs:
        hh, ww = hh // 2, ww // 2
        if use:
            rnn_states.append((torch.zeros(B, hh, ww, oc, dtype=dt), torch.zeros(B, hh, ww, oc, dtype=dt)))
    for oc, use in dec_specs:
        hh, ww = hh * 2, ww * 2
        if use:
            rnn_states.append((torch.zeros(B, hh, ww, oc, dtype=dt), torch.zeros(B, hh, ww, oc, dtype=dt)))
    states = dict(gen_image=torch.zeros(B, H, W, C, dtype=dt), conv_rnn_states=rnn_states,
                  last_images=[images[0]] * hp.last_frames, all_images=images)
    if 'zs' in inputs and hp.use_rnn_z:
        states['rnn_z_state'] = (torch.zeros(B, hp.nz, dtype=dt), torch.zeros(B, hp.nz, dtype=dt))
    outs = []
    for t in range(T - 1):
        inp = dict(images=images[t])
        if 'actions' in inputs:
            inp['actions'] = inputs['actions'][t]
        if 'zs' in inputs:
            inp['zs'] = inputs['zs'][t]
        tap = {} if taps is not None else None
        o, states = savp_cell_step(V, hp, scope, t, inp, images[0], states, ground_truth[t], tap)
        if taps is not None:
            taps.append(tap)
        outs.append(o)
    return {k: torch.stack([o[k] for o in outs], dim=0) for k in outs[0]}


def pix_generator_given_z(V, hp, inputs, ground_truth, scope=P.SCOPE):
    """savp_pix_oracle.generator_given_z for every slot layout: the maps take the slots of the images (:598-621), the
    transforms act on the selected maps of the last F steps, last_pix_distribs (:349-351, 408-410)."""
    plain = {k: v for k, v in inputs.items() if k != 'pix_distribs'}
    taps = []
    out = O.generator_given_z(V, hp, plain, ground_truth, scope=scope, taps=taps)
    if 'pix_distribs' not in inputs:
        return out
    pix = inputs['pix_distribs']
    B, ctx, G = pix.shape[1], hp.context_frames, hp.num_transformed_images
    gen_prev = torch.zeros_like(pix[0])
    last = [pix[0]] * hp.last_frames
    gens, trs = [], []
    for t, tap in enumerate(taps):
        p = torch.where(ground_truth[t].view(B, 1, 1, 1), pix[t], gen_prev)
        last = last[1:] + [p]
        slots = []
        for src in sources(hp):
            if src[0] == 'transform':
                j, k = src[1], src[2]
                if tap['flows'] is not None:
                    slots.append(O.image_warp(last[j], tap['flows'][..., k]))
                else:
                    slots.append(O.apply_cdna_kernels(last[j], tap['kernels'][..., j * G:(j + 1) * G])[k - j * G])
            else:
                slots.append({'prev': p, 'first': pix[0], 'last': pix[ctx - 1], 'last_context': pix[min(t, ctx - 1)],
                              'scratch': p}.get(src[0]) if src[0] != 'context' else pix[src[1]])
        masks = out['masks'][t][..., 0, :]
        gen = sum(tr * masks[..., k:k + 1] for k, tr in enumerate(slots))
        gen_prev = gen / gen.sum(dim=(1, 2), keepdim=True)
        gens.append(gen_prev)
        trs.append(torch.stack(slots, dim=-1))
    out['gen_pix_distribs'] = torch.stack(gens)
    out['transformed_pix_distribs'] = torch.stack(trs)
    return out


@contextmanager
def variant(hp):
    with R.variant(hp):
        saved = O.savp_cell_step, O.generator_given_z, P.generator_given_z
        O.savp_cell_step, O.generator_given_z, P.generator_given_z = savp_cell_step, generator_given_z, pix_generator_given_z
        try:
            yield
        finally:
            O.savp_cell_step, O.generator_given_z, P.generator_given_z = saved


def pix_generator(V, hp, inputs, noise, ground_truth):
    """savp_pix_oracle.generator (the images and the maps of both unrolls) for every slot layout."""
    with variant(hp):
        return P.generator(V, hp, inputs, noise, ground_truth)


def generator(V, hp, inputs, noise, ground_truth, taps=None):
    with variant(hp):
        return O.generator(V, hp, inputs, noise, ground_truth, taps)


def train_step(params, opt, hp, inputs, noise, step, sampling=None):
    with variant(hp):
        return O.train_step(params, opt, hp, inputs, noise, step, sampling)


def init_params(hp, image_shape, batch=1, action_dim=0, seed=0, dtype=torch.float32):
    with variant(hp):
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
