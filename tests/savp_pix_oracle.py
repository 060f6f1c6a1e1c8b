"""CPU reference of the pixel-distribution path (savp_model.py:408-410, 598-621, 648-653; tf_utils.py:562-585), built on
the SAVP oracle (oracle/savp_oracle.py) without changing it.

The maps never feed back into the images, so the image unroll is the oracle's own `generator_given_z`, run with taps; the
maps are then advected step by step with that unroll's CDNA kernels (from the tap) or flows (recomputed from the tap's top
layer with the same oracle ops and variables, hence the same values) and its softmax masks.  Every output of the oracle is
returned unchanged, plus gen_pix_distribs / transformed_pix_distribs (and the _enc versions of the posterior unroll)."""
from collections import OrderedDict

import torch

from oracle import savp_oracle as O

SCOPE = 'generator/rnn/savp_cell'


def pixel_distribution(pos, height, width):
    """tf_utils.pixel_distribution (tf_utils.py:562-585): pos [N,2] = (y, x) -> [N,H,W] bilinear weights on the four
    neighbours of the position.  Each neighbour is a one-hot of the FLAT index y*W + x over H*W entries, so x = W lands on
    column 0 of the next row and an index outside [0, H*W) contributes nothing."""
    n = pos.shape[0]
    y, x = pos[:, 0], pos[:, 1]
    x0, y0 = torch.floor(x).long(), torch.floor(y).long()
    x1, y1 = x0 + 1, y0 + 1
    rows = torch.arange(n)

    def one_hot(idx):
        out = torch.zeros(n, height * width, dtype=pos.dtype)
        ok = (idx >= 0) & (idx < height * width)
        out[rows[ok], idx[ok]] = 1
        return out.reshape(n, height, width)
    x0f, x1f, y0f, y1f = x0.to(pos.dtype), x1.to(pos.dtype), y0.to(pos.dtype), y1.to(pos.dtype)
    wa = ((x1f - x) * (y1f - y))[:, None, None]
    wb = ((x1f - x) * (y - y0f))[:, None, None]
    wc = ((x - x0f) * (y1f - y))[:, None, None]
    wd = ((x - x0f) * (y - y0f))[:, None, None]
    return (wa * one_hot(y0 * width + x0) + wb * one_hot(y1 * width + x0) + wc * one_hot(y0 * width + x1)
            + wd * one_hot(y1 * width + x1))


def step_flows(V, hp, tap, scope=SCOPE):
    """The flows of one cell step (savp_model.py:522-530), [B,H,W,2,nk], from the step's top decoder layer."""
    layers = tap['layers']
    nl, top = len(layers), layers[-1][-1]
    B, H, W = top.shape[:3]
    nk = hp.last_frames * hp.num_transformed_images

    def conv3x3(name, x, oc):
        k = V.get('%s/%s/conv2d/kernel' % (scope, name), (3, 3, x.shape[-1], oc))
        b = V.get('%s/%s/conv2d/bias' % (scope, name), (oc,), 'zeros')
        return O.conv2d_tf(x, k, padding='SAME', bias=b)
    h = conv3x3('h%d_flow' % nl, top, hp.ngf)
    g = V.get('%s/h%d_flow/InstanceNorm/gamma' % (scope, nl), (hp.ngf,), 'ones')
    be = V.get('%s/h%d_flow/InstanceNorm/beta' % (scope, nl), (hp.ngf,), 'zeros')
    h = torch.relu(O.instance_norm(h, g, be))
    return conv3x3('flows', h, 2 * nk).reshape(B, H, W, 2, nk)


def pix_step(hp, pix_t, gen_prev, first_pix, ground_truth_t, masks, kernels=None, flows=None):
    """One step of the map path.  pix_t / gen_prev / first_pix [B,H,W,D]; masks [B,H,W,L] (the images' softmax masks);
    kernels [B,kh,kw,nk] (CDNA) or flows [B,H,W,2,nk].  Returns (gen_pix [B,H,W,D], transformed [B,H,W,D,L])."""
    B = pix_t.shape[0]
    pix = torch.where(ground_truth_t.view(B, 1, 1, 1), pix_t, gen_prev)                       # :408-410
    if flows is not None:                                                                       # :598-604
        tpix = [O.image_warp(pix, flows[..., k]) for k in range(flows.shape[-1])]
    else:
        tpix = O.apply_cdna_kernels(pix, kernels)
    tpix = tpix + [pix, first_pix, pix]                                     # :606-621 (scratch slot: the map)
    gen = sum(tr * masks[..., k:k + 1] for k, tr in enumerate(tpix))                           # :648-652
    gen = gen / gen.sum(dim=(1, 2), keepdim=True)                                              # :653
    return gen, torch.stack(tpix, dim=-1)


def generator_given_z(V, hp, inputs, ground_truth, scope=SCOPE):
    """O.generator_given_z + the maps.  inputs as the oracle's, plus pix_distribs [T,B,H,W,D]."""
    plain = {k: v for k, v in inputs.items() if k != 'pix_distribs'}
    taps = []
    out = O.generator_given_z(V, hp, plain, ground_truth, scope=scope, taps=taps)
    if 'pix_distribs' not in inputs:
        return out
    pix = inputs['pix_distribs']
    gen_prev = torch.zeros_like(pix[0])                    # zero state; never read: ground_truth[0] is True (context)
    gens, trs = [], []
    for t, tap in enumerate(taps):
        flows = step_flows(V, hp, tap, scope) if hp.transformation == 'flow' else None
        gen_prev, tr = pix_step(hp, pix[t], gen_prev, pix[0], ground_truth[t], out['masks'][t][..., 0, :],
                                kernels=tap['kernels'], flows=flows)
        gens.append(gen_prev)
        trs.append(tr)
    out['gen_pix_distribs'] = torch.stack(gens)
    out['transformed_pix_distribs'] = torch.stack(trs)
    return out


def generator(V, hp, inputs, noise, ground_truth):
    """O.generator (generator_fn, savp_model.py:699-768) + the maps of both unrolls."""
    if hp.nz == 0:
        return generator_given_z(V, hp, inputs, ground_truth)
    z_mu, z_lss = O.posterior(V, hp, inputs)
    zs_post = z_mu + torch.sqrt(torch.exp(z_lss)) * noise['eps']             # :712
    zs_prior = torch.cat([zs_post[:hp.context_frames - 1], noise['z_prior']], dim=0)   # :724-725
    out_enc = generator_given_z(V, hp, dict(inputs, zs=zs_post), ground_truth)          # :730
    out = generator_given_z(V, hp, dict(inputs, zs=zs_prior), ground_truth)             # :732
    outputs = OrderedDict(out)
    outputs['zs_mu_enc'] = z_mu
    outputs['zs_log_sigma_sq_enc'] = z_lss
    for k, v in out_enc.items():
        outputs[k + '_enc'] = v
    return outputs
