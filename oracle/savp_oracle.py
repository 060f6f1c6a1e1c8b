"""CPU ORACLE for the SAVP training hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product path (video_prediction_b200/) never does.

PARITY STATUS: "parity unpinned" by reference-owned golden vectors.  The reference
(alexlee-gk/video_prediction @ df43be59) ships NO tests and NO fixtures for this path and its
arithmetic lives in TensorFlow 1.x (requirements.txt:1, `tensorflow-gpu>=1.9.0`), which cannot
be installed or imported in this image.  This file restates the reference's Python line by line
and TF's published op semantics (SAME padding rule, cross-correlation, conv2d_transpose ==
conv dgrad, fused_batch_norm training-mode biased variance, TF1 Adam).  It is pinned by
  (i)  the reference's two docstring identities (ops.py:652-679, ops.py:799-817), and
  (ii) an independent second restatement (tests/test_oracle.py: direct-loop numpy versions of
       conv / transposed conv / CDNA / instance norm) plus fp64-vs-fp32 agreement.

Layout conventions follow the reference: activations NHWC / NDHWC, time-major [T,B,...] inside
the path, conv filters HWIO, conv2d_transpose filters [kh,kw,Cout,Cin].  Every function cites the
reference file:line it restates (paths relative to the reference's video_prediction/ package).

All randomness (weights, eps, prior z, scheduled-sampling mask, discriminator clip offsets) is an
explicit input so that the CUDA path and the oracle see identical numbers.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

RELU_SHIFT = 1e-12  # models/savp_model.py:18


# --------------------------------------------------------------------------------------------
# variable store (stands in for tf.get_variable + variable scopes)
# --------------------------------------------------------------------------------------------
def truncated_normal(rng: np.random.Generator, shape, stddev):
    """tf.truncated_normal_initializer: N(0, stddev) re-sampled outside 2 stddev."""
    x = rng.standard_normal(size=shape)
    bad = np.abs(x) > 2.0
    while bad.any():
        x[bad] = rng.standard_normal(size=int(bad.sum()))
        bad = np.abs(x) > 2.0
    return (x * stddev).astype(np.float64)


class Vars:
    """Get-or-create variable store.  `params` maps full TF-style names to tensors.

    If `rng` is given, missing variables are created with the reference's initializers
    (kernels: truncated normal sigma 0.02, ops.py:9/517/768, rnn_ops.py:120; biases zero; gamma 1,
    beta 0; spectral-norm u: truncated normal sigma 1, ops.py:1027)."""

    def __init__(self, params=None, rng=None, dtype=torch.float32):
        self.params = OrderedDict() if params is None else params
        self.rng = rng
        self.dtype = dtype
        self.trainable = OrderedDict()  # name -> bool

    def get(self, name, shape, init='kernel', trainable=True):
        if name not in self.params:
            if self.rng is None:
                raise KeyError('missing variable %s' % name)
            shape = tuple(int(s) for s in shape)
            if init == 'kernel':
                v = truncated_normal(self.rng, shape, 0.02)
            elif init == 'zeros':
                v = np.zeros(shape)
            elif init == 'ones':
                v = np.ones(shape)
            elif init == 'u':
                v = truncated_normal(self.rng, shape, 1.0)
            else:
                raise ValueError(init)
            self.params[name] = torch.tensor(v, dtype=self.dtype)
        self.trainable[name] = trainable
        p = self.params[name]
        assert tuple(p.shape) == tuple(shape), (name, tuple(p.shape), tuple(shape))
        return p


# --------------------------------------------------------------------------------------------
# TF op semantics
# --------------------------------------------------------------------------------------------
def same_pads(in_size, k, s):
    """TF SAME padding (ops.py:100-107 mirrors it): extra pad goes at the end."""
    out = -(-in_size // s)
    total = max((out - 1) * s + k - in_size, 0)
    return total // 2, total - total // 2


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


# ---- optional emulation of the CUDA path's tensor-core arithmetic --------------------------------
# The sm_90a engine feeds fp32 operands to the TF32 tensor-core MMAs, which read only the top 19 bits
# of each operand (sign, 8 exponent, 10 mantissa bits) and accumulate in fp32.  With
# `set_tf32_emulation('trunc')` every convolution of the oracle (forward AND its autograd backward:
# dgrad sees tf32(dy) x tf32(W), wgrad sees tf32(x) x tf32(dy)) quantises its operands the same way, so a
# difference between the CUDA path and this oracle that is NOT explained by operand rounding shows up
# at fp32-summation-order level.  Default None = the reference's plain fp32 arithmetic.
_TF32 = dict(mode=None, exempt=(), weight_mode='rna')


def set_tf32_emulation(mode, exempt=(), weight_mode='rna'):
    """mode: quantisation of the ACTIVATION-side operands (x in the forward, dy in dgrad, x and dy in wgrad), which the
    tensor core reads raw from fp32 memory: None | 'trunc' (drop the low 13 mantissa bits) | 'rna' (round to nearest,
    ties away).  weight_mode: quantisation of the filter operand of forward and dgrad -- the CUDA path rounds weights
    with cvt.rna.tf32.f32 when it packs them (csrc/pack.cu), independent of what the tensor core does.
    'bf16' (round to nearest even at 8 significant bits) is not a mode of the CUDA path: it is what kind::f16 operands would
    see, used by tests/measure_bf16_tolerance.py to show why the engine multiplies in TF32.
    exempt: iterable of substrings; a conv called with a `tag` containing one of them stays exact
    (layers the CUDA path runs on fp32 CUDA cores)."""
    assert mode in (None, 'trunc', 'rna', 'bf16') and weight_mode in ('trunc', 'rna', 'bf16')
    _TF32['mode'] = mode
    _TF32['exempt'] = tuple(exempt)
    _TF32['weight_mode'] = weight_mode


def tf32_quantize(x, mode=None):
    mode = mode or _TF32['mode']
    if mode is None:
        return x
    x32 = x.detach().to(torch.float32).contiguous()
    xi = x32.view(torch.int32)
    if mode == 'bf16':
        return x32.to(torch.bfloat16).to(torch.float32).to(x.dtype)
    if mode == 'rna':
        xi = (xi + 0x1000) & ~0x1FFF
    else:
        xi = xi & ~0x1FFF
    return xi.view(torch.float32).to(x.dtype)


class _QuantConv(torch.autograd.Function):
    """y = fn(q(x), q(w)); backward re-runs fn on the quantised operands with q(dy) as the cotangent."""

    @staticmethod
    def forward(ctx, x, w, fn):
        ctx.fn = fn
        ctx.save_for_backward(x, w)
        return fn(tf32_quantize(x), tf32_quantize(w, _TF32['weight_mode']))

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        with torch.enable_grad():
            xq = tf32_quantize(x).requires_grad_(True)
            wq = tf32_quantize(w, _TF32['weight_mode']).requires_grad_(True)   # dgrad reads the packed (rna) weights
            y = ctx.fn(xq, wq)
            dx, dw = torch.autograd.grad(y, (xq, wq), tf32_quantize(dy))
        return dx, dw, None


def _conv_op(fn, x, w, tag=''):
    if _TF32['mode'] is None or tag.startswith('exact:') or any(e in tag for e in _TF32['exempt']):
        return fn(x, w)
    return _QuantConv.apply(x, w, fn)


def conv2d_tf(x, kernel, strides=(1, 1), padding='SAME', bias=None, tag=''):
    """tf.nn.conv2d on NHWC input with HWIO filter (cross-correlation).  ops.py:494-550."""
    kh, kw = kernel.shape[:2]
    sh, sw = strides
    xn = _nchw(x)
    if padding == 'SAME':
        pt, pb = same_pads(x.shape[1], kh, sh)
        pl, pr = same_pads(x.shape[2], kw, sw)
        xn = F.pad(xn, (pl, pr, pt, pb))
    elif padding == 'FULL':
        xn = F.pad(xn, (kw - 1, kw - 1, kh - 1, kh - 1))
    elif padding != 'VALID':
        raise ValueError(padding)
    y = _conv_op(lambda a, k: F.conv2d(a, k.permute(3, 2, 0, 1), stride=(sh, sw)), xn, kernel, tag)
    y = _nhwc(y)
    if bias is not None:
        y = y + bias
    return y


def conv3d_tf_valid(x, kernel, strides, bias=None, tag=''):
    """tf.nn.conv3d VALID on NDHWC input with [kt,kh,kw,Cin,Cout] filter.  ops.py:764-777."""
    xn = x.permute(0, 4, 1, 2, 3)
    y = _conv_op(lambda a, k: F.conv3d(a, k.permute(4, 3, 0, 1, 2), stride=tuple(strides)), xn, kernel, tag)
    y = y.permute(0, 2, 3, 4, 1)
    if bias is not None:
        y = y + bias
    return y


def lrelu(x, alpha):
    """ops.py:895-903."""
    return torch.maximum(alpha * x, x)


def dense(x, kernel, bias=None):
    """ops.py:5-16."""
    y = x @ kernel
    if bias is not None:
        y = y + bias
    return y


def instance_norm(x, gamma, beta, eps=1e-6):
    """layers/normalization.py:34-196: per-(n,c) mean / biased variance over all spatial dims
    (fused_batch_norm training mode on the [1,HW,..,N*C] view, :146-170), eps 1e-6 (:37)."""
    dims = tuple(range(1, x.dim() - 1))
    mean = x.mean(dim=dims, keepdim=True)
    var = ((x - mean) ** 2).mean(dim=dims, keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) * gamma + beta


def pooled_kernel(kernel):
    """ops.py:838-842: avg-pool(2x2, stride 1, FULL zero padding) applied to the KERNEL."""
    kh, kw, ci, co = kernel.shape
    k = kernel.permute(2, 3, 0, 1).reshape(1, ci * co, kh, kw)
    k = F.avg_pool2d(F.pad(k, (1, 1, 1, 1)), 2, stride=1)
    return k.reshape(ci, co, kh + 1, kw + 1).permute(2, 3, 0, 1)


def conv_pool2d(x, kernel, bias):
    """ops.py:795-856 with strides=(2,2), SAME, avg pool."""
    return conv2d_tf(x, pooled_kernel(kernel), strides=(2, 2), padding='SAME', bias=bias)


def bilinear_kernel_2x():
    """ops.py:592-600 for strides (2,2): outer([.25,.75,.75,.25])."""
    s = np.array([2, 2])
    ks = 2 * s - s % 2
    center = s - (ks % 2 == 1) - 0.5 * (ks % 2 != 1)
    v = 1 - abs(np.arange(ks[0]) - center[0]) / s[0]
    h = 1 - abs(np.arange(ks[1]) - center[1]) / s[1]
    return v[:, None] * h[None, :]


def upsampled_kernel(kernel):
    """ops.py:698-704: FULL cross-correlation of the 4x4 bilinear kernel with the conv kernel.
    Returns kernel_up [6,6,Cout,Cin] (conv2d_transpose filter layout)."""
    kh, kw, ci, co = kernel.shape
    b2 = torch.tensor(bilinear_kernel_2x(), dtype=kernel.dtype, device=kernel.device)
    kt = kernel.permute(0, 1, 3, 2).reshape(kh, kw, 1, co * ci)       # kernel_reshaped
    up = conv2d_tf(b2[None, :, :, None], kt, padding='FULL', tag='exact:weight-prep')   # [1,6,6,co*ci]
    return up.reshape(up.shape[1], up.shape[2], co, ci)


def upsample_conv2d(x, kernel, bias):
    """ops.py:643-719 with strides=(2,2): conv2d_transpose(x, kernel_up, stride 2, SAME)+bias.
    conv2d_transpose == gradient of the stride-2 SAME conv (k=6 on 2H -> pad 2/2)."""
    kup = upsampled_kernel(kernel)                                     # [6,6,co,ci]
    y = _conv_op(lambda a, k: F.conv_transpose2d(a, k.permute(3, 2, 0, 1), stride=2, padding=2), _nchw(x), kup)
    return _nhwc(y) + bias


def tile_concat_z(h, z):
    """ops.tile_concat([h, z[:,None,None,:]], axis=-1)  (ops.py:968-1006)."""
    if z is None or z.shape[-1] == 0:
        return h
    zt = z[:, None, None, :].expand(h.shape[0], h.shape[1], h.shape[2], z.shape[-1])
    return torch.cat([h, zt], dim=-1)


def identity_kernel(kernel_size):
    """models/savp_model.py:968-980."""
    kh, kw = kernel_size
    k = np.zeros(kernel_size)

    def cs(n):
        return slice(n // 2 - 1, n // 2 + 1) if n % 2 == 0 else slice(n // 2, n // 2 + 1)
    k[cs(kh), cs(kw)] = 1.0
    return k / k.sum()


def apply_cdna_kernels(image, kernels):
    """models/savp_model.py:893-923.  image [B,H,W,C], kernels [B,kh,kw,K] ->
    list of K tensors [B,H,W,C]; SYMMETRIC pad (pad2d, ops.py:129-157) then per-sample
    cross-correlation applied identically to every colour channel."""
    b, h, w, c = image.shape
    _, kh, kw, nk = kernels.shape
    pt, pb = same_pads(h, kh, 1)
    pl, pr = same_pads(w, kw, 1)
    # SYMMETRIC == reflect including the edge pixel
    xp = image
    top = xp[:, :pt].flip(1)
    bot = xp[:, h - pb:].flip(1)
    xp = torch.cat([top, xp, bot], dim=1)
    left = xp[:, :, :pl].flip(2)
    right = xp[:, :, w - pr:].flip(2)
    xp = torch.cat([left, xp, right], dim=2)
    # channels-as-batch, batch-as-channel depthwise conv
    xin = xp.permute(3, 0, 1, 2)                                    # [C,B,Hp,Wp]
    wk = kernels.permute(0, 3, 1, 2).reshape(b * nk, 1, kh, kw)     # out ch = b*nk + k
    y = F.conv2d(xin, wk, groups=b)                                 # [C, B*K, H, W]
    y = y.reshape(c, b, nk, h, w).permute(2, 1, 3, 4, 0)            # [K,B,H,W,C]
    return list(y.unbind(0))


def image_warp(im, flow):
    """flow_ops.py:4-79: backward bilinear warp, indices clipped to the image."""
    b, h, w, c = im.shape
    fl = torch.floor(flow)
    wgt = flow - fl
    fx = fl[..., 0].long()
    fy = fl[..., 1].long()
    xw, yw = wgt[..., 0:1], wgt[..., 1:2]
    gx = torch.arange(w, device=im.device).view(1, 1, w).expand(b, h, w)
    gy = torch.arange(h, device=im.device).view(1, h, 1).expand(b, h, w)
    x0 = (gx + fx).clamp(0, w - 1)
    x1 = (gx + fx + 1).clamp(0, w - 1)
    y0 = (gy + fy).clamp(0, h - 1)
    y1 = (gy + fy + 1).clamp(0, h - 1)
    bi = torch.arange(b, device=im.device).view(b, 1, 1).expand(b, h, w)
    Ia, Ib, Ic, Id = im[bi, y0, x0], im[bi, y1, x0], im[bi, y0, x1], im[bi, y1, x1]
    return (1 - xw) * (1 - yw) * Ia + (1 - xw) * yw * Ib + xw * (1 - yw) * Ic + xw * yw * Id


def spectral_normed_weight(W, u):
    """ops.py:1020-1049, num_iters=1, differentiable through the iteration (no stop_gradient).
    Returns (W_bar, u_final)."""
    Wr = W.reshape(-1, W.shape[-1])

    def l2n(v, eps=1e-12):
        return v / (v.norm() + eps)
    v = l2n(u @ Wr.t())
    u1 = l2n(v @ Wr)
    sigma = (v @ Wr @ u1.t()).squeeze()
    return W / sigma, u1


# --------------------------------------------------------------------------------------------
# hparams (defaults: base_model.py:92-96, 363-399; savp_model.py:781-821)
# --------------------------------------------------------------------------------------------
DEFAULT_HPARAMS = dict(
    context_frames=-1, sequence_length=-1, repeat=1,
    batch_size=16, lr=0.001, end_lr=0.0, decay_steps=(200000, 300000), lr_boundaries=(0,),
    max_steps=300000, beta1=0.9, beta2=0.999, clip_length=10,
    l1_weight=1.0, l2_weight=0.0, vgg_cdist_weight=0.0, feature_l2_weight=0.0, ae_l2_weight=0.0,
    state_weight=0.0, tv_weight=0.0,
    image_sn_gan_weight=0.0, image_sn_vae_gan_weight=0.0,
    images_sn_gan_weight=0.0, images_sn_vae_gan_weight=0.0,
    video_sn_gan_weight=0.0, video_sn_vae_gan_weight=0.0,
    gan_feature_l2_weight=0.0, gan_feature_cdist_weight=0.0,
    vae_gan_feature_l2_weight=0.0, vae_gan_feature_cdist_weight=0.0,
    gan_loss_type='LSGAN', joint_gan_optimization=False,
    kl_weight=0.0, kl_anneal='linear', kl_anneal_k=-1.0, kl_anneal_steps=(50000, 100000),
    z_l1_weight=0.0,
    n_layers=3, ndf=32, norm_layer='instance', use_same_discriminator=False, ngf=32,
    downsample_layer='conv_pool2d', upsample_layer='upsample_conv2d', activation_layer='relu',
    transformation='cdna', kernel_size=(5, 5), dilation_rate=(1, 1), where_add='all',
    use_tile_concat=True, learn_initial_state=False, rnn='lstm', conv_rnn='lstm',
    conv_rnn_norm_layer='instance', num_transformed_images=4, last_frames=1,
    prev_image_background=True, first_image_background=True, last_image_background=False,
    last_context_image_background=False, context_images_background=False,
    generate_scratch_image=True, dependent_mask=True,
    schedule_sampling='inverse_sigmoid', schedule_sampling_k=900.0,
    schedule_sampling_steps=(0, 100000), use_e_rnn=False, learn_prior=False, nz=8, num_samples=8,
    nef=64, use_rnn_z=True, ablation_conv_rnn_norm=False, ablation_rnn=False,
)


class HP(dict):
    __getattr__ = dict.__getitem__


def make_hparams(**overrides):
    hp = HP(DEFAULT_HPARAMS)
    for k, v in overrides.items():
        if k not in hp:
            raise ValueError('unknown hparam %s' % k)
        hp[k] = v
    return hp


def layer_specs(hp, height, width):
    """models/savp_model.py:182-232."""
    s = min(height, width)
    g = hp.ngf
    if s >= 256:
        enc = [(g, False), (g * 2, False), (g * 4, True), (g * 8, True), (g * 8, True)]
        dec = [(g * 8, True), (g * 4, True), (g * 2, False), (g, False), (g, False)]
    elif s >= 128:
        enc = [(g, False), (g * 2, True), (g * 4, True), (g * 8, True)]
        dec = [(g * 8, True), (g * 4, True), (g * 2, False), (g, False)]
    elif s >= 64:
        enc = [(g, True), (g * 2, True), (g * 4, True)]
        dec = [(g * 2, True), (g, True), (g, False)]
    elif s >= 32:
        enc = [(g, True), (g * 2, True)]
        dec = [(g, True), (g, False)]
    else:
        raise NotImplementedError
    return enc, dec


# --------------------------------------------------------------------------------------------
# ConvLSTM cell, dense LSTM cell
# --------------------------------------------------------------------------------------------
def conv_lstm_cell(V, scope, inputs, state, filters):
    """rnn_ops.BasicConv2DLSTMCell.call (rnn_ops.py:137-171) with normalizer_fn=instance norm,
    separate_norms=False (savp_model.py:386-390), kernel 5x5, forget_bias 1."""
    c, h = state
    args = torch.cat([inputs, h], dim=-1)                                    # rnn_ops.py:143
    kernel = V.get(scope + '/kernel', (5, 5, args.shape[-1], 4 * filters))   # :118-120
    concat = conv2d_tf(args, kernel, padding='SAME')                         # :121 (no bias: normed)
    g1 = V.get(scope + '/input_transform_forget_output/gamma', (4 * filters,), 'ones')
    b1 = V.get(scope + '/input_transform_forget_output/beta', (4 * filters,), 'zeros')
    concat = instance_norm(concat, g1, b1)                                   # :148-149
    i, j, f, o = torch.split(concat, filters, dim=-1)                        # :150
    new_c = c * torch.sigmoid(f + 1.0) + torch.sigmoid(i) * torch.tanh(j)    # :157-162
    g2 = V.get(scope + '/state/gamma', (filters,), 'ones')
    b2 = V.get(scope + '/state/beta', (filters,), 'zeros')
    new_c = instance_norm(new_c, g2, b2)                                     # :163-164
    new_h = torch.tanh(new_c) * torch.sigmoid(o)                             # :165
    return new_h, (new_c, new_h)


def dense_lstm_cell(V, scope, x, state, units):
    """tf.nn.rnn_cell.LSTMCell(units, name='basic_lstm_cell') (savp_model.py:354-362):
    gates i,j,f,o from [x,h] @ kernel + bias; forget_bias 1; state (c,h)."""
    c, h = state
    kernel = V.get(scope + '/kernel', (x.shape[-1] + units, 4 * units))
    bias = V.get(scope + '/bias', (4 * units,), 'zeros')
    gates = torch.cat([x, h], dim=-1) @ kernel + bias
    i, j, f, o = torch.split(gates, units, dim=-1)
    new_c = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)
    new_h = torch.tanh(new_c) * torch.sigmoid(o)
    return new_h, (new_c, new_h)


# --------------------------------------------------------------------------------------------
# SAVPCell.call (savp_model.py:393-686) and the unroll (:689-696)
# --------------------------------------------------------------------------------------------
def savp_cell_step(V, hp, scope, t, inp, first_image, states, ground_truth_t, tap=None):
    """One timestep.  inp: dict images[B,H,W,C], optional actions[B,A], zs[B,nz].
    ground_truth_t: bool[B].  Default hparams only (cdna, instance norm, tile-concat 'all')."""
    B, H, W, C = inp['images'].shape
    enc_specs, dec_specs = layer_specs(hp, H, W)
    gt = ground_truth_t.view(B, 1, 1, 1)
    image = torch.where(gt, inp['images'], states['gen_image'])              # :406
    # state_action_z (:414-444)
    saz = []
    if 'actions' in inp:
        saz.append(inp['actions'])
    new_states = dict(states)
    if 'zs' in inp:
        if hp.use_rnn_z:                                                     # :424-432
            rnn_z, rz_state = dense_lstm_cell(V, scope + '/lstm_z/basic_lstm_cell', inp['zs'],
                                              states['rnn_z_state'], hp.nz)
            new_states['rnn_z_state'] = rz_state
            saz.append(rnn_z)
        else:
            saz.append(inp['zs'])
    saz = torch.cat(saz, dim=-1) if saz else None

    layers = []
    new_rnn = []
    rnn_states = states['conv_rnn_states']
    for i, (oc, use_rnn) in enumerate(enc_specs):                            # :448-483
        if i == 0:
            h = torch.cat([image, first_image], dim=-1)                      # :451
            ks = 5
        else:
            h = layers[-1][-1]
            ks = 3
        h = tile_concat_z(h, saz)                                            # :456-458
        kin = h.shape[-1]
        k = V.get('%s/h%d/conv_pool2d/kernel' % (scope, i), (ks, ks, kin, oc))
        b = V.get('%s/h%d/conv_pool2d/bias' % (scope, i), (oc,), 'zeros')
        h = conv_pool2d(h, k, b)                                             # :461-462
        g = V.get('%s/h%d/InstanceNorm/gamma' % (scope, i), (oc,), 'ones')
        be = V.get('%s/h%d/InstanceNorm/beta' % (scope, i), (oc,), 'zeros')
        h = torch.relu(instance_norm(h, g, be))                              # :463-464
        if use_rnn:
            rh = tile_concat_z(h, saz)                                       # :467-469
            rh, st = conv_lstm_cell(V, '%s/lstm_h%d/basic_conv2dlstm_cell' % (scope, i), rh,
                                    rnn_states[len(new_rnn)], oc)            # :480-482
            new_rnn.append(st)
            layers.append((h, rh))
        else:
            layers.append((h,))
    n_enc = len(layers)
    for i, (oc, use_rnn) in enumerate(dec_specs):                            # :486-518
        li = len(layers)
        if i == 0:
            h = layers[-1][-1]
        else:
            h = torch.cat([layers[-1][-1], layers[n_enc - i - 1][-1]], dim=-1)   # :491
        h = tile_concat_z(h, saz)
        kin = h.shape[-1]
        k = V.get('%s/h%d/upsample_conv2d/kernel' % (scope, li), (3, 3, kin, oc))
        b = V.get('%s/h%d/upsample_conv2d/bias' % (scope, li), (oc,), 'zeros')
        h = upsample_conv2d(h, k, b)                                         # :497-498
        g = V.get('%s/h%d/InstanceNorm/gamma' % (scope, li), (oc,), 'ones')
        be = V.get('%s/h%d/InstanceNorm/beta' % (scope, li), (oc,), 'zeros')
        h = torch.relu(instance_norm(h, g, be))
        if use_rnn:
            rh = tile_concat_z(h, saz)
            rh, st = conv_lstm_cell(V, '%s/lstm_h%d/basic_conv2dlstm_cell' % (scope, li), rh,
                                    rnn_states[len(new_rnn)], oc)
            new_rnn.append(st)
            layers.append((h, rh))
        else:
            layers.append((h,))
    assert len(new_rnn) == len(rnn_states)                                   # :519
    nl = len(layers)
    top = layers[-1][-1]

    def conv3x3(name, x, oc):
        k = V.get('%s/%s/conv2d/kernel' % (scope, name), (3, 3, x.shape[-1], oc))
        b = V.get('%s/%s/conv2d/bias' % (scope, name), (oc,), 'zeros')
        return conv2d_tf(x, k, padding='SAME', bias=b)

    def norm_relu(name, x):
        g = V.get('%s/%s/InstanceNorm/gamma' % (scope, name), (x.shape[-1],), 'ones')
        be = V.get('%s/%s/InstanceNorm/beta' % (scope, name), (x.shape[-1],), 'zeros')
        return torch.relu(instance_norm(x, g, be))

    kh, kw = hp.kernel_size
    nk = hp.last_frames * hp.num_transformed_images
    kernels = flows = None
    if hp.transformation == 'flow':
        # flow heads (:522-530): flows [B,H,W,2*nk] reshaped to [B,H,W,2,nk] -> flow k = channels (k, nk + k)
        h_flow = norm_relu('h%d_flow' % nl, conv3x3('h%d_flow' % nl, top, hp.ngf))
        flows = conv3x3('flows', h_flow, 2 * nk).reshape(B, H, W, 2, nk)
    elif hp.transformation == 'cdna':
        # cdna kernels (:546-559)
        smallest = layers[n_enc - 1][-1]
        flat = smallest.reshape(B, -1)
        dk = V.get(scope + '/cdna_kernels/dense/kernel', (flat.shape[1], kh * kw * nk))
        db = V.get(scope + '/cdna_kernels/dense/bias', (kh * kw * nk,), 'zeros')
        kernels = dense(flat, dk, db).reshape(B, kh, kw, nk)
        kernels = kernels + torch.tensor(identity_kernel((kh, kw)), dtype=kernels.dtype, device=kernels.device)[None, :, :, None]
        kernels = torch.relu(kernels - RELU_SHIFT) + RELU_SHIFT                  # :558
        kernels = kernels / kernels.sum(dim=(1, 2), keepdim=True)                # :559
    else:
        raise ValueError('Invalid transformation %s' % hp.transformation)    # :545

    # scratch image (:561-572)
    h_scratch = norm_relu('h%d_scratch' % nl, conv3x3('h%d_scratch' % nl, top, hp.ngf))
    scratch = torch.sigmoid(conv3x3('scratch_image', h_scratch, C))
    # transformed images (:574-596): 4 CDNA, prev image, first image, scratch
    if flows is not None:
        warped = [image_warp(image, flows[..., k]) for k in range(nk)]       # apply_flows (:955-965)
    else:
        warped = apply_cdna_kernels(image, kernels)
    transformed = warped + [image, first_image, scratch]
    # masks (:623-635)
    h_masks = norm_relu('h%d_masks' % nl, conv3x3('h%d_masks' % nl, top, hp.ngf))
    h_masks = torch.cat([h_masks] + transformed, dim=-1)                     # :632 dependent_mask
    mask_logits = conv3x3('masks', h_masks, len(transformed))
    masks = torch.softmax(mask_logits, dim=-1)                               # :634
    gen_image = sum(tr * masks[..., k:k + 1] for k, tr in enumerate(transformed))   # :645-646
    if tap is not None:
        tap.update(dict(image=image, kernels=kernels, scratch=scratch, mask_logits=mask_logits,
                        layers=layers, rnn_z=saz))
    new_states.update(gen_image=gen_image, conv_rnn_states=new_rnn)
    outputs = dict(gen_images=gen_image,
                   transformed_images=torch.stack(transformed, dim=-1),
                   masks=torch.stack([masks[..., k:k + 1] for k in range(masks.shape[-1])], dim=-1))
    return outputs, new_states


def generator_given_z(V, hp, inputs, ground_truth, scope='generator/rnn/savp_cell', taps=None):
    """generator_given_z_fn (savp_model.py:689-696) + zero_state (:344-352).
    inputs: images[T,B,H,W,C] (+actions[T-1,B,A], zs[T-1,B,nz]); ground_truth bool[T-1,B]."""
    images = inputs['images']
    T = hp.sequence_length
    B, H, W, C = images.shape[1:]
    enc_specs, dec_specs = layer_specs(hp, H, W)
    dt = images.dtype
    rnn_states = []
    hh, ww = H, W
    for oc, use in enc_specs:
        hh //= 2
        ww //= 2
        if use:
            rnn_states.append((torch.zeros(B, hh, ww, oc, dtype=dt), torch.zeros(B, hh, ww, oc, dtype=dt)))
    for oc, use in dec_specs:
        hh *= 2
        ww *= 2
        if use:
            rnn_states.append((torch.zeros(B, hh, ww, oc, dtype=dt), torch.zeros(B, hh, ww, oc, dtype=dt)))
    states = dict(gen_image=torch.zeros(B, H, W, C, dtype=dt), conv_rnn_states=rnn_states)
    if 'zs' in inputs and hp.use_rnn_z:
        states['rnn_z_state'] = (torch.zeros(B, hp.nz, dtype=dt), torch.zeros(B, hp.nz, dtype=dt))
    outs = []
    for t in range(T - 1):                                                   # maybe_pad_or_slice to T-1
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


def ground_truth_mask(hp, batch, sampling=None):
    """savp_model.py:309-334: context frames always ground truth; afterwards `sampling`
    (bool [T-1-context, B], explicit input) or all-False (mode != 'train' / schedule 'none')."""
    n = hp.sequence_length - 1 - hp.context_frames
    ctx = torch.ones(hp.context_frames, batch, dtype=torch.bool)
    rest = torch.zeros(n, batch, dtype=torch.bool) if sampling is None else sampling.bool()
    return torch.cat([ctx, rest], dim=0)


# --------------------------------------------------------------------------------------------
# posterior encoder (savp_model.py:21-51, networks.py:12-32)
# --------------------------------------------------------------------------------------------
def encoder_net(V, scope, x, nef, n_layers):
    """networks.encoder: x [N,H,W,Cin] -> [N, nef*4]."""
    def conv(name, x, oc):
        k = V.get('%s/%s/conv2d/kernel' % (scope, name), (4, 4, x.shape[-1], oc))
        b = V.get('%s/%s/conv2d/bias' % (scope, name), (oc,), 'zeros')
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))                                    # networks.py:15,18
        return conv2d_tf(xp, k, strides=(2, 2), padding='VALID', bias=b)
    h = lrelu(conv('layer_1', x, nef), 0.2)
    for i in range(1, n_layers):
        name = 'layer_%d' % (i + 1)
        oc = nef * min(2 ** i, 4)
        c = conv(name, h, oc)
        g = V.get('%s/%s/InstanceNorm/gamma' % (scope, name), (oc,), 'ones')
        be = V.get('%s/%s/InstanceNorm/beta' % (scope, name), (oc,), 'zeros')
        h = lrelu(instance_norm(c, g, be), 0.2)
    return h.mean(dim=(1, 2))                                                # networks.py:30-31


def posterior(V, hp, inputs, scope='generator/encoder'):
    images = inputs['images']
    T, B = images.shape[:2]
    pairs = torch.cat([images[:-1], images[1:]], dim=-1)                     # savp_model.py:23
    if 'actions' in inputs:
        a = inputs['actions'][:T - 1, :, None, None, :].expand(T - 1, B, images.shape[2], images.shape[3], -1)
        pairs = torch.cat([pairs, a], dim=-1)                                # :24-26
    flat = pairs.reshape((-1,) + tuple(pairs.shape[2:]))
    h = encoder_net(V, scope, flat, hp.nef, hp.n_layers)
    mk = V.get(scope + '/z_mu/dense/kernel', (h.shape[-1], hp.nz))
    mb = V.get(scope + '/z_mu/dense/bias', (hp.nz,), 'zeros')
    sk = V.get(scope + '/z_log_sigma_sq/dense/kernel', (h.shape[-1], hp.nz))
    sb = V.get(scope + '/z_log_sigma_sq/dense/bias', (hp.nz,), 'zeros')
    z_mu = dense(h, mk, mb).reshape(T - 1, B, hp.nz)
    z_lss = dense(h, sk, sb).clamp(-10, 10).reshape(T - 1, B, hp.nz)         # :49
    return z_mu, z_lss


def generator(V, hp, inputs, noise, ground_truth, taps=None):
    """generator_fn (savp_model.py:699-768), without the visualisation-only samples unroll.
    noise: dict eps[T-1,B,nz], z_prior[T-context,B,nz] (only if nz>0)."""
    if hp.nz == 0:
        return generator_given_z(V, hp, inputs, ground_truth, taps=taps)
    z_mu, z_lss = posterior(V, hp, inputs)
    zs_post = z_mu + torch.sqrt(torch.exp(z_lss)) * noise['eps']             # :712
    zs_prior = torch.cat([zs_post[:hp.context_frames - 1], noise['z_prior']], dim=0)   # :724-725
    ip = dict(inputs)
    ip['zs'] = zs_post
    out_enc = generator_given_z(V, hp, ip, ground_truth)                     # :730
    ip = dict(inputs)
    ip['zs'] = zs_prior
    out = generator_given_z(V, hp, ip, ground_truth, taps=taps)              # :732
    outputs = OrderedDict(out)
    outputs['zs_mu_enc'] = z_mu
    outputs['zs_log_sigma_sq_enc'] = z_lss
    for k, v in out_enc.items():
        outputs[k + '_enc'] = v
    return outputs


# --------------------------------------------------------------------------------------------
# discriminator (savp_model.py:88-166, networks.py:72-108)
# --------------------------------------------------------------------------------------------
VIDEO_D_LAYERS = [  # (name, out mult of ndf, kernel, strides)   networks.py:83-102
    ('sn_conv0_0', 1, 3, (1, 1, 1)), ('sn_conv0_1', 2, 4, (1, 2, 2)),
    ('sn_conv1_0', 2, 3, (1, 1, 1)), ('sn_conv1_1', 4, 4, (1, 2, 2)),
    ('sn_conv2_0', 4, 3, (1, 1, 1)), ('sn_conv2_1', 8, 4, (2, 2, 2)),
    ('sn_conv3_0', 8, 3, (1, 1, 1)),
]


def video_sn_discriminator(V, scope, clips, ndf, u_out=None):
    """networks.video_sn_discriminator.  clips time-major [T,B,H,W,C]; returns 7 feature maps
    [B,T',H',W',C'] (batch-major here; the reference transposes back to time-major, :107, which
    does not change any loss) and logits [B,1]."""
    x = clips.permute(1, 0, 2, 3, 4)
    feats = []
    for name, mult, k, strides in VIDEO_D_LAYERS:
        oc = ndf * mult
        W = V.get('%s/%s/conv3d/kernel' % (scope, name), (k, k, k, x.shape[-1], oc))
        u = V.get('%s/%s/conv3d/u' % (scope, name), (1, oc), 'u', trainable=False)
        b = V.get('%s/%s/conv3d/bias' % (scope, name), (oc,), 'zeros')
        Wb, u1 = spectral_normed_weight(W, u)
        if u_out is not None:
            u_out['%s/%s/conv3d/u' % (scope, name)] = u1.detach()
        xp = F.pad(x, (0, 0, 1, 1, 1, 1, 1, 1))                              # networks.py:76-81
        x = lrelu(conv3d_tf_valid(xp, Wb, strides, b, tag='%s/%s' % (scope, name)), 0.1)
        feats.append(x)
    flat = x.reshape(x.shape[0], -1)
    W = V.get('%s/sn_fc4/dense/kernel' % scope, (flat.shape[1], 1))
    u = V.get('%s/sn_fc4/dense/u' % scope, (1, 1), 'u', trainable=False)
    b = V.get('%s/sn_fc4/dense/bias' % scope, (1,), 'zeros')
    Wb, u1 = spectral_normed_weight(W, u)
    if u_out is not None:
        u_out['%s/sn_fc4/dense/u' % scope] = u1.detach()
    logits = dense(flat, Wb, b)
    return feats, logits


IMAGE_D_LAYERS = [  # networks.py:45-63
    ('sn_conv0_0', 1, 3, (1, 1)), ('sn_conv0_1', 2, 4, (2, 2)), ('sn_conv1_0', 2, 3, (1, 1)), ('sn_conv1_1', 4, 4, (2, 2)),
    ('sn_conv2_0', 4, 3, (1, 1)), ('sn_conv2_1', 8, 4, (2, 2)), ('sn_conv3_0', 8, 3, (1, 1)),
]


def image_sn_discriminator(V, scope, images, ndf, u_out=None):
    """networks.image_sn_discriminator (networks.py:35-69): images [B,H,W,C] -> 7 feature maps + logits [B,1]."""
    x = images
    feats = []
    for name, mult, k, strides in IMAGE_D_LAYERS:
        oc = ndf * mult
        W = V.get('%s/%s/conv2d/kernel' % (scope, name), (k, k, x.shape[-1], oc))
        u = V.get('%s/%s/conv2d/u' % (scope, name), (1, oc), 'u', trainable=False)
        b = V.get('%s/%s/conv2d/bias' % (scope, name), (oc,), 'zeros')
        Wb, u1 = spectral_normed_weight(W, u)
        if u_out is not None:
            u_out['%s/%s/conv2d/u' % (scope, name)] = u1.detach()
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))                                    # networks.py:38-43
        x = lrelu(conv2d_tf(xp, Wb, strides=strides, padding='VALID', bias=b, tag='%s/%s' % (scope, name)), 0.1)
        feats.append(x)
    flat = x.reshape(x.shape[0], -1)
    W = V.get('%s/sn_fc4/dense/kernel' % scope, (flat.shape[1], 1))
    u = V.get('%s/sn_fc4/dense/u' % scope, (1, 1), 'u', trainable=False)
    b = V.get('%s/sn_fc4/dense/bias' % scope, (1,), 'zeros')
    Wb, u1 = spectral_normed_weight(W, u)
    if u_out is not None:
        u_out['%s/sn_fc4/dense/u' % scope] = u1.detach()
    return feats, dense(flat, Wb, b)


def gather_clip(targets, t_start, clip_length):
    """savp_model.py:97-102: per-sample clip of clip_length frames starting at t_start[b]."""
    T, B = targets.shape[:2]
    idx = t_start.view(1, B) + torch.arange(clip_length).view(-1, 1)         # [clip,B]
    return targets[idx, torch.arange(B).view(1, B)]


def discriminator(V, hp, inputs, gen_outputs, t_starts, u_out=None):
    """discriminator_fn / discriminator_given_video_fn (savp_model.py:88-166): image_sn (one sampled frame per video) and
    video_sn (a clip) discriminators; the per-frame `images_sn` variant is not restated.  t_starts: dict with int64[B]
    entries 'real','fake' (+ 'enc_real','enc_fake' if nz>0) = clip offsets, and 'image_real', ... = sampled frame indices."""
    out = OrderedDict()
    real = inputs['images'][1:]
    has_image = bool(hp.image_sn_gan_weight or hp.image_sn_vae_gan_weight)
    has_video = bool(hp.video_sn_gan_weight or hp.video_sn_vae_gan_weight)

    def run(prefix, video, key, suffix):
        if has_image:
            B = video.shape[1]
            frame = video[t_starts['image_' + key], torch.arange(B)]             # savp_model.py:93-94
            feats, logits = image_sn_discriminator(V, prefix + '/image', frame, hp.ndf, u_out)
            out['discrim_image_sn_logits' + suffix] = logits
            for i, f in enumerate(feats):
                out['discrim_image_sn_feature%d%s' % (i, suffix)] = f
        if has_video:
            clip = gather_clip(video, t_starts[key], hp.clip_length)
            feats, logits = video_sn_discriminator(V, prefix + '/video', clip, hp.ndf, u_out)
            out['discrim_video_sn_logits' + suffix] = logits
            for i, f in enumerate(feats):
                out['discrim_video_sn_feature%d%s' % (i, suffix)] = f
    if not (has_image or has_video):
        return out
    if hp.nz:
        run('discriminator/encoder', real, 'enc_real', '_enc_real')
        run('discriminator/encoder', gen_outputs['gen_images_enc'], 'enc_fake', '_enc_fake')
    run('discriminator', real, 'real', '_real')
    run('discriminator', gen_outputs['gen_images'], 'fake', '_fake')
    return out


# --------------------------------------------------------------------------------------------
# losses (losses.py:6-67; base_model.py:733-852) and schedules (base_model.py:286-319)
# --------------------------------------------------------------------------------------------
def l1_loss(pred, target):
    return (target - pred).abs().mean()


def l2_loss(pred, target):
    return ((target - pred) ** 2).mean()


def cosine_distance(a, b):
    def nrm(t):
        return t / (t.norm(dim=-1, keepdim=True) + 1e-10)
    return ((nrm(a) - nrm(b)) ** 2).sum(dim=-1).mean() / 2.0


def gan_loss(logits, label, kind):
    if kind == 'LSGAN':
        return ((logits - label) ** 2).mean()
    if kind == 'GAN':
        return F.binary_cross_entropy_with_logits(logits, torch.full_like(logits, label))
    if kind == 'SNGAN':
        return F.softplus(logits).mean() if label == 0.0 else F.softplus(-logits).mean()
    raise ValueError(kind)


def kl_loss(mu, lss):
    return -0.5 * (1 + lss - mu ** 2 - torch.exp(lss)).sum(dim=-1).mean()


def learning_rate(hp, step):
    if any(hp.lr_boundaries):
        vals = hp.lr * 0.1 ** np.arange(len(hp.lr_boundaries) + 1)
        return float(vals[int(np.searchsorted(np.array(hp.lr_boundaries), step, side='right'))])
    if any(hp.decay_steps):
        s0, s1 = hp.decay_steps
        if s0 == s1:
            sched = 0.0 if step < s0 else 1.0
        else:
            sched = (min(max(step, s0), s1) - s0) / float(s1 - s0)
        return hp.lr + (hp.end_lr - hp.lr) * sched
    return hp.lr


def kl_weight(hp, step):
    if not hp.kl_weight:
        return None
    if hp.kl_anneal == 'none':
        return hp.kl_weight
    if hp.kl_anneal == 'sigmoid':
        k = hp.kl_anneal_k
        return hp.kl_weight / (1 + k * math.exp(-step / k))
    if hp.kl_anneal == 'linear':
        s0, s1 = hp.kl_anneal_steps
        return hp.kl_weight * (min(max(step, s0), s1) - s0) / float(s1 - s0)
    raise NotImplementedError


def generator_losses(hp, inputs, outputs, step):
    """base_model.py:733-829 (terms used by the shipped hparams)."""
    L = OrderedDict()
    gen = outputs.get('gen_images_enc', outputs['gen_images'])
    target = inputs['images'][1:]
    if hp.l1_weight:
        L['gen_l1_loss'] = (l1_loss(gen, target), hp.l1_weight)
    if hp.l2_weight:
        L['gen_l2_loss'] = (l2_loss(gen, target), hp.l2_weight)
    for infix, w_gan, w_vae in (('_image_sn', hp.image_sn_gan_weight, hp.image_sn_vae_gan_weight),
                                ('_video_sn', hp.video_sn_gan_weight, hp.video_sn_vae_gan_weight)):
        if w_gan:
            L['gen%s_gan_loss' % infix] = (gan_loss(outputs['discrim%s_logits_fake' % infix], 1.0, hp.gan_loss_type), w_gan)
            if hp.gan_feature_cdist_weight:
                sm = sum(cosine_distance(outputs['discrim%s_feature%d_fake' % (infix, i)],
                                         outputs['discrim%s_feature%d_real' % (infix, i)]) for i in range(7))
                L['gen%s_gan_feature_cdist_loss' % infix] = (sm, hp.gan_feature_cdist_weight)
        if w_vae and hp.nz:
            L['gen%s_vae_gan_loss' % infix] = (gan_loss(outputs['discrim%s_logits_enc_fake' % infix], 1.0, hp.gan_loss_type), w_vae)
            if hp.vae_gan_feature_cdist_weight:
                sm = sum(cosine_distance(outputs['discrim%s_feature%d_enc_fake' % (infix, i)],
                                         outputs['discrim%s_feature%d_enc_real' % (infix, i)]) for i in range(7))
                L['gen%s_vae_gan_feature_cdist_loss' % infix] = (sm, hp.vae_gan_feature_cdist_weight)
    if hp.kl_weight:
        L['gen_kl_loss'] = (kl_loss(outputs['zs_mu_enc'], outputs['zs_log_sigma_sq_enc']), kl_weight(hp, step))
    return L


def discriminator_losses(hp, outputs):
    """base_model.py:831-852."""
    L = OrderedDict()
    t = hp.gan_loss_type
    for infix, w_gan, w_vae in (('_image_sn', hp.image_sn_gan_weight, hp.image_sn_vae_gan_weight),
                                ('_video_sn', hp.video_sn_gan_weight, hp.video_sn_vae_gan_weight)):
        if w_gan:
            L['discrim%s_gan_loss' % infix] = (gan_loss(outputs['discrim%s_logits_real' % infix], 1.0, t) +
                                               gan_loss(outputs['discrim%s_logits_fake' % infix], 0.0, t), w_gan)
        if w_vae and hp.nz:
            L['discrim%s_vae_gan_loss' % infix] = (gan_loss(outputs['discrim%s_logits_enc_real' % infix], 1.0, t) +
                                                   gan_loss(outputs['discrim%s_logits_enc_fake' % infix], 0.0, t), w_vae)
    return L


def total_loss(L):
    return sum(l * w for l, w in L.values()) if L else torch.zeros(())


def adam_tf(p, g, m, v, lr, b1, b2, t, eps=1e-8):
    """tf.train.AdamOptimizer update (epsilon-hat form), t = 1-based step count."""
    lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    return p - lr_t * m / (torch.sqrt(v) + eps), m, v


# --------------------------------------------------------------------------------------------
# one full training step (base_model.py:402-516: tower_fn + single-GPU build_graph)
# --------------------------------------------------------------------------------------------
def train_step(params, opt, hp, inputs, noise, step, sampling=None):
    """params: OrderedDict name->tensor (leaf, no grad).  opt: dict with 'm','v' dicts and 't'.
    noise: eps, z_prior, and t_start dicts 'd_pre' / 'd_post' (clip offsets for the two
    discriminator_fn instantiations, base_model.py:414-419).
    Order (non-joint): u <- u' ; D loss -> D grads -> Adam(D); D forward again with updated D
    weights -> g_loss_post -> G grads -> Adam(G).  Spectral-norm u: every forward of this step
    reads the start-of-step u; u' is stored at the end (UPDATE_OPS, ops.py:1046-1048).
    Returns dict with losses, grads, new params/opt state, outputs."""
    dt = next(iter(params.values())).dtype
    P = OrderedDict((k, v.clone().requires_grad_(True)) for k, v in params.items())
    V = Vars(P, None, dt)
    B = inputs['images'].shape[1]
    gt = ground_truth_mask(hp, B, sampling)
    gen_out = generator(V, hp, inputs, noise, gt)
    g_names = [k for k in P if k.startswith('generator/')]
    d_names = [k for k in P if k.startswith('discriminator/') and not k.endswith('/u')]
    res = dict(outputs=gen_out)
    lr = learning_rate(hp, step)
    t = opt['t'] + 1
    newp = OrderedDict((k, v.detach()) for k, v in P.items())
    has_d = bool(hp.video_sn_gan_weight or hp.video_sn_vae_gan_weight or hp.image_sn_gan_weight or hp.image_sn_vae_gan_weight)
    u_new = {}
    if has_d:
        gen_det = {k: v.detach() for k, v in gen_out.items()}
        d_out = discriminator(V, hp, inputs, gen_det, noise['d_pre'], u_new)
        d_losses = discriminator_losses(hp, d_out)
        d_loss = total_loss(d_losses)
        d_grads = torch.autograd.grad(d_loss, [P[k] for k in d_names], allow_unused=True)
        res.update(d_losses={k: float(l.detach()) for k, (l, w) in d_losses.items()}, d_loss=float(d_loss.detach()),
                   d_grads=OrderedDict(zip(d_names, d_grads)), d_outputs=d_out)
        for k, g in zip(d_names, d_grads):
            if g is None:
                continue
            newp[k], opt['m'][k], opt['v'][k] = adam_tf(newp[k], g, opt['m'][k], opt['v'][k], lr,
                                                        hp.beta1, hp.beta2, t)
        # post-update discriminator forward (fresh variable reads, tf_utils.replace_read_ops)
        P2 = OrderedDict(P)
        for k in d_names:
            P2[k] = newp[k]
        V2 = Vars(P2, None, dt)
        d_post = discriminator(V2, hp, inputs, gen_out, noise['d_post'])
        allout = OrderedDict(gen_out)
        allout.update(d_post)
    else:
        allout = gen_out
    g_losses = generator_losses(hp, inputs, allout, step)
    g_loss = total_loss(g_losses)
    g_grads = torch.autograd.grad(g_loss, [P[k] for k in g_names], allow_unused=True)
    for k, g in zip(g_names, g_grads):
        if g is None:
            continue
        newp[k], opt['m'][k], opt['v'][k] = adam_tf(newp[k], g, opt['m'][k], opt['v'][k], lr,
                                                    hp.beta1, hp.beta2, t)
    for k, u in u_new.items():
        newp[k] = u
    opt['t'] = t
    res.update(g_losses={k: float(l.detach()) for k, (l, w) in g_losses.items()}, g_loss=float(g_loss.detach()),
               g_grads=OrderedDict(zip(g_names, g_grads)), params=newp, lr=lr)
    return res


def init_params(hp, image_shape, batch=1, action_dim=0, seed=0, dtype=torch.float32):
    """Create every variable of the path with the reference's initializers by tracing one tiny
    forward (the tf.get_variable creation order), returning OrderedDict name -> tensor."""
    rng = np.random.default_rng(seed)
    V = Vars(None, rng, dtype)
    T = hp.sequence_length
    H, W, C = image_shape
    inputs = dict(images=torch.zeros(T, batch, H, W, C, dtype=dtype))
    if action_dim:
        inputs['actions'] = torch.zeros(T - 1, batch, action_dim, dtype=dtype)
    noise = dict(eps=torch.zeros(T - 1, batch, hp.nz, dtype=dtype),
                 z_prior=torch.zeros(T - hp.context_frames, batch, hp.nz, dtype=dtype))
    with torch.no_grad():
        saved = hp.sequence_length
        gt = ground_truth_mask(hp, batch)
        out = generator(V, hp, inputs, noise, gt)
        if hp.video_sn_gan_weight or hp.video_sn_vae_gan_weight or hp.image_sn_gan_weight or hp.image_sn_vae_gan_weight:
            z = torch.zeros(batch, dtype=torch.long)
            discriminator(V, hp, inputs, out, dict(real=z, fake=z, enc_real=z, enc_fake=z, image_real=z, image_fake=z,
                                                   image_enc_real=z, image_enc_fake=z))
        assert hp.sequence_length == saved
    return V.params, V.trainable


def make_synthetic_inputs(hp, batch, image_shape, action_dim=0, seed=0, dtype=torch.float32,
                          smooth=True):
    """SURVEY 8(d) synthetic inputs: moving-blob videos in [0,1] (smooth=True) or U[0,1)."""
    rng = np.random.default_rng(seed + 1000)
    T = hp.sequence_length
    H, W, C = image_shape
    if smooth:
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
        imgs = np.zeros((T, batch, H, W, C))
        for b in range(batch):
            for blob in range(3):
                cx, cy = rng.uniform(0.2, 0.8, 2) * (W, H)
                vx, vy = rng.uniform(-2.0, 2.0, 2)
                rad = rng.uniform(0.08, 0.2) * min(H, W)
                col = rng.uniform(0.2, 1.0, C)
                for t in range(T):
                    d2 = (xx - (cx + vx * t)) ** 2 + (yy - (cy + vy * t)) ** 2
                    imgs[t, b] += np.exp(-d2 / (2 * rad * rad))[..., None] * col
        imgs = np.clip(imgs * 0.6 + 0.1 * rng.uniform(size=imgs.shape), 0, 1)
    else:
        imgs = rng.uniform(size=(T, batch, H, W, C))
    inputs = dict(images=torch.tensor(imgs, dtype=dtype))
    if action_dim:
        inputs['actions'] = torch.tensor(rng.standard_normal((T - 1, batch, action_dim)), dtype=dtype)
    noise = dict(
        eps=torch.tensor(rng.standard_normal((T - 1, batch, max(hp.nz, 1)))[..., :hp.nz], dtype=dtype),
        z_prior=torch.tensor(rng.standard_normal((T - hp.context_frames, batch, max(hp.nz, 1)))[..., :hp.nz], dtype=dtype))
    hi = T - 1 - hp.clip_length + 1
    if hi >= 1:
        for which in ('d_pre', 'd_post'):
            noise[which] = {k: torch.tensor(rng.integers(0, hi, size=batch), dtype=torch.long)
                            for k in ('real', 'fake', 'enc_real', 'enc_fake')}
        for which in ('d_pre', 'd_post'):      # t_sample of the image discriminators (drawn after, so earlier fixtures keep their values)
            noise[which].update({'image_' + k: torch.tensor(rng.integers(0, T - 1, size=batch), dtype=torch.long)
                                 for k in ('real', 'fake', 'enc_real', 'enc_fake')})
    return inputs, noise
