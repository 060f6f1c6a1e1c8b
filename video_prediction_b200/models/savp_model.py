"""SAVP model on H100: host-side orchestration of the sm_90a kernels in libvp_b200.so.

Mirrors `SAVPVideoPredictionModel` of the reference (video_prediction/models/savp_model.py:771-855):
same constructor, same default hparams (:779-822), same deprecated-key handling (:824-846), same
`build_graph(inputs)` entry and `outputs['gen_images']` (batch-major [B,T-1,H,W,C]).

What differs is everything below that surface: there is no TF graph.  `build_graph` lays the whole
unroll out in HBM as time-stacked channels-last buffers ([T-1, NB, H, W, C']) whose channel layout
*is* the concatenation each convolution reads (image | first image | z), (features | z | h_prev),
(features | skip | z): producers write straight into their consumers' slices, `tile_concat` is a
broadcast store, and the posterior and prior unrolls (savp_model.py:730-732, shared weights) run as
one batch NB = 2B.  All FLOP-carrying ops are tensor-core implicit GEMMs (csrc/igemm.cu); the rest are
HBM-bound kernels (csrc/elementwise.cu).  PyTorch only owns memory and streams.
"""
from __future__ import annotations

import itertools
import os
from collections import OrderedDict

import numpy as np
import torch

from .. import dp
from .. import lib as L
from .base_model import VideoPredictionModel
from .savp_train import TrainMixin

RELU_SHIFT = 1e-12


def _ceil4(v):
    return (v + 3) // 4 * 4


class ConcatSpec(object):
    """Channel layout of a concat buffer: segments (name, valid, alloc); offsets are multiples of 4.
    `cmap[i]` = index in the reference's concatenated tensor feeding internal channel i, or -1."""

    def __init__(self, segs):
        self.segs = []
        off, ref = 0, 0
        cmap = []
        for name, valid in segs:
            alloc = _ceil4(valid)
            self.segs.append((name, off, valid, alloc))
            cmap += list(range(ref, ref + valid)) + [-1] * (alloc - valid)
            off += alloc
            ref += valid
        self.cstride = off
        self.ref_channels = ref
        self.cmap = cmap

    def off(self, name):
        for n, o, v, a in self.segs:
            if n == name:
                return o
        raise KeyError(name)

    def valid(self, name):
        for n, o, v, a in self.segs:
            if n == name:
                return v
        raise KeyError(name)


class ConvLayer(object):
    """One convolution of the path (generator, posterior encoder and discriminator alike): reference-layout parameters +
    packed tensor-core weights.  `spec` is the ConcatSpec of the input buffer, or (ci_ref, ci_int, cmap) given directly
    (cmap None = identity).  `inv_scale` (optional device scalar, the spectral-norm sigma) divides the weights in every pack.
    In the fp32-exact mode (`model.exact`) every call runs as three TF32 passes (conv3x) against the residual packs.
    `prefilled`: the forward's output already holds an addend when the layer runs (the dense term of a conditioning site
    without tile-concat), which the epilogue adds before the bias and the activation."""

    def __init__(self, model, wname, bname, k, kind, stride, pad, transposed, spec, co, inv_scale=None, gates=False,
                 prefilled=False):
        self.model, self.wname, self.bname = model, wname, bname
        self.prefilled = prefilled
        self.k, self.kind, self.stride, self.pad, self.transposed = k, kind, stride, pad, transposed
        self.co, self.inv_scale = co, inv_scale
        self.ci_ref, self.ci_int, cmap = (spec.ref_channels, spec.cstride, spec.cmap) if isinstance(spec, ConcatSpec) else spec
        if kind == L.WKIND_POOLED:
            self.ke = (1, k[1] + 1, k[2] + 1)
        elif kind == L.WKIND_UPSAMPLED:
            self.ke = (1, k[1] + 3, k[2] + 3)
        else:
            self.ke = k
        # without a depth extent every leading dim of a buffer folds into n; a 3-D convolution keeps the depth axis
        self.nd = 3 if (self.ke[0], stride[0], pad[0]) == (1, 1, 0) else 4
        self.geom = L.geom(self.ke, stride, pad, transposed)
        self.cmap = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device=model.device)
        # gates: the forward packs of a norm-free ConvLSTM interleave its four gates for the cell epilogue (lstm_fwd)
        self.fwd_layout = L.WLAYOUT_FWD | (L.WLAYOUT_GATES if gates else 0)
        self.wp, self.n_pad, self.kc = self._alloc(self.fwd_layout)
        self.wp_lo = self._alloc(self.fwd_layout | L.WLAYOUT_RESIDUAL)[0] if model.exact else None
        self.wpd = self.wpd_lo = None

    def _alloc(self, layout):
        n_pad, kc, total = L.pack_dims(self.k, self.ci_int, self.co, self.kind, layout)
        return torch.empty(total, device=self.model.device), n_pad, kc

    def _view(self, t):
        return t.view((-1,) + tuple(t.shape[-self.nd:]))

    def prepare_backward(self):
        self.geom_bwd = L.geom(self.ke, self.stride, self.pad, not self.transposed)
        self.wpd, self.n_pad_d, self.kc_d = self._alloc(L.WLAYOUT_DGRAD)
        self.wpd_lo = self._alloc(L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL)[0] if self.model.exact else None
        self.dwp = torch.zeros_like(self.wp)

    def pack_jobs(self):
        """PackPlan entries that fill every packed buffer of this layer from its reference-layout weights."""
        w = self.model.params[self.wname]
        bufs = ((self.fwd_layout, self.wp), (self.fwd_layout | L.WLAYOUT_RESIDUAL, self.wp_lo),
                (L.WLAYOUT_DGRAD, self.wpd), (L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL, self.wpd_lo))
        return [(w, self.k, self.ci_ref, self.co, self.kind, layout, self.ci_int, self.cmap, self.inv_scale, out)
                for layout, out in bufs if out is not None]

    def fwd(self, x, out, out_off=0, out_c=None, act=L.ACT_NONE, alpha=0.0, split_k=0):
        """x: stacked buffer [.., (d,) h, w, cstride] (any leading dims)."""
        x = self._view(x)
        xv = L.tensor_view(x, self.ci_int)
        ov = L.tensor_view(self._view(out), self.co if out_c is None else out_c, out_off)
        bias = self.model.params[self.bname] if self.bname else None
        if self.model.exact:
            conv3x(x, self.ci_int, self.geom, self.wp, self.wp_lo, self.n_pad, self.kc, ov, bias, act, alpha, self.prefilled)
            return
        if self.prefilled:      # out = act(out + conv + bias): needs an unsplit call
            L.conv_igemm(xv, self.geom, self.wp, self.n_pad, self.kc, ov, bias, act, alpha, 1, 2)
            return
        L.conv_igemm(xv, self.geom, self.wp, self.n_pad, self.kc, ov, bias, act, alpha, split_k)

    def lstm_fwd(self, x, z, c_prev, c_new, h_dests):
        """One norm-free ConvLSTM step from the GATES packs: z = conv(x) + bias (natural gate order), c_new and h (to the
        (address, cstride) slices h_dests) from the engine's epilogue.  fp32-exact mode: two partial passes add into a
        zeroed z, the third adds the residual-weight pass and runs the cell.  A prefilled z keeps its addend: every pass
        adds to it."""
        x = self._view(x)
        xv = L.tensor_view(x, self.ci_int)
        cell = (z, self.model.params[self.bname], c_prev, c_new, h_dests)
        if self.model.exact:
            if not self.prefilled:
                z.zero_()
            L.conv_lstm_fwd(xv, self.geom, self.wp, self.n_pad, self.kc, *cell, accumulate=1)
            L.conv_lstm_fwd(L.tensor_view(L.tf32_residual(x), self.ci_int), self.geom, self.wp, self.n_pad, self.kc, *cell,
                            accumulate=1)
            L.conv_lstm_fwd(xv, self.geom, self.wp_lo, self.n_pad, self.kc, *cell, accumulate=2)
            return
        L.conv_lstm_fwd(xv, self.geom, self.wp, self.n_pad, self.kc, *cell, accumulate=2 if self.prefilled else 0)

    def dgrad(self, dy, dx, dy_c=None, accumulate=False, act_y=None, addend=None, act=L.ACT_NONE, alpha=0.0):
        """dx[.., ci_int] (+)= conv^T(dy): the same engine with the transposed flag flipped.  With act_y, the output of the
        activation `act` that produced this layer's input: dx = (conv^T(dy) + addend) * act'(act_y), fused into the epilogue."""
        dy, dx = self._view(dy), self._view(dx)
        dyv, dxv = L.tensor_view(dy, self.co if dy_c is None else dy_c), L.tensor_view(dx, self.ci_int)
        aux = None if act_y is None else (act_y.data_ptr(), 0 if addend is None else addend.data_ptr(), act)
        if self.model.exact:
            conv3x(dy, dyv.c, self.geom_bwd, self.wpd, self.wpd_lo, self.n_pad_d, self.kc_d, dxv, None, L.ACT_NONE, alpha,
                   accumulate, aux)
        elif aux is None:
            L.conv_igemm(dyv, self.geom_bwd, self.wpd, self.n_pad_d, self.kc_d, dxv, None, L.ACT_NONE, 0.0,
                         1 if accumulate else 0, accumulate)
        else:
            L.conv_igemm_actgrad(dyv, self.geom_bwd, self.wpd, self.n_pad_d, self.kc_d, dxv, aux[0], aux[1], act, alpha,
                                 2 if accumulate else 0)

    def wgrad(self, x, dy, dy_c=None, dw=None):
        """dw (default grads[w]) += dL/dw from ONE GEMM over every position of the (time-stacked) tensors."""
        x, dy = self._view(x), self._view(dy)
        xv = L.tensor_view(x, self.ci_int)
        dyv = L.tensor_view(dy, self.co if dy_c is None else dy_c)
        self.dwp.zero_()
        L.conv_wgrad(xv, dyv, self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
        if self.model.exact:      # + x_lo^T dy + x^T dy_lo
            L.conv_wgrad(L.tensor_view(L.tf32_residual(x), self.ci_int), dyv, self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
            L.conv_wgrad(xv, L.tensor_view(L.tf32_residual(dy), dyv.c), self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
        L.unpack_wgrad(self.dwp, self.k, self.ci_ref, self.co, self.kind, self.model.grads[self.wname] if dw is None else dw,
                       self.n_pad, self.kc, ci_int=self.ci_int, cmap=self.cmap)


def conv3x(x, c, geom, wp, wp_lo, n_pad, kc, ov, bias, act, alpha, accumulate=False, aux=None):
    """fp32-exact convolution on the TF32 tensor cores (VP_EXACT=1): x = x_hi + x_lo (x_hi = what the tensor core reads),
    W = W_hi + W_lo (W_hi = the packed, rounded weights);  out = act(x_hi W_hi + x_lo W_hi + x_hi W_lo + bias), the dropped
    x_lo W_lo term is 2^-21 relative.  aux = (act_output_addr, addend_addr, act): the fused activation-gradient epilogue."""
    xv = L.tensor_view(x, c)
    L.conv_igemm(xv, geom, wp, n_pad, kc, ov, None, L.ACT_NONE, 0.0, 1, 1 if accumulate else 0)
    L.conv_igemm(L.tensor_view(L.tf32_residual(x), c), geom, wp, n_pad, kc, ov, None, L.ACT_NONE, 0.0, 1, 1)
    if aux is None:
        L.conv_igemm(xv, geom, wp_lo, n_pad, kc, ov, bias, act, alpha, 1, 2)
    else:
        L.conv_igemm_actgrad(xv, geom, wp_lo, n_pad, kc, ov, aux[0], aux[1], aux[2], alpha, accumulate=2)


class NormSite(object):
    """One conv -> norm_layer -> activation site (ops.get_norm_layer, ops.py:1062-1073): h{i}, conv_h{i}, the h_flow /
    h_scratch / h_masks heads and posterior encoder layers 2 and up.  'instance' and 'layer' run the convolution into the `pre`
    buffer and the norm kernel from there into the output slice; 'none' has the convolution's epilogue apply bias +
    activation straight into that slice, and the backward takes the activation gradient from the output.

    Buffers are Bf keys (x: the convolution's input, read by the weight gradient; out: the output slice at channel out_off),
    their gradients the Gb key 'd' + pre.  They are indexed by step, and t=None is the whole buffer (the posterior encoder
    runs every step at once); `rows` = samples per call.  A prefilled convolution (a conditioning site without tile-concat)
    has its dense term (kernel `zname`) in `zdense`: (kernel, buffer, channel offset, channels, Gb key of its gradient)."""

    def __init__(self, model, conv, scope, x, pre, stats, out, out_off, rows, act, alpha=0.0, zname=None):
        self.model, self.conv, self.scope = model, conv, scope
        self.x, self.pre, self.dpre, self.stats, self.out, self.out_off = x, pre, 'd' + pre, stats, out, out_off
        pb = model.Bf[pre]
        self.rows, self.positions, self.c = rows, pb.shape[-3] * pb.shape[-2], conv.co
        self.out_cs = model.Bf[out].shape[-1]
        self.act, self.alpha = act, alpha
        self.norm = model.norm_scope and '%s/%s' % (scope, model.norm_scope)      # variable scope, None for 'none'
        self.zdense = None
        if conv.prefilled:      # the dense term lands where the convolution writes
            self.zdense = (zname,) + ((model.Bf[out], out_off) if self.norm is None else (pb, 0)) + (self.c, self.dpre)

    @staticmethod
    def _at(bufs, key, t):
        return bufs[key] if t is None else bufs[key][t]

    def _out(self, t):
        return self._at(self.model.Bf, self.out, t).data_ptr() + 4 * self.out_off

    def conv_fwd(self, x, t):
        """The convolution of step t on its input x."""
        if self.norm is None:
            self.conv.fwd(x, self._at(self.model.Bf, self.out, t), out_off=self.out_off, act=self.act, alpha=self.alpha)
        else:
            self.conv.fwd(x, self._at(self.model.Bf, self.pre, t))

    def norm_fwd(self, t):
        """out = act(norm(pre)) of step t; nothing to do for 'none'."""
        if self.norm is None:
            return
        m, c = self.model, self.c
        fn = L.inorm_act if m.hparams.norm_layer == 'instance' else L.lnorm_act
        fn(self._at(m.Bf, self.pre, t).data_ptr(), c, self._out(t), self.out_cs, self.rows, self.positions, c,
           m.params[self.norm + '/gamma'], m.params[self.norm + '/beta'], self.act, self.alpha, self._at(m.Bf, self.stats, t))

    def bwd(self, t, srcs, dx, accumulate=False):
        """dpre of step t from the gradient sources `srcs` [(address, cstride)] of the output, summed in that order
        (accumulating the norm's gamma / beta gradients), then dx (+)= conv^T(dpre)."""
        m, c = self.model, self.c
        dpre = self._at(m.Gb, self.dpre, t)
        dp = dpre.data_ptr()
        if self.norm is None:
            rows = self.rows * self.positions
            if len(srcs) > 2:            # act_bwd adds two sources: fold the others into dpre first
                L.axpy_channels(srcs[0][0], srcs[0][1], dp, c, rows, c, accumulate=False)
                for a, cs in srcs[1:-1]:
                    L.axpy_channels(a, cs, dp, c, rows, c)
                srcs = [(dp, c), srcs[-1]]
            b = srcs[1] if len(srcs) > 1 else (0, c)
            L.act_bwd(self._out(t), self.out_cs, srcs[0][0], srcs[0][1], b[0], b[1], dp, c, rows, c, self.act, self.alpha)
        else:
            fn = L.inorm_act_bwd if m.hparams.norm_layer == 'instance' else L.lnorm_act_bwd
            P, Gp, nm = m.params, m.grads, self.norm
            fn(self._at(m.Bf, self.pre, t).data_ptr(), c, srcs, dp, c, self.rows, self.positions, c, P[nm + '/gamma'],
               P[nm + '/beta'], self._at(m.Bf, self.stats, t), self.act, self.alpha, Gp[nm + '/gamma'], Gp[nm + '/beta'])
        self.conv.dgrad(dpre, dx, accumulate=accumulate)

    def param_grads(self):
        """The weight gradient over every step (one GEMM), then the bias gradient."""
        m = self.model
        dy = m.Gb[self.dpre]
        self.conv.wgrad(m.Bf[self.x], dy)
        L.colsum(dy.data_ptr(), self.c, m.grads[self.conv.bname], 1, dy.numel() // self.c, self.c)


# The generator's h{i} convolutions (savp_model.py:394-397, 461-464, 494-500; ops.get_downsample_layer /
# get_upsample_layer, ops.py:1077-1098): name -> (variable scope, weight kind, pad before, transposed), all with stride 2.
# The kernel is [k, k, cin, oc] -- deconv2d's is [3, 3, oc, cin], conv2d_transpose's filter layout.
#   conv_pool2d:  SAME conv + 2x2 average pool, folded into one (k+1)x(k+1) stride-2 conv (pad before k // 2)
#   conv2d:       k x k stride-2 SAME conv; SAME on an even extent pads (k-2) // 2 before, the rest after
#   upsample_conv2d: bilinear 2x upsample + 3x3 conv, folded into one 6x6 transposed conv (pad 2)
#   deconv2d:     3x3 stride-2 conv2d_transpose, the adjoint of the 2H -> H SAME conv (pad 0 before, 1 after)
# The _v2 recipes compute the same functions as the v1 layers with the v1 variables (ops.py:643-680, 795-820), so they
# run on the v1 packs.
DOWNSAMPLE_LAYERS = {
    'conv_pool2d': ('conv_pool2d', L.WKIND_POOLED, lambda k: k // 2, False),
    'conv_pool2d_v2': ('conv_pool2d', L.WKIND_POOLED, lambda k: k // 2, False),
    'conv2d': ('conv2d', L.WKIND_PLAIN, lambda k: (k - 2) // 2, False),
}
UPSAMPLE_LAYERS = {
    'upsample_conv2d': ('upsample_conv2d', L.WKIND_UPSAMPLED, lambda k: 2, True),
    'upsample_conv2d_v2': ('upsample_conv2d', L.WKIND_UPSAMPLED, lambda k: 2, True),
    'deconv2d': ('deconv2d', L.WKIND_DECONV, lambda k: 0, True),
}
# activation_layer (ops.get_activation_layer, ops.py:1052-1059): the activation of every norm_layer site of the generator
# (h{i} and the h_flow / h_scratch / h_masks heads); the posterior encoder keeps its leaky relu
ACTIVATIONS = {'relu': L.ACT_RELU, 'elu': L.ACT_ELU}


class SAVPVideoPredictionModel(TrainMixin, VideoPredictionModel):
    def __init__(self, *args, **kwargs):
        super(SAVPVideoPredictionModel, self).__init__(*args, **kwargs)
        self.deterministic = not self.hparams.nz
        self.device = None
        self.params = None
        self.grads = None
        self.built = False
        self.Sd = 0                      # robot-state dimensions, from build_graph's inputs
        self.world_size = 1
        self.rank = 0
        self.random_seed = 0
        self.use_cuda_graph = False      # train_step(): capture the device part of the step once, then replay it
        self._pending_params = None
        self.g_adam_t = self.d_adam_t = 0
        self.dnets = OrderedDict()

    # ------------------------------------------------------------------ hparams (savp_model.py:779-846)
    def get_default_hparams_dict(self):
        default_hparams = super(SAVPVideoPredictionModel, self).get_default_hparams_dict()
        hparams = dict(
            l1_weight=1.0, l2_weight=0.0, n_layers=3, ndf=32, norm_layer='instance', use_same_discriminator=False,
            ngf=32, downsample_layer='conv_pool2d', upsample_layer='upsample_conv2d', activation_layer='relu',
            transformation='cdna', kernel_size=(5, 5), dilation_rate=(1, 1), where_add='all', use_tile_concat=True,
            learn_initial_state=False, rnn='lstm', conv_rnn='lstm', conv_rnn_norm_layer='instance',
            num_transformed_images=4, last_frames=1, prev_image_background=True, first_image_background=True,
            last_image_background=False, last_context_image_background=False, context_images_background=False,
            generate_scratch_image=True, dependent_mask=True, schedule_sampling='inverse_sigmoid',
            schedule_sampling_k=900.0, schedule_sampling_steps=(0, 100000), use_e_rnn=False, learn_prior=False, nz=8,
            num_samples=8, nef=64, use_rnn_z=True, ablation_conv_rnn_norm=False, ablation_rnn=False,
        )
        return dict(itertools.chain(default_hparams.items(), hparams.items()))

    def parse_hparams(self, hparams_dict, hparams):
        deprecated = ['num_gpus', 'e_net', 'd_conditional', 'd_downsample_layer', 'd_net', 'd_use_gt_inputs',
                      'acvideo_gan_weight', 'acvideo_vae_gan_weight', 'image_gan_weight', 'image_vae_gan_weight',
                      'tuple_gan_weight', 'tuple_vae_gan_weight', 'gan_weight', 'vae_gan_weight', 'video_gan_weight',
                      'video_vae_gan_weight']
        hparams_dict = dict(hparams_dict or {})
        for key in deprecated:
            hparams_dict.pop(key, None)
        return super(SAVPVideoPredictionModel, self).parse_hparams(hparams_dict, hparams)

    def _check_supported(self):
        """Every hparam the reference acts on is either implemented here or refused: nothing is accepted and ignored."""
        hp = self.hparams
        if hp.where_add not in ('input', 'all', 'middle'):
            raise ValueError('Invalid where_add %s' % hp.where_add)  # savp_model.py:176-177
        if hp.schedule_sampling not in ('none', 'inverse_sigmoid', 'linear'):
            raise NotImplementedError('schedule_sampling=%r' % (hp.schedule_sampling,))     # savp_model.py:332-333
        if hp.gan_loss_type not in ('LSGAN', 'GAN', 'SNGAN'):
            raise ValueError('Unknown GAN loss type %s' % hp.gan_loss_type)                 # losses.py:52-53
        for key, table in (('downsample', DOWNSAMPLE_LAYERS), ('upsample', UPSAMPLE_LAYERS), ('activation', ACTIVATIONS)):
            if getattr(hp, key + '_layer') not in table:      # ops.get_*_layer (ops.py:1052-1098)
                raise ValueError('Invalid %s layer %s' % (key, getattr(hp, key + '_layer')))
        unsupported = []
        for key, want in (('conv_rnn', 'lstm'), ('use_e_rnn', False), ('learn_prior', False),
                          ('joint_gan_optimization', False), ('use_same_discriminator', False)):
            # (`repeat` is accepted with any value: train.py sets it to the dataset's time_shift (train.py:160) and no model
            #  code of the reference reads it, base_model.py:90-95)
            if getattr(hp, key) != want:
                unsupported.append('%s=%r' % (key, getattr(hp, key)))
        if hp.rnn not in ('lstm', 'gru'):      # the z cell (savp_model.py:354-362)
            unsupported.append('rnn=%r' % (hp.rnn,))
        # the normaliser of every convolution outside the ConvLSTM cells (savp_model.py:394, ops.py:1062-1073): instance,
        # layer or none; 'batch' would need moving averages and a train / test switch
        if hp.norm_layer not in ('instance', 'layer', 'none'):
            unsupported.append('norm_layer=%r' % (hp.norm_layer,))
        # the ConvLSTM's normalisation (savp_model.py:370-390): instance norms inside the cell, none, or (ablation) one
        # instance norm on the cell's output
        if hp.conv_rnn_norm_layer not in ('instance', 'none'):
            unsupported.append('conv_rnn_norm_layer=%r' % (hp.conv_rnn_norm_layer,))
        elif hp.ablation_conv_rnn_norm and hp.conv_rnn_norm_layer == 'none' and not hp.ablation_rnn:
            raise ValueError('ablation_conv_rnn_norm=True needs a conv_rnn_norm_layer to apply to the cell output, got '
                             "'none'")   # the reference calls None(h) (savp_model.py:380-383)
        if hp.transformation not in ('cdna', 'flow'):
            unsupported.append('transformation=%r' % (hp.transformation,))
        # the compositing stage (savp_model.py:239-246, 561-653): L = num_masks slots, the first nk of them transforms
        if hp.last_frames < 0 or hp.num_transformed_images < 0:
            unsupported.append('last_frames=%r, num_transformed_images=%r' % (hp.last_frames, hp.num_transformed_images))
        comp = self.compositing(hp)
        if not comp['L']:       # savp_model.py:641-644
            raise ValueError('Either one of the following should be true: last_frames and num_transformed_images, '
                             'first_image_background, prev_image_background, generate_scratch_image')
        if comp['nk'] > L.SLOT_MAX_TRANSFORMS or comp['L'] > L.SLOT_MAX_LAYERS:
            unsupported.append('last_frames * num_transformed_images=%d (at most %d) with %d compositing layers (at most %d)'
                               % (comp['nk'], L.SLOT_MAX_TRANSFORMS, comp['L'], L.SLOT_MAX_LAYERS))
        if tuple(hp.dilation_rate) != (1, 1):
            unsupported.append('dilation_rate=%r' % (hp.dilation_rate,))
        if self.mode == 'train':
            # loss terms of base_model.py:733-852 that are not built: refuse instead of silently dropping them
            for key in ('vgg_cdist_weight', 'feature_l2_weight', 'ae_l2_weight', 'state_weight', 'tv_weight', 'z_l1_weight',
                        'gan_feature_l2_weight', 'vae_gan_feature_l2_weight'):
                if getattr(hp, key):
                    unsupported.append('%s=%r' % (key, getattr(hp, key)))
            if hp.kl_weight and hp.kl_anneal not in ('none', 'sigmoid', 'linear'):
                unsupported.append('kl_anneal=%r' % (hp.kl_anneal,))
        if unsupported:
            raise NotImplementedError('hparams outside the H100 hot path (SURVEY.md 8f): ' + ', '.join(unsupported))

    @staticmethod
    def compositing(hp):
        """The slot layout of the compositing stage (savp_model.py:239-246, 574-596): nk transforms of the F most recent
        images (F = last_frames, oldest first; none unless last_frames and num_transformed_images), then the backgrounds in
        the reference's order -- 'prev' (the step's input image), 'first' (images[0]), 'last' (images[context_frames-1]),
        'last_context' (images[min(t, context_frames-1)]), ('context', i) (images[i], i < context_frames) -- then the
        scratch image.  L = every slot; masks exist only for L > 1."""
        nk = hp.last_frames * hp.num_transformed_images if (hp.last_frames and hp.num_transformed_images) else 0
        ctx = hp.context_images_background
        bgs = (['prev'] if hp.prev_image_background else []) + (['first'] if hp.first_image_background and not ctx else []) + \
              (['last'] if hp.last_image_background and not ctx else []) + \
              (['last_context'] if hp.last_context_image_background and not ctx else []) + \
              ([('context', i) for i in range(hp.context_frames)] if ctx else [])
        scratch = bool(hp.generate_scratch_image)
        return dict(nk=nk, F=hp.last_frames if nk else 1, bgs=bgs, scratch=scratch, L=nk + len(bgs) + int(scratch),
                    prev_slot=nk + bgs.index('prev') if 'prev' in bgs else -1)

    @property
    def cell_norm(self):
        """True: the reference's default ConvLSTM, with instance norms inside the cell.  False: the norm-free cell
        (conv_rnn_norm_layer='none', or the ablation_conv_rnn_norm form), whose gate math runs in the engine's epilogue."""
        return self.hparams.conv_rnn_norm_layer == 'instance' and not self.hparams.ablation_conv_rnn_norm

    @property
    def z_cell(self):
        """The cell rnn_z comes from (savp_model.py:424-432): 'lstm' / 'gru' (`rnn`), 'fc' (ablation_rnn: tanh(dense(z))), or
        None -- no z, or use_rnn_z=False, where the zs themselves go into the tile-concat vector."""
        hp = self.hparams
        if not hp.nz or not hp.use_rnn_z:
            return None
        return 'fc' if hp.ablation_rnn else hp.rnn

    @property
    def norm_scope(self):
        """Variable scope of the normaliser at the norm_layer sites (h0.., the h_flow / h_scratch / h_masks heads, encoder
        layers 2..): the default scope of the layer ops.get_norm_layer picks (ops.py:1062-1073), or None for
        norm_layer='none' (tf.identity, no variables).  The ConvLSTM's own norms follow conv_rnn_norm_layer instead."""
        return {'instance': 'InstanceNorm', 'layer': 'LayerNorm'}.get(self.hparams.norm_layer)

    @property
    def site_act(self):
        """The activation of the generator's norm_layer sites (activation_layer)."""
        return ACTIVATIONS[self.hparams.activation_layer]

    def _zsite(self, li, rnn=False):
        """How the conditioning vector state_action_z = [actions | state | rnn_z] reaches a site of generator layer li
        (savp_model.py:456-518): the h{li} convolution (rnn=False) or the layer's ConvLSTM / conv_h site (rnn=True).
        'tile' (use_tile_concat): tiled over space as extra input channels of the convolution; 'dense': the convolution reads
        the spatial input alone and dense(v) is added to its output before the norm (_maybe_tile_concat_layer, :983-993;
        the ConvLSTM's `weights`, rnn_ops.py:128-146); None: the site does not see the vector.  where_add='all' feeds every
        site, 'input' h0 alone, 'middle' the first decoder layer alone."""
        hp = self.hparams
        if rnn:
            takes = hp.where_add == 'all'
        else:
            takes = hp.where_add == 'all' or li == {'input': 0, 'middle': len(self.enc_specs)}[hp.where_add]
        if not takes:
            return None
        return 'tile' if hp.use_tile_concat else 'dense'

    def _zdense_name(self, li, rnn=False):
        """The [Zc, site channels] kernel of the dense term of a 'dense' site (no bias)."""
        sc = 'generator/rnn/savp_cell'
        if not rnn:
            return '%s/h%d/dense/kernel' % (sc, li)
        if self.hparams.ablation_rnn:
            return '%s/conv_h%d/dense/kernel' % (sc, li)
        return '%s/lstm_h%d/basic_conv2dlstm_cell/weights' % (sc, li)

    def _hconv_layer(self, li, cin, oc):
        """(scope, kernel shape, weight kind, kernel size, pad before, transposed) of the h{li} convolution with cin input
        channels (tile-concat included)."""
        hp = self.hparams
        if li < len(self.enc_specs):
            ks = 5 if li == 0 else 3
            scope, kind, pad, transposed = DOWNSAMPLE_LAYERS[hp.downsample_layer]
        else:
            ks = 3
            scope, kind, pad, transposed = UPSAMPLE_LAYERS[hp.upsample_layer]
        shape = (ks, ks, oc, cin) if kind == L.WKIND_DECONV else (ks, ks, cin, oc)
        return '%s/h%d/%s' % ('generator/rnn/savp_cell', li, scope), shape, kind, ks, pad(ks), transposed

    # ------------------------------------------------------------------ structure (savp_model.py:182-232)
    @staticmethod
    def layer_specs(ngf, height, width):
        s = min(height, width)
        g = ngf
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

    def _generator_plan(self):
        """The generator's layers from the hparams and shapes alone (no device): per layer li its oc, use (ConvLSTM after
        the h{li} site), output and input extents h, w / ih, iw, zin / zr (_zsite of the h{li} and the recurrent site),
        in_spec (the h{li} input: image | first image, or x | skip, then z when tile-concatenated), hconv (_hconv_layer)
        and, with use, the recurrent site: rin_spec (x | z for conv_h{li}, x | z | h for the ConvLSTM), its scope rname,
        its kernel / bias names and its output channels rco."""
        hp = self.hparams
        sc = 'generator/rnn/savp_cell'
        n_enc = len(self.enc_specs)
        plan = []
        h, w = self.H, self.W

        def zseg(form):     # the z segment of a site's input when it tile-concatenates the vector
            return [('z', self.Zc)] if (self.Zc and form == 'tile') else []
        for li, (oc, use) in enumerate(self.enc_specs + self.dec_specs):
            is_enc = li < n_enc
            d = dict(li=li, oc=oc, use=use, is_enc=is_enc, ih=h, iw=w, zin=self._zsite(li),
                     zr=self._zsite(li, rnn=True) if use else None)
            h, w = (h // 2, w // 2) if is_enc else (h * 2, w * 2)
            d['h'], d['w'] = h, w
            if li == 0:
                segs = [('image', self.C), ('first', self.C)]
            elif is_enc or li == n_enc:
                segs = [('x', plan[-1]['oc'])]
            else:       # skip connection: decoder layer n_enc + i reads layer n_enc - i - 1
                segs = [('x', plan[-1]['oc']), ('skip', plan[2 * n_enc - li - 1]['oc'])]
            d['in_spec'] = ConcatSpec(segs + zseg(d['zin']))
            d['hconv'] = self._hconv_layer(li, d['in_spec'].ref_channels, oc)
            if use:
                if hp.ablation_rnn:     # the stateless conv_h{li} site (savp_model.py:472-475)
                    d['rname'] = '%s/conv_h%d' % (sc, li)
                    d['rin_spec'] = ConcatSpec([('x', oc)] + zseg(d['zr']))
                    d['rkernel'], d['rbias'], d['rco'] = d['rname'] + '/conv2d/kernel', d['rname'] + '/conv2d/bias', oc
                else:                   # the norm-free cell's gate convolution has a bias (rnn_ops.py:122-125)
                    d['rname'] = '%s/lstm_h%d/basic_conv2dlstm_cell' % (sc, li)
                    d['rin_spec'] = ConcatSpec([('x', oc)] + zseg(d['zr']) + [('h', oc)])
                    d['rkernel'], d['rco'] = d['rname'] + '/kernel', 4 * oc
                    d['rbias'] = None if self.cell_norm else d['rname'] + '/bias'
            plan.append(d)
        return plan

    def _generator_param_specs(self):
        """name -> (shape, init) with the reference's variable scopes (generator/...)."""
        hp = self.hparams
        C, A = self.C, self.A
        specs = OrderedDict()
        Zc = self.Zc
        if hp.nz:
            sc = 'generator/encoder'
            cin = 2 * C + A
            for i in range(hp.n_layers):
                oc = hp.nef * min(2 ** i, 4)
                specs['%s/layer_%d/conv2d/kernel' % (sc, i + 1)] = ((4, 4, cin, oc), 'kernel')
                specs['%s/layer_%d/conv2d/bias' % (sc, i + 1)] = ((oc,), 'zeros')
                if i > 0 and self.norm_scope:
                    specs['%s/layer_%d/%s/gamma' % (sc, i + 1, self.norm_scope)] = ((oc,), 'ones')
                    specs['%s/layer_%d/%s/beta' % (sc, i + 1, self.norm_scope)] = ((oc,), 'zeros')
                cin = oc
            for nm in ('z_mu', 'z_log_sigma_sq'):
                specs['%s/%s/dense/kernel' % (sc, nm)] = ((cin, hp.nz), 'kernel')
                specs['%s/%s/dense/bias' % (sc, nm)] = ((hp.nz,), 'zeros')
        sc = 'generator/rnn/savp_cell'
        nz = hp.nz
        if self.z_cell == 'lstm':
            specs[sc + '/lstm_z/basic_lstm_cell/kernel'] = ((2 * nz, 4 * nz), 'kernel')
            specs[sc + '/lstm_z/basic_lstm_cell/bias'] = ((4 * nz,), 'zeros')
        elif self.z_cell == 'gru':     # GRUCell (TF >= 1.9): the gate bias starts at 1
            specs[sc + '/gru_z/gru_cell/gates/kernel'] = ((2 * nz, 2 * nz), 'kernel')
            specs[sc + '/gru_z/gru_cell/gates/bias'] = ((2 * nz,), 'ones')
            specs[sc + '/gru_z/gru_cell/candidate/kernel'] = ((2 * nz, nz), 'kernel')
            specs[sc + '/gru_z/gru_cell/candidate/bias'] = ((nz,), 'zeros')
        elif self.z_cell == 'fc':
            specs[sc + '/fc_z/dense/kernel'] = ((nz, nz), 'kernel')
            specs[sc + '/fc_z/dense/bias'] = ((nz,), 'zeros')

        def norm(name, c):
            specs[name + '/gamma'] = ((c,), 'ones')
            specs[name + '/beta'] = ((c,), 'zeros')

        def site_norm(site, c):
            if self.norm_scope:
                norm('%s/%s' % (site, self.norm_scope), c)

        def zdense(d, c, rnn=False):
            # created after the site's convolution and before its norm, as the reference does; [0, c] without a vector
            if d['zr' if rnn else 'zin'] == 'dense':
                specs[self._zdense_name(d['li'], rnn)] = ((Zc, c), 'kernel')
        plan = self._generator_plan()
        for d in plan:
            li, oc = d['li'], d['oc']
            scope, shape = d['hconv'][:2]
            specs[scope + '/kernel'] = (shape, 'kernel')
            specs[scope + '/bias'] = ((oc,), 'zeros')
            zdense(d, oc)
            site_norm('%s/h%d' % (sc, li), oc)
            if not d['use']:
                continue
            specs[d['rkernel']] = ((5, 5, d['rin_spec'].ref_channels, d['rco']), 'kernel')
            if d['rbias']:
                specs[d['rbias']] = ((d['rco'],), 'zeros')
            zdense(d, d['rco'], rnn=True)
            if hp.ablation_rnn:     # conv 5x5 + norm_layer + activation_layer, no state
                site_norm(d['rname'], oc)
            elif self.cell_norm:
                norm(d['rname'] + '/input_transform_forget_output', 4 * oc)
                norm(d['rname'] + '/state', oc)
            elif hp.ablation_conv_rnn_norm:      # instance norm of the cell output h (savp_model.py:380-383)
                norm('%s/lstm_h%d/InstanceNorm' % (sc, li), oc)
        nl = len(plan)
        kh, kw = hp.kernel_size
        comp = self.compositing(hp)
        nk, nlayers = comp['nk'], comp['L']
        small = plan[len(self.enc_specs) - 1]
        top = plan[-1]['oc']
        if nk and hp.transformation == 'flow':     # savp_model.py:522-530: flow heads instead of the CDNA kernel dense layer
            specs['%s/h%d_flow/conv2d/kernel' % (sc, nl)] = ((3, 3, top, hp.ngf), 'kernel')
            specs['%s/h%d_flow/conv2d/bias' % (sc, nl)] = ((hp.ngf,), 'zeros')
            site_norm('%s/h%d_flow' % (sc, nl), hp.ngf)
            specs[sc + '/flows/conv2d/kernel'] = ((3, 3, hp.ngf, 2 * nk), 'kernel')
            specs[sc + '/flows/conv2d/bias'] = ((2 * nk,), 'zeros')
        elif nk:
            specs[sc + '/cdna_kernels/dense/kernel'] = ((small['h'] * small['w'] * small['oc'], kh * kw * nk), 'kernel')
            specs[sc + '/cdna_kernels/dense/bias'] = ((kh * kw * nk,), 'zeros')
        heads = (['h%d_scratch' % nl] if comp['scratch'] else []) + (['h%d_masks' % nl] if nlayers > 1 else [])
        for nm in heads:
            specs['%s/%s/conv2d/kernel' % (sc, nm)] = ((3, 3, top, hp.ngf), 'kernel')
            specs['%s/%s/conv2d/bias' % (sc, nm)] = ((hp.ngf,), 'zeros')
            site_norm('%s/%s' % (sc, nm), hp.ngf)
        if comp['scratch']:
            specs[sc + '/scratch_image/conv2d/kernel'] = ((3, 3, hp.ngf, C), 'kernel')
            specs[sc + '/scratch_image/conv2d/bias'] = ((C,), 'zeros')
        if nlayers > 1:     # dependent_mask: the masks conv also reads every slot (savp_model.py:630-633)
            specs[sc + '/masks/conv2d/kernel'] = ((3, 3, hp.ngf + (nlayers * C if hp.dependent_mask else 0), nlayers), 'kernel')
            specs[sc + '/masks/conv2d/bias'] = ((nlayers,), 'zeros')
        if self.Sd:       # savp_model.py:655-658: the next robot state from [actions | state]
            specs[sc + '/state_pred/dense/kernel'] = ((A + self.Sd, self.Sd), 'kernel')
            specs[sc + '/state_pred/dense/bias'] = ((self.Sd,), 'zeros')
        for name, shape, _, _ in self._initial_state_specs():
            specs[name] = (shape, 'zeros')
        return specs

    def _initial_state_specs(self):
        """learn_initial_state (savp_model.py:263-307, 344-348): [(name, shape, state, li)] in the order of nest.flatten of
        {'conv_rnn_states': [LSTMStateTuple(c, h) per ConvLSTM, in layer order], 'rnn_z_state': (c, h) of lstm_z or h of
        gru_z} -- dict keys sorted, so the ConvLSTMs first.  `state` names the buffer the variable initialises: 'c' / 'h' of
        generator layer li, 'zc' / 'zh'.  No ConvLSTM entries under ablation_rnn, no z entry without a z RNN."""
        hp = self.hparams
        if not hp.learn_initial_state:
            return []
        leaves = []
        if not hp.ablation_rnn:
            for d in self._generator_plan():
                if d['use']:
                    leaves += [((d['h'], d['w'], d['oc']), what, d['li']) for what in ('c', 'h')]
        if self.z_cell in ('lstm', 'gru'):
            leaves += [((hp.nz,), 'zc', -1)] if self.z_cell == 'lstm' else []
            leaves.append(((hp.nz,), 'zh', -1))
        return [('generator/initial_state_%d/initial_state' % k, shape, what, li) for k, (shape, what, li) in enumerate(leaves)]

    # ------------------------------------------------------------------ build
    def build_graph(self, inputs):
        """inputs: dict with 'images' [B,T,H,W,C] (torch / numpy, batch-major as in base_model.py:467)
        and optionally 'actions' [B,T-1,A], 'states' [B,T,Sd] (robot states: tile-concatenated into every convolution
        input after the actions and predicted as gen_states) and 'pix_distribs' [B,T,H,W,D] (D designated-pixel
        probability maps, moved with the images: gen_pix_distribs / transformed_pix_distribs in `outputs`).  Allocates
        parameters (reference initialisers) unless `set_params` was called, and all activation buffers."""
        super(SAVPVideoPredictionModel, self).build_graph(inputs)
        if not torch.cuda.is_available():
            raise RuntimeError('video_prediction_b200 needs a CUDA device (sm_90a); there is no CPU fallback')
        L.lib()  # fail loudly if the CUDA library is missing
        self._check_supported()
        self.exact = L.exact_mode()     # the arithmetic of every convolution of this model, fixed when its buffers are laid out
        hp = self.hparams
        # data parallelism (base_model.py:517-646): one process per GPU.  torchrun's env gives rank / world; with the
        # reference's `num_gpus` > 1 the batch in `inputs` is the GLOBAL batch and every rank takes its shard
        # (tf.split of the global batch, :523-527); with num_gpus <= 1 under torchrun each rank feeds its own batch.
        self.rank, _local, self.world_size = dp.init_from_env()
        if self.num_gpus and self.num_gpus > 1:
            if self.world_size != self.num_gpus:
                raise ValueError('num_gpus=%d needs %d processes (torchrun --nproc-per-node), found WORLD_SIZE=%d'
                                 % (self.num_gpus, self.num_gpus, self.world_size))
            self._shard = dp.shard_batch(int(inputs['images'].shape[0]), self.rank, self.world_size)
            inputs = {k: v[self._shard] for k, v in inputs.items()}
        else:
            self._shard = None
        self.device = torch.device('cuda', torch.cuda.current_device())
        imgs = inputs['images']
        B, T, H, W, C = [int(s) for s in imgs.shape]
        if T < hp.sequence_length:
            raise ValueError('images have %d frames, sequence_length is %d' % (T, hp.sequence_length))
        self.B, self.T, self.H, self.W, self.C = B, hp.sequence_length, H, W, C
        self.A = int(inputs['actions'].shape[-1]) if 'actions' in inputs else 0
        self.D = self._pix_distribs_depth(inputs)
        self.Sd = self._states_dim(inputs)
        self.S = self.T - 1
        self.Zc = self.A + self.Sd + (hp.nz if hp.nz else 0)     # tile-concat vector [actions | state | rnn_z]
        self.NB = 2 * B if hp.nz else B
        self.enc_specs, self.dec_specs = self.layer_specs(hp.ngf, H, W)
        total_stride = 2 ** len(self.enc_specs)
        if (H % total_stride) or (W % total_stride):
            raise ValueError('The image has dimension (%d, %d), but it should be divisible by the total stride, '
                             'which is %d.' % (H, W, total_stride))
        if C > 3:
            raise NotImplementedError('at most 3 colour channels (pixels are stored as float4 with one padding lane)')
        self.param_specs = self._generator_param_specs()
        if self.mode == 'train':
            self.param_specs.update(self._discriminator_param_specs())
        self._alloc_params()
        self.init_params(seed=0)
        if self._pending_params is not None:
            self._apply_params(self._pending_params)
            self._pending_params = None
        if self.world_size > 1:     # replicas start from rank 0's variables (post_init_ops, base_model.py:640-646)
            dp.broadcast_state([self.g_flat, self.d_flat] + [v for k, v in self.params.items() if k.endswith('/u')])
        self._allreduce = dp.make_allreduce()
        # VP_DP_BUCKETS=1: per-tower / per-layer all-reduces overlapped with the backward pass (dp.GradientReducer); the default
        # is two flat all-reduces (one per optimizer), which cost the fewest NCCL launches
        self._reducer = dp.GradientReducer(self.device) if (self.world_size > 1 and os.environ.get('VP_DP_BUCKETS', '0') == '1') else None
        self._build_generator()
        if self.mode == 'train':
            self._build_discriminator()
            self._build_training()
        self.built = True
        self.set_inputs(inputs)

    @staticmethod
    def _pix_distribs_depth(inputs):
        """D of inputs['pix_distribs'] [B,T,H,W,D] (0 without the key); the maps must cover the images' frames."""
        if 'pix_distribs' not in inputs:
            return 0
        pd, im = inputs['pix_distribs'], inputs['images']
        if len(pd.shape) != 5 or tuple(pd.shape[:4]) != tuple(im.shape[:4]):
            raise ValueError('pix_distribs must be [B, T, H, W, D] with B, T, H, W of the images %s, got %s'
                             % (tuple(im.shape), tuple(pd.shape)))
        if int(pd.shape[4]) < 1:
            raise ValueError('pix_distribs need at least one designated pixel (D >= 1), got shape %s' % (tuple(pd.shape),))
        return int(pd.shape[4])

    @staticmethod
    def _states_dim(inputs):
        """Sd of inputs['states'] [B,T,Sd] (0 without the key); the states must cover the images' frames."""
        if 'states' not in inputs:
            return 0
        st, im = inputs['states'], inputs['images']
        if len(st.shape) != 3 or tuple(st.shape[:2]) != tuple(im.shape[:2]):
            raise ValueError('states must be [B, T, Sd] with B, T of the images %s, got %s' % (tuple(im.shape), tuple(st.shape)))
        if int(st.shape[2]) < 1:
            raise ValueError('states need at least one dimension (Sd >= 1), got shape %s' % (tuple(st.shape),))
        return int(st.shape[2])

    def _alloc_params(self):
        """Flat fp32 buffers (one per optimizer: generator / discriminator, base_model.py:486-487) with
        per-variable views under the reference's variable names; same for gradients and Adam slots."""
        dev = self.device
        gn = [(k, v) for k, v in self.param_specs.items() if k.startswith('generator/')]
        dn = [(k, v) for k, v in self.param_specs.items() if k.startswith('discriminator/') and v[1] != 'u']
        un = [(k, v) for k, v in self.param_specs.items() if v[1] == 'u']
        self.params, self.grads = OrderedDict(), OrderedDict()

        def flat(items):
            sizes = [(int(np.prod(shape)) + 3) // 4 * 4 for _, (shape, _) in items]   # keep every view 16B aligned
            buf = torch.zeros(max(sum(sizes), 4), device=dev, dtype=torch.float32)
            grad = torch.zeros_like(buf)
            off = 0
            for (name, (shape, _)), sz in zip(items, sizes):
                n = int(np.prod(shape))
                self.params[name] = buf[off:off + n].view(shape)
                self.grads[name] = grad[off:off + n].view(shape)
                off += sz
            return buf, grad
        self.g_flat, self.g_grad = flat(gn)
        self.g_m, self.g_v = torch.zeros_like(self.g_flat), torch.zeros_like(self.g_flat)
        self.d_flat, self.d_grad = flat(dn)
        self.d_m, self.d_v = torch.zeros_like(self.d_flat), torch.zeros_like(self.d_flat)
        for name, (shape, _) in un:
            self.params[name] = torch.zeros(shape, device=dev, dtype=torch.float32)

    def init_params(self, seed=0):
        """Reference initialisers: kernels truncated-normal(0.02), biases 0, gamma 1 / beta 0, u truncated-normal(1)."""
        rng = np.random.default_rng(seed)
        vals = OrderedDict()

        def tn(shape, std):
            x = rng.standard_normal(size=shape)
            bad = np.abs(x) > 2.0
            while bad.any():
                x[bad] = rng.standard_normal(size=int(bad.sum()))
                bad = np.abs(x) > 2.0
            return (x * std).astype(np.float32)
        for name, (shape, init) in self.param_specs.items():
            if init == 'kernel':
                vals[name] = tn(shape, 0.02)
            elif init == 'u':
                vals[name] = tn(shape, 1.0)
            elif init == 'ones':
                vals[name] = np.ones(shape, np.float32)
            else:
                vals[name] = np.zeros(shape, np.float32)
        self._apply_params(vals)

    def _apply_params(self, values):
        for name, v in values.items():
            if name not in self.params:
                continue        # e.g. discriminator variables offered to a test-mode model
            t = v.detach().to(dtype=torch.float32, device='cpu').clone() if torch.is_tensor(v) else torch.from_numpy(np.array(v, dtype=np.float32))
            if tuple(t.shape) != tuple(self.params[name].shape):
                raise ValueError('shape mismatch for %s: %s vs %s' % (name, tuple(t.shape), tuple(self.params[name].shape)))
            self.params[name].copy_(t.to(self.device))

    def set_params(self, values):
        """values: name -> array/tensor with the reference's variable names and shapes."""
        if not self.built and self.params is None:
            self._pending_params = dict(values)
            return
        self._apply_params(values)
        if self.built:
            self._pack_all()

    # ------------------------------------------------------------------ checkpoints (base_model.py:229-246, train.py:242, 349)
    def saveable_state(self):
        """What tf.train.Saver(model.saveable_variables) stores: global_step + every variable (reference names) + both
        optimizers' slots."""
        st = OrderedDict(global_step=np.int64(self.global_step))
        for k, v in self.params.items():
            st['var/' + k] = v.detach().cpu().numpy()
        if self.mode == 'train':
            for nm in ('g_m', 'g_v', 'd_m', 'd_v'):
                st['adam/' + nm] = getattr(self, nm).detach().cpu().numpy()
            st['adam/t'] = np.array([self.g_adam_t, self.d_adam_t], np.int64)
        return st

    def save(self, output_dir, prefix='model'):
        """Writes `<output_dir>/<prefix>-<global_step>.npz` (+ a `checkpoint` text file naming the latest, as tf.train.Saver
        does), keeping the two most recent (train.py:231 max_to_keep=2).  Returns the path."""
        import os
        os.makedirs(output_dir, exist_ok=True)
        path = os.path.join(output_dir, '%s-%d.npz' % (prefix, self.global_step))
        np.savez(path, **self.saveable_state())
        with open(os.path.join(output_dir, 'checkpoint'), 'w') as f:
            f.write('model_checkpoint_path: "%s"\n' % os.path.basename(path))
        old = sorted((p for p in os.listdir(output_dir) if p.startswith(prefix + '-') and p.endswith('.npz')),
                     key=lambda p: int(p[len(prefix) + 1:-4]))
        for p in old[:-2]:
            os.remove(os.path.join(output_dir, p))
        return path

    @staticmethod
    def latest_checkpoint(checkpoint):
        """A checkpoint name, or a directory holding a `checkpoint` state file (tf.train.latest_checkpoint).  Both this
        package's `.npz` checkpoints and TensorFlow bundles (`<prefix>.index` + `.data-*`) are resolved."""
        import os
        from .. import tf_checkpoint as T
        if checkpoint and os.path.isdir(checkpoint):
            idx = os.path.join(checkpoint, 'checkpoint')
            if os.path.exists(idx):
                with open(idx) as f:
                    name = f.readline().split('"')[1]
                path = name if os.path.isabs(name) else os.path.join(checkpoint, name)
                if os.path.exists(path) or T.is_tf_checkpoint(path):
                    return path
            return T.latest_checkpoint(checkpoint)
        return checkpoint

    @staticmethod
    def restore_to_checkpoint_mapping(restore_name, checkpoint_var_names):
        """savp_model.py:848-855: checkpoints written before the cell was renamed use the scope 'dna_cell'."""
        restore_name = restore_name.split(':')[0]
        if restore_name not in checkpoint_var_names:
            restore_name = restore_name.replace('savp_cell', 'dna_cell')
        return restore_name

    def _view_of(self, flat_like, flat, name):
        """The slice of a buffer parallel to `flat` (gradients, Adam slots) that belongs to variable `name`."""
        v = self.params[name]
        o = (v.data_ptr() - flat.data_ptr()) // 4
        return flat_like[o:o + v.numel()].view(v.shape)

    def restore(self, sess=None, checkpoints=None, restore_to_checkpoint_mapping=None):
        """base_model.py:229-246 + SAVP's name mapping (savp_model.py:848-855).  `sess` is accepted for call compatibility
        and ignored.  Restores every variable present in both the model and the checkpoint(s) -- this package's .npz files or
        TensorFlow checkpoints of the reference (tf_checkpoint.py) -- reports the rest as get_checkpoint_restore_saver does
        (tf_utils.py:543-557), global_step unless several checkpoints are given, and the Adam slots."""
        import math
        import os
        import sys
        from .. import tf_checkpoint as T
        if not checkpoints:
            return
        if not isinstance(checkpoints, (list, tuple)):
            checkpoints = [checkpoints]
        skip_global_step = len(checkpoints) > 1
        mapping = restore_to_checkpoint_mapping or self.restore_to_checkpoint_mapping
        for ck in checkpoints:
            path = self.latest_checkpoint(ck)
            if path is None or not (os.path.exists(path) or T.is_tf_checkpoint(path)):
                raise FileNotFoundError('no checkpoint found at %s' % ck)
            slots, adam_t = None, None
            if T.is_tf_checkpoint(path):
                vals, missing, unused, extra = T.load_variables(path, list(self.params), mapping)
                gstep, slots = extra['global_step'], extra['slots']
                if extra['beta1_power'] and 0 < extra['beta1_power'] < 1 and 0 < self.hparams.beta1 < 1:
                    t = int(round(math.log(extra['beta1_power']) / math.log(self.hparams.beta1))) - 1    # beta1_power = beta1^(t+1)
                    adam_t = (t, t)
            else:
                data = np.load(path)
                names = set(k[4:] for k in data.files if k.startswith('var/'))
                vals = OrderedDict((k, data['var/' + mapping(k, names)]) for k in self.params if mapping(k, names) in names)
                missing = [k for k in self.params if k not in vals]
                unused = sorted(names - set(mapping(k, names) for k in vals))
                gstep = int(data['global_step']) if 'global_step' in data.files else None
                if self.mode == 'train' and 'adam/t' in data.files:
                    for nm in ('g_m', 'g_v', 'd_m', 'd_v'):
                        buf = getattr(self, nm)
                        if ('adam/' + nm) in data.files and data['adam/' + nm].shape == tuple(buf.shape):
                            buf.copy_(torch.from_numpy(data['adam/' + nm]).to(self.device))
                    adam_t = tuple(int(v) for v in data['adam/t'])
            if missing:
                sys.stderr.write('global variables that were not restored because they are not in the checkpoint:\n' +
                                 ''.join('     %s\n' % k for k in sorted(missing)))
            if unused:
                sys.stderr.write('checkpoint variables that were not used for restoring because they are not in the graph:\n' +
                                 ''.join('     %s\n' % k for k in unused))
            self.set_params(vals)
            if not skip_global_step and gstep is not None:
                self.global_step = gstep
            if self.mode == 'train' and slots is not None:
                for slot, gbuf, dbuf in (('m', self.g_m, self.d_m), ('v', self.g_v, self.d_v)):
                    for name, arr in slots[slot].items():
                        flat, like = (self.g_flat, gbuf) if name.startswith('generator/') else (self.d_flat, dbuf)
                        if not name.endswith('/u'):
                            self._view_of(like, flat, name).copy_(torch.from_numpy(np.array(arr, order="C")).to(self.device))
            if self.mode == 'train' and adam_t is not None:
                self.g_adam_t, self.d_adam_t = adam_t

    def _flat_range(self, flat, names):
        """[lo, hi) element range of `flat` covered by the variables `names` (views of the flat buffer)."""
        lo, hi = None, None
        for n in names:
            v = self.params[n]
            o = (v.data_ptr() - flat.data_ptr()) // 4
            lo = o if lo is None else min(lo, o)
            hi = o + v.numel() if hi is None else max(hi, o + v.numel())
        return (lo or 0), (hi or 0)

    def get_params(self):
        return OrderedDict((k, v.detach().cpu().numpy()) for k, v in self.params.items())

    def _z(self, *shape):
        return torch.zeros(*shape, device=self.device, dtype=torch.float32)

    def _norm_stats(self, *lead_and_c):
        """Per-call statistics of a NormSite: [.., c, 2] (instance), [.., 2] (layer) or empty (none)."""
        lead, c = lead_and_c[:-1], lead_and_c[-1]
        return self._z(*lead, *{'instance': (c, 2), 'layer': (2,)}.get(self.hparams.norm_layer, (0,)))

    def _build_generator(self):
        hp = self.hparams
        S, NB, H, W, C, Zc = self.S, self.NB, self.H, self.W, self.C, self.Zc
        sc = 'generator/rnn/savp_cell'
        n_enc = len(self.enc_specs)
        act = self.site_act
        self.convs = []
        self.Bf = {}   # name -> stacked buffer
        Bf = self.Bf
        self.comp = comp = self.compositing(hp)
        self.nk, self.nlayers = comp['nk'], comp['L']
        self.kh, self.kw = hp.kernel_size
        self.flow = hp.transformation == 'flow' and self.nk > 0      # the flow heads
        self.cdna = hp.transformation == 'cdna' and self.nk > 0      # the CDNA kernel dense layer
        # the use_tile_concat=False sites (NormSite.zdense entries, and the ConvLSTMs' gate buffers): dense(v) is broadcast
        # into the convolution's output before it runs, for every step at once (_broadcast_z)
        self.zdense = []
        # the z segments of the tile-concat inputs: zvec is broadcast into them (_broadcast_z), and their gradients are
        # summed over space into dzvec
        self.ztiles = []
        self.gl = gl = self._generator_plan()
        self.nl = nl = len(gl)

        def slot(key, spec, seg):       # a segment of a concat buffer: (Bf key, Gb key, channel offset, cstride)
            return key, 'd' + key, spec.off(seg), spec.cstride
        for d in gl:
            li, oc, use, hh, ww = d['li'], d['oc'], d['use'], d['h'], d['w']
            sp, rsp = d['in_spec'], d.get('rin_spec')
            Bf['in%d' % li] = self._z(S, NB, d['ih'], d['iw'], sp.cstride)
            scope, _, kind, ks, pb, transposed = d['hconv']
            d['conv'] = ConvLayer(self, scope + '/kernel', scope + '/bias', (1, ks, ks), kind, (1, 2, 2), (0, pb, pb), transposed,
                                  sp, oc, prefilled=bool(Zc) and d['zin'] == 'dense')
            self.convs.append(d['conv'])
            Bf['pre%d' % li] = self._z(S, NB, hh, ww, oc)
            Bf['nst%d' % li] = self._norm_stats(S, NB, oc)
            if use:
                # c[t], the h slot of rin[t]: the state entering step t of a ConvLSTM; conv_h{li} has no state
                Bf['rin%d' % li] = self._z(S if hp.ablation_rnn else S + 1, NB, hh, ww, rsp.cstride)
                d['rconv'] = ConvLayer(self, d['rkernel'], d['rbias'], (1, 5, 5), L.WKIND_PLAIN, (1, 1, 1), (0, 2, 2), False,
                                       rsp, d['rco'], gates=not (hp.ablation_rnn or self.cell_norm),
                                       prefilled=bool(Zc) and d['zr'] == 'dense')
                self.convs.append(d['rconv'])
            if use and hp.ablation_rnn:
                Bf['rpre%d' % li] = self._z(S, NB, hh, ww, oc)
                Bf['rnst%d' % li] = self._norm_stats(S, NB, oc)
                Bf['out%d' % li] = self._z(S, NB, hh, ww, oc)
            elif use:
                Bf['gpre%d' % li] = self._z(S, NB, hh, ww, 4 * oc)
                Bf['c%d' % li] = self._z(S + 1, NB, hh, ww, oc)
                if hp.learn_initial_state:
                    Bf['h0_%d' % li] = self._z(NB, hh, ww, oc)         # the learned h state tiled over the rows
                if self.cell_norm:
                    Bf['gst1_%d' % li] = self._z(S, NB, 4 * oc, 2)
                    Bf['gst2_%d' % li] = self._z(S, NB, oc, 2)
                elif hp.ablation_conv_rnn_norm:
                    # IN(h): the layer's output, copied to its consumers; the raw h is the recurrent state only
                    Bf['out%d' % li] = self._z(S, NB, hh, ww, oc)
                    Bf['hst%d' % li] = self._z(S, NB, oc, 2)
                d['rec'] = slot('rin%d' % li, rsp, 'h')
            else:
                Bf['out%d' % li] = self._z(S, NB, hh, ww, oc)
            # the h{li} site writes the 'x' slot of the recurrent site's input, or the layer's own output
            out = ('rin%d' % li, rsp.off('x')) if use else ('out%d' % li, 0)
            d['site'] = NormSite(self, d['conv'], '%s/h%d' % (sc, li), 'in%d' % li, 'pre%d' % li, 'nst%d' % li, *out, NB, act,
                                 zname=self._zdense_name(li))
            zd = [d['site'].zdense]
            if use and hp.ablation_rnn:
                d['rsite'] = NormSite(self, d['rconv'], d['rname'], 'rin%d' % li, 'rpre%d' % li, 'rnst%d' % li, 'out%d' % li, 0,
                                      NB, act, zname=self._zdense_name(li, rnn=True))
                zd.append(d['rsite'].zdense)
            elif use and d['rconv'].prefilled:
                zd.append((self._zdense_name(li, rnn=True), Bf['gpre%d' % li], 0, 4 * oc, 'dgpre%d' % li))
            d['zdense'] = [z for z in zd if z]
            self.zdense += d['zdense']
            for form, key, spec in ((d['zin'], 'in%d' % li, sp), (d['zr'], 'rin%d' % li, rsp)):
                if Zc and form == 'tile':
                    self.ztiles.append(slot(key, spec, 'z'))
            # the consumers of the layer's output, in the order the forward writes them and the backward sums their
            # gradients: the next layer's 'x' slot (after the top layer, the heads, which read its out buffer: no forward
            # copy), the skip slot of decoder layer 2 n_enc - 1 - li, the CDNA kernel layer's flattened input.  A ConvLSTM
            # also feeds its own h slot of step t + 1 (d['rec']): first in the forward, last in the backward.
            d['wires'] = [slot('in%d' % (li + 1), gl[li + 1]['in_spec'], 'x') if li + 1 < nl else (None, 'dtop', 0, oc)]
            if li < n_enc - 1:
                j = 2 * n_enc - 1 - li
                d['wires'].append(slot('in%d' % j, gl[j]['in_spec'], 'skip'))
            if li == n_enc - 1 and self.cdna:
                d['wires'].append(('small', 'dsmall', 0, oc))
        if self.cdna:
            sl = gl[n_enc - 1]
            Bf['small'] = self._z(S, NB, sl['h'] * sl['w'] * sl['oc'])
            Bf['kraw'] = self._z(S, NB, self.kh * self.kw * self.nk)
            Bf['kern'] = self._z(S, NB, self.kh * self.kw * self.nk)
        # the masks-conv input: h_masks, then the L slots (the scratch image last)
        self.mk_spec = ConcatSpec([('hm', hp.ngf)] + [('l%d' % l, C) for l in range(self.nlayers)])
        if self.flow:
            Bf['fpre'] = self._z(S, NB, H, W, hp.ngf)
            Bf['fst'] = self._norm_stats(S, NB, hp.ngf)
            Bf['hf'] = self._z(S, NB, H, W, hp.ngf)
            Bf['flows'] = self._z(S, NB, H, W, _ceil4(2 * self.nk))
        Bf['spre'] = self._z(S, NB, H, W, hp.ngf)
        Bf['mpre'] = self._z(S, NB, H, W, hp.ngf)
        Bf['sst'] = self._norm_stats(S, NB, hp.ngf)
        Bf['mst'] = self._norm_stats(S, NB, hp.ngf)
        Bf['hs'] = self._z(S, NB, H, W, hp.ngf)
        Bf['mk'] = self._z(S, NB, H, W, self.mk_spec.cstride)
        top_spec = ConcatSpec([('x', gl[-1]['oc'])])
        hs_spec = ConcatSpec([('x', hp.ngf)])

        def head(nm, pre, stats, out, out_off=0):       # a 3x3 site on the top layer's output
            conv = ConvLayer(self, '%s/%s/conv2d/kernel' % (sc, nm), '%s/%s/conv2d/bias' % (sc, nm), (1, 3, 3), L.WKIND_PLAIN,
                             (1, 1, 1), (0, 1, 1), False, top_spec, hp.ngf)
            return NormSite(self, conv, '%s/%s' % (sc, nm), 'out%d' % (nl - 1), pre, stats, out, out_off, NB, act)
        self.scratch_site = head('h%d_scratch' % nl, 'spre', 'sst', 'hs') if comp['scratch'] else None
        self.hmasks_site = head('h%d_masks' % nl, 'mpre', 'mst', 'mk', self.mk_spec.off('hm')) if self.nlayers > 1 else None
        self.conv_scratch = self.scratch_site and self.scratch_site.conv
        self.conv_hmasks = self.hmasks_site and self.hmasks_site.conv
        self.conv_simg = self.conv_masks = None
        if comp['scratch']:
            self.conv_simg = ConvLayer(self, sc + '/scratch_image/conv2d/kernel', sc + '/scratch_image/conv2d/bias',
                                       (1, 3, 3), L.WKIND_PLAIN, (1, 1, 1), (0, 1, 1), False, hs_spec, C)
        if self.nlayers > 1:
            # independent masks read h_masks alone: the slot channels of the buffer get zero weights (cmap -1)
            msp = self.mk_spec
            mspec = msp if hp.dependent_mask else (hp.ngf, msp.cstride, list(range(hp.ngf)) + [-1] * (msp.cstride - hp.ngf))
            self.conv_masks = ConvLayer(self, sc + '/masks/conv2d/kernel', sc + '/masks/conv2d/bias', (1, 3, 3), L.WKIND_PLAIN,
                                        (1, 1, 1), (0, 1, 1), False, mspec, self.nlayers)
        self.convs += [c for c in (self.conv_scratch, self.conv_hmasks, self.conv_simg, self.conv_masks) if c is not None]
        if self.flow:
            self.hflow_site = head('h%d_flow' % nl, 'fpre', 'fst', 'hf')
            self.conv_hflow = self.hflow_site.conv
            self.conv_flows = ConvLayer(self, sc + '/flows/conv2d/kernel', sc + '/flows/conv2d/bias', (1, 3, 3), L.WKIND_PLAIN,
                                        (1, 1, 1), (0, 1, 1), False, hs_spec, 2 * self.nk)
            self.convs += [self.conv_hflow, self.conv_flows]
        self.mc = max(8, _ceil4(self.nlayers))     # channel stride of the mask logits and masks
        Bf['mlog'] = self._z(S, NB, H, W, self.mc)
        Bf['masks'] = self._z(S, NB, H, W, self.mc)
        Bf['gen'] = self._z(S, NB, H, W, 4)
        Bf['img'] = self._z(S, NB, H, W, 4)
        Bf['x'] = self._z(self.T, NB, H, W, 4)
        Bf['sel'] = torch.ones(S, NB, device=self.device, dtype=torch.int32)
        if self.D:
            # pixel distributions (savp_model.py:408-410, 598-653): ground truth, generated maps and the nlayers transformed
            # maps of every channel, each map padded to Dp channels
            Dp = _ceil4(self.D)
            Bf['pix'] = self._z(self.T, NB, H, W, Dp)
            Bf['gpix'] = self._z(S, NB, H, W, Dp)
            Bf['tpix'] = self._z(S, NB, H, W, self.nlayers * Dp)
            if self.comp['F'] > 1:      # the selected map of every step: the history of the later steps' transforms
                Bf['ppix'] = self._z(S, NB, H, W, Dp)
        if Zc:
            Bf['zvec'] = self._z(S, NB, _ceil4(Zc))
        if self.zdense:      # dense(v) of one site at a time, [S * NB, site channels]
            Bf['zw'] = self._z(S * NB, max(s[3] for s in self.zdense))
        if self.Sd:
            Bf['states'] = self._z(S, NB, self.Sd)     # ground-truth states of both unrolls
            Bf['gstates'] = self._z(S, NB, self.Sd)    # predicted states (savp_model.py:655-658)
        if hp.nz:
            nz = hp.nz
            Bf['zs'] = self._z(S, NB, nz)             # zs fed to the two unrolls (posterior | prior)
            if self.z_cell in ('lstm', 'gru'):
                Bf['zcat'] = self._z(S, NB, 2 * nz)   # [z_t, h_{t-1}] of the dense LSTM / the GRU's gates layer on z
                Bf['zgates'] = self._z(S, NB, (4 if self.z_cell == 'lstm' else 2) * nz)
                Bf['zh'] = self._z(S + 1, NB, nz)
            if self.z_cell == 'lstm':
                Bf['zc'] = self._z(S + 1, NB, nz)
            elif self.z_cell == 'gru':
                Bf['zccat'] = self._z(S, NB, 2 * nz)  # [z_t, r * h_{t-1}] of the candidate layer
                Bf['zcand'] = self._z(S, NB, nz)
            elif self.z_cell == 'fc':
                Bf['zfc'] = self._z(S, NB, nz)        # dense(z) before the tanh
            self._build_posterior()
        self._plan_packs()

    def _build_posterior(self):
        hp = self.hparams
        S, B, H, W, C, A = self.S, self.B, self.H, self.W, self.C, self.A
        sc = 'generator/encoder'
        Bf = self.Bf
        segs = [('a', C), ('b', C)] + ([('act', A)] if A else [])
        self.pair_spec = ConcatSpec(segs)
        Bf['pairs'] = self._z(S * B, H, W, self.pair_spec.cstride)
        if A:
            Bf['actions'] = self._z(S, B, A)             # the actions the posterior tile-concatenates (savp_model.py:24-26)
        self.enc_layers = []
        spec = self.pair_spec
        hh, ww = H, W
        for i in range(hp.n_layers):
            oc = hp.nef * min(2 ** i, 4)
            hh, ww = hh // 2, ww // 2
            conv = ConvLayer(self, '%s/layer_%d/conv2d/kernel' % (sc, i + 1), '%s/layer_%d/conv2d/bias' % (sc, i + 1),
                             (1, 4, 4), L.WKIND_PLAIN, (1, 2, 2), (0, 1, 1), False, spec, oc)
            self.convs.append(conv)
            Bf['epre%d' % i] = self._z(S * B, hh, ww, oc)
            el = dict(conv=conv, oc=oc, h=hh, w=ww)
            if i > 0:       # layer 1 has no norm: its leaky relu runs in the convolution's epilogue, into epre0
                Bf['eact%d' % i] = self._z(S * B, hh, ww, oc)
                Bf['est%d' % i] = self._norm_stats(S * B, oc)
                el['site'] = NormSite(self, conv, '%s/layer_%d' % (sc, i + 1), 'eact%d' % (i - 1) if i > 1 else 'epre0',
                                      'epre%d' % i, 'est%d' % i, 'eact%d' % i, 0, S * B, L.ACT_LRELU, 0.2)
            self.enc_layers.append(el)
            spec = ConcatSpec([('x', oc)])
        Bf['epool'] = self._z(S * B, self.enc_layers[-1]['oc'])
        Bf['zmu'] = self._z(S, B, hp.nz)
        Bf['zlss'] = self._z(S, B, hp.nz)
        Bf['zpost'] = self._z(S, B, hp.nz)
        Bf['eps'] = self._z(S, B, hp.nz)
        Bf['zprior'] = self._z(self.T - hp.context_frames, B, hp.nz)

    def _plan_packs(self):
        """One PackPlan over every packed buffer of the generator / encoder convolutions, built when the layers are and again
        when prepare_backward has added the dgrad buffers; runs it once to fill the new buffers."""
        self._pack_plan = L.PackPlan([job for c in self.convs for job in c.pack_jobs()])
        self._pack_all()

    def _pack_all(self):
        """Repacks every generator / encoder convolution weight (after an optimizer step or set_params): one launch."""
        self._pack_plan.run()

    # ------------------------------------------------------------------ inputs
    def set_inputs(self, inputs, noise=None, sampling=None):
        """Stages a batch: images [B,T,H,W,C] -> time-major, colour-padded, duplicated for the two
        unrolls.  noise: dict eps [T-1,B,nz], z_prior [T-context,B,nz] (time-major, as the oracle);
        sampling: bool [T-1-context, B] (or [.., 2B]: posterior | prior unroll) scheduled-sampling mask; None = drawn from
        the schedule (savp_model.py:309-334: Bernoulli(p(global_step)) in train mode, all False otherwise); False = all False."""
        hp = self.hparams
        Bf = self.Bf
        dev = self.device
        B, T, S, C = self.B, self.T, self.S, self.C
        if getattr(self, '_shard', None) is not None and int(inputs['images'].shape[0]) != B:
            inputs = {k: v[self._shard] for k, v in inputs.items()}
            noise, sampling = self._shard_noise(noise), self._shard_cols(sampling)
        imgs = torch.as_tensor(inputs['images']).to(dev, torch.float32)[:, :T]
        x = imgs.permute(1, 0, 2, 3, 4)
        Bf['x'].zero_()
        Bf['x'][:, :B, :, :, :C] = x
        if self.NB > B:
            Bf['x'][:, B:, :, :, :C] = x
        if self.A:
            act = torch.as_tensor(inputs['actions']).to(dev, torch.float32)[:, :S].permute(1, 0, 2)
            if hp.nz:        # a static buffer: the captured training step re-reads it on every replay
                Bf['actions'].copy_(act)
            Bf['zvec'][:, :B, :self.A] = act
            if self.NB > B:
                Bf['zvec'][:, B:, :self.A] = act
        if self._states_dim(inputs) != self.Sd:
            raise ValueError('the model was built %s states; the inputs must match'
                             % ('with %d-dimensional' % self.Sd if self.Sd else 'without'))
        if self.Sd:
            st = torch.as_tensor(inputs['states']).to(dev, torch.float32)[:, :S].permute(1, 0, 2)
            Bf['states'][:, :B] = st
            if self.NB > B:
                Bf['states'][:, B:] = st
        if self._pix_distribs_depth(inputs) != self.D:
            raise ValueError('the model was built %s pix_distribs; the inputs must match'
                             % ('with %d-channel' % self.D if self.D else 'without'))
        if self.D:
            pd = torch.as_tensor(inputs['pix_distribs']).to(dev, torch.float32)[:, :T].permute(1, 0, 2, 3, 4)
            Bf['pix'][:, :B, ..., :self.D] = pd
            if self.NB > B:
                Bf['pix'][:, B:, ..., :self.D] = pd
        sel = torch.ones(S, self.NB, dtype=torch.int32)
        n_free = S - hp.context_frames
        if sampling is None:
            sampling = self.draw_scheduled_sampling()
        elif sampling is False:       # explicit "never feed ground truth after the context frames"
            sampling = None
        if sampling is not None and n_free > 0:
            sm = torch.as_tensor(sampling).to(torch.int32)
            if sm.numel() == n_free * B:          # one mask for both unrolls (what the oracle takes)
                sm = sm.reshape(n_free, B)
                sm = torch.cat([sm, sm], dim=1) if self.NB > B else sm
            sel[hp.context_frames:] = sm.reshape(n_free, self.NB)
        else:
            sel[hp.context_frames:] = 0
        Bf['sel'].copy_(sel)
        if hp.nz:
            if noise is None:
                g = torch.Generator(device='cpu').manual_seed(self._seed('noise'))
                noise = dict(eps=torch.randn(S, B, hp.nz, generator=g),
                             z_prior=torch.randn(T - hp.context_frames, B, hp.nz, generator=g))
            Bf['eps'].copy_(torch.as_tensor(noise['eps']).to(dev, torch.float32))
            Bf['zprior'].copy_(torch.as_tensor(noise['z_prior']).to(dev, torch.float32))

    def redraw_step_randomness(self, noise=None, sampling=None):
        """A step on resident inputs still draws fresh eps / z_prior and a fresh scheduled-sampling mask (tf.random_normal
        / tf.multinomial are re-evaluated by every sess.run)."""
        hp, Bf = self.hparams, self.Bf
        n_free = self.S - hp.context_frames
        if self.mode == 'train' and n_free > 0 and (sampling is not None or hp.schedule_sampling != 'none'):
            if sampling is None:
                sm = self.draw_scheduled_sampling()
            else:
                sm = None if sampling is False else torch.as_tensor(sampling).to(torch.int32)
            sel = torch.ones(self.S, self.NB, dtype=torch.int32)
            if sm is None:
                sel[hp.context_frames:] = 0
            else:
                if sm.numel() == n_free * self.B and self.NB > self.B:
                    sm = torch.cat([sm.reshape(n_free, self.B)] * 2, dim=1)
                sel[hp.context_frames:] = sm.reshape(n_free, self.NB)
            Bf['sel'].copy_(sel)
        if hp.nz:
            if noise is None or 'eps' not in noise:
                g = torch.Generator(device='cpu').manual_seed(self._seed('noise'))
                noise = dict(eps=torch.randn(self.S, self.B, hp.nz, generator=g),
                             z_prior=torch.randn(self.T - hp.context_frames, self.B, hp.nz, generator=g))
            Bf['eps'].copy_(torch.as_tensor(noise['eps']).to(self.device, torch.float32))
            Bf['zprior'].copy_(torch.as_tensor(noise['z_prior']).to(self.device, torch.float32))

    def _shard_cols(self, t):
        """A [.., global batch] tensor (time-major noise / masks) -> this rank's columns."""
        if t is None or t is False or getattr(self, '_shard', None) is None:
            return t
        t = torch.as_tensor(t)
        return t[:, self._shard] if t.dim() >= 2 and t.shape[1] == self.B * self.world_size else t

    def _shard_noise(self, noise):
        """Explicit noise given for the GLOBAL batch (num_gpus > 1): eps / z_prior [T', B_global, nz] and the discriminators'
        offsets [B_global] are cut to this rank's shard like the inputs."""
        if noise is None or getattr(self, '_shard', None) is None:
            return noise
        out = {}
        for k, v in noise.items():
            if isinstance(v, dict):
                out[k] = {kk: (torch.as_tensor(vv)[self._shard] if torch.as_tensor(vv).shape[0] == self.B * self.world_size else vv)
                          for kk, vv in v.items()}
            else:
                out[k] = self._shard_cols(v)
        return out

    def _seed(self, what, extra=0):
        """Host RNG seeds: distinct per purpose, step, data-parallel rank and `extra` (e.g. discriminator scope)."""
        tag = {'noise': 1, 'sampling': 2, 'clips': 3}[what]
        return (((self.random_seed * 1000003 + self.global_step) * 4099 + getattr(self, 'rank', 0)) * 131 + tag) * 8191 + extra

    def schedule_sampling_prob(self, step=None):
        """P(feed ground truth) after the context frames (savp_model.py:313-323), evaluated on the host for `step`."""
        import math
        hp = self.hparams
        step = self.global_step if step is None else step
        if hp.schedule_sampling == 'none' or self.mode != 'train':
            return 0.0
        if hp.schedule_sampling == 'inverse_sigmoid':
            k, start = float(hp.schedule_sampling_k), hp.schedule_sampling_steps[0]
            if step < start:
                return 1.0
            e = (step - start) / k
            return k / (k + math.exp(e)) if e < 700 else 0.0
        if hp.schedule_sampling == 'linear':
            start, end = hp.schedule_sampling_steps
            st = min(max(step, start), end)
            return 1.0 - float(st - start) / float(end - start)
        raise NotImplementedError

    def draw_scheduled_sampling(self):
        """ground_truth_sampling [T-1-context, NB] (savp_model.py:309-331): Bernoulli(prob(global_step)) per (frame,
        sample), drawn independently for the two unrolls (each generator_given_z_fn builds its own SAVPCell, :689-696);
        all False once prob < 0.001 (:327-330), in test mode and for schedule 'none'.  None = all False."""
        hp = self.hparams
        prob = self.schedule_sampling_prob()
        n_free = self.S - hp.context_frames
        if prob < 0.001 or n_free <= 0:
            return None
        g = torch.Generator(device='cpu').manual_seed(self._seed('sampling'))
        return (torch.rand(n_free, self.NB, generator=g) < prob).to(torch.int32)

    # ------------------------------------------------------------------ forward
    def _posterior_forward(self):
        hp = self.hparams
        Bf = self.Bf
        S, B, H, W, C, A = self.S, self.B, self.H, self.W, self.C, self.A
        ps = self.pair_spec
        rows = S * B * H * W
        x = Bf['x']
        # image pairs concat([x_t, x_{t+1}]) (savp_model.py:23) for the first B samples of each frame
        for t in range(S):
            dst = Bf['pairs'][t * B:(t + 1) * B]
            L.copy_channels(x[t].data_ptr(), 4, dst.data_ptr() + 4 * ps.off('a'), ps.cstride, B * H * W, 4)
            L.copy_channels(x[t + 1].data_ptr(), 4, dst.data_ptr() + 4 * ps.off('b'), ps.cstride, B * H * W, 4)
        if A:
            L.broadcast_channels(Bf['actions'], A, Bf['pairs'].data_ptr() + 4 * ps.off('act'), ps.cstride, S * B, H * W, A)
        cur = Bf['pairs']
        for i, el in enumerate(self.enc_layers):
            if i == 0:
                el['conv'].fwd(cur, Bf['epre0'], act=L.ACT_LRELU, alpha=0.2)      # networks.py:17-20
                cur = Bf['epre0']
            else:
                el['site'].conv_fwd(cur, None)
                el['site'].norm_fwd(None)
                cur = Bf['eact%d' % i]
        last = self.enc_layers[-1]
        L.avgpool(cur, last['oc'], Bf['epool'], S * B, last['h'] * last['w'], last['oc'])
        P = self.params
        sc = 'generator/encoder'
        L.dense_fwd(Bf['epool'], last['oc'], P[sc + '/z_mu/dense/kernel'], P[sc + '/z_mu/dense/bias'], Bf['zmu'], hp.nz,
                    S * B, last['oc'], hp.nz)
        L.dense_fwd(Bf['epool'], last['oc'], P[sc + '/z_log_sigma_sq/dense/kernel'], P[sc + '/z_log_sigma_sq/dense/bias'],
                    Bf['zlss'], hp.nz, S * B, last['oc'], hp.nz)
        L.sample_z(Bf['zmu'], Bf['zlss'], Bf['eps'], Bf['zpost'], S * B * hp.nz)
        # zs for the two unrolls: posterior half, prior half = [z_post[:ctx-1], z_prior] (savp_model.py:724-725)
        nz = hp.nz
        zs = Bf['zs']
        for t in range(S):
            L.copy_channels(Bf['zpost'][t].data_ptr(), nz, zs[t, :B].data_ptr(), nz, B, nz)
            src = Bf['zpost'][t] if t < hp.context_frames - 1 else Bf['zprior'][t - (hp.context_frames - 1)]
            L.copy_channels(src.data_ptr(), nz, zs[t, B:].data_ptr(), nz, B, nz)

    def _rnn_z_forward(self):
        """The z cell (savp_model.py:424-432): independent of the images, so the whole chain runs first
        and every tile_concat of (actions, rnn_z) becomes one broadcast store per concat buffer."""
        hp = self.hparams
        Bf = self.Bf
        S, NB, nz, off = self.S, self.NB, hp.nz, self.A + self.Sd
        P = self.params
        Zp = _ceil4(self.Zc)
        zv = Bf['zvec'].data_ptr() + 4 * off
        if self.z_cell is None:        # use_rnn_z=False: the zs are the rnn_z lanes
            L.copy_channels(Bf['zs'].data_ptr(), nz, zv, Zp, S * NB, nz)
            return
        if self.z_cell == 'fc':        # fc_z: tanh(dense(z)) of every step at once
            b = 'generator/rnn/savp_cell/fc_z/dense'
            L.dense_fwd(Bf['zs'], nz, P[b + '/kernel'], P[b + '/bias'], Bf['zfc'], nz, S * NB, nz, nz)
            L.act_fwd(Bf['zfc'].data_ptr(), nz, zv, Zp, S * NB, nz, L.ACT_TANH)
            return
        if self.z_cell == 'gru':
            self._gru_z_forward()
            return
        b = 'generator/rnn/savp_cell/lstm_z/basic_lstm_cell'
        if hp.learn_initial_state:
            self._load_initial_states(conv=False)
        else:
            Bf['zc'][0].zero_()
            Bf['zh'][0].zero_()
        for t in range(S):
            L.copy_channels(Bf['zs'][t].data_ptr(), nz, Bf['zcat'][t].data_ptr(), 2 * nz, NB, nz)
            L.copy_channels(Bf['zh'][t].data_ptr(), nz, Bf['zcat'][t].data_ptr() + 4 * nz, 2 * nz, NB, nz)
            L.dense_fwd(Bf['zcat'][t], 2 * nz, P[b + '/kernel'], P[b + '/bias'], Bf['zgates'][t], 4 * nz, NB, 2 * nz, 4 * nz)
            L.lstm_cell_fwd(Bf['zgates'][t], Bf['zc'][t], Bf['zc'][t + 1], Bf['zh'][t + 1], NB, nz)
            L.copy_channels(Bf['zh'][t + 1].data_ptr(), nz, Bf['zvec'][t].data_ptr() + 4 * off, Zp, NB, nz)

    def _gru_z_forward(self):
        """GRUCell on z (TF >= 1.9): r, u = sigmoid([z, h] Wg + bg); h' = u h + (1 - u) tanh([z, r h] Wc + bc)."""
        Bf, P = self.Bf, self.params
        S, NB, nz, off = self.S, self.NB, self.hparams.nz, self.A + self.Sd
        b = 'generator/rnn/savp_cell/gru_z/gru_cell'
        Zp = _ceil4(self.Zc)
        if self.hparams.learn_initial_state:
            self._load_initial_states(conv=False)
        else:
            Bf['zh'][0].zero_()
        for t in range(S):
            L.copy_channels(Bf['zs'][t].data_ptr(), nz, Bf['zcat'][t].data_ptr(), 2 * nz, NB, nz)
            L.copy_channels(Bf['zh'][t].data_ptr(), nz, Bf['zcat'][t].data_ptr() + 4 * nz, 2 * nz, NB, nz)
            L.dense_fwd(Bf['zcat'][t], 2 * nz, P[b + '/gates/kernel'], P[b + '/gates/bias'], Bf['zgates'][t], 2 * nz, NB, 2 * nz,
                        2 * nz)
            L.copy_channels(Bf['zs'][t].data_ptr(), nz, Bf['zccat'][t].data_ptr(), 2 * nz, NB, nz)
            L.gru_cell_fwd(0, Bf['zgates'][t], Bf['zh'][t], None, Bf['zccat'][t].data_ptr() + 4 * nz, 2 * nz, None, NB, nz)
            L.dense_fwd(Bf['zccat'][t], 2 * nz, P[b + '/candidate/kernel'], P[b + '/candidate/bias'], Bf['zcand'][t], nz, NB,
                        2 * nz, nz)
            L.gru_cell_fwd(1, Bf['zgates'][t], Bf['zh'][t], Bf['zcand'][t], 0, 0, Bf['zh'][t + 1], NB, nz)
            L.copy_channels(Bf['zh'][t + 1].data_ptr(), nz, Bf['zvec'][t].data_ptr() + 4 * off, Zp, NB, nz)

    def _state_pred_forward(self):
        """Robot states (savp_model.py:411-412, 655-658): like rnn_z independent of the images, so one launch runs the
        recurrence of every step and row before the tile-concats; it reads the scheduled-sampling mask `sel` of this step."""
        Bf, P = self.Bf, self.params
        sc = 'generator/rnn/savp_cell/state_pred/dense'
        L.state_pred_fwd(Bf['sel'], Bf['states'], self.Sd, P[sc + '/kernel'], P[sc + '/bias'], Bf['zvec'], _ceil4(self.Zc),
                         Bf['gstates'], self.S, self.NB, self.A, self.Sd)

    def _broadcast_z(self):
        if not self.Zc:
            return
        Bf = self.Bf
        S, NB, Zc = self.S, self.NB, self.Zc
        Zp = _ceil4(Zc)
        for key, _, off, cs in self.ztiles:
            buf = Bf[key]
            L.broadcast_channels(Bf['zvec'], Zp, buf.data_ptr() + 4 * off, cs, S * NB, buf.shape[2] * buf.shape[3], Zc)
        # the sites without tile-concat: their convolution's output starts as dense(v) of its step and row, and the
        # convolution adds to it (ConvLayer.prefilled)
        for name, buf, off, c, _ in self.zdense:
            L.dense_fwd(Bf['zvec'], Zp, self.params[name], None, Bf['zw'], c, S * NB, Zc, c)
            L.broadcast_channels(Bf['zw'], c, buf.data_ptr() + 4 * off, buf.shape[-1], S * NB, buf.shape[-2] * buf.shape[-3], c)

    def _addr(self, wire, t, grad=False):
        """(address, cstride) at step t of a channel slot (Bf key, Gb key, channel offset, cstride): the forward buffer's,
        or (grad) its gradient's."""
        bufs = self.Gb if grad else self.Bf
        return bufs[wire[int(grad)]][t].data_ptr() + 4 * wire[2], wire[3]

    def _consumers(self, d, t, grad=False):
        """The slots of the consumers of generator layer d's output at step t (d['wires']): where the forward copies it,
        or (grad) the gradients the backward sums, in that order."""
        return [self._addr(w, t, grad) for w in d['wires'] if w[int(grad)]]

    def _gen_step(self, t):
        hp = self.hparams
        Bf, P = self.Bf, self.params
        NB, H, W, C = self.NB, self.H, self.W, self.C
        sc = 'generator/rnn/savp_cell'
        HW = H * W
        # image = where(ground_truth[t], x_t, gen_{t-1})  (savp_model.py:406)
        if t == 0:
            L.copy_channels(Bf['x'][0].data_ptr(), 4, Bf['img'][0].data_ptr(), 4, NB * HW, 4)
        else:
            L.select_rows(Bf['sel'][t], Bf['x'][t], Bf['gen'][t - 1], Bf['img'][t], NB, HW * 4)
        sp = self.gl[0]['in_spec']
        L.copy_channels(Bf['img'][t].data_ptr(), 4, Bf['in0'][t].data_ptr() + 4 * sp.off('image'), sp.cstride, NB * HW, 4)
        L.copy_channels(Bf['x'][0].data_ptr(), 4, Bf['in0'][t].data_ptr() + 4 * sp.off('first'), sp.cstride, NB * HW, 4)
        for d in self.gl:
            li, oc, hh, ww = d['li'], d['oc'], d['h'], d['w']
            d['site'].conv_fwd(Bf['in%d' % li][t], t)
            d['site'].norm_fwd(t)
            if d['use'] and hp.ablation_rnn:
                d['rsite'].conv_fwd(Bf['rin%d' % li][t], t)
                d['rsite'].norm_fwd(t)
            elif d['use']:
                rin, gpre, b = Bf['rin%d' % li][t], Bf['gpre%d' % li][t], d['rname']
                h = [self._addr(d['rec'], t + 1)]
                if self.cell_norm:
                    d['rconv'].fwd(rin, gpre)
                    L.lstm_gates_fwd(gpre, NB, hh * ww, oc, Bf['c%d' % li][t],
                                     P[b + '/input_transform_forget_output/gamma'], P[b + '/input_transform_forget_output/beta'],
                                     P[b + '/state/gamma'], P[b + '/state/beta'], Bf['c%d' % li][t + 1],
                                     h + self._consumers(d, t), Bf['gst1_%d' % li][t], Bf['gst2_%d' % li][t])
                    continue
                if not hp.ablation_conv_rnn_norm:
                    d['rconv'].lstm_fwd(rin, gpre, Bf['c%d' % li][t], Bf['c%d' % li][t + 1], h + self._consumers(d, t))
                    continue
                # the cell writes h, its instance norm the layer's output
                d['rconv'].lstm_fwd(rin, gpre, Bf['c%d' % li][t], Bf['c%d' % li][t + 1], h)
                nm = '%s/lstm_h%d/InstanceNorm' % (sc, li)
                L.inorm_act(*h[0], Bf['out%d' % li][t].data_ptr(), oc, NB, hh * ww, oc, P[nm + '/gamma'], P[nm + '/beta'],
                            L.ACT_NONE, 0.0, Bf['hst%d' % li][t])
            out = Bf['out%d' % li][t]
            for addr, cs in self._consumers(d, t):
                L.copy_channels(out.data_ptr(), oc, addr, cs, NB * hh * ww, oc)
        nk, kh, kw = self.nk, self.kh, self.kw
        top = Bf['out%d' % (self.nl - 1)][t]
        if self.flow:
            # flow heads (savp_model.py:522-530): h_flow = relu(IN(conv3x3(top))), flows = conv3x3(h_flow) [.., 2, nk]
            self.hflow_site.conv_fwd(top, t)
            self.hflow_site.norm_fwd(t)
            self.conv_flows.fwd(Bf['hf'][t], Bf['flows'][t], out_c=2 * nk)
        elif self.cdna:
            # cdna kernels (savp_model.py:546-559)
            small = Bf['small'][t]
            K = small.shape[1]
            Bf['kraw'][t].zero_()
            L.dense_fwd(small, K, P[sc + '/cdna_kernels/dense/kernel'], P[sc + '/cdna_kernels/dense/bias'], Bf['kraw'][t],
                        kh * kw * nk, NB, K, kh * kw * nk, k_splits=32)
            L.cdna_kernel_norm(Bf['kraw'][t], Bf['kern'][t], NB, kh, kw, nk)
        # heads: both convolutions, then both norms
        mk = Bf['mk'][t]
        msp = self.mk_spec
        heads = [s for s in (self.scratch_site, self.hmasks_site) if s]
        for s in heads:
            s.conv_fwd(top, t)
        for s in heads:
            s.norm_fwd(t)
        if self.conv_simg:      # scratch image -> last layer slot (savp_model.py:570-572, 595-596)
            self.conv_simg.fwd(Bf['hs'][t], mk, out_off=msp.off('l%d' % (self.nlayers - 1)), out_c=C, act=L.ACT_SIGMOID)
        # transformed images of the history, then the backgrounds (savp_model.py:574-594)
        frames, _ = self._history(t)
        L.slots(frames, nk, self._backgrounds(t), mk.data_ptr() + 4 * msp.off('l0'), msp.cstride, NB, H, W,
                kernels=Bf['kern'][t] if self.cdna else None, kh=kh, kw=kw, flows=Bf['flows'][t] if self.flow else None,
                flows_cs=Bf['flows'].shape[-1] if self.flow else 0)
        # masks + compositing (savp_model.py:623-646); a single layer has the mask 1 = softmax of one zero logit
        if self.conv_masks:
            self.conv_masks.fwd(mk, Bf['mlog'][t], out_c=self.nlayers)
        L.composite(Bf['mlog'][t], self.mc, mk.data_ptr() + 4 * msp.off('l0'), msp.cstride, Bf['masks'][t], self.mc, Bf['gen'][t],
                    NB * HW, self.nlayers)
        if self.D:
            # pixel distributions (savp_model.py:408-410, 598-621, 648-653): same selection, transformation and masks
            # the same slots from the maps (savp_model.py:598-621): history maps for the transforms, ground-truth maps or
            # the step's selected map (0) as backgrounds
            Dp = Bf['gpix'].shape[-1]
            pix, ppix = Bf['pix'], Bf.get('ppix')
            hist = [(ppix[s] if s >= 0 else pix[0]).data_ptr() for s in range(t - self.comp['F'] + 1, t)]
            bgs = [0 if b == 'prev' else a for b, a in zip(self.comp['bgs'], self._backgrounds(t, pix))]
            L.pix_slots_fwd(Bf['sel'][t], pix[t].data_ptr(), Dp, Bf['gpix'][t - 1].data_ptr() if t else 0, hist, nk, bgs,
                            self.comp['scratch'], Bf['masks'][t], self.mc, Bf['gpix'][t].data_ptr(), Dp, Bf['tpix'][t].data_ptr(),
                            self.nlayers * Dp, Dp, ppix[t].data_ptr() if ppix is not None else 0, NB, H, W, self.D,
                            kernels=Bf['kern'][t] if self.cdna else None, kh=kh, kw=kw,
                            flows=Bf['flows'][t] if self.flow else None, flows_cs=Bf['flows'].shape[-1] if self.flow else 0)

    def _history(self, t):
        """(device addresses, gradient addresses) of the F images the transforms of step t read, oldest first
        (savp_model.py:349-351, 407): img_s for s = t-F+1 .. t, the first ground-truth image for s < 0, which takes no
        gradient."""
        Bf = self.Bf
        F = self.comp['F']
        frames, dframes = [], []
        G = getattr(self, 'Gb', None)
        for s in range(t - F + 1, t + 1):
            frames.append(Bf['img'][s].data_ptr() if s >= 0 else Bf['x'][0].data_ptr())
            dframes.append(G['dimg'][s].data_ptr() if (G is not None and s >= 0) else 0)
        return frames, dframes

    def _backgrounds(self, t, x=None):
        """Device addresses of the background slots of step t, in slot order (savp_model.py:581-594), taken from the
        ground-truth frames x (default the images) and, for 'prev', the step's input image."""
        x, ctx = self.Bf['x'] if x is None else x, self.hparams.context_frames
        src = {'prev': self.Bf['img'][t], 'first': x[0], 'last': x[ctx - 1], 'last_context': x[t if t < ctx else ctx - 1]}
        return [(x[b[1]] if isinstance(b, tuple) else src[b]).data_ptr() for b in self.comp['bgs']]

    def _initial_state_slot(self, what, li, grad=False):
        """Where the learned initial state (what, li) of _initial_state_specs is tiled to, or (grad) where its gradient is
        summed from: the t = 0 state buffer c[0], zc[0], zh[0] or, for a ConvLSTM's h, the contiguous h0 buffer; then, for
        h, the strided h slot (d['rec']) that h0 is copied into / from, else None."""
        bufs, p = (self.Gb, 'd') if grad else (self.Bf, '')
        if what == 'h':
            return bufs[p + 'h0_%d' % li], self.gl[li]['rec']
        return bufs[p + ('c%d' % li if what == 'c' else what)][0], None

    def _load_initial_states(self, conv):
        """The learned initial states (learn_initial_state), tiled over the NB rows into the t = 0 state buffers: the ConvLSTMs'
        c[0] and the h slot of rin[0] (conv=True), or the z cell's zc[0] / zh[0] (conv=False).  Runs inside the step, so that a
        captured graph reads the variables Adam has updated."""
        for name, _, what, li in self._initial_state_specs():
            if what.startswith('z') == conv:
                continue
            v = self.params[name]
            n = v.numel()
            dst, h_slot = self._initial_state_slot(what, li)
            L.copy_channels(v.data_ptr(), 0, dst.data_ptr(), n, self.NB, n)
            if h_slot:
                d = self.gl[li]
                L.copy_channels(dst.data_ptr(), d['oc'], *self._addr(h_slot, 0), self.NB * d['h'] * d['w'], d['oc'])

    def generator_forward(self, collect=True):
        hp = self.hparams
        if hp.nz:
            self._posterior_forward()
            self._rnn_z_forward()
        if self.Sd:
            self._state_pred_forward()
        self._broadcast_z()
        if hp.learn_initial_state:
            self._load_initial_states(conv=True)
        else:
            for d in self.gl:
                if d['use'] and not hp.ablation_rnn:
                    li = d['li']
                    self.Bf['c%d' % li][0].zero_()
                    sp = d['rin_spec']
                    # h state entering step 0 is zero (zero_state, savp_model.py:344-352)
                    z = self.Bf['rin%d' % li][0]
                    z[..., sp.off('h'):sp.off('h') + d['oc']] = 0
        for t in range(self.S):
            self._gen_step(t)
        if collect:
            self._collect_outputs()

    def predict(self, inputs, noise=None):
        """sess.run(model.outputs['gen_images'], feed_dict=inputs) of generate.py:166-168: stages the batch, runs the
        generator forward with a fresh noise draw and returns gen_images [B, T-1, H, W, C] as a numpy array."""
        self.set_inputs(inputs, noise)
        self.generator_forward()
        return self.outputs['gen_images'].detach().cpu().numpy()

    def eval_outputs_and_metrics(self, inputs, num_samples=None, noise_seed=0):
        """base_model.py:132-227 (eval_outputs_and_metrics_fn) for mode 'test' / 'val': `num_samples` stochastic predictions of
        the batch (a fresh prior draw each), per-(sample, future frame) psnr / mse / ssim, and for every metric the worst /
        average / best prediction per video, chosen by the metric's mean over the future frames (sort_criterion, :168-169).
        Deterministic models (nz = 0) are evaluated once.  Returns (eval_outputs, eval_metrics) with the reference's keys,
        batch-major ([B, T-1, ...] images, [B, future] metrics); lpips / eval_diversity need downloaded weights and are absent."""
        from .. import metrics as M
        hp = self.hparams
        num_samples = 1 if self.deterministic else (num_samples or self.eval_num_samples)
        future = self.T - hp.context_frames
        images = torch.as_tensor(inputs['images']).to(self.device, torch.float32)[:, :self.T]
        target = images[:, -future:]
        acc = {}
        base_step = self.global_step
        for si in range(num_samples):
            self.global_step = noise_seed * 1000003 + si          # the host RNG seed of the prior draw mixes in global_step
            self.set_inputs(inputs)
            self.generator_forward()
            gen = self.outputs['gen_images'].clone()              # [B, T-1, H, W, C]
            pred = gen[:, -future:]
            for name, fn in M.METRIC_FNS:
                m = fn(target, pred)                              # [B, future]
                if si == 0:
                    acc[name] = dict(min=m.clone(), max=m.clone(), sum=m.clone(), gmin=gen.clone(), gmax=gen.clone(), gsum=gen.clone())
                    continue
                a = acc[name]
                crit, cmin, cmax = m.mean(dim=1), a['min'].mean(dim=1), a['max'].mean(dim=1)
                lo, hi = crit < cmin, crit > cmax
                a['min'][lo], a['gmin'][lo] = m[lo], gen[lo]
                a['max'][hi], a['gmax'][hi] = m[hi], gen[hi]
                a['sum'] += m
                a['gsum'] += gen
        self.global_step = base_step
        eval_outputs, eval_metrics = OrderedDict(eval_images=images), OrderedDict()
        for name, _ in M.METRIC_FNS:
            a = acc[name]
            if self.deterministic:
                eval_outputs['eval_gen_images'] = a['gmax']
            else:
                eval_outputs['eval_gen_images_%s/min' % name] = a['gmin']
                eval_outputs['eval_gen_images_%s/avg' % name] = a['gsum'] / float(num_samples)
                eval_outputs['eval_gen_images_%s/max' % name] = a['gmax']
            eval_metrics['eval_%s/min' % name] = a['min']
            eval_metrics['eval_%s/avg' % name] = a['sum'] / float(num_samples)
            eval_metrics['eval_%s/max' % name] = a['max']
        self.eval_outputs, self.eval_metrics = eval_outputs, eval_metrics
        return eval_outputs, eval_metrics

    def outputs_time_major(self, key):
        """One generator output straight from the device buffers, time-major as generator_fn returns it (no copy)."""
        B, C, Bf = self.B, self.C, self.Bf
        nz = bool(self.hparams.nz)
        if key == 'gen_images':
            return Bf['gen'][:, B:, ..., :C] if nz else Bf['gen'][..., :C]
        if key == 'gen_images_enc':
            return Bf['gen'][:, :B, ..., :C]
        if key == 'zs_mu_enc':
            return Bf['zmu']
        if key == 'zs_log_sigma_sq_enc':
            return Bf['zlss']
        raise KeyError(key)

    def _collect_outputs(self):
        B, C = self.B, self.C
        Bf = self.Bf
        out = OrderedDict()
        gen = Bf['gen'][..., :C]                       # [S, NB, H, W, C] time-major
        nlay = self.nlayers
        msp = self.mk_spec
        tr = torch.stack([Bf['mk'][..., msp.off('l%d' % l):msp.off('l%d' % l) + C] for l in range(nlay)], dim=-1)
        masks = Bf['masks'][..., :nlay].unsqueeze(-2)  # [S,NB,H,W,1,L]
        if self.hparams.nz:
            out['gen_images_enc'] = gen[:, :B].permute(1, 0, 2, 3, 4)
            out['gen_images'] = gen[:, B:].permute(1, 0, 2, 3, 4)
            out['transformed_images'] = tr[:, B:].permute(1, 0, 2, 3, 4, 5)
            out['masks'] = masks[:, B:].permute(1, 0, 2, 3, 4, 5)
            out['zs_mu_enc'] = Bf['zmu'].permute(1, 0, 2)
            out['zs_log_sigma_sq_enc'] = Bf['zlss'].permute(1, 0, 2)
        else:
            out['gen_images'] = gen.permute(1, 0, 2, 3, 4)
            out['transformed_images'] = tr.permute(1, 0, 2, 3, 4, 5)
            out['masks'] = masks.permute(1, 0, 2, 3, 4, 5)
        if self.Sd:
            gst = Bf['gstates'].permute(1, 0, 2)                                                   # [NB,S,Sd]
            if self.hparams.nz:
                out['gen_states_enc'] = gst[:B]
                gst = gst[B:]
            out['gen_states'] = gst
        if self.D:
            D, S, NB, H, W = self.D, self.S, self.NB, self.H, self.W
            gpix = Bf['gpix'][..., :D]                                                             # [S,NB,H,W,D]
            tpix = Bf['tpix'].view(S, NB, H, W, nlay, -1)[..., :D].transpose(-1, -2)               # [S,NB,H,W,D,L]
            if self.hparams.nz:
                out['gen_pix_distribs_enc'] = gpix[:, :B].permute(1, 0, 2, 3, 4)
                out['transformed_pix_distribs_enc'] = tpix[:, :B].permute(1, 0, 2, 3, 4, 5)
                gpix, tpix = gpix[:, B:], tpix[:, B:]
            out['gen_pix_distribs'] = gpix.permute(1, 0, 2, 3, 4)
            out['transformed_pix_distribs'] = tpix.permute(1, 0, 2, 3, 4, 5)
        self.outputs = out
        self.gen_images = out['gen_images']
