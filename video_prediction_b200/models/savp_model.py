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
    """One convolution of the path: reference-layout parameters + packed tensor-core weights."""

    def __init__(self, model, wname, bname, k, kind, stride, pad, transposed, spec, co):
        self.model, self.wname, self.bname = model, wname, bname
        self.k, self.kind, self.stride, self.pad, self.transposed = k, kind, stride, pad, transposed
        self.spec, self.co = spec, co
        self.ci_ref, self.ci_int = spec.ref_channels, spec.cstride
        if kind == L.WKIND_POOLED:
            self.ke = (1, k[1] + 1, k[2] + 1)
        elif kind == L.WKIND_UPSAMPLED:
            self.ke = (1, k[1] + 3, k[2] + 3)
        else:
            self.ke = k
        self.geom = L.geom(self.ke, stride, pad, transposed)
        self.cmap = torch.tensor(spec.cmap, dtype=torch.int32, device=model.device)
        self.wp = None
        self.n_pad = self.kc = None

    def pack(self):
        w = self.model.params[self.wname]
        self.wp, self.n_pad, self.kc = L.pack_weights(w, self.k, self.ci_ref, self.co, self.kind, L.WLAYOUT_FWD,
                                                      ci_int=self.ci_int, cmap=self.cmap, out=self.wp)
        if L.exact_mode():      # fp32-exact 3xTF32 mode: the part of the weights the TF32 rounding dropped
            self.wp_lo, _, _ = L.pack_weights(w, self.k, self.ci_ref, self.co, self.kind, L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL,
                                              ci_int=self.ci_int, cmap=self.cmap, out=getattr(self, 'wp_lo', None))

    def prepare_backward(self):
        self.geom_bwd = L.geom(self.ke, self.stride, self.pad, not self.transposed)
        self.wpd = self.dwp = None
        self.pack_bwd()
        self.dwp = torch.zeros(L.eff_taps(self.k, self.kind) * self.n_pad * self.kc * 32, device=self.model.device)

    def pack_bwd(self):
        w = self.model.params[self.wname]
        self.wpd, self.n_pad_d, self.kc_d = L.pack_weights(w, self.k, self.ci_ref, self.co, self.kind, L.WLAYOUT_DGRAD,
                                                          ci_int=self.ci_int, cmap=self.cmap, out=getattr(self, 'wpd', None))
        if L.exact_mode():
            self.wpd_lo, _, _ = L.pack_weights(w, self.k, self.ci_ref, self.co, self.kind, L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL,
                                               ci_int=self.ci_int, cmap=self.cmap, out=getattr(self, 'wpd_lo', None))

    def dgrad(self, dy, dx, dy_c=None, accumulate=False):
        """dx[.., ci_int] (+)= conv^T(dy): the same engine with the transposed flag flipped."""
        dy4 = dy.view((-1,) + tuple(dy.shape[-3:]))
        dyv = L.tensor_view(dy4, self.co if dy_c is None else dy_c)
        dxv = L.tensor_view(dx.view((-1,) + tuple(dx.shape[-3:])), self.ci_int)
        if L.exact_mode():
            conv3x(dy4, dyv.c, self.geom_bwd, self.wpd, self.wpd_lo, self.n_pad_d, self.kc_d, dxv, None, L.ACT_NONE, 0.0,
                   accumulate)
            return
        L.conv_igemm(dyv, self.geom_bwd, self.wpd, self.n_pad_d, self.kc_d, dxv, None, L.ACT_NONE, 0.0, 1 if accumulate else 0,
                     accumulate)

    def wgrad(self, x, dy, dy_c=None):
        """grads[w] += dL/dw from ONE GEMM over every position of the (time-stacked) tensors."""
        x4, dy4 = x.reshape((-1,) + tuple(x.shape[-3:])), dy.reshape((-1,) + tuple(dy.shape[-3:]))
        xv = L.tensor_view(x4, self.ci_int)
        dyv = L.tensor_view(dy4, self.co if dy_c is None else dy_c)
        self.dwp.zero_()
        L.conv_wgrad(xv, dyv, self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
        if L.exact_mode():      # + x_lo^T dy + x^T dy_lo
            L.conv_wgrad(L.tensor_view(L.tf32_residual(x4), self.ci_int), dyv, self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
            L.conv_wgrad(xv, L.tensor_view(L.tf32_residual(dy4), dyv.c), self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
        L.unpack_wgrad(self.dwp, self.k, self.ci_ref, self.co, self.kind, self.model.grads[self.wname], self.n_pad, self.kc,
                       ci_int=self.ci_int, cmap=self.cmap)

    def fwd(self, x, out, out_off=0, out_c=None, act=L.ACT_NONE, alpha=0.0, split_k=0):
        """x: stacked buffer [.., h, w, cstride] (4-D or 5-D torch tensor, leading dims folded into n)."""
        x4 = x.view((-1,) + tuple(x.shape[-3:]))
        xv = L.tensor_view(x4, self.ci_int)
        ov = L.tensor_view(out.view((-1,) + tuple(out.shape[-3:])), self.co if out_c is None else out_c, out_off)
        bias = self.model.params[self.bname] if self.bname else None
        if L.exact_mode():
            conv3x(x4, self.ci_int, self.geom, self.wp, self.wp_lo, self.n_pad, self.kc, ov, bias, act, alpha)
            return
        L.conv_igemm(xv, self.geom, self.wp, self.n_pad, self.kc, ov, bias, act, alpha, split_k)


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


class SAVPVideoPredictionModel(TrainMixin, VideoPredictionModel):
    def __init__(self, *args, **kwargs):
        super(SAVPVideoPredictionModel, self).__init__(*args, **kwargs)
        self.deterministic = not self.hparams.nz
        self.device = None
        self.params = None
        self.grads = None
        self.built = False
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
        unsupported = []
        for key, want in (('where_add', 'all'), ('use_tile_concat', True),
                          ('conv_rnn', 'lstm'), ('rnn', 'lstm'), ('conv_rnn_norm_layer', 'instance'),
                          ('norm_layer', 'instance'), ('downsample_layer', 'conv_pool2d'),
                          ('upsample_layer', 'upsample_conv2d'), ('activation_layer', 'relu'), ('last_frames', 1),
                          ('prev_image_background', True), ('first_image_background', True),
                          ('last_image_background', False), ('last_context_image_background', False),
                          ('context_images_background', False), ('generate_scratch_image', True),
                          ('dependent_mask', True), ('use_e_rnn', False), ('learn_prior', False),
                          ('learn_initial_state', False), ('ablation_conv_rnn_norm', False), ('ablation_rnn', False),
                          ('use_rnn_z', True), ('joint_gan_optimization', False), ('use_same_discriminator', False)):
            # (`repeat` is accepted with any value: train.py sets it to the dataset's time_shift (train.py:160) and no model
            #  code of the reference reads it, base_model.py:90-95)
            if getattr(hp, key) != want:
                unsupported.append('%s=%r' % (key, getattr(hp, key)))
        if hp.transformation not in ('cdna', 'flow'):
            unsupported.append('transformation=%r' % (hp.transformation,))
        if tuple(hp.dilation_rate) != (1, 1):
            unsupported.append('dilation_rate=%r' % (hp.dilation_rate,))
        if self.mode == 'train':
            # loss terms of base_model.py:733-852 that are not built: refuse instead of silently dropping them
            for key in ('vgg_cdist_weight', 'feature_l2_weight', 'ae_l2_weight', 'state_weight', 'tv_weight', 'z_l1_weight',
                        'images_sn_gan_weight', 'images_sn_vae_gan_weight', 'gan_feature_l2_weight',
                        'vae_gan_feature_l2_weight'):
                if getattr(hp, key):
                    unsupported.append('%s=%r' % (key, getattr(hp, key)))
            if hp.kl_weight and hp.kl_anneal not in ('none', 'sigmoid', 'linear'):
                unsupported.append('kl_anneal=%r' % (hp.kl_anneal,))
        if unsupported:
            raise NotImplementedError('hparams outside the H100 hot path (SURVEY.md 8f): ' + ', '.join(unsupported))

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

    def _generator_param_specs(self):
        """name -> (shape, init) with the reference's variable scopes (generator/...)."""
        hp = self.hparams
        H, W, C, A = self.H, self.W, self.C, self.A
        specs = OrderedDict()
        Zc = self.Zc
        enc, dec = self.enc_specs, self.dec_specs
        if hp.nz:
            sc = 'generator/encoder'
            cin = 2 * C + A
            for i in range(hp.n_layers):
                oc = hp.nef * min(2 ** i, 4)
                specs['%s/layer_%d/conv2d/kernel' % (sc, i + 1)] = ((4, 4, cin, oc), 'kernel')
                specs['%s/layer_%d/conv2d/bias' % (sc, i + 1)] = ((oc,), 'zeros')
                if i > 0:
                    specs['%s/layer_%d/InstanceNorm/gamma' % (sc, i + 1)] = ((oc,), 'ones')
                    specs['%s/layer_%d/InstanceNorm/beta' % (sc, i + 1)] = ((oc,), 'zeros')
                cin = oc
            for nm in ('z_mu', 'z_log_sigma_sq'):
                specs['%s/%s/dense/kernel' % (sc, nm)] = ((cin, hp.nz), 'kernel')
                specs['%s/%s/dense/bias' % (sc, nm)] = ((hp.nz,), 'zeros')
        sc = 'generator/rnn/savp_cell'
        if hp.nz:
            specs[sc + '/lstm_z/basic_lstm_cell/kernel'] = ((2 * hp.nz, 4 * hp.nz), 'kernel')
            specs[sc + '/lstm_z/basic_lstm_cell/bias'] = ((4 * hp.nz,), 'zeros')

        def norm(name, c):
            specs[name + '/gamma'] = ((c,), 'ones')
            specs[name + '/beta'] = ((c,), 'zeros')

        def lstm(i, cin, oc):
            b = '%s/lstm_h%d/basic_conv2dlstm_cell' % (sc, i)
            specs[b + '/kernel'] = ((5, 5, cin + Zc + oc, 4 * oc), 'kernel')
            norm(b + '/input_transform_forget_output', 4 * oc)
            norm(b + '/state', oc)
        outs = []
        cin = 2 * C
        for i, (oc, use) in enumerate(enc):
            ks = 5 if i == 0 else 3
            specs['%s/h%d/conv_pool2d/kernel' % (sc, i)] = ((ks, ks, cin + Zc, oc), 'kernel')
            specs['%s/h%d/conv_pool2d/bias' % (sc, i)] = ((oc,), 'zeros')
            norm('%s/h%d/InstanceNorm' % (sc, i), oc)
            if use:
                lstm(i, oc, oc)
            outs.append(oc)
            cin = oc
        n_enc = len(enc)
        for i, (oc, use) in enumerate(dec):
            li = n_enc + i
            cin = outs[-1] if i == 0 else outs[-1] + outs[n_enc - i - 1]
            specs['%s/h%d/upsample_conv2d/kernel' % (sc, li)] = ((3, 3, cin + Zc, oc), 'kernel')
            specs['%s/h%d/upsample_conv2d/bias' % (sc, li)] = ((oc,), 'zeros')
            norm('%s/h%d/InstanceNorm' % (sc, li), oc)
            if use:
                lstm(li, oc, oc)
            outs.append(oc)
        nl = n_enc + len(dec)
        kh, kw = hp.kernel_size
        nk = hp.last_frames * hp.num_transformed_images
        sh = H // (2 ** n_enc)
        sw = W // (2 ** n_enc)
        top = outs[-1]
        if hp.transformation == 'flow':         # savp_model.py:522-530: flow heads instead of the CDNA kernel dense layer
            specs['%s/h%d_flow/conv2d/kernel' % (sc, nl)] = ((3, 3, top, hp.ngf), 'kernel')
            specs['%s/h%d_flow/conv2d/bias' % (sc, nl)] = ((hp.ngf,), 'zeros')
            norm('%s/h%d_flow/InstanceNorm' % (sc, nl), hp.ngf)
            specs[sc + '/flows/conv2d/kernel'] = ((3, 3, hp.ngf, 2 * nk), 'kernel')
            specs[sc + '/flows/conv2d/bias'] = ((2 * nk,), 'zeros')
        else:
            specs[sc + '/cdna_kernels/dense/kernel'] = ((sh * sw * outs[n_enc - 1], kh * kw * nk), 'kernel')
            specs[sc + '/cdna_kernels/dense/bias'] = ((kh * kw * nk,), 'zeros')
        for nm in ('h%d_scratch' % nl, 'h%d_masks' % nl):
            specs['%s/%s/conv2d/kernel' % (sc, nm)] = ((3, 3, top, hp.ngf), 'kernel')
            specs['%s/%s/conv2d/bias' % (sc, nm)] = ((hp.ngf,), 'zeros')
            norm('%s/%s/InstanceNorm' % (sc, nm), hp.ngf)
        specs[sc + '/scratch_image/conv2d/kernel'] = ((3, 3, hp.ngf, C), 'kernel')
        specs[sc + '/scratch_image/conv2d/bias'] = ((C,), 'zeros')
        nlayers = nk + 3
        specs[sc + '/masks/conv2d/kernel'] = ((3, 3, hp.ngf + nlayers * C, nlayers), 'kernel')
        specs[sc + '/masks/conv2d/bias'] = ((nlayers,), 'zeros')
        return specs

    # ------------------------------------------------------------------ build
    def build_graph(self, inputs):
        """inputs: dict with 'images' [B,T,H,W,C] (torch / numpy, batch-major as in base_model.py:467)
        and optionally 'actions' [B,T-1,A].  Allocates parameters (reference initialisers) unless
        `set_params` was called, and all activation buffers."""
        super(SAVPVideoPredictionModel, self).build_graph(inputs)
        if not torch.cuda.is_available():
            raise RuntimeError('video_prediction_b200 needs a CUDA device (sm_90a); there is no CPU fallback')
        L.lib()  # fail loudly if the CUDA library is missing
        self._check_supported()
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
        self.S = self.T - 1
        self.Zc = self.A + (hp.nz if hp.nz else 0)
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

    def _build_generator(self):
        hp = self.hparams
        S, NB, H, W, C, Zc = self.S, self.NB, self.H, self.W, self.C, self.Zc
        sc = 'generator/rnn/savp_cell'
        enc, dec = self.enc_specs, self.dec_specs
        n_enc = len(enc)
        self.convs = []
        self.Bf = {}   # name -> stacked buffer
        Bf = self.Bf
        zseg = [('z', Zc)] if Zc else []
        self.gl = []   # per generator layer dict
        res = [(H >> (i + 1), W >> (i + 1)) for i in range(n_enc)]
        for i in range(len(dec)):
            res.append((res[n_enc - 1][0] << (i + 1), res[n_enc - 1][1] << (i + 1)))
        outs = []
        for li in range(n_enc + len(dec)):
            is_enc = li < n_enc
            oc, use = enc[li] if is_enc else dec[li - n_enc]
            hh, ww = res[li]
            ih, iw = (H, W) if li == 0 else res[li - 1]
            d = dict(li=li, oc=oc, use=use, h=hh, w=ww, is_enc=is_enc)
            if li == 0:
                segs = [('image', C), ('first', C)] + zseg
            elif is_enc or li == n_enc:
                segs = [('x', outs[-1])] + zseg
            else:
                segs = [('x', outs[-1]), ('skip', outs[n_enc - (li - n_enc) - 1])] + zseg
            d['in_spec'] = ConcatSpec(segs)
            Bf['in%d' % li] = self._z(S, NB, ih, iw, d['in_spec'].cstride)
            if is_enc:
                ks = 5 if li == 0 else 3
                pb = (ks + 1 - 2) // 2
                d['conv'] = ConvLayer(self, '%s/h%d/conv_pool2d/kernel' % (sc, li), '%s/h%d/conv_pool2d/bias' % (sc, li),
                                      (1, ks, ks), L.WKIND_POOLED, (1, 2, 2), (0, pb, pb), False, d['in_spec'], oc)
            else:
                d['conv'] = ConvLayer(self, '%s/h%d/upsample_conv2d/kernel' % (sc, li),
                                      '%s/h%d/upsample_conv2d/bias' % (sc, li), (1, 3, 3), L.WKIND_UPSAMPLED, (1, 2, 2),
                                      (0, 2, 2), True, d['in_spec'], oc)
            self.convs.append(d['conv'])
            Bf['pre%d' % li] = self._z(S, NB, hh, ww, oc)
            Bf['nst%d' % li] = self._z(S, NB, oc, 2)
            if use:
                d['rin_spec'] = ConcatSpec([('x', oc)] + zseg + [('h', oc)])
                Bf['rin%d' % li] = self._z(S + 1, NB, hh, ww, d['rin_spec'].cstride)
                b = '%s/lstm_h%d/basic_conv2dlstm_cell' % (sc, li)
                d['rconv'] = ConvLayer(self, b + '/kernel', None, (1, 5, 5), L.WKIND_PLAIN, (1, 1, 1), (0, 2, 2), False,
                                       d['rin_spec'], 4 * oc)
                d['rname'] = b
                self.convs.append(d['rconv'])
                Bf['gpre%d' % li] = self._z(S, NB, hh, ww, 4 * oc)
                Bf['c%d' % li] = self._z(S + 1, NB, hh, ww, oc)      # c[t] = state entering step t
                Bf['gst1_%d' % li] = self._z(S, NB, 4 * oc, 2)
                Bf['gst2_%d' % li] = self._z(S, NB, oc, 2)
            else:
                Bf['out%d' % li] = self._z(S, NB, hh, ww, oc)
            outs.append(oc)
            self.gl.append(d)
        nl = len(self.gl)
        self.nl = nl
        top = outs[-1]
        kh, kw = hp.kernel_size
        nk = hp.last_frames * hp.num_transformed_images
        self.nk, self.kh, self.kw = nk, kh, kw
        self.nlayers = nk + 3
        sl = self.gl[n_enc - 1]
        Bf['small'] = self._z(S, NB, sl['h'] * sl['w'] * sl['oc'])
        Bf['kraw'] = self._z(S, NB, kh * kw * nk)
        Bf['kern'] = self._z(S, NB, kh * kw * nk)
        top_spec = ConcatSpec([('x', top)])
        self.top_spec = top_spec
        self.conv_scratch = ConvLayer(self, '%s/h%d_scratch/conv2d/kernel' % (sc, nl), '%s/h%d_scratch/conv2d/bias' % (sc, nl),
                                      (1, 3, 3), L.WKIND_PLAIN, (1, 1, 1), (0, 1, 1), False, top_spec, hp.ngf)
        self.conv_hmasks = ConvLayer(self, '%s/h%d_masks/conv2d/kernel' % (sc, nl), '%s/h%d_masks/conv2d/bias' % (sc, nl),
                                     (1, 3, 3), L.WKIND_PLAIN, (1, 1, 1), (0, 1, 1), False, top_spec, hp.ngf)
        hs_spec = ConcatSpec([('x', hp.ngf)])
        self.conv_simg = ConvLayer(self, sc + '/scratch_image/conv2d/kernel', sc + '/scratch_image/conv2d/bias',
                                   (1, 3, 3), L.WKIND_PLAIN, (1, 1, 1), (0, 1, 1), False, hs_spec, C)
        self.mk_spec = ConcatSpec([('hm', hp.ngf)] + [('l%d' % l, C) for l in range(self.nlayers)])
        self.conv_masks = ConvLayer(self, sc + '/masks/conv2d/kernel', sc + '/masks/conv2d/bias', (1, 3, 3), L.WKIND_PLAIN,
                                    (1, 1, 1), (0, 1, 1), False, self.mk_spec, self.nlayers)
        self.convs += [self.conv_scratch, self.conv_hmasks, self.conv_simg, self.conv_masks]
        self.flow = hp.transformation == 'flow'
        if self.flow:
            self.conv_hflow = ConvLayer(self, '%s/h%d_flow/conv2d/kernel' % (sc, nl), '%s/h%d_flow/conv2d/bias' % (sc, nl),
                                        (1, 3, 3), L.WKIND_PLAIN, (1, 1, 1), (0, 1, 1), False, top_spec, hp.ngf)
            self.conv_flows = ConvLayer(self, sc + '/flows/conv2d/kernel', sc + '/flows/conv2d/bias', (1, 3, 3), L.WKIND_PLAIN,
                                        (1, 1, 1), (0, 1, 1), False, hs_spec, 2 * nk)
            self.convs += [self.conv_hflow, self.conv_flows]
            Bf['fpre'] = self._z(S, NB, H, W, hp.ngf)
            Bf['fst'] = self._z(S, NB, hp.ngf, 2)
            Bf['hf'] = self._z(S, NB, H, W, hp.ngf)
            Bf['flows'] = self._z(S, NB, H, W, _ceil4(2 * nk))
        Bf['spre'] = self._z(S, NB, H, W, hp.ngf)
        Bf['mpre'] = self._z(S, NB, H, W, hp.ngf)
        Bf['sst'] = self._z(S, NB, hp.ngf, 2)
        Bf['mst'] = self._z(S, NB, hp.ngf, 2)
        Bf['hs'] = self._z(S, NB, H, W, hp.ngf)
        Bf['mk'] = self._z(S, NB, H, W, self.mk_spec.cstride)
        Bf['mlog'] = self._z(S, NB, H, W, 8)
        Bf['masks'] = self._z(S, NB, H, W, 8)
        Bf['gen'] = self._z(S, NB, H, W, 4)
        Bf['img'] = self._z(S, NB, H, W, 4)
        Bf['x'] = self._z(self.T, NB, H, W, 4)
        Bf['sel'] = torch.ones(S, NB, device=self.device, dtype=torch.int32)
        if Zc:
            Bf['zvec'] = self._z(S, NB, _ceil4(Zc))
        if hp.nz:
            nz = hp.nz
            Bf['zs'] = self._z(S, NB, nz)             # zs fed to the two unrolls (posterior | prior)
            Bf['zcat'] = self._z(S, NB, 2 * nz)       # [z_t, h_{t-1}] of the dense LSTM on z
            Bf['zgates'] = self._z(S, NB, 4 * nz)
            Bf['zc'] = self._z(S + 1, NB, nz)
            Bf['zh'] = self._z(S + 1, NB, nz)
            self._build_posterior()
        self._pack_all()

    def _build_posterior(self):
        hp = self.hparams
        S, B, H, W, C, A = self.S, self.B, self.H, self.W, self.C, self.A
        sc = 'generator/encoder'
        Bf = self.Bf
        segs = [('a', C), ('b', C)] + ([('act', A)] if A else [])
        self.pair_spec = ConcatSpec(segs)
        Bf['pairs'] = self._z(S * B, H, W, self.pair_spec.cstride)
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
            if i > 0:
                Bf['eact%d' % i] = self._z(S * B, hh, ww, oc)
                Bf['est%d' % i] = self._z(S * B, oc, 2)
            self.enc_layers.append(dict(conv=conv, oc=oc, h=hh, w=ww))
            spec = ConcatSpec([('x', oc)])
        Bf['epool'] = self._z(S * B, self.enc_layers[-1]['oc'])
        Bf['zmu'] = self._z(S, B, hp.nz)
        Bf['zlss'] = self._z(S, B, hp.nz)
        Bf['zpost'] = self._z(S, B, hp.nz)
        Bf['eps'] = self._z(S, B, hp.nz)
        Bf['zprior'] = self._z(self.T - hp.context_frames, B, hp.nz)

    def _pack_all(self):
        """Repacks every generator / encoder convolution weight after an optimizer step: one table-driven launch once all
        packed buffers exist (the first call creates them layer by layer), per-layer calls in the fp32-exact mode."""
        plan = getattr(self, '_pack_plan', None)
        if plan is not None:
            plan.run()
            return
        for c in self.convs:
            c.pack()
            if getattr(c, 'wpd', None) is not None:
                c.pack_bwd()
        if not L.exact_mode() and os.environ.get('VP_PACK_BATCH', '1') == '1' and all(getattr(c, 'wpd', None) is not None for c in self.convs):
            entries = []
            for c in self.convs:
                w = self.params[c.wname]
                entries.append((w, c.k, c.ci_ref, c.co, c.kind, L.WLAYOUT_FWD, c.ci_int, c.cmap, None, c.wp))
                entries.append((w, c.k, c.ci_ref, c.co, c.kind, L.WLAYOUT_DGRAD, c.ci_int, c.cmap, None, c.wpd))
            self._pack_plan = L.PackPlan(entries)

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
            self._actions = act.contiguous()
            Bf['zvec'][:, :B, :self.A] = act
            if self.NB > B:
                Bf['zvec'][:, B:, :self.A] = act
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
            L.broadcast_channels(self._actions, A, Bf['pairs'].data_ptr() + 4 * ps.off('act'), ps.cstride, S * B, H * W, A)
        cur = Bf['pairs']
        for i, el in enumerate(self.enc_layers):
            pre = Bf['epre%d' % i]
            if i == 0:
                el['conv'].fwd(cur, pre, act=L.ACT_LRELU, alpha=0.2)      # networks.py:17-20
                cur = pre
            else:
                el['conv'].fwd(cur, pre)
                nm = 'generator/encoder/layer_%d/InstanceNorm' % (i + 1)
                L.inorm_act(pre.data_ptr(), el['oc'], Bf['eact%d' % i].data_ptr(), el['oc'], S * B, el['h'] * el['w'],
                            el['oc'], self.params[nm + '/gamma'], self.params[nm + '/beta'], L.ACT_LRELU, 0.2,
                            Bf['est%d' % i])
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
        """Dense LSTM on z (savp_model.py:424-432): independent of the images, so the whole chain runs first
        and every tile_concat of (actions, rnn_z) becomes one broadcast store per concat buffer."""
        hp = self.hparams
        Bf = self.Bf
        S, NB, nz, A = self.S, self.NB, hp.nz, self.A
        P = self.params
        b = 'generator/rnn/savp_cell/lstm_z/basic_lstm_cell'
        Zp = _ceil4(self.Zc)
        Bf['zc'][0].zero_()
        Bf['zh'][0].zero_()
        for t in range(S):
            L.copy_channels(Bf['zs'][t].data_ptr(), nz, Bf['zcat'][t].data_ptr(), 2 * nz, NB, nz)
            L.copy_channels(Bf['zh'][t].data_ptr(), nz, Bf['zcat'][t].data_ptr() + 4 * nz, 2 * nz, NB, nz)
            L.dense_fwd(Bf['zcat'][t], 2 * nz, P[b + '/kernel'], P[b + '/bias'], Bf['zgates'][t], 4 * nz, NB, 2 * nz, 4 * nz)
            L.lstm_cell_fwd(Bf['zgates'][t], Bf['zc'][t], Bf['zc'][t + 1], Bf['zh'][t + 1], NB, nz)
            L.copy_channels(Bf['zh'][t + 1].data_ptr(), nz, Bf['zvec'][t].data_ptr() + 4 * A, Zp, NB, nz)

    def _broadcast_z(self):
        if not self.Zc:
            return
        Bf = self.Bf
        S, NB, Zc = self.S, self.NB, self.Zc
        Zp = _ceil4(Zc)
        for d in self.gl:
            li = d['li']
            buf = Bf['in%d' % li]
            sp = d['in_spec']
            L.broadcast_channels(Bf['zvec'], Zp, buf.data_ptr() + 4 * sp.off('z'), sp.cstride, S * NB,
                                 buf.shape[2] * buf.shape[3], Zc)
            if d['use']:
                buf = Bf['rin%d' % li]
                sp = d['rin_spec']
                L.broadcast_channels(Bf['zvec'], Zp, buf.data_ptr() + 4 * sp.off('z'), sp.cstride, S * NB,
                                     buf.shape[2] * buf.shape[3], Zc)

    def _h_dests(self, li, t):
        """Where the output of generator layer li at step t must land (its consumers' concat slices)."""
        Bf = self.Bf
        d = self.gl[li]
        n_enc = len(self.enc_specs)
        dests = []
        if d['use'] and t + 1 <= self.S:
            sp = d['rin_spec']
            dests.append((Bf['rin%d' % li][t + 1].data_ptr() + 4 * sp.off('h'), sp.cstride))
        if li + 1 < self.nl:
            sp = self.gl[li + 1]['in_spec']
            dests.append((Bf['in%d' % (li + 1)][t].data_ptr() + 4 * sp.off('x'), sp.cstride))
        if li < n_enc - 1:       # skip connection: decoder layer n_enc + i reads layers[n_enc - i - 1]
            i = n_enc - 1 - li
            sp = self.gl[n_enc + i]['in_spec']
            dests.append((Bf['in%d' % (n_enc + i)][t].data_ptr() + 4 * sp.off('skip'), sp.cstride))
        if li == n_enc - 1 and not self.flow:     # flattened input of the CDNA kernel dense layer
            dests.append((Bf['small'][t].data_ptr(), d['oc']))
        return dests

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
            pre = Bf['pre%d' % li][t]
            d['conv'].fwd(Bf['in%d' % li][t], pre)
            nm = '%s/h%d/InstanceNorm' % (sc, li)
            if d['use']:
                rsp = d['rin_spec']
                rin = Bf['rin%d' % li][t]
                L.inorm_act(pre.data_ptr(), oc, rin.data_ptr() + 4 * rsp.off('x'), rsp.cstride, NB, hh * ww, oc,
                            P[nm + '/gamma'], P[nm + '/beta'], L.ACT_RELU, 0.0, Bf['nst%d' % li][t])
                gpre = Bf['gpre%d' % li][t]
                d['rconv'].fwd(rin, gpre)
                b = d['rname']
                L.lstm_gates_fwd(gpre, NB, hh * ww, oc, Bf['c%d' % li][t],
                                 P[b + '/input_transform_forget_output/gamma'], P[b + '/input_transform_forget_output/beta'],
                                 P[b + '/state/gamma'], P[b + '/state/beta'], Bf['c%d' % li][t + 1], self._h_dests(li, t),
                                 Bf['gst1_%d' % li][t], Bf['gst2_%d' % li][t])
            else:
                dests = self._h_dests(li, t)
                out = Bf['out%d' % li][t]
                L.inorm_act(pre.data_ptr(), oc, out.data_ptr(), oc, NB, hh * ww, oc, P[nm + '/gamma'], P[nm + '/beta'],
                            L.ACT_RELU, 0.0, Bf['nst%d' % li][t])
                for addr, cs in dests:
                    L.copy_channels(out.data_ptr(), oc, addr, cs, NB * hh * ww, oc)
        nk, kh, kw = self.nk, self.kh, self.kw
        top = Bf['out%d' % (self.nl - 1)][t] if not self.gl[-1]['use'] else None
        ngf = hp.ngf
        nl = self.nl
        if self.flow:
            # flow heads (savp_model.py:522-530): h_flow = relu(IN(conv3x3(top))), flows = conv3x3(h_flow) [.., 2, nk]
            self.conv_hflow.fwd(top, Bf['fpre'][t])
            nm = '%s/h%d_flow/InstanceNorm' % (sc, nl)
            L.inorm_act(Bf['fpre'][t].data_ptr(), ngf, Bf['hf'][t].data_ptr(), ngf, NB, HW, ngf, P[nm + '/gamma'], P[nm + '/beta'],
                        L.ACT_RELU, 0.0, Bf['fst'][t])
            self.conv_flows.fwd(Bf['hf'][t], Bf['flows'][t], out_c=2 * nk)
        else:
            # cdna kernels (savp_model.py:546-559)
            small = Bf['small'][t]
            K = small.shape[1]
            Bf['kraw'][t].zero_()
            L.dense_fwd(small, K, P[sc + '/cdna_kernels/dense/kernel'], P[sc + '/cdna_kernels/dense/bias'], Bf['kraw'][t],
                        kh * kw * nk, NB, K, kh * kw * nk, k_splits=32)
            L.cdna_kernel_norm(Bf['kraw'][t], Bf['kern'][t], NB, kh, kw, nk)
        # heads
        self.conv_scratch.fwd(top, Bf['spre'][t])
        self.conv_hmasks.fwd(top, Bf['mpre'][t])
        nm = '%s/h%d_scratch/InstanceNorm' % (sc, nl)
        L.inorm_act(Bf['spre'][t].data_ptr(), ngf, Bf['hs'][t].data_ptr(), ngf, NB, HW, ngf, P[nm + '/gamma'],
                    P[nm + '/beta'], L.ACT_RELU, 0.0, Bf['sst'][t])
        mk = Bf['mk'][t]
        msp = self.mk_spec
        nm = '%s/h%d_masks/InstanceNorm' % (sc, nl)
        L.inorm_act(Bf['mpre'][t].data_ptr(), ngf, mk.data_ptr() + 4 * msp.off('hm'), msp.cstride, NB, HW, ngf,
                    P[nm + '/gamma'], P[nm + '/beta'], L.ACT_RELU, 0.0, Bf['mst'][t])
        # scratch image -> last layer slot (savp_model.py:570-572, 595-596)
        self.conv_simg.fwd(Bf['hs'][t], mk, out_off=msp.off('l%d' % (self.nlayers - 1)), out_c=C, act=L.ACT_SIGMOID)
        # transformed images: 4 CDNA (or flow-warped) + prev image + first image (savp_model.py:574-584)
        if self.flow:
            L.flow_apply(Bf['img'][t], Bf['x'][0], Bf['flows'][t], Bf['flows'].shape[-1], mk.data_ptr() + 4 * msp.off('l0'),
                         msp.cstride, NB, H, W, nk)
        else:
            L.cdna_apply(Bf['img'][t], Bf['x'][0], Bf['kern'][t], mk.data_ptr() + 4 * msp.off('l0'), msp.cstride, NB, H, W,
                         kh, kw, nk)
        # masks + compositing (savp_model.py:623-646)
        self.conv_masks.fwd(mk, Bf['mlog'][t], out_c=self.nlayers)
        L.composite(Bf['mlog'][t], 8, mk.data_ptr() + 4 * msp.off('l0'), msp.cstride, Bf['masks'][t], 8, Bf['gen'][t],
                    NB * HW, self.nlayers)

    def generator_forward(self, collect=True):
        hp = self.hparams
        if hp.nz:
            self._posterior_forward()
            self._rnn_z_forward()
        self._broadcast_z()
        for d in self.gl:
            if d['use']:
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
        self.outputs = out
        self.gen_images = out['gen_images']
