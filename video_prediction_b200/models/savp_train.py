"""Training half of the SAVP path on H100: spectrally-normalised video discriminators, losses,
back-propagation through time over the time-stacked buffers, and the two TF-style Adam steps.

Restates the reference's single-tower training graph (base_model.py:402-516): per step
  UPDATE_OPS(u) -> D forward on {enc_real, enc_fake, real, fake} -> d_loss -> D grads -> Adam(D)
  -> D forward again with the updated weights (new clip offsets) -> g_loss_post -> G grads -> Adam(G).
All convolution gradients run on the tensor-core engine: dgrad = the same implicit GEMM with the
transposed-flag flipped and [ci][co] tap matrices; wgrad = one MN-major GEMM per layer over ALL
timesteps of the unroll at once (GEMM-K = (T-1)*NB*H*W pixels) instead of per-step accumulation."""
from __future__ import annotations

from collections import OrderedDict

import os

import numpy as np
import torch

from .. import lib as L

VIDEO_D_LAYERS = [  # networks.py:83-102: (scope, ndf multiplier, kernel, strides (t,h,w))
    ('sn_conv0_0', 1, 3, (1, 1, 1)), ('sn_conv0_1', 2, 4, (1, 2, 2)),
    ('sn_conv1_0', 2, 3, (1, 1, 1)), ('sn_conv1_1', 4, 4, (1, 2, 2)),
    ('sn_conv2_0', 4, 3, (1, 1, 1)), ('sn_conv2_1', 8, 4, (2, 2, 2)),
    ('sn_conv3_0', 8, 3, (1, 1, 1)),
]
IMAGE_D_LAYERS = [  # networks.py:45-63 (image_sn_discriminator): the 2-D analogue, applied to ONE sampled frame per video
    ('sn_conv0_0', 1, 3, (1, 1, 1)), ('sn_conv0_1', 2, 4, (1, 2, 2)),
    ('sn_conv1_0', 2, 3, (1, 1, 1)), ('sn_conv1_1', 4, 4, (1, 2, 2)),
    ('sn_conv2_0', 4, 3, (1, 1, 1)), ('sn_conv2_1', 8, 4, (1, 2, 2)),
    ('sn_conv3_0', 8, 3, (1, 1, 1)),
]

LOSS_SLOTS = ['gen_l1_loss', 'gen_l2_loss', 'gen_kl_loss']
for _kind in ('video', 'image'):
    LOSS_SLOTS += ['gen_%s_sn_gan_loss' % _kind, 'gen_%s_sn_vae_gan_loss' % _kind, 'gen_%s_sn_vae_gan_feature_cdist_loss' % _kind,
                   'gen_%s_sn_gan_feature_cdist_loss' % _kind, 'discrim_%s_sn_gan_loss' % _kind, 'discrim_%s_sn_vae_gan_loss' % _kind]


def _ceil4(v):
    return (v + 3) // 4 * 4


class SNLayer(object):
    """A spectrally-normalised conv3d (or the final dense) of the video discriminator."""

    def __init__(self, model, scope, name, k, stride, cin_ref, cin_int, cmap, co, is_fc=False, fc_in=0, two_d=False):
        self.m, self.is_fc = model, is_fc
        self.k, self.stride, self.co = k, stride, co
        self.two_d = two_d                          # image discriminator: conv2d kernels [k,k,ci,co], no temporal extent
        self.k3 = (1, k, k) if two_d else (k, k, k)
        self.cin_ref, self.cin_int = cin_ref, cin_int
        sub = 'dense' if is_fc else ('conv2d' if two_d else 'conv3d')
        self.wname = '%s/%s/%s/kernel' % (scope, name, sub)
        self.uname = '%s/%s/%s/u' % (scope, name, sub)
        self.bname = '%s/%s/%s/bias' % (scope, name, sub)
        self.rows = fc_in if is_fc else int(np.prod(self.k3)) * cin_ref
        self.cols = co
        dev = model.device
        z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float32)
        self.v, self.s, self.u_new, self.scal = z(self.rows), z(self.cols), z(self.cols), z(4)
        self.gs, self.gt = z(self.cols), z(self.rows)
        self.gwbar = z(self.rows * self.cols)
        self.u_next = z(self.cols)
        self.cmap = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device=dev)
        if not is_fc:
            pad = (0, 1, 1) if two_d else (1, 1, 1)        # tf.pad of 1 on H,W (and T for conv3d) + VALID (networks.py:38-43, 76-81)
            self.geom = L.geom(self.k3, stride, pad, False)
            self.geom_t = L.geom(self.k3, stride, pad, True)
            self.wp = self.wpd = self.dwp = None

    @property
    def sigma(self):
        return self.scal[2:3]

    def sn_forward(self):
        P = self.m.params
        L.spectral_norm_fwd(P[self.wname], P[self.uname], self.rows, self.cols, self.v, self.s, self.u_new, self.scal)

    def pack(self):
        if self.is_fc:
            return
        w = self.m.params[self.wname]
        kk = self.k3
        self.wp, self.n_pad, self.kc = L.pack_weights(w, kk, self.cin_ref, self.co, L.WKIND_PLAIN, L.WLAYOUT_FWD,
                                                      ci_int=self.cin_int, cmap=self.cmap, inv_scale=self.sigma, out=self.wp)
        self.wpd, self.n_pad_d, self.kc_d = L.pack_weights(w, kk, self.cin_ref, self.co, L.WKIND_PLAIN, L.WLAYOUT_DGRAD,
                                                          ci_int=self.cin_int, cmap=self.cmap, inv_scale=self.sigma, out=self.wpd)
        if L.exact_mode():
            self.wp_lo, _, _ = L.pack_weights(w, kk, self.cin_ref, self.co, L.WKIND_PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL,
                                              ci_int=self.cin_int, cmap=self.cmap, inv_scale=self.sigma, out=getattr(self, 'wp_lo', None))
            self.wpd_lo, _, _ = L.pack_weights(w, kk, self.cin_ref, self.co, L.WKIND_PLAIN, L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL,
                                               ci_int=self.cin_int, cmap=self.cmap, inv_scale=self.sigma, out=getattr(self, 'wpd_lo', None))
        if self.dwp is None:
            self.dwp = torch.zeros(int(np.prod(self.k3)) * self.n_pad * self.kc * 32, device=w.device)

    @property
    def cuda_core(self):
        """First layer (3 colour channels -> 32): runs on the CUDA-core kernels of csrc/discrim.cu.  With 4 channels per
        tap the generic tensor-core engine would pad every operand to 32 channels and issue one K = 8 MMA per pipeline stage
        (VP_D0_CUDA_CORE=0 selects the engine for comparison)."""
        if os.environ.get('VP_D0_CUDA_CORE', '1') != '1':
            return False
        return (not self.is_fc) and not self.two_d and self.k == 3 and tuple(self.stride) == (1, 1, 1) and self.cin_ref <= 3 and self.co == 32

    def fwd(self, x, out):
        # the first layer has its own tensor-core kernels (csrc/d0_layer.cu): float4 voxel rows are tensor-core operands as they lie
        # -- forward: overlapping rows x[v-1 .. v+2] = the K = 16 operand of a kernel row, 18 MMAs per 128 voxels against
        # 108 on the generic engine; weight gradient: the overlapping voxels of a halo row as the (dx, ci) x voxel operand.
        # The fp32-exact mode runs the generic engine (3xTF32) and the exact CUDA-core weight gradient.
        if self.cuda_core and not L.exact_mode():
            P = self.m.params
            n, d, h, w = x.shape[:4]
            if os.environ.get('VP_D0_FWD_CUDA_CORE', '0') == '1':
                L.conv3d_c4_fwd(x, P[self.wname], self.sigma, P[self.bname], out, n, d, h, w, self.cin_ref, 0.1)
                return
            if os.environ.get('VP_D0_FWD_ENGINE', '0') != '1' and L.conv3d_c4_fwd_tc_ok(h, w):
                L.conv3d_c4_fwd_tc(x, P[self.wname], self.sigma, P[self.bname], out, n, d, h, w, self.cin_ref, 0.1)
                return
        if L.exact_mode():
            from .savp_model import conv3x
            conv3x(x, self.cin_int, self.geom, self.wp, self.wp_lo, self.n_pad, self.kc, L.tensor_view(out, self.co),
                   self.m.params[self.bname], L.ACT_LRELU, 0.1)
            return
        L.conv_igemm(L.tensor_view(x, self.cin_int), self.geom, self.wp, self.n_pad, self.kc, L.tensor_view(out, self.co),
                     self.m.params[self.bname], L.ACT_LRELU, 0.1)

    def dgrad(self, dy, dx, act_y=None, addend=None):
        """dx = conv^T(dy); with act_y: dx = (conv^T(dy) + addend) * lrelu'(act_y) -- the backward of the previous
        layer's leaky relu fused into the epilogue."""
        dyv, dxv = L.tensor_view(dy, self.co), L.tensor_view(dx, self.cin_int)
        if L.exact_mode():
            from .savp_model import conv3x
            aux = None if act_y is None else (act_y.data_ptr(), addend.data_ptr() if addend is not None else 0, L.ACT_LRELU)
            conv3x(dy, self.co, self.geom_t, self.wpd, self.wpd_lo, self.n_pad_d, self.kc_d, dxv, None, L.ACT_NONE, 0.1, aux=aux)
            return
        if act_y is None:
            L.conv_igemm(dyv, self.geom_t, self.wpd, self.n_pad_d, self.kc_d, dxv, None, L.ACT_NONE, 0.0, 0)
        else:
            L.conv_igemm_actgrad(dyv, self.geom_t, self.wpd, self.n_pad_d, self.kc_d, dxv, act_y.data_ptr(),
                                 addend.data_ptr() if addend is not None else 0, L.ACT_LRELU, 0.1)

    def wgrad(self, x, dy):
        """dW += SN-backward(dL/dWbar) with dL/dWbar from the tensor-core wgrad GEMM."""
        m = self.m
        if self.cuda_core:
            n, d, h, w = x.shape[:4]
            self.gwbar.zero_()
            L.conv3d_c4_wgrad(x, dy, self.gwbar, n, d, h, w, self.cin_ref)
            self.sn_backward()
            return
        self.dwp.zero_()
        xv, dyv = L.tensor_view(x, self.cin_int), L.tensor_view(dy, self.co)
        L.conv_wgrad(xv, dyv, self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
        if L.exact_mode():
            L.conv_wgrad(L.tensor_view(L.tf32_residual(x.contiguous()), self.cin_int), dyv, self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
            L.conv_wgrad(xv, L.tensor_view(L.tf32_residual(dy.contiguous()), self.co), self.geom, self.dwp, self.n_pad, self.kc, split_k=0)
        self.gwbar.zero_()
        L.unpack_wgrad(self.dwp, self.k3, self.cin_ref, self.co, L.WKIND_PLAIN, self.gwbar, self.n_pad, self.kc,
                       ci_int=self.cin_int, cmap=self.cmap)
        self.sn_backward()

    def sn_backward(self):
        P = self.m.params
        L.spectral_norm_bwd(P[self.wname], P[self.uname], self.gwbar, self.rows, self.cols, self.v, self.s, self.scal, self.gs,
                            self.gt, self.m.grads[self.wname])


class TrainMixin(object):
    # ------------------------------------------------------------------ parameter specs
    def _d_towers(self):
        """Discriminator towers of discriminator_fn / discriminator_given_video_fn (savp_model.py:88-166): per enabled kind
        (image: one sampled frame, networks.py:35-69; video: a clip_length clip, networks.py:72-108) one tower in the root
        scope (real / fake = prior-unroll images) and, with nz > 0, one with separate weights under encoder/ (enc_real /
        enc_fake = posterior-unroll images; use_same_discriminator=False).  `images_sn_*` (per-frame discriminator over the
        whole clip) is refused in _check_supported."""
        hp = self.hparams
        towers = []
        for kind, w_gan, w_vae in (('image', hp.image_sn_gan_weight, hp.image_sn_vae_gan_weight),
                                   ('video', hp.video_sn_gan_weight, hp.video_sn_vae_gan_weight)):
            if w_gan or w_vae:
                if hp.nz:
                    towers.append(dict(scope='discriminator/encoder/' + kind, kind=kind, enc=True, weight=w_vae,
                                       cdist=hp.vae_gan_feature_cdist_weight if w_vae else 0.0, keys=('enc_real', 'enc_fake')))
                towers.append(dict(scope='discriminator/' + kind, kind=kind, enc=False, weight=w_gan,
                                   cdist=hp.gan_feature_cdist_weight if w_gan else 0.0, keys=('real', 'fake')))
        return towers

    def _d_scopes(self):
        return [t['scope'] for t in self._d_towers()]

    def _d_shapes(self, kind='video'):
        """Output dims (T',H',W',C') of the 7 conv layers for clips [clip,H,W,C] (image towers: clip = 1, no temporal taps)."""
        hp = self.hparams
        layers = VIDEO_D_LAYERS if kind == 'video' else IMAGE_D_LAYERS
        dims = (hp.clip_length if kind == 'video' else 1, self.H, self.W)
        out = []
        for name, mult, k, st in layers:
            kk, pad = ((k, k, k), (1, 1, 1)) if kind == 'video' else ((1, k, k), (0, 1, 1))
            dims = tuple((d + 2 * p - q) // s + 1 for d, p, q, s in zip(dims, pad, kk, st))
            out.append(dims + (hp.ndf * mult,))
        return out

    def _discriminator_param_specs(self):
        hp = self.hparams
        specs = OrderedDict()
        for tw in self._d_towers():
            scope, kind = tw['scope'], tw['kind']
            shapes = self._d_shapes(kind)
            layers = VIDEO_D_LAYERS if kind == 'video' else IMAGE_D_LAYERS
            sub = 'conv3d' if kind == 'video' else 'conv2d'
            cin = self.C
            for (name, mult, k, st), shp in zip(layers, shapes):
                co = hp.ndf * mult
                kshape = (k, k, k, cin, co) if kind == 'video' else (k, k, cin, co)
                specs['%s/%s/%s/kernel' % (scope, name, sub)] = (kshape, 'kernel')
                specs['%s/%s/%s/u' % (scope, name, sub)] = ((1, co), 'u')
                specs['%s/%s/%s/bias' % (scope, name, sub)] = ((co,), 'zeros')
                cin = co
            f = int(np.prod(shapes[-1]))
            specs['%s/sn_fc4/dense/kernel' % scope] = ((f, 1), 'kernel')
            specs['%s/sn_fc4/dense/u' % scope] = ((1, 1), 'u')
            specs['%s/sn_fc4/dense/bias' % scope] = ((1,), 'zeros')
        return specs

    # ------------------------------------------------------------------ build (training side)
    def _build_discriminator(self):
        hp = self.hparams
        B, H, W, C = self.B, self.H, self.W, self.C
        z = self._z
        self.dnets = OrderedDict()
        for tw in self._d_towers():
            scope, kind = tw['scope'], tw['kind']
            shapes = self._d_shapes(kind)
            layers = VIDEO_D_LAYERS if kind == 'video' else IMAGE_D_LAYERS
            clip_len = hp.clip_length if kind == 'video' else 1
            net = dict(tw, layers=[], feat=[], dfeat=[], dcd=[], clip_len=clip_len)
            cin_ref, cin_int, cmap = C, 4, list(range(C)) + [-1] * (4 - C)
            nb = 2 * B
            net['clip'] = z(nb, clip_len, H, W, 4)
            net['dclip'] = z(nb, clip_len, H, W, 4)
            for (name, mult, k, st), shp in zip(layers, shapes):
                co = hp.ndf * mult
                net['layers'].append(SNLayer(self, scope, name, k, st, cin_ref, cin_int, cmap, co, two_d=(kind == 'image')))
                net['feat'].append(z(nb, *shp))
                net['dfeat'].append(z(nb, *shp))
                net['dcd'].append(z(B, *shp))
                cin_ref, cin_int, cmap = co, co, None
            f = int(np.prod(shapes[-1]))
            net['fc'] = SNLayer(self, scope, 'sn_fc4', 1, None, f, f, None, 1, is_fc=True, fc_in=f)
            net['logits'] = z(nb)
            net['dlogits'] = z(nb)
            net['tstart'] = torch.zeros(2, B, dtype=torch.int32, device=self.device)
            self.dnets[scope] = net

    def _build_training(self):
        """Gradient buffers mirroring the forward buffers (time-stacked) + dgrad weight packs."""
        Bf, z = self.Bf, self._z
        S, NB, H, W = self.S, self.NB, self.H, self.W
        G = self.Gb = {}
        hp = self.hparams
        for d in self.gl:
            li = d['li']
            G['din%d' % li] = torch.zeros_like(Bf['in%d' % li])
            G['dpre%d' % li] = torch.zeros_like(Bf['pre%d' % li])
            if d['use']:
                G['drin%d' % li] = torch.zeros_like(Bf['rin%d' % li])
                G['dgpre%d' % li] = torch.zeros_like(Bf['gpre%d' % li])
                G['dc%d' % li] = torch.zeros_like(Bf['c%d' % li])
        ngf = hp.ngf
        G['dgen'] = z(S, NB, H, W, 4)
        G['dimg'] = z(S, NB, H, W, 4)
        G['dmlog'] = z(S, NB, H, W, 8)
        G['dlay'] = z(S, NB, H, W, 4 * self.nlayers)
        G['dmk'] = torch.zeros_like(Bf['mk'])
        G['dmpre'] = z(S, NB, H, W, ngf)
        G['dspre'] = z(S, NB, H, W, ngf)
        G['dsimg'] = z(S, NB, H, W, 4)
        G['dhs'] = z(S, NB, H, W, ngf)
        G['dtop'] = z(S, NB, H, W, self.gl[-1]['oc'])
        G['dkern'] = torch.zeros_like(Bf['kern'])
        G['dkraw'] = torch.zeros_like(Bf['kraw'])
        G['dsmall'] = torch.zeros_like(Bf['small'])
        if self.flow:
            G['dflows'] = torch.zeros_like(Bf['flows'])
            G['dhf'] = z(S, NB, H, W, ngf)
            G['dfpre'] = z(S, NB, H, W, ngf)
        if self.Zc:
            G['dzvec'] = torch.zeros_like(Bf['zvec'])
        if hp.nz:
            nz = hp.nz
            G['dzh'] = z(S + 1, NB, nz)        # gradient w.r.t. rnn_z h[t+1] (slot t+1)
            G['dzc'] = z(S + 1, NB, nz)
            G['dzgates'] = z(S, NB, 4 * nz)
            G['dzcat'] = z(S, NB, 2 * nz)
            G['dzpost'] = z(S, self.B, nz)
            G['dzmu'] = z(S, self.B, nz)
            G['dzlss'] = z(S, self.B, nz)
            G['depool'] = torch.zeros_like(Bf['epool'])
            for i, el in enumerate(self.enc_layers):
                G['depre%d' % i] = torch.zeros_like(Bf['epre%d' % i])
                if i > 0:
                    G['deact%d' % i] = torch.zeros_like(Bf['eact%d' % i])
        self.loss_vals = z(len(LOSS_SLOTS))
        self._graph, self._eager_steps = None, 0
        self.step_scalars = z(4)      # [lr_t(D), lr_t(G), kl_scale, -]  refreshed from the host every step
        self._scal_host = torch.zeros(4, dtype=torch.float32).pin_memory()
        for c in self.convs:
            c.prepare_backward()

    # ------------------------------------------------------------------ discriminator forward / backward
    def _d_sn_and_pack(self):
        for net in self.dnets.values():
            for lay in net['layers'] + [net['fc']]:
                lay.sn_forward()
                lay.pack()

    def _d_gather(self, net, which, t_real, t_fake, fake_off, rows_real=True):
        """Fills net['clip']: rows [0,B) real clip (optional), rows [B,2B) fake clip."""
        hp = self.hparams
        B, NB, HW = self.B, self.NB, self.H * self.W
        Bf = self.Bf
        if rows_real:
            L.gather_clip(Bf['x'][1:], t_real, net['clip'][:B], B, net['clip_len'], HW, NB, 0)
        L.gather_clip(Bf['gen'], t_fake, net['clip'][B:], B, net['clip_len'], HW, NB, fake_off)

    def _d_forward(self, net, r0, r1):
        """Runs the tower on clip rows [r0, r1)."""
        x = net['clip'][r0:r1]
        for lay, feat in zip(net['layers'], net['feat']):
            lay.fwd(x, feat[r0:r1])
            x = feat[r0:r1]
        fc = net['fc']
        n = r1 - r0
        net['logits'][r0:r1].zero_()
        P = self.params
        L.dense_fwd(x, fc.rows, P[fc.wname], P[fc.bname], net['logits'][r0:r1], 1, n, fc.rows, 1, k_splits=64,
                    inv_scale=fc.sigma)

    def _d_backward(self, net, r0, r1, with_wgrad, to_clip, dcd=None):
        """Back-propagates net['dlogits'][r0:r1] (and optional per-layer feature gradients dcd, rows [0, r1-r0))."""
        P, Gp = self.params, self.grads
        n = r1 - r0
        fc = net['fc']
        feats, dfeats = net['feat'], net['dfeat']
        last = feats[-1][r0:r1]
        L.dense_bwd(last, fc.rows, P[fc.wname], net['dlogits'][r0:r1], 1, n, fc.rows, 1, dx=dfeats[-1][r0:r1], dx_stride=fc.rows,
                    inv_scale=fc.sigma)
        if with_wgrad:
            fc.gwbar.zero_()
            L.dense_bwd(last, fc.rows, P[fc.wname], net['dlogits'][r0:r1], 1, n, fc.rows, 1, dw=fc.gwbar, dbias=Gp[fc.bname])
            fc.sn_backward()
        for l in range(len(feats) - 1, -1, -1):
            lay = net['layers'][l]
            y, dy = feats[l][r0:r1], dfeats[l][r0:r1]
            rows = int(np.prod(y.shape[:-1]))
            co = lay.co
            if l == len(feats) - 1:     # lower layers get their leaky-relu backward fused into the dgrad epilogue below
                extra = dcd[l][:n] if dcd is not None else None
                L.act_bwd(y.data_ptr(), co, dy.data_ptr(), co, extra.data_ptr() if extra is not None else 0, co, dy.data_ptr(), co,
                          rows, co, L.ACT_LRELU, 0.1)
            x = feats[l - 1][r0:r1] if l > 0 else net['clip'][r0:r1]
            if with_wgrad:
                L.colsum(dy.data_ptr(), co, Gp[lay.bname], 1, rows, co)
                lay.wgrad(x, dy)
            if l > 0:
                lay.dgrad(dy, dfeats[l - 1][r0:r1], act_y=feats[l - 1][r0:r1], addend=dcd[l - 1][:n] if dcd is not None else None)
            elif to_clip:
                lay.dgrad(dy, net['dclip'][r0:r1])

    # ------------------------------------------------------------------ generator backward
    def _gen_backward_step(self, t):
        hp = self.hparams
        Bf, G, P, Gp = self.Bf, self.Gb, self.params, self.grads
        NB, H, W, C = self.NB, self.H, self.W, self.C
        HW = H * W
        S = self.S
        sc = 'generator/rnn/savp_cell'
        nl, ngf = self.nl, hp.ngf
        msp = self.mk_spec
        mk, dmk = Bf['mk'][t], G['dmk'][t]
        nlay = self.nlayers
        # compositing + masks conv
        L.composite_bwd(G['dgen'][t], Bf['masks'][t], 8, mk.data_ptr() + 4 * msp.off('l0'), msp.cstride, G['dmlog'][t], 8,
                        G['dlay'][t], 4 * nlay, NB * HW, nlay)
        self.conv_masks.dgrad(G['dmlog'][t], dmk, dy_c=nlay)
        # h_masks branch
        nm = '%s/h%d_masks/InstanceNorm' % (sc, nl)
        L.inorm_act_bwd(Bf['mpre'][t].data_ptr(), ngf, [(dmk.data_ptr() + 4 * msp.off('hm'), msp.cstride)], G['dmpre'][t].data_ptr(),
                        ngf, NB, HW, ngf, P[nm + '/gamma'], P[nm + '/beta'], Bf['mst'][t], L.ACT_RELU, 0.0, Gp[nm + '/gamma'],
                        Gp[nm + '/beta'])
        self.conv_hmasks.dgrad(G['dmpre'][t], G['dtop'][t])
        # scratch branch
        so = msp.off('l%d' % (nlay - 1))
        L.act_bwd(mk.data_ptr() + 4 * so, msp.cstride, dmk.data_ptr() + 4 * so, msp.cstride,
                  G['dlay'][t].data_ptr() + 4 * 4 * (nlay - 1), 4 * nlay, G['dsimg'][t].data_ptr(), 4, NB * HW, C, L.ACT_SIGMOID)
        self.conv_simg.dgrad(G['dsimg'][t], G['dhs'][t], dy_c=C)
        nm = '%s/h%d_scratch/InstanceNorm' % (sc, nl)
        L.inorm_act_bwd(Bf['spre'][t].data_ptr(), ngf, [(G['dhs'][t].data_ptr(), ngf)], G['dspre'][t].data_ptr(), ngf, NB, HW, ngf,
                        P[nm + '/gamma'], P[nm + '/beta'], Bf['sst'][t], L.ACT_RELU, 0.0, Gp[nm + '/gamma'], Gp[nm + '/beta'])
        self.conv_scratch.dgrad(G['dspre'][t], G['dtop'][t], accumulate=True)
        nk, kh, kw = self.nk, self.kh, self.kw
        G['dimg'][t].zero_()
        if self.flow:
            # flow warps (flow_ops.py:4-79) -> flows conv -> h_flow instance norm -> h_flow conv (savp_model.py:522-530)
            L.flow_apply_bwd(Bf['img'][t], Bf['flows'][t], Bf['flows'].shape[-1], dmk.data_ptr() + 4 * msp.off('l0'), msp.cstride,
                             G['dlay'][t].data_ptr(), 4 * nlay, G['dimg'][t], G['dflows'][t], NB, H, W, nk)
            self.conv_flows.dgrad(G['dflows'][t], G['dhf'][t], dy_c=2 * nk)
            nm = '%s/h%d_flow/InstanceNorm' % (sc, nl)
            L.inorm_act_bwd(Bf['fpre'][t].data_ptr(), ngf, [(G['dhf'][t].data_ptr(), ngf)], G['dfpre'][t].data_ptr(), ngf, NB, HW, ngf,
                            P[nm + '/gamma'], P[nm + '/beta'], Bf['fst'][t], L.ACT_RELU, 0.0, Gp[nm + '/gamma'], Gp[nm + '/beta'])
            self.conv_hflow.dgrad(G['dfpre'][t], G['dtop'][t], accumulate=True)
        else:
            # CDNA
            G['dkern'][t].zero_()
            L.cdna_apply_bwd(Bf['img'][t], Bf['kern'][t], dmk.data_ptr() + 4 * msp.off('l0'), msp.cstride, G['dlay'][t].data_ptr(),
                             4 * nlay, G['dimg'][t], G['dkern'][t], NB, H, W, kh, kw, nk)
            L.cdna_kernel_norm_bwd(Bf['kraw'][t], Bf['kern'][t], G['dkern'][t], G['dkraw'][t], NB, kh, kw, nk)
            K = Bf['small'].shape[-1]
            dn = sc + '/cdna_kernels/dense'
            # dx only; dW / dbias of this layer are one GEMM over all time steps in _gen_backward_params
            L.dense_bwd(Bf['small'][t], K, P[dn + '/kernel'], G['dkraw'][t], kh * kw * nk, NB, K, kh * kw * nk, dx=G['dsmall'][t],
                        dx_stride=K)
        # encoder/decoder stack in reverse
        n_enc = len(self.enc_specs)
        for li in range(nl - 1, -1, -1):
            d = self.gl[li]
            oc, hh, ww = d['oc'], d['h'], d['w']
            srcs = []
            if li == nl - 1:
                srcs.append((G['dtop'][t].data_ptr(), oc))
            else:
                sp = self.gl[li + 1]['in_spec']
                srcs.append((G['din%d' % (li + 1)][t].data_ptr() + 4 * sp.off('x'), sp.cstride))
            if li < n_enc - 1:
                i = n_enc - 1 - li
                sp = self.gl[n_enc + i]['in_spec']
                srcs.append((G['din%d' % (n_enc + i)][t].data_ptr() + 4 * sp.off('skip'), sp.cstride))
            if li == n_enc - 1 and not self.flow:
                srcs.append((G['dsmall'][t].data_ptr(), oc))
            nm = '%s/h%d/InstanceNorm' % (sc, li)
            if d['use']:
                rsp = d['rin_spec']
                if t + 1 < S:
                    srcs.append((G['drin%d' % li][t + 1].data_ptr() + 4 * rsp.off('h'), rsp.cstride))
                b = d['rname']
                L.lstm_gates_bwd(Bf['gpre%d' % li][t], NB, hh * ww, oc, Bf['c%d' % li][t],
                                 P[b + '/input_transform_forget_output/gamma'], P[b + '/input_transform_forget_output/beta'],
                                 P[b + '/state/gamma'], P[b + '/state/beta'], Bf['gst1_%d' % li][t], Bf['gst2_%d' % li][t], srcs,
                                 G['dc%d' % li][t + 1] if t + 1 < S else None, G['dgpre%d' % li][t], G['dc%d' % li][t],
                                 Gp[b + '/input_transform_forget_output/gamma'], Gp[b + '/input_transform_forget_output/beta'],
                                 Gp[b + '/state/gamma'], Gp[b + '/state/beta'])
                d['rconv'].dgrad(G['dgpre%d' % li][t], G['drin%d' % li][t])
                srcs = [(G['drin%d' % li][t].data_ptr() + 4 * rsp.off('x'), rsp.cstride)]
            L.inorm_act_bwd(Bf['pre%d' % li][t].data_ptr(), oc, srcs, G['dpre%d' % li][t].data_ptr(), oc, NB, hh * ww, oc,
                            P[nm + '/gamma'], P[nm + '/beta'], Bf['nst%d' % li][t], L.ACT_RELU, 0.0, Gp[nm + '/gamma'],
                            Gp[nm + '/beta'])
            d['conv'].dgrad(G['dpre%d' % li][t], G['din%d' % li][t])
        # gradient w.r.t. the input image of this step: CDNA path + first conv's 'image' slot
        sp = self.gl[0]['in_spec']
        L.axpy_channels(G['din0'][t].data_ptr() + 4 * sp.off('image'), sp.cstride, G['dimg'][t].data_ptr(), 4, NB * HW, 4)
        if t > 0:   # image_t was gen_{t-1} wherever ground truth was not used (sel == 0)
            L.axpy_channels(G['dimg'][t].data_ptr(), 4, G['dgen'][t - 1].data_ptr(), 4, NB * HW, 4, row_mask=Bf['sel'][t],
                            rows_per_mask=HW)

    def _gen_backward_params(self, red=None):
        """Time-batched weight/bias gradients + the z path (dense LSTM on z, posterior encoder).  With a GradientReducer
        (data parallel) every generator layer's slice of the flat gradient buffer is all-reduced as soon as it is final, under
        the weight-gradient GEMMs of the following layers; the remainder goes at the end."""
        done = []                                    # [lo, hi) ranges already exchanged
        self._gen_backward_params_body(red, done)
        if red is not None:
            pos = 0
            for lo, hi in sorted(done) + [(self.g_flat.numel(), self.g_flat.numel())]:
                red.reduce_range(self.g_grad, pos, lo)
                pos = max(pos, hi)

    def _gen_backward_params_body(self, red, done):
        hp = self.hparams
        Bf, G, P, Gp = self.Bf, self.Gb, self.params, self.grads
        S, NB, B, H, W, C = self.S, self.NB, self.B, self.H, self.W, self.C
        rows_top = S * NB * H * W
        sc_cell = 'generator/rnn/savp_cell'
        for d in self.gl:
            li = d['li']
            d['conv'].wgrad(Bf['in%d' % li], G['dpre%d' % li])
            L.colsum(G['dpre%d' % li].data_ptr(), d['oc'], Gp[d['conv'].bname], 1, S * NB * d['h'] * d['w'], d['oc'])
            if d['use']:
                d['rconv'].wgrad(Bf['rin%d' % li][:S], G['dgpre%d' % li])
            if red is not None:
                pre = ('%s/h%d/' % (sc_cell, li), '%s/lstm_h%d/' % (sc_cell, li))
                lo, hi = self._flat_range(self.g_flat, [k for k in P if k.startswith(pre)])
                red.reduce_range(self.g_grad, lo, hi)
                done.append((lo, hi))
        top = Bf['out%d' % (self.nl - 1)]
        ngf = hp.ngf
        self.conv_scratch.wgrad(top, G['dspre'])
        L.colsum(G['dspre'].data_ptr(), ngf, Gp[self.conv_scratch.bname], 1, rows_top, ngf)
        self.conv_hmasks.wgrad(top, G['dmpre'])
        L.colsum(G['dmpre'].data_ptr(), ngf, Gp[self.conv_hmasks.bname], 1, rows_top, ngf)
        self.conv_simg.wgrad(Bf['hs'], G['dsimg'], dy_c=C)
        L.colsum(G['dsimg'].data_ptr(), 4, Gp[self.conv_simg.bname], 1, rows_top, C)
        self.conv_masks.wgrad(Bf['mk'], G['dmlog'], dy_c=self.nlayers)
        L.colsum(G['dmlog'].data_ptr(), 8, Gp[self.conv_masks.bname], 1, rows_top, self.nlayers)
        if self.flow:
            self.conv_hflow.wgrad(top, G['dfpre'])
            L.colsum(G['dfpre'].data_ptr(), ngf, Gp[self.conv_hflow.bname], 1, rows_top, ngf)
            self.conv_flows.wgrad(Bf['hf'], G['dflows'], dy_c=2 * self.nk)
            L.colsum(G['dflows'].data_ptr(), G['dflows'].shape[-1], Gp[self.conv_flows.bname], 1, rows_top, 2 * self.nk)
        else:
            # CDNA kernel dense layer: dW = sum over all time steps of small_t^T dkraw_t, one launch
            Kd = Bf['small'].shape[-1]
            dn = 'generator/rnn/savp_cell/cdna_kernels/dense'
            nkk = self.kh * self.kw * self.nk
            L.dense_bwd(Bf['small'], Kd, P[dn + '/kernel'], G['dkraw'], nkk, S * NB, Kd, nkk, dw=Gp[dn + '/kernel'], dbias=Gp[dn + '/bias'])
        if not self.Zc:
            return
        # tile_concat adjoint: sum the z-slot gradients of every concat buffer over space
        Zc, Zp = self.Zc, _ceil4(self.Zc)
        G['dzvec'].zero_()
        for d in self.gl:
            li = d['li']
            for key, spn in (('din%d' % li, 'in_spec'), ('drin%d' % li, 'rin_spec')):
                if spn == 'rin_spec' and not d['use']:
                    continue
                buf = G[key][:S]
                sp = d[spn]
                L.colsum(buf.data_ptr() + 4 * sp.off('z'), sp.cstride, G['dzvec'], S * NB, buf.shape[2] * buf.shape[3], Zc, out_stride=Zp)
        if not hp.nz:
            return
        nz, A = hp.nz, self.A
        b = 'generator/rnn/savp_cell/lstm_z/basic_lstm_cell'
        G['dzh'].zero_()
        for t in range(S - 1, -1, -1):
            # dh[t+1] = z-slot gradient (rnn_z part) + recurrent part already accumulated in dzh[t+1]
            L.axpy_channels(G['dzvec'][t].data_ptr() + 4 * A, Zp, G['dzh'][t + 1].data_ptr(), nz, NB, nz)
            L.lstm_cell_bwd(Bf['zgates'][t], Bf['zc'][t], Bf['zc'][t + 1], G['dzh'][t + 1], G['dzc'][t + 1] if t + 1 < S else None,
                            G['dzgates'][t], G['dzc'][t], NB, nz)
            L.dense_bwd(Bf['zcat'][t], 2 * nz, P[b + '/kernel'], G['dzgates'][t], 4 * nz, NB, 2 * nz, 4 * nz, dx=G['dzcat'][t],
                        dx_stride=2 * nz, dw=Gp[b + '/kernel'], dbias=Gp[b + '/bias'])
            L.axpy_channels(G['dzcat'][t].data_ptr() + 4 * nz, 2 * nz, G['dzh'][t].data_ptr(), nz, NB, nz)
        # dzs -> posterior sample: posterior half always, prior half for the context steps (savp_model.py:724-725)
        for t in range(S):
            L.axpy_channels(G['dzcat'][t, :B].data_ptr(), 2 * nz, G['dzpost'][t].data_ptr(), nz, B, nz, accumulate=False)
            if t < hp.context_frames - 1:
                L.axpy_channels(G['dzcat'][t, B:].data_ptr(), 2 * nz, G['dzpost'][t].data_ptr(), nz, B, nz)
        L.sample_z_bwd(Bf['zmu'], Bf['zlss'], Bf['eps'], G['dzpost'], G['dzmu'], G['dzlss'], S * B * nz, self.step_scalars[2:3])
        sc = 'generator/encoder'
        last = self.enc_layers[-1]
        oc = last['oc']
        L.dense_bwd(Bf['epool'], oc, P[sc + '/z_mu/dense/kernel'], G['dzmu'], nz, S * B, oc, nz, dx=G['depool'], dx_stride=oc,
                    dw=Gp[sc + '/z_mu/dense/kernel'], dbias=Gp[sc + '/z_mu/dense/bias'])
        L.dense_bwd(Bf['epool'], oc, P[sc + '/z_log_sigma_sq/dense/kernel'], G['dzlss'], nz, S * B, oc, nz, dx=G['depool'],
                    dx_stride=oc, dx_accumulate=True, dw=Gp[sc + '/z_log_sigma_sq/dense/kernel'],
                    dbias=Gp[sc + '/z_log_sigma_sq/dense/bias'])
        n_l = len(self.enc_layers)
        for i in range(n_l - 1, -1, -1):
            el = self.enc_layers[i]
            oc, pos = el['oc'], el['h'] * el['w']
            if i == n_l - 1:
                dact = G['deact%d' % i] if i > 0 else G['depre0']
                L.avgpool_bwd(G['depool'], dact, oc, S * B, pos, oc)
            if i > 0:
                nm = '%s/layer_%d/InstanceNorm' % (sc, i + 1)
                L.inorm_act_bwd(Bf['epre%d' % i].data_ptr(), oc, [(G['deact%d' % i].data_ptr(), oc)], G['depre%d' % i].data_ptr(), oc,
                                S * B, pos, oc, P[nm + '/gamma'], P[nm + '/beta'], Bf['est%d' % i], L.ACT_LRELU, 0.2,
                                Gp[nm + '/gamma'], Gp[nm + '/beta'])
                x_in = Bf['eact%d' % (i - 1)] if i > 1 else Bf['epre0']
                dst = G['deact%d' % (i - 1)] if i > 1 else G['depre0']
                el['conv'].dgrad(G['depre%d' % i], dst)
            else:
                # layer 1 stored the lrelu OUTPUT (activation fused in the conv epilogue)
                L.act_bwd(Bf['epre0'].data_ptr(), oc, G['depre0'].data_ptr(), oc, 0, oc, G['depre0'].data_ptr(), oc, S * B * pos, oc,
                          L.ACT_LRELU, 0.2)
                x_in = Bf['pairs']
            el['conv'].wgrad(x_in, G['depre%d' % i])
            L.colsum(G['depre%d' % i].data_ptr(), oc, Gp[el['conv'].bname], 1, S * B * pos, oc)

    # ------------------------------------------------------------------ one optimisation step
    def _slot(self, name):
        return self.loss_vals[LOSS_SLOTS.index(name):LOSS_SLOTS.index(name) + 1]

    def _set_tstarts(self, noise):
        """Clip offsets t_start[B] in [0, T-1-clip_length] (video towers) / frame indices t_sample[B] in [0, T-2] (image towers)
        of the two discriminator_fn instantiations (pre / post D update; savp_model.py:93-98).  `noise[which][key]` (as the
        oracle takes them: 'real', 'fake', 'enc_real', 'enc_fake' for video, 'image_*' for image towers) overrides the draw."""
        for ti, (scope, net) in enumerate(self.dnets.items()):
            hi = self.S - net['clip_len'] + 1
            for w, which in enumerate(('d_pre', 'd_post')):
                for r, key in enumerate(net['keys']):
                    nkey = key if net['kind'] == 'video' else 'image_' + key
                    if noise is not None and which in noise and nkey in noise[which]:
                        v = torch.as_tensor(noise[which][nkey]).to(torch.int32)
                    else:
                        g = torch.Generator().manual_seed(self._seed('clips', 8 * ti + 2 * w + r))
                        v = torch.randint(0, hi, (self.B,), generator=g, dtype=torch.int32)
                    if 'ts' not in net:
                        net['ts'] = {(a, b): torch.zeros(self.B, dtype=torch.int32, device=self.device)
                                     for a in ('d_pre', 'd_post') for b in (0, 1)}
                    net['ts'][(which, r)].copy_(v)

    def stage_step(self, noise=None):
        """Host-side staging of one step: step-dependent scalars (lr_t, KL weight) and the discriminators' random
        clip offsets are written into static device buffers, so the device part can be a replayed CUDA graph."""
        self._stage_step_scalars()
        if self.dnets:
            self._set_tstarts(noise)

    def train_step(self, inputs=None, noise=None, sampling=None, allreduce=None, staged=False):
        """One optimisation step (D then G, base_model.py:477-516); loss values are left on the device (`losses()`).
        `allreduce(flat_grad)` (optional) is called on the flat discriminator / generator gradient buffers before
        their Adam steps (data parallel, tf_utils.py:450-480).  staged=True: `stage_step()` was already called and
        the caller advances `global_step` (used when the device part is captured into a CUDA graph)."""
        if allreduce is None:
            allreduce = getattr(self, '_allreduce', None)     # data parallel under torchrun (dp.make_allreduce)
        if inputs is not None:
            self.set_inputs(inputs, noise, sampling)
        elif not staged:
            self.redraw_step_randomness(noise, sampling)      # resident inputs: fresh eps / z_prior / sampling mask per step
        if not staged:
            self.stage_step(self._shard_noise(noise))
        if self.use_cuda_graph and not staged and self._eager_steps >= 1 and not L.exact_mode():
            # the device part of the step (~1.5 k launches, no host sync) is captured once and replayed
            if self._graph is None:
                try:
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        self._step_device(allreduce)
                    self._graph = g
                    g.replay()               # capturing only records: this step still has to run
                except Exception as ex:      # noqa: BLE001  (e.g. a collective that cannot be captured): stay eager
                    import sys
                    sys.stderr.write('CUDA graph capture failed (%s); continuing with eager launches\n' % ex)
                    self.use_cuda_graph, self._graph = False, None
                    torch.cuda.synchronize()
                    self._step_device(allreduce)
            else:
                self._graph.replay()
        else:
            self._step_device(allreduce)
            self._eager_steps += 1
        if not staged:
            self.global_step += 1

    def _run_concurrent(self, fns):
        """Runs independent pieces of the step (the two discriminator towers) on forked streams: inside the captured CUDA
        graph they become parallel branches, so the many sub-wave kernels of one tower fill the SMs the other leaves idle.
        Every callable only touches its own tower's buffers, disjoint parameter/gradient ranges and its own loss slots."""
        if len(fns) < 2 or os.environ.get('VP_CONCURRENT_D', '1') != '1':
            for fn in fns:
                fn()
            return
        main = torch.cuda.current_stream()
        if not hasattr(self, '_side_streams'):
            self._side_streams = []
        while len(self._side_streams) < len(fns) - 1:
            self._side_streams.append(torch.cuda.Stream(device=self.device))
        side = self._side_streams[:len(fns) - 1]
        for st in side:
            st.wait_stream(main)
        fns[0]()
        for fn, st in zip(fns[1:], side):
            with torch.cuda.stream(st):
                fn()
        for st in side:
            main.wait_stream(st)

    def _step_device(self, allreduce=None):
        hp = self.hparams
        Bf, G, P = self.Bf, self.Gb, self.params
        B, NB, S, C = self.B, self.NB, self.S, self.C
        HW = self.H * self.W
        self.loss_vals.zero_()
        has_d = bool(self.dnets)
        world = float(self.world_size)
        red = getattr(self, '_reducer', None) if allreduce is not None else None     # bucketed, overlapped all-reduce (dp.py)

        def d_prepare(net):
            # spectral norm + weight packing of one tower (dozens of tiny dependent launches): independent of the generator
            # forward, so it runs as a parallel graph branch underneath it
            for lay in net['layers'] + [net['fc']]:
                lay.sn_forward()
                lay.pack()
                lay.u_next.copy_(lay.u_new)     # UPDATE_OPS (ops.py:1046-1048): u' of the start-of-step weights

        self._run_concurrent([lambda: self.generator_forward(collect=False)] +
                             [(lambda nt=nt: d_prepare(nt)) for nt in self.dnets.values()])
        if has_d:
            self.d_grad.zero_()
            def d_step_tower(scope, net):
                enc, w, kind = net['enc'], net['weight'], net['kind']
                if not w:
                    return      # the reference builds the tower but no loss term reads it (base_model.py:831-852)
                self._d_gather(net, 'pre', net['ts'][('d_pre', 0)], net['ts'][('d_pre', 1)], 0 if enc else (B if hp.nz else 0))
                self._d_forward(net, 0, 2 * B)
                slot = self._slot('discrim_%s_sn_%sgan_loss' % (kind, 'vae_' if enc else ''))
                L.gan_loss(net['logits'][:B], 1.0, B, w, hp.gan_loss_type, net['dlogits'][:B], slot)
                L.gan_loss(net['logits'][B:], 0.0, B, w, hp.gan_loss_type, net['dlogits'][B:], slot)
                self._d_backward(net, 0, 2 * B, with_wgrad=True, to_clip=False)
                if red is not None:      # this tower's gradients are final: exchange them under the other towers' backward
                    lo, hi = self._flat_range(self.d_flat, [k for k in self.params if k.startswith(scope + '/') and not k.endswith('/u')])
                    red.reduce_range(self.d_grad, lo, hi)
            self._run_concurrent([(lambda sc=sc, nt=nt: d_step_tower(sc, nt)) for sc, nt in self.dnets.items()])
            if red is not None:
                red.join()
            elif allreduce is not None:
                allreduce(self.d_grad)
            L.adam(self.d_flat, self.d_grad, self.d_m, self.d_v, self.d_flat.numel(), self.step_scalars[0:1], hp.beta1, hp.beta2,
                   1.0 / world)
            # post-update discriminator forward (fresh reads of the updated variables, tf_utils.replace_read_ops)
            self._d_sn_and_pack()
        # ---- generator loss seeds
        G['dgen'].zero_()
        self.g_grad.zero_()
        r0, r1 = 0, B       # L1/L2 compare gen_images_enc (posterior half) when it exists (base_model.py:737)
        if not hp.nz:
            r1 = NB
        cnt = S * (r1 - r0) * HW * C
        for t in range(S):
            first = True
            for mode, wgt, nm in ((0, hp.l1_weight, 'gen_l1_loss'), (1, hp.l2_weight, 'gen_l2_loss')):
                if wgt:
                    # the first enabled term writes dgen, a second one accumulates into it (mode bit 1)
                    L.pixel_loss(Bf['gen'][t, r0:r1].data_ptr(), 4, Bf['x'][t + 1, r0:r1].data_ptr(), 4, G['dgen'][t, r0:r1].data_ptr(), 4,
                                 (r1 - r0) * HW, C, mode | (0 if first else 2), cnt, wgt, self._slot(nm))
                    first = False
        if hp.kl_weight and hp.nz:
            L.kl_loss(Bf['zmu'], Bf['zlss'], S * B, hp.nz, self._slot('gen_kl_loss'))
        if has_d:
            def g_step_tower(scope, net):
                enc, w, kind, cd_w = net['enc'], net['weight'], net['kind'], net['cdist']
                if not w:
                    return
                foff = 0 if enc else (B if hp.nz else 0)
                need_real = bool(cd_w)
                self._d_gather(net, 'post', net['ts'][('d_post', 0)], net['ts'][('d_post', 1)], foff, rows_real=need_real)
                self._d_forward(net, 0 if need_real else B, 2 * B)
                L.gan_loss(net['logits'][B:], 1.0, B, w, hp.gan_loss_type, net['dlogits'][B:],
                           self._slot('gen_%s_sn_%sgan_loss' % (kind, 'vae_' if enc else '')))
                dcd = None
                if cd_w:
                    dcd = net['dcd']
                    slot = self._slot('gen_%s_sn_%sgan_feature_cdist_loss' % (kind, 'vae_' if enc else ''))
                    for l, feat in enumerate(net['feat']):
                        dcd[l].zero_()
                        co = feat.shape[-1]
                        rows = int(np.prod(feat.shape[1:-1])) * B
                        L.cosine_distance(feat[B:], feat[:B], dcd[l], rows, co, cd_w, slot)
                self._d_backward(net, B, 2 * B, with_wgrad=False, to_clip=True, dcd=dcd)
                # the towers scatter into disjoint sample rows of dgen per unroll; towers of different kinds on the same
                # unroll accumulate (scatter_clip adds)
                L.scatter_clip(net['dclip'][B:], net['ts'][('d_post', 1)], G['dgen'], B, net['clip_len'], HW, NB, foff)
            self._run_concurrent([(lambda sc=sc, nt=nt: g_step_tower(sc, nt)) for sc, nt in self.dnets.items()])
        # ---- BPTT
        for t in range(S - 1, -1, -1):
            self._gen_backward_step(t)
        self._gen_backward_params(red)
        if red is not None:
            red.join()
        elif allreduce is not None:
            allreduce(self.g_grad)
        L.adam(self.g_flat, self.g_grad, self.g_m, self.g_v, self.g_flat.numel(), self.step_scalars[1:2], hp.beta1, hp.beta2, 1.0 / world)
        if has_d:   # every forward of this step read the start-of-step u; store u' now
            for net in self.dnets.values():
                for lay in net['layers'] + [net['fc']]:
                    self.params[lay.uname].view(-1).copy_(lay.u_next)
        self._pack_all()

    def _stage_step_scalars(self):
        """Host -> device: the step-dependent scalars (TF Adam's lr_t for both optimizers, annealed KL weight)."""
        import math
        hp = self.hparams
        step = self.global_step
        self._staged_step = step
        lr = self.learning_rate_at(step)
        if self.dnets:
            self.d_adam_t += 1
        self.g_adam_t += 1

        def lr_t(t):
            return lr * math.sqrt(1.0 - hp.beta2 ** t) / (1.0 - hp.beta1 ** t) if t > 0 else 0.0
        klw = (self.kl_weight_at(step) or 0.0) if (hp.kl_weight and hp.nz) else 0.0
        self._scal_host[0] = lr_t(self.d_adam_t)
        self._scal_host[1] = lr_t(self.g_adam_t)
        self._scal_host[2] = klw / float(self.S * self.B)
        self.step_scalars.copy_(self._scal_host, non_blocking=True)

    def loss_weights(self, step=None):
        """name -> weight of every loss slot at `step` (base_model.py:733-852; the KL weight is annealed, :312-319)."""
        hp = self.hparams
        step = self._staged_step if step is None else step
        kl = (self.kl_weight_at(step) or 0.0) if (hp.kl_weight and hp.nz) else 0.0
        w = OrderedDict([('gen_l1_loss', hp.l1_weight), ('gen_l2_loss', hp.l2_weight), ('gen_kl_loss', kl)])
        for kind, w_gan, w_vae in (('video', hp.video_sn_gan_weight, hp.video_sn_vae_gan_weight),
                                   ('image', hp.image_sn_gan_weight, hp.image_sn_vae_gan_weight)):
            w['gen_%s_sn_gan_loss' % kind] = w_gan
            w['gen_%s_sn_vae_gan_loss' % kind] = w_vae if hp.nz else 0.0
            w['gen_%s_sn_vae_gan_feature_cdist_loss' % kind] = hp.vae_gan_feature_cdist_weight if (w_vae and hp.nz) else 0.0
            w['gen_%s_sn_gan_feature_cdist_loss' % kind] = hp.gan_feature_cdist_weight if w_gan else 0.0
            w['discrim_%s_sn_gan_loss' % kind] = w_gan
            w['discrim_%s_sn_vae_gan_loss' % kind] = w_vae if hp.nz else 0.0
        return w

    @staticmethod
    def split_losses(vals, weights):
        """UNWEIGHTED per-term values of one step + their weights -> (g_losses, d_losses, g_loss, d_loss) as the reference
        exposes them: the dicts hold the unweighted terms, the totals are sum(loss * weight) (base_model.py:461)."""
        g = OrderedDict((k, v) for k, v in vals.items() if k.startswith('gen_') and weights.get(k))
        d = OrderedDict((k, v) for k, v in vals.items() if k.startswith('discrim_') and weights.get(k))
        return (g, d, float(sum(v * weights[k] for k, v in g.items())), float(sum(v * weights[k] for k, v in d.items())))

    def losses(self):
        """Unweighted loss terms of the last step (device -> host read, averaged over data-parallel replicas as
        tf_utils.py:489-490 does); also refreshes g_losses / d_losses / g_loss / d_loss.  The generator's GAN / feature
        terms are the POST-update values (the quantity train_op differentiates, base_model.py:497-503)."""
        lv = self.loss_vals.detach().clone()
        if self.world_size > 1:
            from .. import dp
            dp.mean_scalars(lv)
        vals = lv.cpu().numpy()
        out = OrderedDict((k, float(v)) for k, v in zip(LOSS_SLOTS, vals))
        self.g_losses, self.d_losses, self.g_loss, self.d_loss = self.split_losses(out, self.loss_weights())
        return out
