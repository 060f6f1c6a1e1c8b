"""Host-side mirror of the reference's model base classes (video_prediction/models/base_model.py).

Keeps the constructor signature, hparams defaults/override order, mode / context_frames /
sequence_length validation (base_model.py:20-59), the learning-rate and KL-weight schedules
(:286-319) and the `build_graph(inputs)` entry point (:467).  There is no TF graph: build_graph
allocates device buffers and the compute is the sm_90a kernels in libvp_b200.so."""
from __future__ import annotations

import itertools
import math
import os

import numpy as np

from ..hparams import HParams


class BaseVideoPredictionModel(object):
    def __init__(self, mode='train', hparams_dict=None, hparams=None, num_gpus=None, eval_num_samples=100,
                 eval_num_samples_for_diversity=10, eval_parallel_iterations=1):
        # reference accepts 'train'/'test' (base_model.py:37-38); generate.py passes 'val' too.
        if mode not in ('train', 'val', 'test'):
            raise ValueError('mode must be train or test, but %s given' % mode)
        self.mode = mode
        cuda_visible_devices = os.environ.get('CUDA_VISIBLE_DEVICES', '0')
        max_num_gpus = 0 if cuda_visible_devices == '' else len(cuda_visible_devices.split(','))
        if num_gpus is None:
            num_gpus = max_num_gpus
        elif num_gpus > max_num_gpus:
            raise ValueError('num_gpus=%d is greater than the number of visible devices %d' % (num_gpus, max_num_gpus))
        self.num_gpus = num_gpus
        self.eval_num_samples = eval_num_samples
        self.eval_num_samples_for_diversity = eval_num_samples_for_diversity
        self.eval_parallel_iterations = eval_parallel_iterations
        self.hparams = self.parse_hparams(hparams_dict, hparams)
        if self.hparams.context_frames == -1:
            raise ValueError('Invalid context_frames %r. It might have to be specified.' % self.hparams.context_frames)
        if self.hparams.sequence_length == -1:
            raise ValueError('Invalid sequence_length %r. It might have to be specified.' % self.hparams.sequence_length)
        self.deterministic = True
        self.inputs = None
        self.gen_images = None
        self.outputs = None
        self.metrics = None
        self.eval_outputs = None
        self.eval_metrics = None
        self.saveable_variables = None
        self.post_init_ops = None

    def get_default_hparams_dict(self):
        return dict(context_frames=-1, sequence_length=-1, repeat=1)

    def get_default_hparams(self):
        return HParams(**self.get_default_hparams_dict())

    def parse_hparams(self, hparams_dict, hparams):
        parsed = self.get_default_hparams().override_from_dict(hparams_dict or {})
        if hparams:
            if not isinstance(hparams, (list, tuple)):
                hparams = [hparams]
            for hparam in hparams:
                parsed.parse(hparam)
        return parsed

    def build_graph(self, inputs):
        self.inputs = inputs


class VideoPredictionModel(BaseVideoPredictionModel):
    def __init__(self, generator_scope='generator', discriminator_scope='discriminator', aggregate_nccl=False,
                 mode='train', hparams_dict=None, hparams=None, **kwargs):
        super(VideoPredictionModel, self).__init__(mode, hparams_dict, hparams, **kwargs)
        self.generator_scope = generator_scope
        self.discriminator_scope = discriminator_scope
        self.aggregate_nccl = aggregate_nccl
        self.global_step = 0
        self.g_losses = None
        self.d_losses = None
        self.g_loss = None
        self.d_loss = None
        self.train_op = None

    def get_default_hparams_dict(self):
        default_hparams = super(VideoPredictionModel, self).get_default_hparams_dict()
        hparams = dict(
            batch_size=16, lr=0.001, end_lr=0.0, decay_steps=(200000, 300000), lr_boundaries=(0,),
            max_steps=300000, beta1=0.9, beta2=0.999, context_frames=-1, sequence_length=-1, clip_length=10,
            l1_weight=0.0, l2_weight=1.0, vgg_cdist_weight=0.0, feature_l2_weight=0.0, ae_l2_weight=0.0,
            state_weight=0.0, tv_weight=0.0,
            image_sn_gan_weight=0.0, image_sn_vae_gan_weight=0.0,
            images_sn_gan_weight=0.0, images_sn_vae_gan_weight=0.0,
            video_sn_gan_weight=0.0, video_sn_vae_gan_weight=0.0,
            gan_feature_l2_weight=0.0, gan_feature_cdist_weight=0.0,
            vae_gan_feature_l2_weight=0.0, vae_gan_feature_cdist_weight=0.0,
            gan_loss_type='LSGAN', joint_gan_optimization=False,
            kl_weight=0.0, kl_anneal='linear', kl_anneal_k=-1.0, kl_anneal_steps=(50000, 100000),
            z_l1_weight=0.0,
        )
        return dict(itertools.chain(default_hparams.items(), hparams.items()))

    # ---- schedules (base_model.py:286-319), evaluated on the host for the current global_step
    def learning_rate_at(self, step):
        hp = self.hparams
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

    def kl_weight_at(self, step):
        hp = self.hparams
        if not hp.kl_weight:
            return None
        if hp.kl_anneal == 'none':
            return hp.kl_weight
        if hp.kl_anneal == 'sigmoid':
            k = hp.kl_anneal_k
            if k == -1.0:
                raise ValueError('Invalid kl_anneal_k %d when kl_anneal is sigmoid.' % k)
            return hp.kl_weight / (1 + k * math.exp(-step / k))
        if hp.kl_anneal == 'linear':
            s0, s1 = hp.kl_anneal_steps
            return hp.kl_weight * (min(max(step, s0), s1) - s0) / float(s1 - s0)
        raise NotImplementedError

    @property
    def learning_rate(self):
        return self.learning_rate_at(self.global_step)

    @property
    def kl_weight(self):
        return self.kl_weight_at(self.global_step)
