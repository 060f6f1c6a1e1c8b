"""Dataset registry with the reference's surface (video_prediction/datasets/__init__.py:11-25).

The TFRecord input pipelines sit either side of the H100 hot path (SURVEY.md 8f-3).  The two formats the BASELINE configs
train on are read on the host without TensorFlow (`video_datasets.py`, `tfrecord.py`): BAIR robot pushing (`softmotion` /
`bair`) and KTH (`kth`); the other registered names (JPEG-encoded or unused by any shipped config) raise
NotImplementedError.  `synthetic` is the dataset the hot path is measured on:
seeded videos of the shape the reference datasets deliver (`images` [B,T,H,W,C] f32 in [0,1], optional `actions`
[B,T-1,A]; base_dataset.py:189), generated on the host, so `scripts/train.py --dataset synthetic` and
`scripts/generate.py --dataset synthetic` run end to end without any input files."""
from __future__ import annotations

import numpy as np

from ..hparams import HParams

from .video_datasets import BaseVideoDataset, KTHVideoDataset, SoftmotionVideoDataset, VarLenFeatureVideoDataset, VideoDataset  # noqa: F401

_OUT_OF_SCOPE = {
    'google_robot': 'GoogleRobotVideoDataset', 'sv2p': 'SV2PVideoDataset', 'ucf101': 'UCF101VideoDataset',
    'cartgripper': 'CartgripperVideoDataset',
}
_TFRECORD = {'softmotion': SoftmotionVideoDataset, 'bair': SoftmotionVideoDataset, 'kth': KTHVideoDataset,
             'SoftmotionVideoDataset': SoftmotionVideoDataset, 'KTHVideoDataset': KTHVideoDataset}


class SyntheticVideoDataset(object):
    """Constructor / hparams / make_batch / num_examples_per_epoch mirror BaseVideoDataset (base_dataset.py:14-110, 259-312).
    `input_dir` is accepted and ignored (there are no files)."""

    def __init__(self, input_dir=None, mode='train', num_epochs=None, seed=None, hparams_dict=None, hparams=None):
        if mode not in ('train', 'val', 'test'):
            raise ValueError('Invalid mode %s' % mode)                     # base_dataset.py:36-37
        self.input_dir, self.mode, self.num_epochs, self.seed = input_dir, mode, num_epochs, seed
        self.hparams = self.parse_hparams(hparams_dict, hparams)
        self._epoch_pos = 0
        self._rng = np.random.default_rng((seed or 0) * 3 + {'train': 0, 'val': 1, 'test': 2}[mode])

    def get_default_hparams_dict(self):
        # base_dataset.py:84-96 + the synthetic shape knobs (defaults: the BAIR action-free shape, 2 + 10 frames)
        return dict(crop_size=0, scale_size=0, context_frames=2, sequence_length=12, long_sequence_length=0, frame_skip=0,
                    time_shift=1, force_time_shift=False, shuffle_on_val=False, use_state=False,
                    image_size=(64, 64), channels=3, action_dim=0, num_examples=256, smooth=True)

    def get_default_hparams(self):
        return HParams(**self.get_default_hparams_dict())

    def parse_hparams(self, hparams_dict, hparams):
        parsed = self.get_default_hparams().override_from_dict(hparams_dict or {})
        if hparams:
            for h in (hparams if isinstance(hparams, (list, tuple)) else [hparams]):
                parsed.parse(h)
        if parsed.long_sequence_length == 0:
            parsed.long_sequence_length = parsed.sequence_length            # base_dataset.py:108-109
        return parsed

    def set_sequence_length(self, sequence_length):
        self.hparams.sequence_length = sequence_length

    def num_examples_per_epoch(self):
        return int(self.hparams.num_examples)

    def _videos(self, batch):
        hp = self.hparams
        T, (H, W), C = hp.sequence_length, hp.image_size, hp.channels
        rng = self._rng
        if not hp.smooth:
            return rng.random((batch, T, H, W, C), dtype=np.float32)
        # moving blobs: smooth content so that the CDNA kernels / masks are exercised non-degenerately
        yy, xx = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing='ij')
        t = np.arange(T, dtype=np.float32)[:, None, None]
        out = np.zeros((batch, T, H, W, C), np.float32)
        for b in range(batch):
            for _ in range(3):
                cx, cy = rng.uniform(0.2, 0.8, 2) * (W, H)
                vx, vy = rng.uniform(-2.0, 2.0, 2)
                rad = rng.uniform(0.08, 0.2) * min(H, W)
                col = rng.uniform(0.2, 1.0, C).astype(np.float32)
                d2 = (xx[None] - (cx + vx * t)) ** 2 + (yy[None] - (cy + vy * t)) ** 2
                out[b] += np.exp(-d2 / (2 * rad * rad))[..., None] * col
        return np.clip(out * 0.6 + 0.1 * rng.random(out.shape, dtype=np.float32), 0.0, 1.0)

    def make_batch(self, batch_size):
        """One batch as a dict of numpy arrays (batch-major, base_dataset.py:259-312).  Raises StopIteration after
        num_epochs passes (the reference raises tf.errors.OutOfRangeError)."""
        if self.num_epochs is not None and self._epoch_pos + batch_size > self.num_epochs * self.num_examples_per_epoch():
            raise StopIteration
        self._epoch_pos += batch_size
        hp = self.hparams
        batch = {'images': self._videos(batch_size)}
        if hp.action_dim:
            batch['actions'] = self._rng.standard_normal((batch_size, hp.sequence_length - 1, hp.action_dim)).astype(np.float32)
        return batch


def get_dataset_class(dataset):
    if dataset in ('synthetic', 'SyntheticVideoDataset'):
        return SyntheticVideoDataset
    if dataset in _TFRECORD:
        return _TFRECORD[dataset]
    if dataset in _OUT_OF_SCOPE or dataset in _OUT_OF_SCOPE.values():
        raise NotImplementedError('%s is not built (SURVEY.md 8f-3 covers the BAIR and KTH formats); use --dataset bair | kth | synthetic'
                                  % dataset)
    raise ValueError('Invalid dataset %s' % dataset)                        # datasets/__init__.py:24
