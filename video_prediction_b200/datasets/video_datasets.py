"""The reference's TFRecord video datasets on the host, without TensorFlow (SURVEY.md 8f-3): the BAIR robot-pushing format
(`SoftmotionVideoDataset`, softmotion_dataset.py:10-82: one tf.train.Example per trajectory, one feature per time step,
raw uint8 frames) and the KTH format (`KTHVideoDataset`, kth_dataset.py:16-50: one Example per clip, a variable-length list
of raw frames).  Constructor, hparams, file discovery, filtering, sub-sequence sampling (time shift, frame skip, macro
actions) and batching follow base_dataset.py:12-312; `make_batch(batch_size)` returns one batch per call as a dict of
numpy arrays (`images` [B,T,H,W,C] float32 in [0,1], `actions` [B,T-1,A], `states` [B,T,S], and for BAIR records with
designated pixels `object_pos` [B,T,2D] and `pix_distribs` [B,T,H,W,D]) -- what the model's
`build_graph` / `train_step` take -- and raises StopIteration after `num_epochs` passes."""
from __future__ import annotations

import glob
import os
import re
from collections import OrderedDict

import numpy as np

from ..hparams import HParams
from . import tfrecord


class BaseVideoDataset(object):
    SHUFFLE_BUFFER = 1024                                                   # base_dataset.py:138

    def __init__(self, input_dir, mode='train', num_epochs=None, seed=None, hparams_dict=None, hparams=None):
        self.input_dir = os.path.normpath(os.path.expanduser(input_dir))
        self.mode, self.num_epochs, self.seed = mode, num_epochs, seed
        if mode not in ('train', 'val', 'test'):
            raise ValueError('Invalid mode %s' % mode)
        if not os.path.exists(self.input_dir):
            raise FileNotFoundError('input_dir %s does not exist' % self.input_dir)
        self.filenames = None
        for cand in (self.input_dir, os.path.join(self.input_dir, mode)):   # the records, or the split's sub-directory
            found = glob.glob(os.path.join(cand, '*.tfrecord*'))
            if found:
                self.input_dir, self.filenames = cand, sorted(found)
                break
        if not self.filenames:
            raise FileNotFoundError('No tfrecords were found in %s.' % self.input_dir)
        self.dataset_name = os.path.basename(os.path.split(self.input_dir)[0])
        self.state_like_names_and_shapes = OrderedDict()
        self.action_like_names_and_shapes = OrderedDict()
        self.hparams = self.parse_hparams(hparams_dict, hparams)
        self._rng = np.random.default_rng(seed)
        self._stream = None

    # ------------------------------------------------------------------ hparams (base_dataset.py:57-110)
    def get_default_hparams_dict(self):
        return dict(crop_size=0, scale_size=0, context_frames=1, sequence_length=0, long_sequence_length=0, frame_skip=0,
                    time_shift=1, force_time_shift=False, shuffle_on_val=False, use_state=False)

    def get_default_hparams(self):
        return HParams(**self.get_default_hparams_dict())

    def parse_hparams(self, hparams_dict, hparams):
        parsed = self.get_default_hparams().override_from_dict(hparams_dict or {})
        if hparams:
            for h in (hparams if isinstance(hparams, (list, tuple)) else [hparams]):
                parsed.parse(h)
        if parsed.long_sequence_length == 0:
            parsed.long_sequence_length = parsed.sequence_length
        return parsed

    @property
    def jpeg_encoding(self):
        raise NotImplementedError

    def set_sequence_length(self, sequence_length):
        self.hparams.sequence_length = sequence_length

    def num_examples_per_epoch(self):
        raise NotImplementedError

    # ------------------------------------------------------------------ per-example hooks
    def keep(self, example):
        """base_dataset.py:120-121 (`filter`): every example by default."""
        return True

    def parse(self, example):
        """parsed tf.train.Example -> (state-like sequences, action-like sequences) of ONE sampled sub-sequence."""
        raise NotImplementedError

    # ------------------------------------------------------------------ images (base_dataset.py:157-189)
    def decode_and_preprocess_images(self, buffers, image_shape):
        h, w, c = image_shape
        frames = []
        for buf in buffers:
            if self.jpeg_encoding:
                try:
                    import io
                    from PIL import Image
                except ImportError:
                    raise NotImplementedError('JPEG-encoded frames need PIL, which is not installed')
                img = np.asarray(Image.open(io.BytesIO(buf)))
            else:
                img = np.frombuffer(buf, dtype=np.uint8)
            frames.append(img.reshape(h, w, c))
        video = np.stack(frames)
        crop, scale = self.hparams.crop_size, self.hparams.scale_size
        if crop or scale:
            crop = crop or min(h, w)
            video = _crop_or_pad(video, crop, crop)
            if scale and scale != crop:
                raise NotImplementedError('scale_size != crop_size needs image resampling (tf.image.resize_images), not built')
        return video.astype(np.float32) * np.float32(1.0 / 255.0)          # tf.image.convert_image_dtype

    # ------------------------------------------------------------------ sub-sequence sampling (base_dataset.py:191-229)
    def slice_sequences(self, state_like, action_like, example_sequence_length):
        hp = self.hparams
        T, skip, shift = hp.sequence_length, hp.frame_skip, hp.time_shift
        t_start = 0
        if (shift and self.mode == 'train') or hp.force_time_shift:
            assert shift > 0 and isinstance(shift, int)
            num_shifts = ((example_sequence_length - 1) - (T - 1) * (skip + 1)) // shift
            if num_shifts < 0:
                raise ValueError('example_sequence_length has to be at least %d when sequence_length=%d, frame_skip=%d.'
                                 % ((T - 1) * (skip + 1) + 1, T, skip))
            t_start = int(self._rng.integers(0, num_shifts + 1)) * shift
        s_slice = slice(t_start, t_start + (T - 1) * (skip + 1) + 1, skip + 1)
        a_slice = slice(t_start, t_start + (T - 1) * (skip + 1))
        for name in list(state_like):
            seq = state_like[name][s_slice]
            assert len(seq) == T, (name, len(seq), T)
            state_like[name] = seq
        for name in list(action_like):
            seq = np.asarray(action_like[name][a_slice])
            assert len(seq) == (T - 1) * (skip + 1), (name, len(seq))
            action_like[name] = seq.reshape(T - 1, -1)                     # actions of skipped frames -> one macro action
        return state_like, action_like

    # ------------------------------------------------------------------ record stream + batching (base_dataset.py:129-156)
    def _records(self):
        shuffle = self.mode == 'train' or (self.mode == 'val' and self.hparams.shuffle_on_val)
        epoch = 0
        while self.num_epochs is None or epoch < self.num_epochs:
            files = list(self.filenames)
            if shuffle:
                self._rng.shuffle(files)
            for path in files:
                for rec in tfrecord.read_records(path):
                    ex = tfrecord.parse_example(rec)
                    if self.keep(ex):
                        yield ex
            epoch += 1

    def _shuffled(self):
        shuffle = self.mode == 'train' or (self.mode == 'val' and self.hparams.shuffle_on_val)
        if not shuffle:
            yield from self._records()
            return
        buf = []
        for ex in self._records():                                          # a bounded shuffle buffer, like tf.data's
            if len(buf) < self.SHUFFLE_BUFFER:
                buf.append(ex)
                continue
            i = int(self._rng.integers(0, len(buf)))
            out, buf[i] = buf[i], ex
            yield out
        self._rng.shuffle(buf)
        yield from buf

    def make_batch(self, batch_size):
        if self._stream is None:
            self._stream = self._shuffled()
        rows = []
        for ex in self._stream:
            state_like, action_like = self.parse(ex)
            rows.append(OrderedDict(list(state_like.items()) + list(action_like.items())))
            if len(rows) == batch_size:
                break
        if len(rows) < batch_size:                                          # drop_remainder=True
            raise StopIteration
        return {k: np.stack([np.asarray(r[k], dtype=np.float32) for r in rows]) for k in rows[0]}


def pixel_distribution(pos, height, width):
    """tf_utils.pixel_distribution (tf_utils.py:562-585) in float32: pos [N,2] = (y, x) -> [N,H,W] maps with bilinear
    weights on the four neighbours of the position.  Like the reference, each neighbour is a one-hot of the FLAT index
    y*W + x over H*W entries: x = W lands on column 0 of the next row, and an index outside [0, H*W) adds nothing."""
    pos = np.asarray(pos, np.float32)
    n = pos.shape[0]
    y, x = pos[:, 0], pos[:, 1]
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    x0f, x1f, y0f, y1f = (v.astype(np.float32) for v in (x0, x1, y0, y1))
    out = np.zeros((n, height * width), np.float32)
    for idx, wgt in ((y0 * width + x0, (x1f - x) * (y1f - y)), (y1 * width + x0, (x1f - x) * (y - y0f)),
                     (y0 * width + x1, (x - x0f) * (y1f - y)), (y1 * width + x1, (x - x0f) * (y - y0f))):
        ok = (idx >= 0) & (idx < height * width)
        np.add.at(out, (np.nonzero(ok)[0], idx[ok]), wgt[ok])
    return out.reshape(n, height, width)


def _crop_or_pad(video, th, tw):
    """tf.image.resize_image_with_crop_or_pad on [T,H,W,C]: centred crop and / or zero pad."""
    _, h, w, _ = video.shape
    if h > th:
        o = (h - th) // 2
        video = video[:, o:o + th]
    if w > tw:
        o = (w - tw) // 2
        video = video[:, :, o:o + tw]
    _, h, w, _ = video.shape
    if h < th or w < tw:
        pt, pl = (th - h) // 2, (tw - w) // 2
        video = np.pad(video, ((0, 0), (pt, th - h - pt), (pl, tw - w - pl), (0, 0)))
    return video


class VideoDataset(BaseVideoDataset):
    """One tf.train.Example per trajectory, one feature per time step (`'%d/name'`; base_dataset.py:235-353)."""

    def __init__(self, *args, **kwargs):
        super(VideoDataset, self).__init__(*args, **kwargs)
        self._max_sequence_length = None
        self._first = tfrecord.parse_example(next(tfrecord.read_records(self.filenames[0])))

    def _check_or_infer_shapes(self):
        """Fills in shapes that are None from the first example and finds the trajectory length (base_dataset.py:246-305)."""
        def finish(table, is_state):
            out = OrderedDict()
            for ex_name, (pattern, shape) in table.items():
                rx = re.compile(pattern.replace('%d', r'\d+') + '$')
                names = [n for n in self._first if rx.match(n)]
                if not names:
                    raise ValueError('Could not found any feature with name pattern %s.' % pattern)
                length = len(names) if is_state else len(names) + 1
                self._max_sequence_length = length if self._max_sequence_length is None else min(length, self._max_sequence_length)
                kind, val = self._first[names[0]]
                if kind == 'float':
                    inferred = (len(val),)
                    if shape is not None and tuple(shape) != inferred:
                        raise ValueError('Inferred shape for feature %s is %r but instead got shape %r.' % (names[0], inferred, shape))
                    shape = inferred
                elif kind == 'bytes':
                    inferred = None
                    if not self.jpeg_encoding:
                        side = int(np.sqrt(len(val[0]) // 3))               # raw uint8, square, 3 channels
                        if side * side * 3 == len(val[0]):
                            inferred = (side, side, 3)
                    if shape is None:
                        if inferred is None:
                            raise ValueError('Unable to infer shape for feature %s of size %d.' % (names[0], len(val[0])))
                        shape = inferred
                    elif inferred is not None and tuple(shape) != inferred:
                        raise ValueError('Inferred shape for feature %s is %r but instead got shape %r.' % (names[0], inferred, shape))
                else:
                    raise NotImplementedError(kind)
                out[ex_name] = (pattern, tuple(shape))
            return out
        self.state_like_names_and_shapes = finish(self.state_like_names_and_shapes, True)
        self.action_like_names_and_shapes = finish(self.action_like_names_and_shapes, False)
        if not self.hparams.sequence_length:
            self.hparams.sequence_length = (self._max_sequence_length - 1) // (self.hparams.frame_skip + 1) + 1

    def set_sequence_length(self, sequence_length):
        self.hparams.sequence_length = sequence_length or (self._max_sequence_length - 1) // (self.hparams.frame_skip + 1) + 1

    def parse(self, example):
        L = self._max_sequence_length

        def feature(name):
            if name not in example:
                raise ValueError('Feature with name %s not found in tfrecord. Possible feature names are:\n%s'
                                 % (name, '\n'.join(sorted(example))))
            return example[name][1]
        state_like, action_like = OrderedDict(), OrderedDict()
        for ex_name, (pattern, shape) in self.state_like_names_and_shapes.items():
            if ex_name == 'images':
                state_like[ex_name] = self.decode_and_preprocess_images([feature(pattern % i)[0] for i in range(L)], shape)
            else:
                state_like[ex_name] = np.stack([np.asarray(feature(pattern % i), np.float32).reshape(shape) for i in range(L)])
        for ex_name, (pattern, shape) in self.action_like_names_and_shapes.items():
            action_like[ex_name] = np.stack([np.asarray(feature(pattern % i), np.float32).reshape(shape) for i in range(L - 1)])
        return self.slice_sequences(state_like, action_like, L)


class VarLenFeatureVideoDataset(BaseVideoDataset):
    """One tf.train.Example per clip with a variable number of frames (base_dataset.py:401-453)."""

    def keep(self, example):
        return int(example['sequence_length'][1][0]) >= self.hparams.sequence_length

    def parse(self, example):
        length = int(example['sequence_length'][1][0])
        state_like, action_like = OrderedDict(), OrderedDict()
        image_spec = None
        for ex_name, (name, shape) in self.state_like_names_and_shapes.items():
            if ex_name == 'images':
                state_like[ex_name] = list(example[name][1])
                image_spec = shape
            else:
                state_like[ex_name] = np.asarray(example[name][1], np.float32).reshape((length,) + tuple(shape))
        for ex_name, (name, shape) in self.action_like_names_and_shapes.items():
            action_like[ex_name] = np.asarray(example[name][1], np.float32).reshape((length - 1,) + tuple(shape))
        state_like, action_like = self.slice_sequences(state_like, action_like, length)
        state_like['images'] = self.decode_and_preprocess_images(state_like['images'], image_spec)   # only the sampled slice
        return state_like, action_like


class SoftmotionVideoDataset(VideoDataset):
    """BAIR robot pushing (softmotion_dataset.py:10-82): frames under '%d/image_aux1/encoded' (or image_view0), optional
    '%d/endeffector_pos' (3) and '%d/action' (4) with use_state, and '%d/object_pos' (2D floats: the (y, x) positions of D
    designated pixels) when the records have it, which also yields their maps as `pix_distribs` [T,H,W,D]."""

    def __init__(self, *args, **kwargs):
        super(SoftmotionVideoDataset, self).__init__(*args, **kwargs)
        image_names = set()
        for name in self._first:
            m = re.search(r'\d+/(\w+)/encoded', name)
            if m:
                image_names.add(m.group(1))
        image_name = next((n for n in ('image_aux1', 'image_view0') if n in image_names), None)
        if image_name is None:
            if len(image_names) != 1:
                raise ValueError('The examples have images under more than one name.')
            image_name = image_names.pop()
        self.state_like_names_and_shapes['images'] = ('%%d/%s/encoded' % image_name, None)
        if self.hparams.use_state:
            self.state_like_names_and_shapes['states'] = ('%d/endeffector_pos', (3,))
            self.action_like_names_and_shapes['actions'] = ('%d/action', (4,))
        if any(re.match(r'\d+/object_pos$', name) for name in self._first):       # softmotion_dataset.py:41-42
            self.state_like_names_and_shapes['object_pos'] = ('%d/object_pos', None)
        self._check_or_infer_shapes()
        if 'object_pos' in self.state_like_names_and_shapes:
            h, w, _ = self.state_like_names_and_shapes['images'][1]
            npos = self.state_like_names_and_shapes['object_pos'][1][0]
            if npos % 2:
                raise ValueError('object_pos holds (y, x) pairs; got %d values per frame' % npos)
            crop, scale = self.hparams.crop_size, self.hparams.scale_size
            side = scale or crop or min(h, w)
            if (crop or scale) and (side, side) != (h, w):
                raise NotImplementedError('object_pos with crop_size / scale_size changing the %dx%d frames: how the positions '
                                          'map is not defined' % (h, w))

    def parse(self, example):
        state_like, action_like = super(SoftmotionVideoDataset, self).parse(example)
        if 'object_pos' in state_like:                                      # softmotion_dataset.py:59-68
            h, w, _ = self.state_like_names_and_shapes['images'][1]
            pos = state_like['object_pos'].reshape(len(state_like['object_pos']), -1, 2)
            state_like['pix_distribs'] = np.stack([pixel_distribution(pos[:, i], h, w) for i in range(pos.shape[1])], axis=-1)
        return state_like, action_like

    def get_default_hparams_dict(self):
        d = super(SoftmotionVideoDataset, self).get_default_hparams_dict()
        d.update(context_frames=2, sequence_length=12, long_sequence_length=30, time_shift=2)
        return d

    @property
    def jpeg_encoding(self):
        return False

    def num_examples_per_epoch(self):
        count = 0
        for filename in self.filenames:                                     # traj_<first>_to_<last>.tfrecords
            m = re.search(r'traj_(\d+)_to_(\d+).tfrecords', os.path.basename(filename))
            if m is None:
                return sum(1 for f in self.filenames for _ in tfrecord.read_records(f))
            count += int(m.group(2)) - int(m.group(1)) + 1
        return count


class KTHVideoDataset(VarLenFeatureVideoDataset):
    """KTH actions (kth_dataset.py:16-50): 'images/encoded' = raw uint8 frames, 'sequence_length', 'height', 'width', 'channels'."""

    def __init__(self, *args, **kwargs):
        super(KTHVideoDataset, self).__init__(*args, **kwargs)
        first = tfrecord.parse_example(next(tfrecord.read_records(self.filenames[0])))
        shape = tuple(int(first[k][1][0]) for k in ('height', 'width', 'channels'))
        self.state_like_names_and_shapes['images'] = ('images/encoded', shape)

    def get_default_hparams_dict(self):
        d = super(KTHVideoDataset, self).get_default_hparams_dict()
        d.update(context_frames=10, sequence_length=20, long_sequence_length=40, force_time_shift=True, shuffle_on_val=True,
                 use_state=False)
        return d

    @property
    def jpeg_encoding(self):
        return False

    def num_examples_per_epoch(self):
        path = os.path.join(self.input_dir, 'sequence_lengths.txt')
        if os.path.exists(path):
            with open(path) as f:
                lengths = [int(line.strip()) for line in f if line.strip()]
        else:
            lengths = [int(tfrecord.parse_example(r)['sequence_length'][1][0]) for fn in self.filenames for r in tfrecord.read_records(fn)]
        return int(np.sum(np.asarray(lengths) >= self.hparams.sequence_length))
