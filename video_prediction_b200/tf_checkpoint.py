"""Reader for TensorFlow checkpoints ("tensor bundle", V2: `<prefix>.index` + `<prefix>.data-00000-of-0000N`) without
TensorFlow -- SURVEY.md 8f-1: lets the pretrained SAVP weights the reference distributes
(pretrained_models/download_model.sh) drive the H100 path through `model.restore()`.

Formats restated from TensorFlow's published sources (tensorflow/core/util/tensor_bundle/tensor_bundle.{h,cc},
tensorflow/core/lib/io/table*.cc, tensorflow/core/protobuf/tensor_bundle.proto, tensor_shape.proto):

  .index   a LevelDB-style immutable table.  48-byte footer = metaindex BlockHandle + index BlockHandle (varint64 offset, size),
           zero padding, magic 0xdb4775248b80fb57 (little endian).  A block = prefix-compressed entries
           (varint32 shared, varint32 non_shared, varint32 value_len, key delta, value) followed by the uint32 restart offsets
           and their count; every block is followed by a 1-byte compression type (0 = none, 1 = snappy) and a 4-byte masked
           crc32c that are not part of its BlockHandle size.  The index block maps separator keys to the BlockHandles of the
           data blocks; the data blocks map variable names to serialized BundleEntryProto; the entry with the empty key is
           the BundleHeaderProto (num_shards, endianness, version).
  BundleEntryProto: 1 dtype (DataType enum), 2 shape (TensorShapeProto: repeated 2 dim { 1 size }), 3 shard_id, 4 offset,
           5 size, 6 crc32c (fixed32), 7 slices (partitioned variables: not supported here).
  .data-*  the raw little-endian tensor bytes at [offset, offset + size).

PARITY STATUS: no TensorFlow-written checkpoint exists in this environment (no network, no TF); tests/test_tf_checkpoint.py
round-trips through an independent writer of the same published format, so the reader is "unpinned" against real files."""
from __future__ import annotations

import glob
import os
import re
import struct
from collections import OrderedDict

import numpy as np

TABLE_MAGIC = 0xdb4775248b80fb57
# tensorflow/core/framework/types.proto DataType -> numpy
DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64, 10: np.bool_,
          17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}


def _varint(buf, pos):
    result, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7


def _block_handle(buf, pos):
    off, pos = _varint(buf, pos)
    size, pos = _varint(buf, pos)
    return (off, size), pos


def _read_block(data, handle):
    off, size = handle
    ctype = data[off + size]
    if ctype == 1:
        raise NotImplementedError('snappy-compressed table block (TensorFlow writes checkpoint indexes uncompressed)')
    if ctype != 0:
        raise ValueError('unknown block compression type %d' % ctype)
    return data[off:off + size]


def _block_entries(block):
    """(key, value) pairs of one table block (prefix-compressed keys)."""
    n_restarts = struct.unpack_from('<I', block, len(block) - 4)[0]
    limit = len(block) - 4 - 4 * n_restarts
    pos, key = 0, b''
    while pos < limit:
        shared, pos = _varint(block, pos)
        non_shared, pos = _varint(block, pos)
        vlen, pos = _varint(block, pos)
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        yield key, bytes(block[pos:pos + vlen])
        pos += vlen


def _parse_proto(buf):
    """Minimal protobuf wire-format walk: field number -> list of raw values (varint int / bytes / fixed)."""
    out, pos = {}, 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        field, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from('<Q', buf, pos)[0]
            pos += 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            v = bytes(buf[pos:pos + ln])
            pos += ln
        elif wt == 5:
            v = struct.unpack_from('<I', buf, pos)[0]
            pos += 4
        else:
            raise ValueError('unsupported protobuf wire type %d' % wt)
        out.setdefault(field, []).append(v)
    return out


def _parse_entry(value):
    f = _parse_proto(value)
    shape = []
    if 2 in f:
        for dim in _parse_proto(f[2][0]).get(2, []):
            d = _parse_proto(dim).get(1, [0])[0]
            shape.append(d - (1 << 64) if d >= (1 << 63) else d)
    return dict(dtype=f.get(1, [0])[0], shape=tuple(shape), shard_id=f.get(3, [0])[0], offset=f.get(4, [0])[0],
                size=f.get(5, [0])[0], crc32c=f.get(6, [0])[0], sliced=7 in f)


class CheckpointReader(object):
    """`tf.pywrap_tensorflow.NewCheckpointReader` work-alike (tf_utils.py:531-533): get_variable_to_shape_map(), has_tensor(),
    get_tensor()."""

    def __init__(self, prefix):
        self.prefix = prefix
        with open(prefix + '.index', 'rb') as fh:
            data = fh.read()
        if len(data) < 48 or struct.unpack_from('<Q', data, len(data) - 8)[0] != TABLE_MAGIC:
            raise ValueError('%s.index is not a TensorFlow checkpoint index (bad table magic)' % prefix)
        footer = data[len(data) - 48:]
        _, pos = _block_handle(footer, 0)                 # metaindex (unused by the bundle format)
        index_handle, _ = _block_handle(footer, pos)
        self.entries, self.header = OrderedDict(), None
        for _, handle_bytes in _block_entries(_read_block(data, index_handle)):
            handle, _ = _block_handle(handle_bytes, 0)
            for key, value in _block_entries(_read_block(data, handle)):
                if key == b'':
                    h = _parse_proto(value)
                    self.header = dict(num_shards=h.get(1, [1])[0], endianness=h.get(2, [0])[0])
                else:
                    self.entries[key.decode()] = _parse_entry(value)
        if self.header is None:
            raise ValueError('%s.index has no bundle header entry' % prefix)
        if self.header['endianness'] != 0:
            raise NotImplementedError('big-endian checkpoint')
        self._shards = {}

    def get_variable_to_shape_map(self):
        return OrderedDict((k, list(e['shape'])) for k, e in self.entries.items())

    def has_tensor(self, name):
        return name in self.entries

    def _shard(self, shard_id):
        if shard_id not in self._shards:
            path = '%s.data-%05d-of-%05d' % (self.prefix, shard_id, self.header['num_shards'])
            self._shards[shard_id] = np.memmap(path, dtype=np.uint8, mode='r')
        return self._shards[shard_id]

    def get_tensor(self, name):
        e = self.entries[name]
        if e['sliced']:
            raise NotImplementedError('partitioned variable %s' % name)
        if e['dtype'] not in DTYPES:
            raise NotImplementedError('dtype %d of %s' % (e['dtype'], name))
        raw = self._shard(e['shard_id'])[e['offset']:e['offset'] + e['size']]
        return np.frombuffer(bytes(raw), dtype=DTYPES[e['dtype']]).reshape(e['shape'])


def latest_checkpoint(checkpoint_dir):
    """tf.train.latest_checkpoint: the prefix named by `<dir>/checkpoint` (model_checkpoint_path: "..."), else the
    `model-<step>.index` with the largest step."""
    state = os.path.join(checkpoint_dir, 'checkpoint')
    if os.path.exists(state):
        with open(state) as fh:
            m = re.search(r'model_checkpoint_path:\s*"([^"]+)"', fh.read())
        if m:
            p = m.group(1)
            p = p if os.path.isabs(p) else os.path.join(checkpoint_dir, p)
            if os.path.exists(p + '.index'):
                return p
    cands = glob.glob(os.path.join(checkpoint_dir, '*.index'))
    if not cands:
        return None

    def step(p):
        m = re.search(r'-(\d+)\.index$', p)
        return int(m.group(1)) if m else -1
    return max(cands, key=step)[:-len('.index')]


def is_tf_checkpoint(path):
    return path is not None and os.path.exists(path + '.index')


def load_variables(prefix, wanted, mapping=None):
    """name -> array for the variables in `wanted` found in the checkpoint.  `mapping(name, checkpoint_names)` is the
    reference's restore_to_checkpoint_mapping (default: identity; SAVP falls back from 'savp_cell' to the historical
    'dna_cell' scope, savp_model.py:848-855).  Also returns global_step and the Adam slots under the reference's slot names
    (`<var>/Adam`, `<var>/Adam_1`, `beta1_power`) when present, and the lists the reference prints (tf_utils.py:543-557)."""
    reader = CheckpointReader(prefix)
    names = set(reader.entries)
    mapping = mapping or (lambda n, _: n)
    found, missing = OrderedDict(), []
    slots = dict(m=OrderedDict(), v=OrderedDict())
    for name in wanted:
        ck = mapping(name, names)
        if ck in names:
            found[name] = reader.get_tensor(ck)
            for slot, suffix in (('m', '/Adam'), ('v', '/Adam_1')):
                if ck + suffix in names:
                    slots[slot][name] = reader.get_tensor(ck + suffix)
        else:
            missing.append(name)
    used = set(mapping(n, names) for n in found)
    unused = sorted(n for n in names if n not in used and not n.endswith(('/Adam', '/Adam_1')) and
                    n not in ('global_step', 'beta1_power', 'beta2_power'))
    extra = dict(global_step=int(reader.get_tensor('global_step')) if 'global_step' in names else None, slots=slots,
                 beta1_power=float(reader.get_tensor('beta1_power')) if 'beta1_power' in names else None)
    return found, missing, unused, extra
