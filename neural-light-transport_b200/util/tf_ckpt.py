"""Reader (and a minimal writer, for round-trip tests and export) of TensorFlow "tensor bundle" checkpoints, so that
the released NLT weights -- `tf.train.Checkpoint(step=, optimizer=, net=model)` files, nlt/trainvali.py:134-141,
restored by nlt/nlt_test.py:61-75 -- can drive this repo's model without TensorFlow (SURVEY.md 8f row N4).

Format (public, TensorFlow `tensor_bundle` + LevelDB table format; restated here, TensorFlow is not installable
offline so no TF-written file could be used to pin this reader -- the tests round-trip files written by
`write_bundle` below, which follows the same specification):

  <prefix>.index                 a LevelDB-format sorted string table: data blocks of prefix-compressed
                                 (key, value) entries + restart array, an index block of block handles, a 48-byte
                                 footer ending in the magic 0xdb4775248b80fb57; every block is followed by a 1-byte
                                 compression type (0 none, 1 snappy) and a 4-byte masked CRC32C.
                                 key ""  -> BundleHeaderProto {num_shards=1, endianness=2, version=3}
                                 key k   -> BundleEntryProto {dtype=1, shape=2, shard_id=3, offset=4, size=5, crc32c=6}
  <prefix>.data-00000-of-00001   raw little-endian tensor bytes, addressed by (shard_id, offset, size)

Object-graph keys of the reference model (Keras tracking of `net_<network>_layer<i>`, nlt/models/base.py:79-101):
  net/net_query_layer0/kernel/.ATTRIBUTES/VARIABLE_VALUE                          bare Conv2D (levels 0 and 13)
  net/net_query_layer3/layer_with_weights-1/bias/.ATTRIBUTES/VARIABLE_VALUE       j-th conv of a Sequential block
  .../kernel/.OPTIMIZER_SLOT/optimizer/{m,v,vhat}/.ATTRIBUTES/VARIABLE_VALUE      Adam slots; optimizer/iter/...
  net/net_query_layer7/layer_with_weights-0/layer_with_weights-0/kernel/...       `pool != None`: the conv of the up
                                                                                  block's nested upconv Sequential
                                                                                  (conv0; the two deconvs are -1, -2)
The nested upconv keys follow from Keras's `layer_with_weights-N` tracking of a Sequential inside a Sequential
(nlt/networks/elements.py:42-48 inside convnet.py:66-75); like the rest of this reader they are unpinned, since no
TF-written checkpoint of a pooling network exists offline.
"""
import os
import re
import struct

import numpy as np

_MAGIC = 0xdb4775248b80fb57
_SUFFIX = '/.ATTRIBUTES/VARIABLE_VALUE'
# tensorflow/core/framework/types.proto
_DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64, 10: np.bool_,
           17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}
_DTYPE_CODES = {np.dtype(v): k for k, v in _DTYPES.items()}


# ---------------------------------------------------------------------------------------------
# varints / protobuf wire format (only what the two bundle messages need)
# ---------------------------------------------------------------------------------------------
def _varint(buf, pos):
    out = shift = 0
    while True:
        b = buf[pos]
        pos += 1
        out |= (b & 0x7f) << shift
        if not b & 0x80:
            return out, pos
        shift += 7


def _enc_varint(v):
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _parse_fields(buf):
    """[(field number, wire type, value)] of one protobuf message (value: int or bytes)."""
    pos, out = 0, []
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        num, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from('<Q', buf, pos)[0]
            pos += 8
        elif wt == 2:
            n, pos = _varint(buf, pos)
            v = bytes(buf[pos:pos + n])
            pos += n
        elif wt == 5:
            v = struct.unpack_from('<I', buf, pos)[0]
            pos += 4
        else:
            raise ValueError('unsupported protobuf wire type %d' % wt)
        out.append((num, wt, v))
    return out


def _parse_entry(buf):
    e = {'dtype': 0, 'shape': [], 'shard_id': 0, 'offset': 0, 'size': 0, 'sliced': False}
    for num, _, v in _parse_fields(buf):
        if num == 1:
            e['dtype'] = v
        elif num == 2:      # TensorShapeProto: repeated Dim dim = 2 { int64 size = 1 }
            for n2, _, v2 in _parse_fields(v):
                if n2 == 2:
                    size = 0
                    for n3, _, v3 in _parse_fields(v2):
                        if n3 == 1:
                            size = v3
                    e['shape'].append(size)
        elif num == 3:
            e['shard_id'] = v
        elif num == 4:
            e['offset'] = v
        elif num == 5:
            e['size'] = v
        elif num == 7:
            e['sliced'] = True
    return e


# ---------------------------------------------------------------------------------------------
# snappy (raw format) decompression -- LevelDB tables may compress blocks with it
# ---------------------------------------------------------------------------------------------
def _snappy_decompress(buf):
    n, pos = _varint(buf, 0)
    out = bytearray()
    while pos < len(buf):
        tag = buf[pos]
        pos += 1
        kind = tag & 3
        if kind == 0:                       # literal
            ln = tag >> 2
            if ln >= 60:
                nb = ln - 59
                ln = int.from_bytes(buf[pos:pos + nb], 'little')
                pos += nb
            ln += 1
            out += buf[pos:pos + ln]
            pos += ln
            continue
        if kind == 1:
            ln = ((tag >> 2) & 7) + 4
            off = ((tag >> 5) << 8) | buf[pos]
            pos += 1
        elif kind == 2:
            ln = (tag >> 2) + 1
            off = buf[pos] | (buf[pos + 1] << 8)
            pos += 2
        else:
            ln = (tag >> 2) + 1
            off = int.from_bytes(buf[pos:pos + 4], 'little')
            pos += 4
        if off == 0 or off > len(out):
            raise ValueError('corrupt snappy stream')
        for _ in range(ln):                 # overlapping copies are legal
            out.append(out[-off])
    if len(out) != n:
        raise ValueError('snappy: length mismatch')
    return bytes(out)


# ---------------------------------------------------------------------------------------------
# LevelDB table
# ---------------------------------------------------------------------------------------------
def _read_block(data, offset, size):
    raw = data[offset:offset + size]
    ctype = data[offset + size]
    if ctype == 1:
        raw = _snappy_decompress(raw)
    elif ctype != 0:
        raise ValueError('unknown block compression %d' % ctype)
    n_restarts = struct.unpack_from('<I', raw, len(raw) - 4)[0]
    end = len(raw) - 4 - 4 * n_restarts
    pos, key, out = 0, b'', []
    while pos < end:
        shared, pos = _varint(raw, pos)
        non_shared, pos = _varint(raw, pos)
        vlen, pos = _varint(raw, pos)
        key = key[:shared] + bytes(raw[pos:pos + non_shared])
        pos += non_shared
        out.append((key, bytes(raw[pos:pos + vlen])))
        pos += vlen
    return out


def read_index(path):
    """{key (str): BundleEntry dict} of `<prefix>.index` (the header entry "" is dropped)."""
    data = open(path, 'rb').read()
    if len(data) < 48 or struct.unpack_from('<Q', data, len(data) - 8)[0] != _MAGIC:
        raise ValueError('%s is not a TensorFlow checkpoint index (bad table magic)' % path)
    footer = data[-48:]
    _, p = _varint(footer, 0)               # metaindex handle (unused)
    _, p = _varint(footer, p)
    ioff, p = _varint(footer, p)
    isize, p = _varint(footer, p)
    entries = {}
    for _, handle in _read_block(data, ioff, isize):
        boff, q = _varint(handle, 0)
        bsize, q = _varint(handle, q)
        for key, val in _read_block(data, boff, bsize):
            if key:
                entries[key.decode()] = _parse_entry(val)
    return entries


def load_bundle(prefix):
    """{variable key: ndarray} of every dense numeric tensor of the checkpoint `prefix` (e.g. '.../ckpt-43')."""
    entries = read_index(prefix + '.index')
    shards = {}
    out = {}
    n_shards = max([e['shard_id'] for e in entries.values()] + [0]) + 1
    for key, e in entries.items():
        if e['sliced'] or e['dtype'] not in _DTYPES:
            continue                        # string tensors (the object graph), partitioned variables
        sid = e['shard_id']
        if sid not in shards:
            cands = [f for f in os.listdir(os.path.dirname(prefix) or '.')
                     if re.fullmatch(re.escape(os.path.basename(prefix)) + r'\.data-%05d-of-\d{5}' % sid, f)]
            if not cands:
                raise FileNotFoundError('%s.data-%05d-of-%05d' % (prefix, sid, n_shards))
            shards[sid] = np.memmap(os.path.join(os.path.dirname(prefix) or '.', cands[0]), dtype=np.uint8, mode='r')
        dt = np.dtype(_DTYPES[e['dtype']])
        raw = np.asarray(shards[sid][e['offset']:e['offset'] + e['size']])
        arr = raw.view(dt.newbyteorder('<')).reshape(e['shape'])
        out[key] = np.array(arr, dtype=dt)
    return out


def load_nlt_state(prefix):
    """A released NLT checkpoint as the key set of util/ckpt.py ('net/net_query_layer3/conv0/kernel', optimizer slots,
    'optimizer/iterations', 'step')."""
    raw = load_bundle(prefix)
    state = {}
    pat = re.compile(r'^net/(net_\w+?_layer\d+)/(?:layer_with_weights-(\d+)/)?(?:layer_with_weights-0/)?(kernel|bias)'
                     r'(?:/\.OPTIMIZER_SLOT/optimizer/(m|v|vhat))?' + re.escape(_SUFFIX) + '$')
    for key, arr in raw.items():
        m = pat.match(key)
        if m:
            layer, j, leaf, slot = m.group(1), int(m.group(2) or 0), m.group(3), m.group(4)
            ours = '%s/conv%d/%s' % (layer, j, leaf)
            state[('optimizer/%s/%s' % (slot, ours)) if slot else ('net/' + ours)] = arr.astype(np.float32)
        elif key == 'optimizer/iter' + _SUFFIX:
            state['optimizer/iterations'] = np.int64(arr)
        elif key == 'step' + _SUFFIX:
            state['step'] = np.int64(arr)
    if not any(k.startswith('net/') for k in state):
        raise ValueError('no NLT network variables (net/net_<network>_layer<i>/...) found in %s' % prefix)
    return state


# ---------------------------------------------------------------------------------------------
# writer (single shard, uncompressed blocks, like TensorFlow's BundleWriter)
# ---------------------------------------------------------------------------------------------
def _crc32c_table():
    tab = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82f63b78 if c & 1 else c >> 1
        tab.append(c)
    return tab


_CRC_TAB = None


def _masked_crc32c(data):
    global _CRC_TAB
    if _CRC_TAB is None:
        _CRC_TAB = _crc32c_table()
    c = 0xffffffff
    for b in data:
        c = _CRC_TAB[(c ^ b) & 0xff] ^ (c >> 8)
    c ^= 0xffffffff
    return ((((c >> 15) | (c << 17)) & 0xffffffff) + 0xa282ead8) & 0xffffffff


def _field(num, wt, payload):
    return _enc_varint((num << 3) | wt) + payload


def _enc_entry(dtype_code, shape, offset, size):
    dims = b''.join(_field(2, 2, (lambda d: _enc_varint(len(d)) + d)(_field(1, 0, _enc_varint(int(s))))) for s in shape)
    msg = _field(1, 0, _enc_varint(dtype_code)) + _field(2, 2, _enc_varint(len(dims)) + dims)
    if offset:
        msg += _field(4, 0, _enc_varint(offset))
    msg += _field(5, 0, _enc_varint(size))
    return msg


def _build_block(items, restart_interval=16):
    out, restarts, prev = bytearray(), [], b''
    for i, (key, val) in enumerate(items):
        shared = 0
        if i % restart_interval == 0:
            restarts.append(len(out))
        else:
            while shared < min(len(prev), len(key)) and prev[shared] == key[shared]:
                shared += 1
        out += _enc_varint(shared) + _enc_varint(len(key) - shared) + _enc_varint(len(val)) + key[shared:] + val
        prev = key
    for r in restarts or [0]:
        out += struct.pack('<I', r)
    out += struct.pack('<I', len(restarts) or 1)
    return bytes(out)


def write_bundle(prefix, tensors, block_entries=32):
    """Writes {key: ndarray} as `<prefix>.index` + `<prefix>.data-00000-of-00001`."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    keys = sorted(tensors)
    data, entries = bytearray(), []
    header = _field(1, 0, _enc_varint(1)) + _field(2, 0, _enc_varint(0)) + \
        _field(3, 2, (lambda v: _enc_varint(len(v)) + v)(_field(1, 0, _enc_varint(1))))     # num_shards 1, LITTLE, version 1
    entries.append((b'', header))
    for k in keys:
        a = np.ascontiguousarray(tensors[k])
        raw = a.astype(a.dtype.newbyteorder('<')).tobytes()
        entries.append((k.encode(), _enc_entry(_DTYPE_CODES[a.dtype], a.shape, len(data), len(raw))))
        data += raw
    with open(prefix + '.data-00000-of-00001', 'wb') as f:
        f.write(bytes(data))
    table, index_items = bytearray(), []

    def emit(block):
        off = len(table)
        table.extend(block)
        table.extend(bytes([0]) + struct.pack('<I', _masked_crc32c(block + bytes([0]))))
        return _enc_varint(off) + _enc_varint(len(block))
    for i in range(0, len(entries), block_entries):
        chunk = entries[i:i + block_entries]
        index_items.append((chunk[-1][0], emit(_build_block(chunk))))
    meta = emit(_build_block([]))
    index = emit(_build_block(index_items, restart_interval=1))
    footer = (meta + index).ljust(40, b'\x00') + struct.pack('<Q', _MAGIC)
    table.extend(footer)
    with open(prefix + '.index', 'wb') as f:
        f.write(bytes(table))


def save_nlt_state(prefix, state):
    """Inverse of load_nlt_state: our key set -> the reference's object-graph keys (export to a TF-readable bundle)."""
    out = {}
    for k, v in state.items():
        if k == 'step':
            out['step' + _SUFFIX] = np.int64(v)
        elif k == 'optimizer/iterations':
            out['optimizer/iter' + _SUFFIX] = np.int64(v)
        else:
            m = re.match(r'^(?:optimizer/(m|v|vhat)/|net/)(net_\w+?_layer\d+)/conv(\d+)/(kernel|bias)$', k)
            if not m:
                continue
            slot, layer, j, leaf = m.groups()
            # a bare Conv2D layer (one conv in the block) has no layer_with_weights level; a three-conv up block
            # (pool != None) starts with the nested upconv Sequential, whose conv is its layer_with_weights-0
            single = not any(kk.endswith('%s/conv1/kernel' % layer) for kk in state)
            nested = j == '0' and any(kk.endswith('%s/conv2/kernel' % layer) for kk in state)
            path = 'net/%s/%s%s%s' % (layer, '' if single else 'layer_with_weights-%s/' % j,
                                      'layer_with_weights-0/' if nested else '', leaf)
            if slot:
                path += '/.OPTIMIZER_SLOT/optimizer/' + slot
            out[path + _SUFFIX] = np.asarray(v, dtype=np.float32)
    write_bundle(prefix, out)
