"""TensorFlow checkpoint-V2 ("tensor bundle") reader / writer without TensorFlow, plus the variable-name map between the
reference's TF graph and this repo's flat parameter buffers (SURVEY.md §8f.1).

The reference saves / restores with `tf.train.Saver` (tacotron/train.py:153-155,205-215,377-380; wavenet_vocoder/train.py:75-83,
262-276,330-334): a checkpoint is `<prefix>.index` + `<prefix>.data-00000-of-00001` + the `checkpoint` state file. Neither TensorFlow
nor any checkpoint of the reference exists in this image, so the on-disk format below is a restatement of the published
TensorBundle layout (tensorflow/core/util/tensor_bundle, tensorflow/core/lib/io/{table,block,format}, the LevelDB table
format) — verified here only by round trips, the CRC-32C known answers and hand-assembled blocks (tests/test_tf_bundle_cpu.py):

  <prefix>.index   LevelDB-format sorted table.  key ""          -> BundleHeaderProto {num_shards=1, endianness=0, version{producer=1}}
                                                 key <var name>  -> BundleEntryProto  {dtype=1, shape=2, shard_id=3, offset=4, size=5,
                                                                                       crc32c=6 (fixed32, masked)}
                   block = entries (varint shared | varint non_shared | varint value_len | key delta | value) + uint32 restarts[] +
                   uint32 n_restarts; every block is followed by a 5-byte trailer (compression type, masked crc32c of block+type);
                   file ends with a 48-byte footer (metaindex handle, index handle, padding, magic 0xdb4775248b80fb57).
  <prefix>.data-00000-of-00001   the tensors' raw little-endian bytes at BundleEntryProto.offset.

Tensor LAYOUTS need no conversion: the flat buffers of this repo already hold every variable in the TensorFlow layout
(conv kernels [kw, in, out], dense / LSTM kernels [in, out]; DESIGN.md §3)."""
import os
import struct

import numpy as np

# ---------------------------------------------------------------------------------------------------------------------
# CRC-32C (Castagnoli), masked as leveldb / TensorFlow do
# ---------------------------------------------------------------------------------------------------------------------
_CRC_TABLE = None


def _crc_table():
    global _CRC_TABLE
    if _CRC_TABLE is None:
        t = np.zeros(256, dtype=np.uint32)
        for i in range(256):
            c = i
            for _ in range(8):
                c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
            t[i] = c
        _CRC_TABLE = t
    return _CRC_TABLE


_GF2_SHIFT = {}


def _gf2_mat_times(mat, vec):
    out, i = 0, 0
    while vec:
        if vec & 1:
            out ^= mat[i]
        vec >>= 1
        i += 1
    return out


def _gf2_shift_matrix(nbytes):
    """32x32 GF(2) matrix (list of 32 column words) that advances a raw CRC register over `nbytes` zero bytes"""
    if nbytes in _GF2_SHIFT:
        return _GF2_SHIFT[nbytes]
    # one zero BIT: reflected polynomial shift
    m = [0x82F63B78] + [1 << (i - 1) for i in range(1, 32)]
    def square(a):
        return [_gf2_mat_times(a, a[i]) for i in range(32)]
    m = square(square(square(m)))          # 8 bits = one byte
    res, n = None, nbytes
    while n:
        if n & 1:
            res = m if res is None else [_gf2_mat_times(m, res[i]) for i in range(32)]
        n >>= 1
        if n:
            m = square(m)
    _GF2_SHIFT[nbytes] = res
    return res


def crc32c(data, crc=0):
    """CRC-32C of a bytes-like object (init / final xor 0xffffffff). Large buffers are processed as 4096 independent lanes
    stepped together through numpy table look-ups and then folded with the GF(2) zero-shift matrix (CRCs are linear)."""
    buf = np.frombuffer(memoryview(data).cast("B"), dtype=np.uint8)
    table = _crc_table()
    n = buf.size
    reg = (crc ^ 0xFFFFFFFF) & 0xFFFFFFFF
    LANES = 4096
    if n >= LANES * 64:
        chunk = n // LANES
        body = buf[:chunk * LANES].reshape(LANES, chunk)
        regs = np.zeros(LANES, dtype=np.uint32)
        regs[0] = reg
        for j in range(chunk):
            regs = table[(regs ^ body[:, j]) & 0xFF] ^ (regs >> np.uint32(8))
        shift = _gf2_shift_matrix(chunk)
        acc = 0
        for r in regs.tolist():
            acc = _gf2_mat_times(shift, acc) ^ r
        reg = acc
        buf = buf[chunk * LANES:]
    tl = table.tolist()
    for b in buf.tolist():
        reg = tl[(reg ^ b) & 0xFF] ^ (reg >> 8)
    return reg ^ 0xFFFFFFFF


def mask_crc(crc):
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def unmask_crc(m):
    rot = (m - 0xA282EAD8) & 0xFFFFFFFF
    return ((rot >> 17) | (rot << 15)) & 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------------------
# varints + the three protobuf messages the bundle needs
# ---------------------------------------------------------------------------------------------------------------------
def _put_varint(out, v):
    v &= (1 << 64) - 1
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)


def _get_varint(buf, pos):
    shift = result = 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7


def _pb_fields(buf):
    """yield (field number, wire type, value) of one serialized message"""
    pos, n = 0, len(buf)
    while pos < n:
        tag, pos = _get_varint(buf, pos)
        f, w = tag >> 3, tag & 7
        if w == 0:
            v, pos = _get_varint(buf, pos)
        elif w == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        elif w == 2:
            ln, pos = _get_varint(buf, pos)
            v = bytes(buf[pos:pos + ln])
            pos += ln
        elif w == 5:
            v = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        else:
            raise ValueError("unsupported protobuf wire type %d" % w)
        yield f, w, v


# tensorflow/core/framework/types.proto
DT_FLOAT, DT_DOUBLE, DT_INT32, DT_UINT8, DT_INT16, DT_INT8, DT_INT64, DT_BOOL = 1, 2, 3, 4, 5, 6, 9, 10
_NP_OF_DT = {DT_FLOAT: np.float32, DT_DOUBLE: np.float64, DT_INT32: np.int32, DT_UINT8: np.uint8, DT_INT16: np.int16,
             DT_INT8: np.int8, DT_INT64: np.int64, DT_BOOL: np.bool_}
_DT_OF_NP = {np.dtype(v): k for k, v in _NP_OF_DT.items()}


def _encode_shape(shape):
    out = bytearray()
    for d in shape:                          # TensorShapeProto.dim = 2 { size = 1 }
        dim = bytearray()
        if d:
            dim.append(0x08)
            _put_varint(dim, d)
        out.append(0x12)
        _put_varint(out, len(dim))
        out += dim
    return bytes(out)


def _decode_shape(buf):
    shape = []
    for f, _, v in _pb_fields(buf):
        if f == 2:
            size = 0
            for g, _, u in _pb_fields(v):
                if g == 1:
                    size = u if u < (1 << 63) else u - (1 << 64)
            shape.append(size)
    return tuple(shape)


def _encode_entry(dtype, shape, offset, size, crc_masked):
    out = bytearray()
    out.append(0x08)
    _put_varint(out, dtype)
    sh = _encode_shape(shape)
    out.append(0x12)
    _put_varint(out, len(sh))
    out += sh
    # shard_id = 0 is the proto3 default and is not serialised
    if offset:
        out.append(0x20)
        _put_varint(out, offset)
    if size:
        out.append(0x28)
        _put_varint(out, size)
    out.append(0x35)
    out += struct.pack("<I", crc_masked)
    return bytes(out)


def _decode_entry(buf):
    e = {"dtype": 0, "shape": (), "shard_id": 0, "offset": 0, "size": 0, "crc32c": None, "slices": 0}
    for f, _, v in _pb_fields(buf):
        if f == 1:
            e["dtype"] = v
        elif f == 2:
            e["shape"] = _decode_shape(v)
        elif f == 3:
            e["shard_id"] = v
        elif f == 4:
            e["offset"] = v
        elif f == 5:
            e["size"] = v
        elif f == 6:
            e["crc32c"] = v
        elif f == 7:
            e["slices"] += 1
    return e


def _encode_header(num_shards=1):
    out = bytearray([0x08])
    _put_varint(out, num_shards)              # endianness LITTLE = 0: default, omitted
    out += bytes([0x1A, 0x02, 0x08, 0x01])    # version { producer: 1 }
    return bytes(out)


def _decode_header(buf):
    h = {"num_shards": 0, "endianness": 0}
    for f, _, v in _pb_fields(buf):
        if f == 1:
            h["num_shards"] = v
        elif f == 2:
            h["endianness"] = v
    return h


# ---------------------------------------------------------------------------------------------------------------------
# LevelDB-format table
# ---------------------------------------------------------------------------------------------------------------------
_MAGIC = 0xDB4775248B80FB57
_RESTART_INTERVAL = 16
_BLOCK_SIZE = 262144                          # tensorflow/core/lib/io/table_options.h default


class _BlockBuilder(object):
    def __init__(self):
        self.buf = bytearray()
        self.restarts = [0]
        self.counter = 0
        self.last_key = b""

    def add(self, key, value):
        shared = 0
        if self.counter < _RESTART_INTERVAL:
            m = min(len(key), len(self.last_key))
            while shared < m and key[shared] == self.last_key[shared]:
                shared += 1
        else:
            self.restarts.append(len(self.buf))
            self.counter = 0
        _put_varint(self.buf, shared)
        _put_varint(self.buf, len(key) - shared)
        _put_varint(self.buf, len(value))
        self.buf += key[shared:]
        self.buf += value
        self.last_key = key
        self.counter += 1

    def size(self):
        return len(self.buf) + 4 * len(self.restarts) + 4

    def finish(self):
        out = bytes(self.buf)
        out += b"".join(struct.pack("<I", r) for r in self.restarts)
        out += struct.pack("<I", len(self.restarts))
        return out


def _shortest_separator(a, b):
    """leveldb BytewiseComparator::FindShortestSeparator: a short key k with a <= k < b"""
    m = min(len(a), len(b))
    i = 0
    while i < m and a[i] == b[i]:
        i += 1
    if i < m and a[i] < 0xFF and a[i] + 1 < b[i]:
        return a[:i] + bytes([a[i] + 1])
    return a


def _short_successor(a):
    for i, c in enumerate(a):
        if c != 0xFF:
            return a[:i] + bytes([c + 1])
    return a


def _handle(offset, size):
    out = bytearray()
    _put_varint(out, offset)
    _put_varint(out, size)
    return bytes(out)


def write_table(path, items, block_size=_BLOCK_SIZE):
    """items: iterable of (key bytes, value bytes) in strictly increasing key order"""
    out = bytearray()
    index = _BlockBuilder()

    def emit(block_bytes):
        off = len(out)
        out.extend(block_bytes)
        out.append(0)                                                     # kNoCompression
        out.extend(struct.pack("<I", mask_crc(crc32c(block_bytes + b"\x00"))))
        return off, len(block_bytes)

    block, pending, last = _BlockBuilder(), None, None
    for key, value in items:
        if last is not None and key <= last:
            raise ValueError("table keys must be strictly increasing")
        if pending is not None:
            index.add(_shortest_separator(pending[0], key), _handle(*pending[1]))
            pending = None
        block.add(key, value)
        last = key
        if block.size() >= block_size:
            pending = (last, emit(block.finish()))
            block = _BlockBuilder()
    if block.buf:
        pending = (last, emit(block.finish()))
    if pending is not None:
        index.add(_short_successor(pending[0]), _handle(*pending[1]))
    meta = emit(_BlockBuilder().finish())
    idx = emit(index.finish())
    footer = bytearray(_handle(*meta) + _handle(*idx))
    footer += bytes(40 - len(footer))
    footer += struct.pack("<Q", _MAGIC)
    out += footer
    with open(path, "wb") as f:
        f.write(out)


def _snappy_decompress(src):
    n, pos = _get_varint(src, 0)
    out = bytearray()
    while pos < len(src):
        tag = src[pos]
        pos += 1
        kind = tag & 3
        if kind == 0:
            ln = tag >> 2
            if ln >= 60:
                nb = ln - 59
                ln = int.from_bytes(src[pos:pos + nb], "little")
                pos += nb
            ln += 1
            out += src[pos:pos + ln]
            pos += ln
            continue
        if kind == 1:
            ln = ((tag >> 2) & 7) + 4
            off = ((tag >> 5) << 8) | src[pos]
            pos += 1
        elif kind == 2:
            ln = (tag >> 2) + 1
            off = src[pos] | (src[pos + 1] << 8)
            pos += 2
        else:
            ln = (tag >> 2) + 1
            off = int.from_bytes(src[pos:pos + 4], "little")
            pos += 4
        if off == 0 or off > len(out):
            raise ValueError("corrupt snappy block")
        for _ in range(ln):                     # overlapping copies are legal
            out.append(out[-off])
    if len(out) != n:
        raise ValueError("snappy length mismatch")
    return bytes(out)


def _read_block(data, offset, size, verify=True):
    body = data[offset:offset + size]
    ctype = data[offset + size]
    stored = struct.unpack_from("<I", data, offset + size + 1)[0]
    if verify and unmask_crc(stored) != crc32c(data[offset:offset + size + 1]):
        raise ValueError("table block checksum mismatch at offset %d" % offset)
    if ctype == 1:
        body = _snappy_decompress(body)
    elif ctype != 0:
        raise ValueError("unknown block compression type %d" % ctype)
    return body


def _block_entries(block):
    n_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    end = len(block) - 4 - 4 * n_restarts
    pos, key = 0, b""
    while pos < end:
        shared, pos = _get_varint(block, pos)
        non_shared, pos = _get_varint(block, pos)
        vlen, pos = _get_varint(block, pos)
        key = key[:shared] + bytes(block[pos:pos + non_shared])
        pos += non_shared
        yield key, bytes(block[pos:pos + vlen])
        pos += vlen


def read_table(path, verify=True):
    """-> list of (key, value) in key order"""
    data = open(path, "rb").read()
    if len(data) < 48 or struct.unpack_from("<Q", data, len(data) - 8)[0] != _MAGIC:
        raise ValueError("%s is not a TensorFlow/LevelDB table (bad magic)" % path)
    footer = data[-48:]
    _, p = _get_varint(footer, 0)
    _, p = _get_varint(footer, p)
    ioff, p = _get_varint(footer, p)
    isize, p = _get_varint(footer, p)
    out = []
    for _, h in _block_entries(_read_block(data, ioff, isize, verify)):
        boff, q = _get_varint(h, 0)
        bsize, q = _get_varint(h, q)
        out.extend(_block_entries(_read_block(data, boff, bsize, verify)))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# bundles
# ---------------------------------------------------------------------------------------------------------------------
def write_bundle(prefix, tensors):
    """tensors: {name: array-like}. Writes <prefix>.index and <prefix>.data-00000-of-00001 (one shard, no compression)."""
    os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
    items = [(b"", _encode_header())]
    offset = 0
    with open(prefix + ".data-00000-of-00001", "wb") as f:
        for name in sorted(tensors, key=lambda s: s.encode()):
            a = np.asarray(tensors[name])
            if a.dtype not in _DT_OF_NP:
                raise ValueError("dtype %s of %r has no bundle encoding here" % (a.dtype, name))
            raw = np.ascontiguousarray(a).astype(a.dtype.newbyteorder("<"), copy=False).tobytes()
            f.write(raw)
            items.append((name.encode(), _encode_entry(_DT_OF_NP[a.dtype], a.shape, offset, len(raw), mask_crc(crc32c(raw)))))
            offset += len(raw)
    write_table(prefix + ".index", items)


def list_bundle(prefix, verify=True):
    """-> {name: entry dict(dtype, shape, shard_id, offset, size, crc32c)}"""
    rows = read_table(prefix + ".index", verify)
    if not rows or rows[0][0] != b"":
        raise ValueError("bundle index has no header entry")
    header = _decode_header(rows[0][1])
    if header["endianness"] != 0:
        raise ValueError("big-endian bundles are not supported")
    out = {k.decode(): _decode_entry(v) for k, v in rows[1:]}
    for e in out.values():
        e["num_shards"] = header["num_shards"]
    return out


def read_bundle(prefix, names=None, verify=True):
    """-> {name: numpy array}. `names` restricts what is loaded; sliced (partitioned) variables are rejected."""
    entries = list_bundle(prefix, verify)
    out, shards = {}, {}
    for name, e in entries.items():
        if names is not None and name not in names:
            continue
        if e["slices"]:
            raise ValueError("%s is a partitioned variable (slices): not supported" % name)
        if e["dtype"] not in _NP_OF_DT:
            raise ValueError("%s has unsupported dtype enum %d" % (name, e["dtype"]))
        sid = e["shard_id"]
        if sid not in shards:
            shards[sid] = np.memmap("%s.data-%05d-of-%05d" % (prefix, sid, e["num_shards"]), dtype=np.uint8, mode="r")
        raw = shards[sid][e["offset"]:e["offset"] + e["size"]]
        if verify and e["crc32c"] is not None and unmask_crc(e["crc32c"]) != crc32c(raw):
            raise ValueError("tensor %s: data checksum mismatch" % name)
        dt = np.dtype(_NP_OF_DT[e["dtype"]]).newbyteorder("<")
        out[name] = np.frombuffer(bytes(raw), dtype=dt).reshape(e["shape"]).astype(_NP_OF_DT[e["dtype"]], copy=True)
    return out


def write_checkpoint_state(save_dir, latest_name, all_names=None):
    """the `checkpoint` text proto tf.train.Saver maintains (CheckpointState)"""
    with open(os.path.join(save_dir, "checkpoint"), "w") as f:
        f.write('model_checkpoint_path: "%s"\n' % latest_name)
        for n in (all_names or [latest_name]):
            f.write('all_model_checkpoint_paths: "%s"\n' % n)


def read_checkpoint_state(save_dir):
    p = os.path.join(save_dir, "checkpoint")
    if not os.path.isfile(p):
        return None
    for line in open(p):
        line = line.strip()
        if line.startswith("model_checkpoint_path:"):
            return line.split(":", 1)[1].strip().strip('"')
    return None


# ---------------------------------------------------------------------------------------------------------------------
# variable-name map: this repo's tensor names (t2_taco_param_info / t2_wn_param_info) <-> the reference graph's variables
# ---------------------------------------------------------------------------------------------------------------------
def tacotron_tf_name(name):
    """engine tensor name -> variable name in the reference graph (scope `Tacotron_model/inference`, tacotron/train.py:79,
    tacotron/models/tacotron.py:104). Decoder-side variables are created inside dynamic_decode's `decoder` scope
    (tacotron.py:169-173): the prenet (modules.py:243-246), the MultiRNNCell (modules.py:274-282), the projections
    (modules.py:302-305,335-337) and the attention's per-step layers (attention.py:183 `Location_Sensitive_Attention`);
    `memory_layer` is built in BahdanauAttention.__init__ (attention.py:152-157), i.e. outside `decoder`."""
    P = "Tacotron_model/inference/"
    head, _, leaf = name.rpartition("/")
    if name == "inputs_embedding":
        return P + name
    for block in ("encoder_convolutions", "postnet_convolutions"):
        if head.startswith(block + "/conv_layer_"):
            i = head.rsplit("_", 1)[1]
            sub = "conv1d" if leaf in ("kernel", "bias") else "batch_normalization"
            return "%s%s/conv_layer_%s_%s/%s/%s" % (P, block, i, block, sub, leaf)
    if head in ("encoder_LSTM/fw", "encoder_LSTM/bw"):
        d = head[-2:]
        return "%sencoder_LSTM/bidirectional_rnn/%s/encoder_%s_LSTM/%s" % (P, d, d, leaf)
    if name.startswith("attention/memory_layer/"):
        return P + "memory_layer/" + leaf
    if name.startswith("attention/"):
        return P + "decoder/Location_Sensitive_Attention/" + name[len("attention/"):]
    if head.startswith("decoder_prenet/"):
        return P + "decoder/" + name
    if head.startswith("decoder_LSTM/cell_"):
        i = int(head.rsplit("_", 1)[1])
        return "%sdecoder/decoder_LSTM/multi_rnn_cell/cell_%d/decoder_LSTM_%d/%s" % (P, i - 1, i, leaf)
    if head in ("linear_transform_projection", "stop_token_projection"):
        return "%sdecoder/%s/projection_%s/%s" % (P, head, head, leaf)
    if head in ("postnet_projection", "cbhg_linear_specs_projection"):
        return "%s%s/projection_%s/%s" % (P, head, head, leaf)
    if head.startswith("CBHG_postnet"):
        # modules.py:19-78 under variable_scope('CBHG_postnet'): conv1d() scopes wrap tf.layers.conv1d / batch_normalization
        # (modules.py:379-391), highway layers are named '<scope>_highwaynet_<i>' (:33), the GRU cells '<scope>_forward_RNN' /
        # '<scope>_backward_RNN' inside bidirectional_dynamic_rnn's fw / bw scopes (:34-35,69-75), the width adapter is tf.layers.dense
        parts = head.split("/")
        if parts[1] in ("conv_bank", "proj1", "proj2"):
            sub = "conv1d" if leaf in ("kernel", "bias") else "batch_normalization"
            return "%s%s/%s/%s" % (P, head, sub, leaf)
        if parts[1].startswith("highwaynet_"):
            return "%sCBHG_postnet/CBHG_postnet_%s/%s/%s" % (P, parts[1], parts[2], leaf)
        if parts[1] in ("forward_RNN", "backward_RNN"):
            d = "fw" if parts[1].startswith("forward") else "bw"
            return "%sCBHG_postnet/bidirectional_rnn/%s/CBHG_postnet_%s/%s/%s" % (P, d, parts[1], parts[2], leaf)
        return P + name
    raise KeyError("no TensorFlow name known for engine tensor %r" % name)


def wavenet_tf_name(name, upsample_type="SubPixel"):
    """engine tensor name -> variable name in the reference graph (scope `WaveNet_model/inference`, wavenet_vocoder/train.py:169,
    wavenet.py:269). Every convolution of the reference is a keras Wrapper around a tf.layers conv that is built directly
    (modules.py:253-268), so its variables land in `<calling scope>/<layer name>/{kernel,bias}`: the residual blocks call
    their convs inside `variable_scope('ResidualConv1DGLU_<l>')` (modules.py:482) with layer names
    `residual_block_<role>_conv_ResidualConv1DGLU_<l>` (modules.py:412-450); first / last convs are named at wavenet.py:109-149;
    the upsampling layers `<Type>_layer_<i>` at wavenet.py:176-192. The saver of the reference stores the EMA shadow next to each
    variable as `<name>/ExponentialMovingAverage` (wavenet_vocoder/train.py:75-83). The speaker embedding is created outside the
    `inference` scope (modules.py:12-21): `WaveNet_model/gc_embedding`."""
    if name == "gc_embedding":
        return "WaveNet_model/gc_embedding"
    P = "WaveNet_model/inference/"
    head, _, leaf = name.rpartition("/")
    parts = head.split("/")
    if parts[0].startswith("ResidualConv1DGLU_") and len(parts) == 2:
        return "%s%s/%s_%s/%s" % (P, parts[0], parts[1], parts[0], leaf)
    if parts[0].startswith("local_conditioning_upsampling_"):
        i = int(parts[0].rsplit("_", 1)[1]) - 1
        kind = {"2D": "ConvTranspose2D", "1D": "ConvTranspose1D", "Resize": "ResizeConvolution"}.get(upsample_type, "SubPixelConvolution")
        return "%s%s_layer_%d/%s" % (P, kind, i, leaf)
    return P + name


def engine_name(tf_name):
    """inverse of tacotron_tf_name / wavenet_tf_name for a variable name WITHOUT slot suffix; None when the name is not a model
    variable of either graph (optimizer scalars, `global_step`, unrelated scopes). Outer scopes in front of `inference/` are ignored."""
    import re
    if tf_name == "WaveNet_model/gc_embedding" or tf_name.endswith("/WaveNet_model/gc_embedding"):
        return "gc_embedding"
    if "/inference/" not in tf_name:
        return None
    outer, tail = tf_name.split("/inference/", 1)
    if outer.endswith("WaveNet_model"):
        m = re.fullmatch(r"(ResidualConv1DGLU_\d+)/(residual_block_\w+?_conv)_\1/(\w+)", tail)
        if m:
            return "%s/%s/%s" % m.groups()
        m = re.fullmatch(r"(?:SubPixelConvolution|ConvTranspose2D|ConvTranspose1D|ResizeConvolution)_layer_(\d+)/(\w+)", tail)
        if m:
            return "local_conditioning_upsampling_%d/%s" % (int(m.group(1)) + 1, m.group(2))
        return tail
    m = re.fullmatch(r"(encoder_convolutions|postnet_convolutions)/conv_layer_(\d+)_\1/(?:conv1d|batch_normalization)/(\w+)", tail)
    if m:
        return "%s/conv_layer_%s/%s" % m.groups()
    m = re.fullmatch(r"encoder_LSTM/bidirectional_rnn/(fw|bw)/encoder_\1_LSTM/(\w+)", tail)
    if m:
        return "encoder_LSTM/%s/%s" % m.groups()
    m = re.fullmatch(r"decoder/decoder_LSTM/multi_rnn_cell/cell_\d+/decoder_LSTM_(\d+)/(\w+)", tail)
    if m:
        return "decoder_LSTM/cell_%s/%s" % m.groups()
    m = re.fullmatch(r"(CBHG_postnet/(?:conv_bank/conv1d_\d+|proj\d))/(?:conv1d|batch_normalization)/(\w+)", tail)
    if m:
        return "%s/%s" % m.groups()
    m = re.fullmatch(r"CBHG_postnet/CBHG_postnet_(highwaynet_\d+)/(H|T)/(\w+)", tail)
    if m:
        return "CBHG_postnet/%s/%s/%s" % m.groups()
    m = re.fullmatch(r"CBHG_postnet/bidirectional_rnn/(?:fw|bw)/CBHG_postnet_((?:forward|backward)_RNN)/(gates|candidate)/(\w+)", tail)
    if m:
        return "CBHG_postnet/%s/%s/%s" % m.groups()
    m = re.fullmatch(r"(?:decoder/)?(\w+)/projection_\1/(\w+)", tail)
    if m:
        return "%s/%s" % m.groups()
    if tail.startswith("memory_layer/"):
        return "attention/" + tail
    if tail.startswith("decoder/Location_Sensitive_Attention/"):
        return "attention/" + tail[len("decoder/Location_Sensitive_Attention/"):]
    if tail.startswith("decoder/decoder_prenet/"):
        return tail[len("decoder/"):]
    return tail


_SLOTS = (("/Adam_1", "adam_v"), ("/Adam", "adam_m"), ("/ExponentialMovingAverage", "ema"))


def load_as_engine_dicts(prefix, verify=True):
    """TF-V2 checkpoint -> (variables {engine name: array}, state {'global_step', 'adam_m', 'adam_v', 'ema'}) — the same
    structure t2_checkpoint.load returns for the native .npz files."""
    arrays = read_bundle(prefix, verify=verify)
    variables, state = {}, {"global_step": int(arrays.get("global_step", 0)), "adam_m": {}, "adam_v": {}, "ema": {}}
    for k, a in arrays.items():
        for suffix, tag in _SLOTS:
            if k.endswith(suffix):
                n = engine_name(k[:-len(suffix)])
                if n is not None:
                    state[tag][n] = a
                break
        else:
            n = engine_name(k)
            if n is not None:
                variables[n] = a
    return variables, state


def _name_fn(model, eng):
    if model == "Tacotron":
        return tacotron_tf_name
    kind = getattr(getattr(eng, "hp", None), "upsample_type", "SubPixel")
    return lambda n: wavenet_tf_name(n, kind)


def export_tf(prefix, model, eng, global_step=None):
    """Write a TF-V2 checkpoint of a product engine (t2.tacotron.Tacotron | t2.wavenet.WaveNet) under the reference's names:
    variables, Adam slots (`<var>/Adam`, `<var>/Adam_1`), WaveNet EMA shadows and `global_step`."""
    to_tf = _name_fn(model, eng)
    out = {}
    for k, v in eng.export_params().items():
        out[to_tf(k)] = np.asarray(v, dtype=np.float32)
    trainable = {t[0] for t in eng.tensors if (len(t) < 4 or t[3])}
    for buf, suffix in ((getattr(eng, "m", None), "/Adam"), (getattr(eng, "v", None), "/Adam_1"),
                        (getattr(eng, "ema", None), "/ExponentialMovingAverage")):
        if buf is None:
            continue
        for k, v in eng.unflatten(buf).items():
            if k in trainable:
                out[to_tf(k) + suffix] = np.asarray(v, dtype=np.float32)
    out["global_step"] = np.asarray(int(eng.global_step if global_step is None else global_step), dtype=np.int32)
    write_bundle(prefix, out)
    return sorted(out)


def import_tf(prefix, model, eng, use_ema=False, strict=True):
    """Load a TF-V2 checkpoint written by the reference (or by export_tf) into a product engine. Names are matched exactly
    first, then by unique suffix (checkpoints written under another outer scope). use_ema: take the
    `/ExponentialMovingAverage` shadows as the weights (what the reference's WaveNet synthesizer restores).
    -> (loaded names, missing engine tensors)"""
    import torch
    to_tf = _name_fn(model, eng)
    entries = list_bundle(prefix)
    keys = list(entries)

    def find(tf_name):
        if tf_name in entries:
            return tf_name
        tail = tf_name.split("/inference/", 1)[-1]
        cands = [k for k in keys if k.endswith("/" + tail) or k == tail]
        return cands[0] if len(cands) == 1 else None

    want, slots = {}, {}
    for t in eng.tensors:
        name = t[0]
        base = to_tf(name)
        key = find(base + "/ExponentialMovingAverage") if use_ema else None
        key = key or find(base)
        if key is not None:
            want[name] = key
        for tag, suffix in (("m", "/Adam"), ("v", "/Adam_1"), ("ema", "/ExponentialMovingAverage")):
            k = find(base + suffix)
            if k is not None:
                slots.setdefault(tag, {})[name] = k
    missing = [t[0] for t in eng.tensors if t[0] not in want]
    if strict and missing:
        raise KeyError("checkpoint %s lacks %d variables, e.g. %s" % (prefix, len(missing), missing[:3]))
    needed = set(want.values()) | {k for d in slots.values() for k in d.values()} | ({"global_step"} & set(keys))
    arrays = read_bundle(prefix, names=needed)
    current = eng.export_params()
    for name, key in want.items():
        a = arrays[key]
        if tuple(a.shape) != tuple(current[name].shape):
            raise ValueError("%s: checkpoint shape %s != model shape %s" % (key, a.shape, tuple(current[name].shape)))
        current[name] = torch.from_numpy(a.astype(np.float32))
    eng.load_params(current)

    def flat(d):
        buf = torch.zeros(eng.n_params, dtype=torch.float32)
        for t in eng.tensors:
            if t[0] in d:
                a = torch.from_numpy(arrays[d[t[0]]].astype(np.float32)).reshape(-1)
                buf[t[1]:t[1] + a.numel()] = a
        return buf.to(eng.device)
    if "m" in slots and "v" in slots:
        eng.m, eng.v = flat(slots["m"]), flat(slots["v"])
    if "ema" in slots and hasattr(eng, "ema"):
        eng.ema = flat(slots["ema"])
    if "global_step" in arrays:
        eng.global_step = int(arrays["global_step"])
    return sorted(want.values()), missing


if __name__ == "__main__":
    import sys
    for name, e in sorted(list_bundle(sys.argv[1]).items()):
        print("%-110s %-8s %s" % (name, np.dtype(_NP_OF_DT.get(e["dtype"], np.void)).name, e["shape"]))
