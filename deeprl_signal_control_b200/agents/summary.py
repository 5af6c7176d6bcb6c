"""TensorBoard event files without tensorflow, tensorboard or protobuf: the scalars the reference's `main.py train` writes
with `tf.summary.FileWriter(dirs['log'])` (utils.py:129-140, agents/policies.py:62-72, 331-338).

    w = SummaryWriter(log_dir)            # <log_dir>/events.out.tfevents.<time>.<host>
    w.add_scalar('train_reward', -412.5, step=720)
    w.close()
    read_scalars(w.path)                  # {'train_reward': [(wall_time, 720, -412.5)]}

The file is a sequence of TFRecords (uint64 length, masked CRC32C of the length, the record, masked CRC32C of the record,
little-endian), each an `Event` protocol buffer encoded by hand: first `file_version: "brain.Event:2"`, then one event
per `add_scalars` call, `{wall_time, step, summary {value {tag, simple_value}}}`, the form of TF1's `tf.summary.scalar`.
`tensorboard --logdir <agent>/log` and the reference's `extract_tensorboard.py` read it.

`summary_name` and `a2c_events` / `iql_events` say which tags the training driver writes and at which steps.
"""
from __future__ import annotations

import os
import socket
import struct
import time

import numpy as np

_CRC_TABLE = []
for _n in range(256):
    _c = _n
    for _ in range(8):
        _c = (_c >> 1) ^ 0x82F63B78 if _c & 1 else _c >> 1       # CRC-32C (Castagnoli), reflected
    _CRC_TABLE.append(_c)


def crc32c(data: bytes) -> int:
    crc = 0xFFFFFFFF
    t = _CRC_TABLE
    for b in data:
        crc = t[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def masked_crc32c(data: bytes) -> int:
    """The TFRecord checksum: the CRC rotated right by 15 bits plus 0xa282ead8."""
    c = crc32c(data)
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


# ---- protocol-buffer wire format: only what Event / Summary / Summary.Value need ------------------------------------
def _varint(n: int) -> bytes:
    n &= (1 << 64) - 1                                             # int64: two's complement, ten bytes when negative
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _key(field: int, wire: int) -> bytes:
    return _varint(field << 3 | wire)


def _bytes_field(field: int, data: bytes) -> bytes:
    return _key(field, 2) + _varint(len(data)) + data


def encode_event(wall_time: float, step: int = 0, values=None, file_version: str | None = None) -> bytes:
    """Event{wall_time = 1 (double), step = 2 (int64), file_version = 3 (string), summary = 5 (Summary)};
    Summary{repeated value = 1}; Summary.Value{tag = 1 (string), simple_value = 2 (float)}."""
    out = _key(1, 1) + struct.pack('<d', float(wall_time)) + _key(2, 0) + _varint(int(step))
    if file_version is not None:
        out += _bytes_field(3, file_version.encode())
    if values:
        summ = b''.join(_bytes_field(1, _bytes_field(1, str(tag).encode()) + _key(2, 5) + struct.pack('<f', float(v)))
                        for tag, v in values.items())
        out += _bytes_field(5, summ)
    return out


def _fields(buf: bytes):
    """(field, wire type, value) of every field of one message: ints for varints, bytes otherwise."""
    i, n = 0, len(buf)
    while i < n:
        key, i = _read_varint(buf, i)
        field, wire = key >> 3, key & 7
        if wire == 0:
            v, i = _read_varint(buf, i)
        elif wire == 1:
            v, i = buf[i:i + 8], i + 8
        elif wire == 2:
            ln, i = _read_varint(buf, i)
            v, i = buf[i:i + ln], i + ln
        elif wire == 5:
            v, i = buf[i:i + 4], i + 4
        else:
            raise ValueError('unsupported protobuf wire type %d' % wire)
        if i > n:
            raise ValueError('truncated protobuf message')
        yield field, wire, v


def _read_varint(buf: bytes, i: int):
    shift = result = 0
    while True:
        if i >= len(buf):
            raise ValueError('truncated varint')
        b = buf[i]
        i += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, i
        shift += 7


def decode_event(buf: bytes):
    """(wall_time, step, file_version or None, [(tag, simple_value)]) of one Event; values without simple_value are
    skipped."""
    wall_time, step, version, values = 0.0, 0, None, []
    for f, w, v in _fields(buf):
        if f == 1 and w == 1:
            wall_time = struct.unpack('<d', v)[0]
        elif f == 2 and w == 0:
            step = v - (1 << 64) if v >= 1 << 63 else v
        elif f == 3 and w == 2:
            version = v.decode()
        elif f == 5 and w == 2:
            for sf, sw, sv in _fields(v):
                if sf != 1 or sw != 2:
                    continue
                tag, val = None, None
                for vf, vw, vv in _fields(sv):
                    if vf == 1 and vw == 2:
                        tag = vv.decode()
                    elif vf == 2 and vw == 5:
                        val = struct.unpack('<f', vv)[0]
                if tag is not None and val is not None:
                    values.append((tag, val))
    return wall_time, step, version, values


def read_records(path):
    """The records of a TFRecord file, both checksums of each verified (ValueError on a mismatch or a cut record)."""
    with open(path, 'rb') as f:
        data = f.read()
    i, out = 0, []
    while i < len(data):
        if i + 12 > len(data):
            raise ValueError('%s: truncated record header at byte %d' % (path, i))
        head = data[i:i + 8]
        (n,) = struct.unpack('<Q', head)
        (crc_len,) = struct.unpack('<I', data[i + 8:i + 12])
        if crc_len != masked_crc32c(head):
            raise ValueError('%s: bad length checksum at byte %d' % (path, i))
        if i + 12 + n + 4 > len(data):
            raise ValueError('%s: truncated record at byte %d' % (path, i))
        rec = data[i + 12:i + 12 + n]
        (crc_data,) = struct.unpack('<I', data[i + 12 + n:i + 16 + n])
        if crc_data != masked_crc32c(rec):
            raise ValueError('%s: bad data checksum at byte %d' % (path, i))
        out.append(rec)
        i += 16 + n
    return out


def read_scalars(path):
    """{tag: [(wall_time, step, value)]} of an event file, in file order (values are float32, returned as float)."""
    out = {}
    for rec in read_records(path):
        wall_time, step, _, values = decode_event(rec)
        for tag, v in values:
            out.setdefault(tag, []).append((wall_time, step, v))
    return out


def event_files(log_dir):
    """The event files of a directory, sorted by name (that is, by creation time)."""
    return sorted(os.path.join(log_dir, f) for f in os.listdir(log_dir) if f.startswith('events.out.tfevents.'))


class SummaryWriter:
    """tf.summary.FileWriter's scalar path: `<log_dir>/events.out.tfevents.<time>.<host>`, opened on construction with
    its file_version event.  An existing file of the same name is never overwritten: a numeric suffix is added."""

    def __init__(self, log_dir):
        os.makedirs(log_dir, exist_ok=True)
        base = os.path.join(log_dir, 'events.out.tfevents.%010d.%s' % (int(time.time()), socket.gethostname()))
        path, k = base, 0
        while True:
            try:
                self._f = open(path, 'xb')
                break
            except FileExistsError:
                k += 1
                path = '%s.%d' % (base, k)
        self.path = path
        self._write(encode_event(time.time(), 0, file_version='brain.Event:2'))
        self.flush()

    def _write(self, rec: bytes):
        head = struct.pack('<Q', len(rec))
        self._f.write(head + struct.pack('<I', masked_crc32c(head)) + rec + struct.pack('<I', masked_crc32c(rec)))

    def add_scalars(self, values: dict, step: int, wall_time: float | None = None):
        """One event holding several scalars at one step (the reference's merged summaries)."""
        self._write(encode_event(time.time() if wall_time is None else wall_time, step, values))

    def add_scalar(self, tag: str, value: float, step: int, wall_time: float | None = None):
        self.add_scalars({tag: value}, step, wall_time)

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


# ---- what the training driver writes --------------------------------------------------------------------------------
def summary_name(agent: str, policy: str = 'lstm', model_type: str | None = None) -> str:
    """The scope of agent 0's policy, whose scalars the reference writes (agents/policies.py:77, 168, 216, 261, 343, 386;
    agents/models.py names agent i '%da'): lstm / fplstm (ia2c / ma2c), fc / fpfc (FC policy), dqn / lr (IQL)."""
    if agent in ('ia2c', 'ma2c'):
        base = 'fc' if policy == 'fc' else 'lstm'
        return ('fp' + base if agent == 'ma2c' else base) + '_0a'
    return ('dqn' if model_type == 'dqn' else 'lr') + '_0a'


def a2c_values(name: str, rec):
    """The four scalars of one A2C update from its record (policy, value, entropy loss, pre-clip gradient norm)
    (agents/policies.py:62-72): total_loss = policy + value + entropy in float32, as the TF graph adds them."""
    p, v, e, g = (np.float32(x) for x in rec[:4])
    return {'loss/%s_policy_loss' % name: p, 'loss/%s_value_loss' % name: v,
            'loss/%s_total_loss' % name: np.float32(np.float32(p + v) + e), 'train/%s_gradnorm' % name: g}


def a2c_events(name: str, rec, first_step: int, n_step: int):
    """[(step, values)] of one episode set's A2C updates: rec [n_updates, 4], update j at first_step + j * n_step (the
    global step of its backward, utils.py:288-291)."""
    return [(int(first_step + j * n_step), a2c_values(name, rec[j])) for j in range(len(rec))]


def iql_events(name: str, rec, ran, first_step: int, n_step: int):
    """[(step, values)] of one episode set's IQL updates: rec [n_updates, rounds, 4] of (loss, q, tq, gradnorm),
    round k of update j at first_step + j * n_step + k (agents/models.py:337-345); an update that did not run (the
    replay buffer held fewer than batch_size entries) writes nothing."""
    out = []
    for j in range(len(rec)):
        if not ran[j]:
            continue
        for k in range(len(rec[j])):
            loss, q, tq, g = (np.float32(x) for x in rec[j][k][:4])
            out.append((int(first_step + j * n_step + k), {'train/%s_loss' % name: loss, 'train/%s_q' % name: q,
                                                          'train/%s_tq' % name: tq, 'train/%s_gradnorm' % name: g}))
    return out
