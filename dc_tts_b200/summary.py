"""TensorBoard summaries without TensorFlow: what the reference's `tf.summary.scalar` / `tf.summary.image` /
`tf.summary.merge_all` (train.py:100-104,115-118,123,134) produce and what its `tf.train.Supervisor` (train.py:144) writes
to `logdir` -- serialized `Summary` protobufs inside `Event` records in an `events.out.tfevents.<secs>.<host>` file.

Records use TFRecord framing: uint64 length, masked CRC-32C of the length, the data, masked CRC-32C of the data (the
CRC-32C and its mask are checkpoint.py's, which reads TF's tensor bundles).  `read_events` parses such a file back and
verifies every checksum.

`audio` (the trainer's samples) is written from the same recollection of TF 1.x's Summary protobuf, also unchecked.

`image` follows TF 1.x's image summary op for float input, as recalled (not checked against TF): min and max over the
finite pixels; if min >= 0 the pixels are scaled by 255 / max, otherwise by 127 / max|x| and offset by 128 (a scale of 0
when that maximum is below 1e-6); the result is truncated to uint8, non-finite pixels become 255; 8-bit grayscale PNG.
"""
import os
import socket
import struct
import time
import zlib

import numpy as np

from .checkpoint import _proto_bytes_field, _proto_fields, _proto_varint_field, _put_varint, crc32c, mask_crc

FILE_VERSION = b"brain.Event:2"


# ------------------------------------------------------------------------------------ protobuf encoding
def _fixed32_field(field, v):
    return _put_varint((field << 3) | 5) + struct.pack("<f", float(v))


def _fixed64_field(field, v):
    return _put_varint((field << 3) | 1) + struct.pack("<d", float(v))


def _value(tag, body):
    """Summary.value (field 1): Value {tag = 1; simple_value = 2 | image = 4}."""
    return _proto_bytes_field(1, _proto_bytes_field(1, tag.encode()) + body)


def scalar(tag, value):
    """Serialized `Summary` with one scalar, as sess.run(tf.summary.scalar(tag, value)) returns it."""
    return _value(tag, _fixed32_field(2, np.float32(value)))


def png(pixels):
    """PNG bytes of uint8 pixels: (H, W) grayscale or (H, W, 3) RGB, no filtering, zlib-compressed."""
    px = np.ascontiguousarray(pixels, np.uint8)
    h, w = px.shape[:2]
    color = 0 if px.ndim == 2 else 2
    raw = b"".join(b"\x00" + px[r].tobytes() for r in range(h))

    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xffffffff)
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, color, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def image_pixels(array):
    """The uint8 pixels TF 1.x's image summary makes of one float (H, W) image (see the module docstring)."""
    x = np.asarray(array, np.float32)
    finite = np.isfinite(x)
    lo = float(x[finite].min()) if finite.any() else 0.0
    hi = float(x[finite].max()) if finite.any() else 0.0
    if lo >= 0:
        scale, offset = (np.float32(0) if hi < 1e-6 else np.float32(255) / np.float32(hi)), np.float32(0)
    else:
        m = max(abs(lo), abs(hi))
        scale, offset = (np.float32(0) if m < 1e-6 else np.float32(127) / np.float32(m)), np.float32(128)
    v = np.where(finite, x, np.float32(0)) * scale + offset
    out = np.clip(v, 0, 255).astype(np.uint8)
    out[~finite] = 255
    return out


def image(tag, array, max_outputs=3):
    """Serialized `Summary` of tf.summary.image(tag, array) for float images: array (n, H, W) or (n, H, W, 1); the first
    `max_outputs` images, tagged `<tag>/image/<i>` (`<tag>/image` when max_outputs is 1)."""
    a = np.asarray(array, np.float32)
    if a.ndim == 4:
        if a.shape[-1] != 1:
            raise ValueError("image: only one channel is supported, got shape %s" % (a.shape,))
        a = a[..., 0]
    if a.ndim != 3:
        raise ValueError("image: expected (n, H, W) or (n, H, W, 1), got shape %s" % (np.shape(array),))
    out = b""
    for i in range(min(len(a), max_outputs)):
        h, w = a[i].shape
        img = (_proto_varint_field(1, h) + _proto_varint_field(2, w) + _proto_varint_field(3, 1) +
               _proto_bytes_field(4, png(image_pixels(a[i]))))
        out += _value(tag + ("/image" if max_outputs == 1 else "/image/%d" % i), _proto_bytes_field(4, img))
    return out


def wav_bytes(wav, sample_rate):
    """A mono 16-bit PCM WAV file of float samples in [-1, 1] (clipped, scaled by 32767 and rounded)."""
    pcm = np.round(np.clip(np.asarray(wav, np.float32), -1.0, 1.0) * 32767.0).astype("<i2").tobytes()
    fmt = struct.pack("<HHIIHH", 1, 1, int(sample_rate), 2 * int(sample_rate), 2, 16)
    return (b"RIFF" + struct.pack("<I", 36 + len(pcm)) + b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt +
            b"data" + struct.pack("<I", len(pcm)) + pcm)


def audio(tag, wav, sample_rate):
    """Serialized `Summary` with one audio clip, tagged `<tag>/audio/0` as tf.summary.audio(tag, ..., max_outputs=1) names
    it: Value.audio (field 6) = {sample_rate, num_channels 1, length_frames, 16-bit PCM WAV bytes (wav_bytes),
    content_type "audio/wav"}.  Written from the TF 1.x protobuf definitions as recalled, not checked against TF."""
    n = int(np.asarray(wav).shape[0])
    body = (_fixed32_field(1, sample_rate) + _proto_varint_field(2, 1) + _proto_varint_field(3, n) +
            _proto_bytes_field(4, wav_bytes(wav, sample_rate)) + _proto_bytes_field(5, b"audio/wav"))
    return _value(tag + "/audio/0", _proto_bytes_field(6, body))


def merge(*summaries):
    """tf.summary.merge: the values of several serialized Summaries in one (protobuf messages concatenate)."""
    return b"".join(summaries)


def train_summary(num, losses, target, output, lr):
    """What sess.run(g.merged) returns for the reference's training graph (train.py:100-104,115-118,123, in the order
    merge_all collects them): the losses, the first utterance's ground truth `target` and network output `output`
    ((B, T, C) arrays: mels and Y for num = 1, mags and Z for num = 2) transposed to (1, C, T) images, and `lr`."""
    gt, hat = np.asarray(target[:1], np.float32), np.asarray(output[:1], np.float32)
    if num == 1:
        parts = [scalar("train/loss_mels", losses["loss_mels"]), scalar("train/loss_bd1", losses["loss_bd1"]),
                 scalar("train/loss_att", losses["loss_att"]),
                 image("train/mel_gt", gt.transpose(0, 2, 1)), image("train/mel_hat", hat.transpose(0, 2, 1))]
    else:
        parts = [scalar("train/loss_mags", losses["loss_mags"]), scalar("train/loss_bd2", losses["loss_bd2"]),
                 image("train/mag_gt", gt.transpose(0, 2, 1)), image("train/mag_hat", hat.transpose(0, 2, 1))]
    return merge(*parts, scalar("lr", lr))


# ------------------------------------------------------------------------------------ event files
def _record(data):
    n = struct.pack("<Q", len(data))
    return n + struct.pack("<I", mask_crc(crc32c(n))) + data + struct.pack("<I", mask_crc(crc32c(data)))


class FileWriter:
    """tf.summary.FileWriter(logdir): a new `events.out.tfevents.<secs>.<host>` file whose first event carries the file
    version; add_summary(summary bytes, step) appends one event with the wall time."""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        now = time.time()
        base = os.path.join(logdir, "events.out.tfevents.%010d.%s" % (int(now), socket.gethostname()))
        self.path, n = base, 0
        while os.path.exists(self.path):         # a second writer in the same second must not overwrite the first file
            n += 1
            self.path = "%s.%d" % (base, n)
        self._f = open(self.path, "xb")
        self._write(_fixed64_field(1, now) + _proto_bytes_field(3, FILE_VERSION))

    def _write(self, event):
        self._f.write(_record(event))

    def add_summary(self, summary, global_step):
        self._write(_fixed64_field(1, time.time()) + _proto_varint_field(2, int(global_step)) + _proto_bytes_field(5, summary))

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.close()


def parse_summary(buf):
    """Summary bytes -> [(tag, float) for scalars, (tag, {height, width, colorspace, png}) for images or
    (tag, {sample_rate, num_channels, length_frames, wav, content_type}) for audio]."""
    out = []
    for field, _, val in _proto_fields(buf):
        if field != 1:
            continue
        tag, v = None, None
        for f, wt, x in _proto_fields(val):
            if f == 1:
                tag = x.decode()
            elif f == 2 and wt == 5:
                v = struct.unpack("<f", struct.pack("<I", x))[0]
            elif f == 4:
                img = {1: "height", 2: "width", 3: "colorspace", 4: "png"}
                v = {img[k]: y for k, _, y in _proto_fields(x) if k in img}
            elif f == 6:
                au = {1: "sample_rate", 2: "num_channels", 3: "length_frames", 4: "wav", 5: "content_type"}
                v = {au[k]: y for k, _, y in _proto_fields(x) if k in au}
                if "sample_rate" in v:
                    v["sample_rate"] = struct.unpack("<f", struct.pack("<I", v["sample_rate"]))[0]
        out.append((tag, v))
    return out


def read_events(path):
    """The events of a TFRecord event file as dicts {wall_time, step, file_version?, summary?}; raises on a bad checksum."""
    data = open(path, "rb").read()
    pos, events = 0, []
    while pos < len(data):
        n = struct.unpack_from("<Q", data, pos)[0]
        if struct.unpack_from("<I", data, pos + 8)[0] != mask_crc(crc32c(data[pos:pos + 8])):
            raise ValueError("%s: bad length checksum at offset %d" % (path, pos))
        body = data[pos + 12:pos + 12 + n]
        if len(body) != n or struct.unpack_from("<I", data, pos + 12 + n)[0] != mask_crc(crc32c(body)):
            raise ValueError("%s: bad data checksum at offset %d" % (path, pos))
        pos += 16 + n
        ev = {"step": 0}
        for field, _, v in _proto_fields(body):
            if field == 1:
                ev["wall_time"] = struct.unpack("<d", struct.pack("<Q", v))[0]
            elif field == 2:
                ev["step"] = v
            elif field == 3:
                ev["file_version"] = v.decode()
            elif field == 5:
                ev["summary"] = parse_summary(v)
        events.append(ev)
    return events
