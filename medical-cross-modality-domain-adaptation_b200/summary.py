"""TensorBoard event files without TensorFlow: what `tf.summary.FileWriter(dir)` + `add_summary(scalar_summary_op, step)` +
`add_summary(image_summary_op, step)` leave on disk (adversarial.py:664-697, 807-808, 989-991; source_segmenter.py:394-409,
452-453, 537-539, 568-570).

An event file is a TFRecord stream (the framing `tfrecord.write_record` already implements: u64 length, masked CRC32C of the length,
payload, masked CRC32C of the payload -- CRC32C from libpnp_io.so) of serialized `tensorflow.Event` messages.  The fields needed
are encoded by hand from event.proto / summary.proto:

    Event   { double wall_time = 1; int64 step = 2; oneof what { string file_version = 3; Summary summary = 5; } }
    Summary { repeated Value value = 1; }      Value { string tag = 1; float simple_value = 2; Image image = 4; }
    Image   { int32 height = 1; int32 width = 2; int32 colorspace = 3; bytes encoded_image_string = 4; }

The first record of a file is the version event `brain.Event:2`, as TensorFlow writes it.  Image summaries carry 8-bit grayscale
PNGs (`encode_png`, stdlib zlib) of the uint8 panels that functional.image_summary renders on the GPU, tagged as TF-1.4's
ImageSummaryOp tags them (`image_tags`).  The `graph=sess.graph` GraphDef event is not written.  tests/test_summary_cpu.py and
tests/test_image_summary_cpu.py read the files back with the `tensorboard` package's own loader."""
import os
import socket
import struct
import time
import zlib

from .tfrecord import _enc_varint, _ld, masked_crc


def _key(field, wire):
    return _enc_varint((field << 3) | wire)


def encode_scalar_summary(scalars):
    """Summary message with one Value per (tag, number) pair, in the given order (the order of the merged summary op)"""
    out = b""
    for tag, v in scalars:
        value = _ld(1, str(tag).encode("utf-8")) + _key(2, 5) + struct.pack("<f", float(v))
        out += _ld(1, value)
    return out


def _png_chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def encode_png(u8_hw):
    """8-bit grayscale PNG (colour type 0) of a uint8 [H, W] array: every row with filter byte 0 (none), one IDAT deflated at
    zlib's default level (TF's png encoder runs with compression = -1, the same default)"""
    import numpy as np
    a = np.ascontiguousarray(u8_hw, dtype=np.uint8)
    if a.ndim != 2 or a.shape[0] < 1 or a.shape[1] < 1:
        raise ValueError("encode_png: expected a non-empty uint8 [H, W] array, got shape %s" % (a.shape,))
    h, w = a.shape
    raw = np.zeros((h, w + 1), np.uint8)
    raw[:, 1:] = a
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)
    return (b"\x89PNG\r\n\x1a\n" + _png_chunk(b"IHDR", ihdr) + _png_chunk(b"IDAT", zlib.compress(raw.tobytes(), -1))
            + _png_chunk(b"IEND", b""))


def image_tags(name, n):
    """the tags TF-1.4's ImageSummaryOp gives the first n images of a batch when max_images > 1: '<name>/image/<i>'"""
    return ["%s/image/%d" % (name, i) for i in range(n)]


def encode_image_summary(images):
    """Summary message with one Value{tag, image} per (tag, uint8 [H, W] panel) pair, in the given order (colorspace 1 = depth 1)"""
    out = b""
    for tag, u8 in images:
        h, w = u8.shape
        img = (_key(1, 0) + _enc_varint(int(h)) + _key(2, 0) + _enc_varint(int(w)) + _key(3, 0) + _enc_varint(1)
               + _ld(4, encode_png(u8)))
        out += _ld(1, _ld(1, str(tag).encode("utf-8")) + _ld(4, img))
    return out


def encode_event(wall_time, step=None, file_version=None, summary=None):
    ev = _key(1, 1) + struct.pack("<d", float(wall_time))
    if step is not None:
        ev += _key(2, 0) + _enc_varint(int(step) & 0xFFFFFFFFFFFFFFFF)
    if file_version is not None:
        ev += _ld(3, file_version.encode("utf-8"))
    if summary is not None:
        ev += _ld(5, summary)
    return ev


def frame(payload):
    head = struct.pack("<Q", len(payload))
    return head + struct.pack("<I", masked_crc(head)) + payload + struct.pack("<I", masked_crc(payload))


class FileWriter(object):
    """tf.summary.FileWriter for scalar and image summaries: `events.out.tfevents.<seconds>.<hostname>` under `logdir`, appended and flushed per call."""

    def __init__(self, logdir, filename_suffix=""):
        os.makedirs(logdir, exist_ok=True)
        self.logdir = logdir
        now = time.time()
        self.path = os.path.join(logdir, "events.out.tfevents.%010d.%s.%d%s" % (int(now), socket.gethostname(), os.getpid(),
                                                                              filename_suffix))
        self._f = open(self.path, "ab")
        self._f.write(frame(encode_event(now, file_version="brain.Event:2")))
        self._f.flush()

    def add_scalars(self, scalars, step, wall_time=None):
        """one Event carrying every (tag, value) pair: what add_summary(sess.run(tf.summary.merge(scalar_summaries)), step) writes.
        `scalars`: dict (insertion order kept) or a list of pairs."""
        items = list(scalars.items()) if hasattr(scalars, "items") else list(scalars)
        ev = encode_event(time.time() if wall_time is None else wall_time, step=step, summary=encode_scalar_summary(items))
        self._f.write(frame(ev))

    def add_images(self, images, step, wall_time=None):
        """one Event carrying every (tag, uint8 [H, W] panel) pair: add_summary(sess.run(tf.summary.merge(image_summaries)), step)"""
        ev = encode_event(time.time() if wall_time is None else wall_time, step=step, summary=encode_image_summary(list(images)))
        self._f.write(frame(ev))

    def add_summary(self, summary, global_step=None):
        """the reference's call shape: `summary` is a serialized Summary message (bytes) or a dict of scalars"""
        if isinstance(summary, (bytes, bytearray)):
            self._f.write(frame(encode_event(time.time(), step=global_step, summary=bytes(summary))))
        else:
            self.add_scalars(summary, global_step)

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.flush()
            self._f.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
