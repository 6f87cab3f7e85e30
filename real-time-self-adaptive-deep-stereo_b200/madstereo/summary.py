"""TensorBoard event files without TensorFlow: what tf.summary.FileWriter writes for scalar and image summaries.

File: `events.out.tfevents.<10-digit unix time>.<hostname>` in the log directory, a sequence of TFRecords
    uint64 length | uint32 masked CRC32C(length) | Event bytes | uint32 masked CRC32C(Event bytes)   (little endian)
whose first Event carries file_version "brain.Event:2" and every later one a Summary at a step.  The protobufs are
hand-encoded (tensorflow/core/util/event.proto, tensorflow/core/framework/summary.proto):
    Event         1: wall_time (double)  2: step (int64)  3: file_version (string)  5: summary (Summary)
    Summary       1: value (repeated Value)
    Value         1: tag (string)  2: simple_value (float)  4: image (Image)
    Image         1: height  2: width  3: colorspace (3 = RGB)  4: encoded_image_string (PNG)

AdaptationSummary is the drivers' --summary on top of it (Stereo_Online_Adaptation.py:131-140,196-199,235-236 and
Stereo_Continual_Adaptation.py:135-145,207-209,259-260 of the reference).
"""
import os
import socket
import struct
import time

import numpy as np

from .tf_checkpoint import _field, _put_varint, crc32c, mask_crc


def _bytes(num, payload):
    return _field(num, 2, _put_varint(len(payload)) + payload)


def _scalar_value(tag, value):
    return _bytes(1, tag.encode()) + _field(2, 5, struct.pack('<f', float(value)))


def _image_value(tag, image):
    """image: uint8 [H,W,3] RGB -> PNG (cv2 encodes BGR, so the channels are reversed on the way in)."""
    import cv2
    img = np.ascontiguousarray(np.asarray(image, dtype=np.uint8))
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('add_image: expected uint8 [height, width, 3], got %s' % (img.shape,))
    ok, png = cv2.imencode('.png', np.ascontiguousarray(img[..., ::-1]))
    if not ok:
        raise RuntimeError('add_image: PNG encoding failed')
    h, w = img.shape[:2]
    msg = _field(1, 0, _put_varint(h)) + _field(2, 0, _put_varint(w)) + _field(3, 0, _put_varint(3)) + _bytes(4, png.tobytes())
    return _bytes(1, tag.encode()) + _bytes(4, msg)


def _event(wall_time, step=0, file_version=None, values=None):
    msg = _field(1, 1, struct.pack('<d', wall_time))
    if step:
        msg += _field(2, 0, _put_varint(step))
    if file_version is not None:
        msg += _bytes(3, file_version.encode())
    if values is not None:
        msg += _bytes(5, b''.join(_bytes(1, v) for v in values))
    return msg


def tfrecord(data):
    """One TFRecord: length, masked CRC32C of the 8 length bytes, data, masked CRC32C of the data."""
    n = struct.pack('<Q', len(data))
    return n + struct.pack('<I', mask_crc(crc32c(n))) + data + struct.pack('<I', mask_crc(crc32c(data)))


class SummaryWriter(object):
    """tf.summary.FileWriter(logdir) with scalar and image summaries.  Values added for the same step go into one Event,
    as tf.summary.merge_all + FileWriter.add_summary(summary, global_step=step) write them; that Event is written when a
    value for another step arrives, on flush() and on close()."""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        now = time.time()
        self.path = os.path.join(logdir, 'events.out.tfevents.%010d.%s' % (int(now), socket.gethostname()))
        self._f = open(self.path, 'wb')
        self._f.write(tfrecord(_event(now, file_version='brain.Event:2')))
        self._step, self._values = None, []

    def _add(self, step, value):
        if self._values and step != self._step:
            self._write_pending()
        self._step = int(step)
        self._values.append(value)

    def add_scalar(self, tag, value, step):
        self._add(step, _scalar_value(tag, value))

    def add_image(self, tag, image, step):
        """image: uint8 [H,W,3] RGB (e.g. madstereo.ops.colorize_summary_image), stored as PNG."""
        self._add(step, _image_value(tag, image))

    def _write_pending(self):
        if self._values:
            self._f.write(tfrecord(_event(time.time(), self._step, values=self._values)))
            self._values = []

    def flush(self):
        self._write_pending()
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self.flush()
            self._f.close()


SUMMARY_EVERY = 100      # the reference fetches the summary op when step % 100 == 0


class AdaptationSummary(object):
    """The reference drivers' --summary: at steps that are multiples of 100, scalars `EPE` and `bad3` and, per map, the image
    `<name>/image` of colorize_img(map, cmap='jet') (image 0 of the batch), in that order, at global_step = step.

    `colorize(map) -> uint8 [H,W,3]` defaults to the device kernel (madstereo.ops.colorize_summary_image, the map copied
    to the current CUDA device if it is not there); tests substitute a host restatement."""

    def __init__(self, logdir, colorize=None):
        self.writer = SummaryWriter(logdir)
        self._colorize = colorize

    @staticmethod
    def due(step):
        return step % SUMMARY_EVERY == 0

    def _image(self, value):
        if self._colorize is not None:
            return self._colorize(value)
        import torch
        from . import ops
        t = value if torch.is_tensor(value) else torch.from_numpy(np.ascontiguousarray(value, dtype=np.float32))
        t = t.to(device=torch.device('cuda', torch.cuda.current_device()), dtype=torch.float32).contiguous()
        return ops.colorize_summary_image(t, cmap='jet').cpu().numpy()

    def add(self, step, epe, bad3, maps):
        """maps: [(name, [B,H,W,1] disparities)] in the reference's summary order."""
        self.writer.add_scalar('EPE', epe, step)
        self.writer.add_scalar('bad3', bad3, step)
        for name, value in maps:
            self.writer.add_image(name + '/image', self._image(value), step)
        self.writer.flush()

    def close(self):
        self.writer.close()
