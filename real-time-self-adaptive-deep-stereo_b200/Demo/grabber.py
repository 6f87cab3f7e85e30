"""Stereo frame grabbers of the live demo: the reference's camera factory (Demo/grabber.py), plus a list-file grabber.

Every grabber is a thread that puts `[2,h,w,3]` uint8 arrays (left, right) on a shared queue.  A grabber whose source
ends puts END_OF_STREAM on the queue and stops.
"""
import abc
import json
import queue
import threading
import time

import numpy as np

END_OF_STREAM = None

_GRABBER_FACTORY = {}


def get_camera(name, frame_queue, config=None, framerate=30):
    """Factory method to construct a camera wrapper."""
    if name not in _GRABBER_FACTORY:
        raise Exception('Unrecognized camera type: {}'.format(name))
    return _GRABBER_FACTORY[name](frame_queue, config=config, framerate=framerate)


def get_available_camera():
    return _GRABBER_FACTORY.keys()


def register_camera_to_factory():
    def decorator(cls):
        _GRABBER_FACTORY[cls._name] = cls
        return cls
    return decorator


class ImageGrabber(threading.Thread, metaclass=abc.ABCMeta):
    """Thread that grabs frames from a camera and loads them in frame_queue.

    frame_queue: synchronised queue where [2,h,w,3] left/right frames are put; config: path to a JSON file of camera
    parameters; framerate: target frames per second (<= 0: no pacing)."""
    needs_config = True

    def __init__(self, frame_queue, config=None, framerate=30):
        threading.Thread.__init__(self, daemon=True)
        self._config = config
        self._connect_to_camera()
        self._buffer = frame_queue
        self._sleeptime = 1.0 / framerate if framerate and framerate > 0 else 0.0
        self._stop_acquire = False

    def stop(self):
        """Stop the acquisition of new frames and end the thread."""
        self._stop_acquire = True

    def _put(self, item):
        # the queue holds one frame: wait for room, but give up when stopped (the consumer may be gone)
        while not self._stop_acquire:
            try:
                self._buffer.put(item, timeout=0.1)
                return True
            except queue.Full:
                pass
        return False

    def run(self):
        """Grab frames and put them on the queue as [2,h,w,c] arrays until stopped or the source ends."""
        try:
            while not self._stop_acquire:
                frames = self._read_frame()
                if frames is None:
                    self._put(END_OF_STREAM)
                    break
                l, r = frames
                if not self._put(np.stack([l, r], axis=0)):
                    break
                if self._sleeptime:
                    time.sleep(self._sleeptime)
        finally:
            self._disconnect_from_camera()

    @abc.abstractmethod
    def _read_frame(self):
        """Read left and right rectified frames and return them (None at the end of the stream)."""

    @abc.abstractmethod
    def _connect_to_camera(self):
        """Connect to the camera."""

    @abc.abstractmethod
    def _disconnect_from_camera(self):
        """Disconnect from the camera."""


@register_camera_to_factory()
class ImageList(ImageGrabber):
    """Replays a `left;right[;...]` list file (the format of Data_utils.data_reader) as uint8 RGB frames.

    config: JSON file {"list": path, "fps": frames per second}; fps 0 (or absent) means no pacing.  A "calibration" key
    is read by the demo, not here: the listed frames are then raw and are rectified on the device."""
    _name = 'ImageList'

    def _connect_to_camera(self):
        from Data_utils import data_reader
        with open(self._config) as f_in:
            cfg = json.load(f_in)
        self._lefts, self._rights, _, _ = data_reader.read_list_file(cfg['list'])
        self._fps = float(cfg.get('fps', 0))
        self._read = data_reader.read_image_u8_from_disc
        self._next = 0

    def __init__(self, frame_queue, config=None, framerate=30):
        ImageGrabber.__init__(self, frame_queue, config=config, framerate=framerate)
        self._sleeptime = 1.0 / self._fps if self._fps > 0 else 0.0      # the list's own pacing replaces --framerate

    def _read_frame(self):
        if self._next >= len(self._lefts):
            return None
        i = self._next
        self._next += 1
        return self._read(self._lefts[i]), self._read(self._rights[i])

    def _disconnect_from_camera(self):
        pass


try:
    import pyzed.sl as sl
except ImportError:
    sl = None

if sl is not None:
    @register_camera_to_factory()
    class ZEDMini(ImageGrabber):
        """Read stereo frames from a ZED Mini stereo camera (BGRA frames; the first three channels are passed on as they
        are, as the reference does)."""
        _name = 'ZED_Mini'
        _key_to_res = {
            '2K': sl.RESOLUTION.RESOLUTION_HD2K,
            '1080p': sl.RESOLUTION.RESOLUTION_HD1080,
            '720p': sl.RESOLUTION.RESOLUTION_HD720,
            'VGA': sl.RESOLUTION.RESOLUTION_VGA,
        }

        def _read_frame(self):
            err = self._cam.grab(self._runtime)
            if err == sl.ERROR_CODE.SUCCESS:
                self._cam.retrieve_image(self._left_frame, sl.VIEW.VIEW_LEFT)
                self._cam.retrieve_image(self._right_frame, sl.VIEW.VIEW_RIGHT)
                return self._left_frame.get_data()[:, :, :3], self._right_frame.get_data()[:, :, :3]

        def _connect_to_camera(self):
            with open(self._config) as f_in:
                self._config = json.load(f_in)
            self._params = sl.InitParameters()
            self._params.camera_resolution = self._key_to_res[self._config['resolution']] if 'resolution' in self._config \
                else sl.RESOLUTION.RESOLUTION_HD720
            self._params.camera_fps = self._config['fps'] if 'fps' in self._config else 30
            self._cam = sl.Camera()
            status = self._cam.open(self._params)
            if status != sl.ERROR_CODE.SUCCESS:
                print(status)
                raise Exception('Unable to connect to Stereo Camera')
            self._runtime = sl.RuntimeParameters()
            self._left_frame = sl.Mat()
            self._right_frame = sl.Mat()

        def _disconnect_from_camera(self):
            self._cam.close()
