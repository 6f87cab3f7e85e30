"""Stereo rectification tables from a calibration file, for `StereoEngine.set_rectification`.

The file is what `cv2.FileStorage` reads and writes (YAML, XML or JSON): `image_width` and `image_height` of the frames
it was calibrated on, the intrinsics `K1 D1 K2 D2` of the left and right camera (pinhole, 4, 5, 8, 12 or 14 distortion
coefficients), and then either

  * `R T` (right camera relative to the left, as `cv2.stereoCalibrate` returns them) and an optional `alpha` (default 0):
    the rectification is computed here with `cv2.stereoRectify(..., flags=CALIB_ZERO_DISPARITY, alpha=alpha)`, or
  * `R1 R2 P1 P2`: a rectification computed elsewhere, used as it is.

The tables are `cv2.initUndistortRectifyMap(K, D, R_i, P_i, size, CV_32FC1)` stacked as float32 [h, w, 2] =
(src_x, src_y) per output pixel.  They are built once on the host; the device only resamples through them, so any model
whose tables are built this way (fisheye included, with `cv2.fisheye.initUndistortRectifyMap`) can be handed to the
engine directly.
"""
import numpy as np

from ._lib import MadStereoError

INTRINSICS = ('K1', 'D1', 'K2', 'D2')
EXTRINSICS = ('R', 'T')
RECTIFICATION = ('R1', 'R2', 'P1', 'P2')


def load_calibration(path):
    """Read a stereo calibration: dict of float64 arrays by key, plus 'size' = (height, width) and 'alpha'."""
    import cv2
    try:
        fs = cv2.FileStorage(str(path), cv2.FILE_STORAGE_READ)
    except cv2.error as ex:
        raise MadStereoError('calibration %s: not a file cv2.FileStorage reads (%s)' % (path, ex))
    if not fs.isOpened():
        raise MadStereoError('calibration %s: cannot be opened' % (path,))
    try:
        def present(k):
            return not fs.getNode(k).isNone()

        rectified = all(present(k) for k in RECTIFICATION)
        need = ('image_width', 'image_height') + INTRINSICS + (RECTIFICATION if rectified else EXTRINSICS)
        missing = [k for k in need if not present(k)]
        if missing:
            raise MadStereoError('calibration %s: missing %s (it needs image_width image_height K1 D1 K2 D2 and either '
                                 'R T or R1 R2 P1 P2)' % (path, ' '.join(missing)))
        calib = {}
        for k in need[2:]:
            m = fs.getNode(k).mat()
            if m is None:
                raise MadStereoError('calibration %s: %s is not a matrix' % (path, k))
            calib[k] = np.asarray(m, np.float64)
        calib['size'] = (int(fs.getNode('image_height').real()), int(fs.getNode('image_width').real()))
        calib['alpha'] = float(fs.getNode('alpha').real()) if present('alpha') else 0.0
    finally:
        fs.release()
    if min(calib['size']) < 1:
        raise MadStereoError('calibration %s: image size %r' % (path, calib['size']))
    return calib


def rectification_maps(calib, frame_size):
    """(map_left, map_right): float32 [h, w, 2] tables for frames of frame_size = (h, w), which must be the size the
    calibration was made for."""
    import cv2
    h, w = (int(v) for v in frame_size)
    if (h, w) != tuple(calib['size']):
        raise MadStereoError('frames are %dx%d but the calibration is for %dx%d frames' % ((h, w) + tuple(calib['size'])))
    size = (w, h)
    if all(k in calib for k in RECTIFICATION):
        r1, r2, p1, p2 = (calib[k] for k in RECTIFICATION)
    else:
        r1, r2, p1, p2 = cv2.stereoRectify(calib['K1'], calib['D1'], calib['K2'], calib['D2'], size, calib['R'], calib['T'],
                                           flags=cv2.CALIB_ZERO_DISPARITY, alpha=calib['alpha'])[:4]
    maps = []
    for k, d, r, p in ((calib['K1'], calib['D1'], r1, p1), (calib['K2'], calib['D2'], r2, p2)):
        mx, my = cv2.initUndistortRectifyMap(k, d, r, p, size, cv2.CV_32FC1)
        maps.append(np.ascontiguousarray(np.stack([mx, my], axis=-1), dtype=np.float32))
    return maps[0], maps[1]
