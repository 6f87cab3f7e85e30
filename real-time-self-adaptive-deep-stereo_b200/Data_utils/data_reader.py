"""Input pipeline of the online-adaptation driver, host side (no TensorFlow).

Mirrors Data_utils/data_reader.py of the reference: `readPFM` (:11-52), `read_list_file` (:54-79: `left;right;gt[;conf]`
per line, ',' or ';' separated, blank lines and '#' comments skipped), image decoding (:81-100: 8-bit images as float32
RGB, first three channels; 16-bit ground-truth PNGs divided by 256, PFM ground truth as is), the ground-truth crop to
the image width (:146) and, for inference/adaptation, the centre crop / zero pad to `crop_shape`
(`tf.image.resize_image_with_crop_or_pad`, :150-151).  `tf.data`'s map + batch(drop_remainder) + prefetch become a
background thread that fills a bounded queue with numpy batches (optionally pinned torch tensors, so that
`OnlineAdaptation.step(prefetch=...)` can overlap the host->device copy with the previous frame).
Augmentation (`augment=True`, training-only in the reference) is outside the adaptation path and not provided.
"""
import os
import queue
import re
import threading

import numpy as np


def readPFM(file):
    """-> (array [H,W,1|3] float32, bottom-up flipped to top-down; scale)."""
    with open(file, 'rb') as f:
        header = f.readline().rstrip()
        if header == b'PF':
            color = True
        elif header == b'Pf':
            color = False
        else:
            raise Exception('Not a PFM file.')
        try:
            width, height = list(map(int, f.readline().split()))
        except Exception:
            raise Exception('Malformed PFM header.')
        scale = float(f.readline().rstrip())
        endian = '<' if scale < 0 else '>'
        scale = abs(scale)
        data = np.fromfile(f, endian + 'f')
    shape = (height, width, 3) if color else (height, width, 1)
    data = np.flipud(np.reshape(data, shape)).astype(np.float32)
    return data, scale


def read_list_file(path_file):
    """-> [left, right, gt, conf] file-name lists."""
    with open(path_file, 'r') as f_in:
        lines = f_in.readlines()
    lines = [x for x in lines if not (x.strip() == '' or x.strip()[0] == '#')]
    left, right, gt, conf = [], [], [], []
    for l in lines:
        to_load = re.split(',|;', l.strip())
        left.append(to_load[0])
        right.append(to_load[1])
        if len(to_load) > 2:
            gt.append(to_load[2])
        if len(to_load) > 3:
            conf.append(to_load[3])
    return left, right, gt, conf


def _imread(path):
    import cv2                                   # host-side decode; the same image ships cv2 on the GPU box
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise Exception('cannot decode image %s' % path)
    if img.dtype == np.uint16 and img.ndim == 3 and img.shape[2] >= 3:
        # a 16-bit COLOUR image: tf.image.decode_image(..., dtype=uint8) hands the reference the top 8 bits
        img = (img >> 8).astype(np.uint8)
    if img.ndim == 2:
        img = img[:, :, None]
    elif img.shape[2] >= 3:                      # OpenCV decodes to BGR(A); TensorFlow to RGB(A)
        img = np.concatenate([img[:, :, 2::-1], img[:, :, 3:]], axis=2)
    return img


def read_image_from_disc(image_path):
    """float32 [H,W,3] RGB (tf.image.decode_image + cast, then `[:, :, :3]`).  Grey images are replicated to 3 channels."""
    img = _imread(image_path).astype(np.float32)
    if img.shape[2] == 1:
        img = np.repeat(img, 3, axis=2)
    return np.ascontiguousarray(img[:, :, :3])


def read_image_u8_from_disc(image_path):
    """uint8 [H,W,3] RGB: the decoded image before the cast of read_image_from_disc (what a camera delivers)."""
    img = _imread(image_path)
    if img.dtype != np.uint8:
        raise Exception('%s is not an 8-bit image' % image_path)
    if img.shape[2] == 1:
        img = np.repeat(img, 3, axis=2)
    return np.ascontiguousarray(img[:, :, :3])


def read_gt_from_disc(gt_path):
    """float32 [H,W,1]: PFM as is; 16-bit PNG / 256; 8-bit PNG as is."""
    if gt_path.lower().endswith('pfm'):
        return readPFM(gt_path)[0][:, :, :1]
    g = _imread(gt_path)
    out = g[:, :, :1].astype(np.float32)
    return out / 256.0 if g.dtype == np.uint16 else out


def resize_image_with_crop_or_pad(img, target_height, target_width):
    """tf.image.resize_image_with_crop_or_pad on [H,W,C]: centre crop, then centre zero-pad (floor division offsets)."""
    h, w = img.shape[0], img.shape[1]
    wd, hd = target_width - w, target_height - h
    oc_w, op_w = max(-wd // 2, 0), max(wd // 2, 0)
    oc_h, op_h = max(-hd // 2, 0), max(hd // 2, 0)
    ch, cw = min(target_height, h), min(target_width, w)
    cropped = img[oc_h:oc_h + ch, oc_w:oc_w + cw]
    out = np.zeros((target_height, target_width) + img.shape[2:], dtype=img.dtype)
    out[op_h:op_h + ch, op_w:op_w + cw] = cropped
    return out


def random_crop(crop_shape, tensor_list, rng=np.random):
    """preprocessing.random_crop (:31-55): one aligned random crop for all tensors."""
    h, w = tensor_list[0].shape[0], tensor_list[0].shape[1]
    max_row = h - crop_shape[0] - 1
    max_col = w - crop_shape[1] - 1
    max_row = max_row if max_row > 0 else 1
    max_col = max_col if max_col > 0 else 1
    r = int(rng.randint(0, max_row)); c = int(rng.randint(0, max_col))
    return [x[r:r + crop_shape[0], c:c + crop_shape[1], :] for x in tensor_list]


class dataset():
    """Reads a stereo dataset described by a list file; iterate to get (left, right, gt) batches:
    float32 arrays [B,H,W,3], [B,H,W,3], [B,H,W,1]."""

    def __init__(self, path_file, batch_size=4, crop_shape=[320, 1216], num_epochs=None, augment=False,
                 is_training=True, shuffle=True, prefetch=30, pin_memory=False, seed=None, proxies=False):
        if not os.path.exists(path_file):
            raise Exception('File not found during dataset construction')
        if augment:
            raise NotImplementedError('augmentation belongs to the training scripts, not to the adaptation path')
        self._path_file = path_file
        self._batch_size = batch_size
        self._crop_shape = list(crop_shape)
        self._num_epochs = num_epochs
        self._shuffle = shuffle
        self._is_training = is_training
        self._prefetch = prefetch
        self._pin = pin_memory
        self._rng = np.random.RandomState(seed)
        left, right, gt, px = read_list_file(path_file)
        # proxies=True: the continual-adaptation list format left;right;gt;proxy (Data_utils/continual_data_reader.py:55-78,
        # :136-160): batches become (left, right, gt, proxy, real_width)
        self._proxies = proxies
        if proxies:
            if len(px) != len(left):
                raise Exception('the list file must name a proxy disparity for every frame (left;right;gt;proxy)')
            self._couples = [[l, r, g, p] for l, r, g, p in zip(left, right, gt, px)]
        else:
            self._couples = [[l, r, g] for l, r, g in zip(left, right, gt)]

    def _load_image(self, files):
        left = read_image_from_disc(files[0])
        right = read_image_from_disc(files[1])
        gt = read_gt_from_disc(files[2])
        gt = gt[:, :left.shape[1], :]                                  # "SGM add some paddings" (:146)
        if self._proxies:
            px = read_gt_from_disc(files[3])[:, :left.shape[1], :]      # 16-bit PNG / 256 or 8-bit, like the ground truth
            real_width = np.float32(left.shape[1])
            if self._is_training:
                left, right, gt = random_crop(self._crop_shape, [left, right, gt], self._rng)
            else:
                left, right, gt, px = [resize_image_with_crop_or_pad(x, self._crop_shape[0], self._crop_shape[1]) for x in (left, right, gt, px)]
            return left, right, gt, px, np.full((1,), real_width, np.float32)
        if self._is_training:
            left, right, gt = random_crop(self._crop_shape, [left, right, gt], self._rng)
        else:
            left, right, gt = [resize_image_with_crop_or_pad(x, self._crop_shape[0], self._crop_shape[1]) for x in (left, right, gt)]
        return left, right, gt

    def __len__(self):
        return len(self._couples)

    def get_max_steps(self):
        return (len(self) * self._num_epochs) // self._batch_size

    def get_couples(self):
        return self._couples

    def _batches(self):
        epoch = 0
        while self._num_epochs is None or epoch < self._num_epochs:
            order = list(range(len(self._couples)))
            if self._shuffle:
                self._rng.shuffle(order)
            for b in range(0, len(order) - self._batch_size + 1, self._batch_size):      # drop_remainder=True
                items = [self._load_image(self._couples[i]) for i in order[b:b + self._batch_size]]
                batch = tuple(np.stack([it[k] for it in items]).astype(np.float32) for k in range(5 if self._proxies else 3))
                if self._pin:
                    import torch
                    batch = tuple(torch.from_numpy(x).pin_memory() for x in batch)
                yield batch
            epoch += 1

    def __iter__(self):
        """Batches in order, produced by a background thread into a queue of `prefetch` entries (tf.data prefetch)."""
        q = queue.Queue(maxsize=max(1, self._prefetch))
        done = object()

        def worker():
            try:
                for b in self._batches():
                    q.put(b)
                q.put(done)
            except BaseException as e:          # surface decode errors in the consumer
                q.put(e)

        threading.Thread(target=worker, daemon=True).start()
        while True:
            item = q.get()
            if item is done:
                return
            if isinstance(item, BaseException):
                raise item
            yield item
