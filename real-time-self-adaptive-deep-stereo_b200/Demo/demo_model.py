"""Real-time self-adaptive stereo thread of the live demo -- the reference's Demo/demo_model.py on the engine.

The TF graph of the reference (input rescale + crop :72-86, network :88-109, Adam train ops :111-170, restore :184-217)
becomes `Nets.get_stereo_net` + `OnlineAdaptation(optimizer='adam')`; the camera frames go to the device as uint8 and are
rescaled / cropped there (`StereoEngine.set_resize`), after an on-device rectification when the camera is calibrated
(`StereoEngine.set_rectification`).  The loop (:233-284) is kept as the reference runs it, quirks
included (see `run`).
"""
import json
import os
import threading
import time

import numpy as np

import grabber

MODES = ('NONE', 'FULL', 'MAD')


def _softmax(x):
    exp = np.exp(x)
    return exp / np.sum(exp, axis=0)


def network_shape(image_shape, crop_shape, camera_shape):
    """(H, W) the network runs at: the crop if enabled, else the rescale target if enabled, else the camera size."""
    if crop_shape[0] is not None:
        return tuple(crop_shape)
    if image_shape[0] is not None:
        return tuple(image_shape)
    return tuple(camera_shape)


def build_engine(model_name, height, width, mode, train_config, learning_rate, ssim_th, image_shape):
    """Network + Adam adaptation on the current CUDA device.  Returns (adapt, fetch): fetch() -> the displayed host copies
    (lefty [1,H,W,3], righty [1,H,W,3], disparity [1,H,W,1]) of the last frame."""
    import torch
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    if not torch.cuda.is_available():
        raise SystemExit('the live demo needs a CUDA device (there is no CPU fallback)')
    dev = torch.device('cuda', torch.cuda.current_device())
    left_buf = torch.zeros(1, height, width, 3, device=dev)
    right_buf = torch.zeros(1, height, width, 3, device=dev)
    net_args = {'left_img': left_buf, 'right_img': right_buf, 'split_layers': [None], 'sequence': True,
                'train_portion': 'BEGIN', 'bulkhead': True if mode == 'MAD' else False}
    net = Nets.get_stereo_net(model_name, net_args)
    if mode == 'MAD':
        # the reference's MAD sampler is PROBABILITY with one block (:147); FULL and NONE use FIXED (:151, :156)
        adapt = OnlineAdaptation(net, mode='MAD', train_config=train_config, lr=learning_rate, sample_mode='PROBABILITY',
                                 num_blocks=1, ssim_th=ssim_th, optimizer='adam')
    else:
        adapt = OnlineAdaptation(net, mode=mode, lr=learning_rate, sample_mode='FIXED', fixed_id=0, ssim_th=ssim_th,
                                 optimizer='adam')
    adapt.engine.set_resize(image_shape if image_shape[0] is not None else (-1, -1))
    disparity = net.get_disparities()[-1]

    def fetch():
        eng = adapt.engine
        return (eng.tensor('raw_left').cpu().numpy(), eng.tensor('raw_right').cpu().numpy(), disparity.numpy())
    return adapt, fetch


def restore_weights(adapt, weight_path):
    """Restore every variable the checkpoint names (weights_utils.get_var_to_restore_list, :196-202), including the Adam
    slots and powers a default tf.train.Saver() writes; they all become the reset snapshot."""
    from Data_utils import weights_utils
    if os.path.isdir(weight_path):
        weight_path = weights_utils.latest_checkpoint(weight_path)
    w = weights_utils.load_weights(weight_path, adapt.get_variable_names())
    if not w:
        raise SystemExit('no variable of the network found in {}'.format(weight_path))
    adapt.load_weights(w, strict=False)
    b1, b2 = adapt.engine.adam_betas[:2]
    state = weights_utils.load_adam_state(weight_path, adapt.trained_variable_shapes(), b1, b2)
    adapt.load_adam_state(state)
    print('Disparity Net Restored?: {}, number of restored variables: {}'.format(True, len(w) + state['found']))


class RealTimeStereo(threading.Thread):
    """Thread that runs real-time self-adaptive stereo on the frames of a camera queue."""
    _camera_window_name_left = "left frame"
    _camera_window_name_right = "right frame"
    _disparity_window_name = "disparity prediction"

    def __init__(self, camera_buffer, model_name='MADNet', weight_path=None, learning_rate=0.0001,
                 block_config_path='../block_config/MadNet_full.json', image_shape=[480, 640], crop_shape=[None, None],
                 SSIMTh=0.5, mode='MAD', output=None, max_frames=None, calibration=None, build=None, log=print):
        """camera_buffer: queue of [2,h,w,3] uint8 frames (grabber.END_OF_STREAM ends the run); weight_path: initial
        weights (required: the TF random initialisers are not reproduced); image_shape / crop_shape: [None, None]
        disables the rescale / the crop; output: directory for the displayed disparity of every frame and log.csv (no
        windows are opened); max_frames: stop after this many frames; calibration: stereo calibration file
        (madstereo.rectify) of a camera that delivers raw frames, which are then rectified on the device;
        build(height, width) -> (adapt, fetch) replaces build_engine (tests)."""
        threading.Thread.__init__(self)
        assert mode in MODES
        if weight_path is None:
            raise SystemExit('--weights is required: the TF random initialisers of the reference are not reproduced')
        self._camera_buffer = camera_buffer
        self._model_name = model_name
        self._weight_path = weight_path
        self._learning_rate = learning_rate
        self._block_config_path = block_config_path
        self._image_shape = list(image_shape)
        self._crop_shape = list(crop_shape)
        self._SSIMTh = SSIMTh
        self._mode = mode
        self._output = output
        self._max_frames = max_frames
        self._build = build
        self._log = log
        self._calibration = None
        if calibration is not None:
            from madstereo.rectify import load_calibration
            self._calibration = load_calibration(calibration)
        self._rectifying = False
        self._stop_flag = False
        self._adapt = None
        self.error = None
        self.records = []
        self._train_config = None
        if mode == 'MAD':
            with open(self._block_config_path) as json_data:
                self._train_config = json.load(json_data)
        self._ready = True
        if self._crop_shape[0] is not None or self._image_shape[0] is not None:
            self._setup(network_shape(self._image_shape, self._crop_shape, None))

    def _setup(self, shape):
        """Build the network at `shape` and restore the weights (the camera size decides it when rescale and crop are off)."""
        h, w = shape
        if self._build is not None:
            self._adapt, self._fetch = self._build(h, w)
        else:
            self._adapt, self._fetch = build_engine(self._model_name, h, w, self._mode, self._train_config,
                                                    self._learning_rate, self._SSIMTh, self._image_shape)
            restore_weights(self._adapt, self._weight_path)
        num_actions = len(self._train_config) if self._mode == 'MAD' else 1
        self._sample_distribution = np.zeros(shape=[num_actions])
        self._loss_t_2 = 0
        self._loss_t_1 = 0
        self._expected_loss = 0
        self._last_trained_blocks = 0
        print('Network Ready')

    def _setup_rectification(self, frame_size):
        """Rectification tables for the camera's frame size (refused when it is not the calibrated size), on the engine."""
        from madstereo.rectify import rectification_maps
        map_left, map_right = rectification_maps(self._calibration, frame_size)
        self._adapt.engine.set_rectification(map_left, map_right)
        self._rectifying = True

    def _setup_gui(self):
        import cv2
        cv2.namedWindow(self._camera_window_name_left, cv2.WINDOW_NORMAL)
        cv2.namedWindow(self._camera_window_name_right, cv2.WINDOW_NORMAL)
        cv2.namedWindow(self._disparity_window_name, cv2.WINDOW_NORMAL)

    def stop(self):
        """Stop the prediction and end the thread."""
        self._stop_flag = True

    def run(self):
        try:
            self._run()
        except BaseException as ex:          # reported by the main thread
            self.error = ex
            self._log('demo stopped by an error: %r' % (ex,))

    def _run(self):
        import cv2
        if self._output is None:
            self._setup_gui()
        else:
            os.makedirs(self._output, exist_ok=True)
            csv = open(os.path.join(self._output, 'log.csv'), 'w')
            csv.write('step,loss,module,reset,step_ms\n')
        # `first` is never set to False in the reference loop (:235-265): loss_t_1 = loss_t_2 = loss on every frame, the
        # gain is always 0, the sample distribution stays at zero and MAD draws its module uniformly.  Kept as is.
        first = True
        it = 0
        while not self._stop_flag and (self._max_frames is None or it < self._max_frames):
            frames = self._camera_buffer.get(block=True)
            if frames is grabber.END_OF_STREAM:
                break
            # frames go to the network in the channel order the grabber delivers (the ZED's BGR is not swapped)
            left_frame = frames[:1]
            right_frame = frames[1:]
            if self._adapt is None:
                self._setup(network_shape(self._image_shape, self._crop_shape, left_frame.shape[1:3]))
            if self._calibration is not None and not self._rectifying:
                self._setup_rectification(left_frame.shape[1:3])

            # the module is drawn from softmax(sample_distribution) inside OnlineAdaptation.step (:243-247)
            self._adapt.sample_distribution = self._sample_distribution.copy()
            t0 = time.perf_counter()
            out = self._adapt.step(left_frame, right_frame)
            step_ms = 1e3 * (time.perf_counter() - t0)
            full_ssim = out['loss']
            train_op_id = out['blocks'][0] if out['blocks'] else 0
            self._log('Step {}: {}'.format(it, full_ssim))

            if self._mode == 'MAD':
                # update sampling probabilities (:261-273)
                if first:
                    self._loss_t_2 = full_ssim
                    self._loss_t_1 = full_ssim
                self._expected_loss = 2 * self._loss_t_1 - self._loss_t_2
                gain_loss = self._expected_loss - full_ssim
                self._sample_distribution = 0.99 * self._sample_distribution
                self._sample_distribution[self._last_trained_blocks] += 0.01 * gain_loss
                self._last_trained_blocks = train_op_id
                self._loss_t_2 = self._loss_t_1
                self._loss_t_1 = full_ssim

            # the reset (loss > SSIMTh -> restore the checkpoint, :275-277) is checked in every mode, inside step()
            if out['reset']:
                self._log('Resetting Network...')

            # show the current prediction (:280-283), computed on the host as the reference does
            lefty, righty, disp_prediction = self._fetch()
            disp_img = cv2.applyColorMap(disp_prediction[0].astype(np.uint8), cv2.COLORMAP_JET)
            self.records.append({'step': it, 'loss': full_ssim, 'module': train_op_id, 'reset': bool(out['reset']),
                                 'step_ms': step_ms, 't': time.perf_counter()})
            if self._output is None:
                cv2.imshow(self._camera_window_name_left, lefty[0].astype(np.uint8))
                cv2.imshow(self._camera_window_name_right, righty[0].astype(np.uint8))
                cv2.imshow(self._disparity_window_name, disp_img)
                cv2.waitKey(1)
            else:
                cv2.imwrite(os.path.join(self._output, 'disparity_{:06d}.png'.format(it)), disp_img)
                csv.write('{},{!r},{},{},{:.3f}\n'.format(it, full_ssim, train_op_id, int(bool(out['reset'])), step_ms))
            it += 1
        if self._output is None:
            cv2.destroyAllWindows()
        else:
            csv.close()

    @property
    def sample_distribution(self):
        return self._sample_distribution
