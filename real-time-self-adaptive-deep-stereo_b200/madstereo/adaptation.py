"""Online adaptation loop — the reference inner loop (Stereo_Online_Adaptation.py:85-128,166-253) on the engine.

Train-op construction follows the reference: for MAD, one train op per side disparity, whose var_list is the
union of `net.get_variables(name)` over the layer names of that block_config group (:110-118); FULL trains
every variable on the full-resolution loss (:126-128); one momentum slot per variable shared by all ops (:85).
Per frame: sample blocks (:181-189) -> one engine step (forward, full-res loss, selected train ops) ->
reward recurrence (:211-224) -> divergence reset (:242-244).

Data parallel (new functionality, SURVEY §8e): one process per GPU.  The adapted module's gradient range and the
loss scalars are exchanged by ONE kernel inside the step's CUDA graph: it all-reduces over NVLink peer memory and
applies the momentum update with the 1/N mean folded in (csrc/dp.cu), so N ranks with one frame each equal the
reference graph at batch N (every loss is a mean over the batch).  Every rank draws the module from an identically
seeded private RNG stream and sees the same all-reduced loss, so no per-step broadcast is needed; the exchange
kernel cross-checks the module id.  If peer mapping is unavailable the torch.distributed all-reduce path remains.
"""
import os

import numpy as np
import torch

from Sampler import sampler_factory
from .engine import MODE_FULL, MODE_MAD, MODE_NONE
from ._lib import MadStereoError


def softmax(x):
    """Stereo_Online_Adaptation.py:25-27."""
    return np.exp(x) / np.sum(np.exp(x), axis=0)


def trained_variable_names(mode, groups, layers):
    """TF variable names some train op trains, in layer order: the union of the MAD groups (lists of layer indices), every
    variable in FULL, none in NONE.  TF creates optimizer slots per var_list of each minimize(), so only these have them.
    layers: objects with .index, .scope and .bias_name (StereoEngine.layers)."""
    if mode == 'NONE':
        return []
    chosen = None if mode == 'FULL' else {i for g in groups for i in g}
    names = []
    for l in layers:
        if chosen is None or l.index in chosen:
            names += [l.scope + '/weights', l.scope + '/' + l.bias_name]
    return names


class OnlineAdaptation(object):
    def __init__(self, net, mode='MAD', train_config=None, lr=0.0001, momentum=0.9, sample_mode='SEQUENTIAL',
                 num_blocks=1, fixed_id=0, sample_frequency=1, ssim_th=0.5, process_group=None,
                 loss='reprojection', decay=0.99, uf=0.01, dilation=1, optimizer='momentum', beta1=0.9, beta2=0.999,
                 epsilon=1e-8, reprojection_scale=1):
        """loss='proxy', decay, uf, dilation: the continual-adaptation variant (Stereo_Continual_Adaptation.py): masked L1 to
        proxy disparities (weights 0.01 full-resolution / FULL, 0.1 per MAD module, :75,112), reward recurrence
        h <- decay*h, h[i] += uf*gain (:232-234), a train op only every `dilation`-th frame (:212).
        optimizer='adam': tf.train.AdamOptimizer(lr) with TF1's defaults, as the live demo adapts (Demo/demo_model.py:163);
        one pair of bias-correction powers shared by every train op.  Single GPU only.
        reprojection_scale: the MAD module losses at 1/reprojection_scale resolution (--reprojectionScale,
        Stereo_Online_Adaptation.py:91-107); no effect under FULL / NONE, as in the reference.  MADNet only."""
        assert mode in ('NONE', 'FULL', 'MAD')
        assert loss in ('reprojection', 'proxy')
        assert optimizer in ('momentum', 'adam')
        self.loss_kind, self.decay, self.uf, self.dilation = loss, float(decay), float(uf), int(dilation)
        self.net, self.engine, self.mode = net, net.engine, mode
        self.lr, self.mu = float(lr), float(momentum)
        self.sample_frequency, self.ssim_th = sample_frequency, ssim_th
        self.pg = process_group
        self.world = 1
        self.rank = 0
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            self.world = torch.distributed.get_world_size(self.pg)
            self.rank = torch.distributed.get_rank(self.pg)
        if optimizer == 'adam' and self.world > 1:
            raise MadStereoError("optimizer='adam' runs on a single GPU: the data-parallel exchange applies momentum only")
        self.optimizer = optimizer
        predictions = net.get_disparities()
        self.groups = []
        if mode == 'MAD':
            if getattr(net, 'bulkhead', True) is not True:
                print('WARNING: MAD adaptation on a net built without bulkhead; the engine always cuts gradients '
                      'between modules in MAD mode (Stereo_Online_Adaptation.py:61)')
            assert train_config is not None
            assert (len(predictions[:-1]) == len(train_config))     # Stereo_Online_Adaptation.py:97
            for layer_to_train in train_config:
                var_accumulator = []
                for name in layer_to_train:
                    var_accumulator += net.get_variables(name)
                idxs = sorted({net.layer_index_of_variable(v) for v in var_accumulator})
                self.groups.append(idxs)
            self.sampler = sampler_factory.get_sampler(sample_mode, num_blocks, fixed_id)
        self.engine.set_groups(self.groups)
        self.engine.bind()
        if loss == 'proxy':
            self.engine.set_loss('proxy')
        if optimizer == 'adam':
            self.engine.set_optimizer('adam', beta1, beta2, epsilon)
        if int(reprojection_scale) < 1:
            raise MadStereoError('reprojection_scale must be >= 1, got %r' % (reprojection_scale,))
        if mode == 'MAD' and int(reprojection_scale) != 1:
            self.engine.set_reprojection_scale(reprojection_scale)
        self._adam_snapshot = None
        self.num_actions = len(self.groups) if mode == 'MAD' else (1 if mode == 'FULL' else 0)
        self.fetch_counter = [0] * self.num_actions
        self.sample_distribution = np.zeros(shape=[self.num_actions])
        self.loss_t_1 = self.loss_t_2 = 0.0
        self.last_trained_blocks = []
        self.blocks_to_train = []
        self.reset_counter = 0
        self.step_count = 0
        self._snapshot = None
        self._stage = None          # device staging buffers + side stream for prefetch()
        self._staged_for = None
        self.dp_peer = False
        self._dp_rng_state = None
        if self.world > 1 and hasattr(self.engine, 'dp_setup') and os.environ.get('MS_DP_IMPL', 'peer') == 'peer':
            self._dp_peer_setup()

    def _dp_peer_setup(self):
        ok = 1
        try:
            self.engine.dp_setup(self.rank, self.world, self.pg)
        except Exception as ex:                       # e.g. CUDA IPC not permitted in this container
            print('WARNING: peer-memory gradient exchange unavailable (%r); using torch.distributed all-reduce' % (ex,))
            ok = 0
        t = torch.tensor([ok], dtype=torch.int32, device=self.engine.device)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MIN, group=self.pg)
        self.dp_peer = bool(int(t.item()))
        if self.dp_peer:
            # a private, identically seeded RNG stream for the module sampler on every rank
            seed = torch.tensor([int(np.random.randint(0, 2 ** 31 - 1))], dtype=torch.int64, device=self.engine.device)
            torch.distributed.broadcast(seed, 0, group=self.pg)
            self._dp_rng_state = np.random.RandomState(int(seed.item())).get_state()

    def _sample_blocks(self, distribution):
        # only the samplers that draw random numbers need the private stream (swapping numpy's global state costs ~50 us)
        if self._dp_rng_state is None or type(self.sampler).__name__ not in ('random_sampler', 'probabilistic_sampler'):
            return [int(b) for b in self.sampler.sample(distribution)]
        outer = np.random.get_state()
        np.random.set_state(self._dp_rng_state)
        try:
            return [int(b) for b in self.sampler.sample(distribution)]
        finally:
            self._dp_rng_state = np.random.get_state()
            np.random.set_state(outer)

    # ---- weights -----------------------------------------------------------------------------------
    def load_weights(self, params, strict=True):
        """params: dict TF-variable-name -> array (HWIO).  Also becomes the snapshot used by the reset.
        strict=False keeps the current value of every variable `params` does not name (partial restore)."""
        if not strict:
            missing = [k for k in self.engine.param_views() if k not in params]
            if missing:
                print('WARNING: %d of %d variables are not in the checkpoint and keep their current values (first: %s); '
                      'the reference would have left them at their initialiser' % (len(missing), len(missing) + len(params), missing[0]))
        self.engine.load_params(params, strict)
        self._snapshot = self.engine.weights.clone()

    def get_variable_names(self):
        """TF variable names (without ':0') in checkpoint order, e.g. model/gc-read-pyramid/conv1/weights."""
        return list(self.engine.param_views().keys())

    def save_weights(self, prefix):
        """Write the current weights as a TensorFlow V2 checkpoint (<prefix>.index / .data-00000-of-00001) that the
        reference's tf.train.Saver can restore: same variable names, HWIO fp32."""
        from .tf_checkpoint import write_checkpoint
        write_checkpoint(prefix, self.engine.export_params())

    def trained_variable_names(self):
        """Variables some train op trains: only these have optimizer slots."""
        return trained_variable_names(self.mode, self.groups, self.engine.layers)

    def trained_variable_shapes(self):
        views = self.engine.param_views()
        return {n: tuple(views[n].shape) for n in self.trained_variable_names()}

    def load_adam_state(self, state):
        """state: Data_utils.weights_utils.load_adam_state(...) -- {'m': {var: array}, 'v': {var: array},
        'powers': (beta1_power, beta2_power) or None, 'found': number of checkpoint entries it came from}.  Writes the
        first moments into the momentum arena, the second moments into the Adam arena and the shared powers.  When the
        checkpoint held any of them they join the reset snapshot: the demo's reset re-runs the same restore, which
        assigns every global variable the checkpoint names (Demo/demo_model.py:198-201)."""
        if self.optimizer != 'adam':
            raise MadStereoError("load_adam_state needs optimizer='adam'")
        eng = self.engine
        mv, vv = eng.param_views(eng.momentum), eng.param_views(eng.adam_v)
        for name, arr in state['m'].items():
            mv[name].copy_(torch.as_tensor(np.asarray(arr, dtype=np.float32)).reshape(mv[name].shape))
        for name, arr in state['v'].items():
            vv[name].copy_(torch.as_tensor(np.asarray(arr, dtype=np.float32)).reshape(vv[name].shape))
        if state.get('powers') is not None:
            eng.adam_powers.copy_(torch.tensor(state['powers'], dtype=torch.float32))
        if state.get('found', 0) > 0:
            self._adam_snapshot = (eng.momentum.clone(), eng.adam_v.clone(), eng.adam_powers.clone())

    def restore(self):
        """restorer.restore(sess, weights) (:242-244): weights only; momentum slots are left untouched.  Under Adam the
        slots and powers are restored too when the checkpoint held them (load_adam_state)."""
        if self._snapshot is None:
            raise MadStereoError('no weight snapshot to restore')
        self.engine.weights.copy_(self._snapshot)
        if self._adam_snapshot is not None:
            for dst, src in zip((self.engine.momentum, self.engine.adam_v, self.engine.adam_powers), self._adam_snapshot):
                dst.copy_(src)
        self.engine.weights_changed()

    # ---- one frame ---------------------------------------------------------------------------------
    def _allreduce(self, t):
        if self.world > 1:
            torch.distributed.all_reduce(t, group=self.pg)

    def prefetch(self, left, right):
        """Start the host->device copy of the NEXT frame on a side stream while the current frame computes (the
        reference overlaps input decoding with sess.run through its tf.data pipeline, Data_utils/data_reader.py).
        The step() call that receives these same tensor objects then only does a device-to-device copy."""
        eng = self.engine
        u8 = eng._is_u8(left) and eng._is_u8(right)
        dt = torch.uint8 if u8 else torch.float32
        resized = u8 and eng.resize_shape is not None     # frames at camera size: staging buffers of the source size
        if resized:
            l, r = eng._u8_source(left), eng._u8_source(right)
        else:
            l, r = (eng._as_u8(left), eng._as_u8(right)) if u8 else (eng._as_f32(left), eng._as_f32(right))
        shape = tuple(l.shape) if resized else (eng.B, eng.H, eng.W, 3)
        if self._stage is None or self._stage[0].dtype != dt or tuple(self._stage[0].shape) != shape:
            self._stage = [torch.empty(shape, dtype=dt, device=eng.device) for _ in range(2)]
            self._copy_stream = torch.cuda.Stream(device=eng.device)
            self._stage_ready = torch.cuda.Event()
            self._stage_free = torch.cuda.Event()
            self._stage_free.record(torch.cuda.current_stream(eng.device))
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._stage_free)      # the previous frame's staging -> input copy is done
            self._stage[0].copy_(l, non_blocking=True)
            self._stage[1].copy_(r, non_blocking=True)
            self._stage_ready.record(self._copy_stream)
        self._staged_for = (left, right, l, r)

    def _set_input(self, left, right):
        eng = self.engine
        st = self._staged_for
        if st is not None and left is st[0] and right is st[1]:
            cur = torch.cuda.current_stream(eng.device)
            cur.wait_event(self._stage_ready)
            eng.set_input(self._stage[0], self._stage[1])
            self._stage_free.record(cur)
            self._staged_for = None
        else:
            eng.set_input(left, right)

    def step(self, left, right, gt=None, want_disp_mask=0, prefetch=None, proxy=None):
        """One frame == one sess.run of the reference loop (Stereo_Online_Adaptation.py:176-253).
        prefetch=(next_left, next_right): start copying the next frame's host buffers while this frame computes."""
        eng = self.engine
        step = self.step_count
        if self.mode == 'MAD' and step % self.sample_frequency == 0:
            distribution = softmax(self.sample_distribution)
            if self.dp_peer:
                blocks = self._sample_blocks(distribution)
            elif self.world > 1:
                blocks = [int(b) for b in self.sampler.sample(distribution)] if self.rank == 0 else [0] * len(
                    self.blocks_to_train or [0] * self.sampler._blocks_to_fetch)
                t = torch.tensor(blocks, dtype=torch.int32, device=eng.device)
                torch.distributed.broadcast(t, 0, group=self.pg)
                blocks = [int(b) for b in t.tolist()]
            else:
                blocks = [int(b) for b in self.sampler.sample(distribution)]
            self.blocks_to_train = blocks
            for l in blocks:
                self.fetch_counter[l] += 1

        self._set_input(left, right)
        if gt is not None:
            eng.set_gt(gt)
        if self.loss_kind == 'proxy':
            if proxy is None:
                raise MadStereoError('loss="proxy" needs the proxy disparities of every frame: step(..., proxy=...)')
            eng.set_proxy(proxy)
        mask = want_disp_mask
        adapt_now = step % self.dilation == 0          # Stereo_Continual_Adaptation.py:212: train ops every `dilation` frames
        gscale = 1.0 / self.world
        solo = self.world == 1
        if self.mode == 'NONE' or not adapt_now:
            eng.run(MODE_NONE, 0, mask, False)
        elif self.mode == 'FULL':
            fused = self.dp_peer
            eng.run(MODE_FULL, 0, mask, 2 if fused else (1 if solo else 0), self.lr, self.mu, gscale)
            if not solo and not fused:
                self._allreduce(eng.grads)
                eng.update(-1, self.lr, self.mu, gscale)
        else:
            for i, b in enumerate(self.blocks_to_train):
                if i == 0:
                    bm = mask
                    for other in self.blocks_to_train[1:]:
                        bm |= 1 << other
                    fused = self.dp_peer and len(self.blocks_to_train) == 1
                    eng.run(MODE_MAD, b, bm, 2 if fused else (1 if solo else 0), self.lr, self.mu, gscale)
                    if fused:
                        break
                else:      # further train ops of the same sess.run: same forward, disjoint variables
                    eng.loss(b, True, 1)
                    eng.backward(MODE_MAD, b)
                if not solo or i > 0:
                    if not solo:
                        lo, hi = eng.group_ranges[b]
                        self._allreduce(eng.grads[lo:hi])
                    eng.update(b, self.lr, self.mu, gscale)
        if gt is not None:
            eng.metrics()
        if prefetch is not None:         # issued AFTER the step's graph launch: the host work of enqueueing the next frame's
            self.prefetch(*prefetch)     # copies (side stream) no longer delays this frame's kernels
        sc = eng.read_scalars()
        new_loss = sc[0]
        fused_loss = self.dp_peer and adapt_now and (self.mode == 'FULL' or (self.mode == 'MAD' and len(self.blocks_to_train) == 1))
        if fused_loss:                  # the exchange kernel already wrote the mean over the ranks
            if new_loss != new_loss:
                raise MadStereoError('data-parallel exchange failed (code %d: 1 = peer timeout, 2 = ranks adapt '
                                     'different modules)' % eng.dp_error())
        elif self.world > 1:
            t = torch.tensor([new_loss], dtype=torch.float64, device=eng.device)
            self._allreduce(t)
            new_loss = float(t.item()) / self.world

        if self.mode == 'MAD':
            if step == 0:
                self.loss_t_2 = new_loss
                self.loss_t_1 = new_loss
            expected_loss = 2 * self.loss_t_1 - self.loss_t_2
            gain_loss = expected_loss - new_loss
            self.sample_distribution = self.decay * self.sample_distribution
            for i in self.last_trained_blocks:
                self.sample_distribution[i] += self.uf * gain_loss
            self.last_trained_blocks = self.blocks_to_train
            self.loss_t_2 = self.loss_t_1
            self.loss_t_1 = new_loss

        did_reset = False
        # (any mode: the reference restores and counts whenever the loss exceeds the threshold, Stereo_Online_Adaptation.py:242-244;
        #  in NONE the weights never moved, so the restore is a no-op and only #resets in stats.csv is affected)
        if new_loss > self.ssim_th and self._snapshot is not None:
            self.restore()
            self.reset_counter += 1
            did_reset = True
        self.step_count += 1
        return {'loss': new_loss, 'train_loss': sc[1], 'epe': sc[2], 'bad3': sc[3],
                'blocks': list(self.blocks_to_train), 'reset': did_reset}
