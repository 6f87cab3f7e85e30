"""Kernel sequence of one engine step, for tests/test_engine_kernels_gpu.py.

For every case below this records the ordered names of the CUDA activities (kernels with their template arguments,
memsets, copies) of one eager step, as torch.profiler sees them.  engine.profile(1) runs the step eagerly on one stream,
so the order is the launch order.  The fixture pins which kernel, and which tile variant, every convolution of the
engine dispatches to: a change to the dispatch or to what the engine allocates shows up as a different sequence.

Needs a GPU and the built library:

    python tests/golden/make_engine_kernels.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200')
OUT = os.path.join(HERE, 'engine_kernels.json')

MAD_ALL = ('none', 'full', 'mad0', 'mad1', 'mad2', 'mad3', 'mad4')
# (name, network, batch, height, width, (radius_d, stride, warping), steps)
CONFIGS = [
    ('madnet_384x1280', 'MADNet', 1, 384, 1280, (2, 1, True), MAD_ALL),
    ('madnet_64x128', 'MADNet', 1, 64, 128, (2, 1, True), MAD_ALL),
    ('madnet_r4s1_warp_384x640', 'MADNet', 1, 384, 640, (4, 1, True), ('full',)),
    ('madnet_r4s2_nowarp_384x640', 'MADNet', 1, 384, 640, (4, 2, False), ('full',)),
    ('madnet_b8_1056x1920', 'MADNet', 8, 1056, 1920, (2, 1, True), ('mad2',)),
    ('dispnet_384x1280', 'Dispnet', 1, 384, 1280, None, ('full',)),
    ('dispnet_128x256', 'Dispnet', 1, 128, 256, None, ('full',)),
]


def _paths():
    for p in (ROOT, PKG):
        if p not in sys.path:
            sys.path.insert(0, p)


def build_engine(net_name, batch, h, w, variant):
    """A bound engine with MADNet's MAD modules (block_config/MadNet_full.json) or DispNet's FULL train op, small random
    weights and a random input pair."""
    _paths()
    import torch
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    g = torch.Generator(device='cuda').manual_seed(7)
    lt = torch.rand(batch, h, w, 3, device='cuda', generator=g) * 255
    rt = torch.rand(batch, h, w, 3, device='cuda', generator=g) * 255
    args = dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True, train_portion='BEGIN')
    if net_name == 'MADNet':
        radius_d, stride, warping = variant
        args.update(bulkhead=True, warping=warping, context_net=True, radius_d=radius_d, stride=stride, is_training=False)
        cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
        net = Nets.get_stereo_net('MADNet', args)
        OnlineAdaptation(net, mode='MAD', train_config=cfg, lr=1e-4, sample_mode='FIXED', fixed_id=0)
    else:
        net = Nets.get_stereo_net('Dispnet', args)
        OnlineAdaptation(net, mode='FULL', lr=1e-4)
    eng = net.engine
    eng.weights.normal_(0.0, 0.02, generator=g)
    eng.weights_changed()
    eng.set_input(lt, rt)
    eng.profile(1)
    return eng


def _run(eng, step):
    mode, group = {'none': (0, 0), 'full': (2, 0)}.get(step, (1, int(step[3:]) if step.startswith('mad') else -1))
    eng.run(mode, group, 0, with_update=True, lr=1e-4)


def cuda_activities(fn):
    """Names of the CUDA activities fn issues, in start order; None if the profiler records none.

    The profiler can miss the first activities of a session when it has run before in the same process, so fn runs
    twice with a torch kernel in between as a marker (the engine's own kernels are all in namespace ms::), and only
    what follows the marker counts."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
        torch.ones(1, device='cuda').add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    names = [e.name for e in ev]
    marks = [i for i, n in enumerate(names) if 'ms::' not in n]
    return names[marks[-1] + 1:] if marks else None


def record_config(cfg):
    """{case name: kernel sequence} of every step of one configuration (not the engine's first step, so that one-time
    work -- the first weight-tile preparation, kernel attributes -- is not part of the sequence)."""
    import torch
    name, net_name, batch, h, w, variant, steps = cfg
    eng = build_engine(net_name, batch, h, w, variant)
    out = {}
    for step in steps:
        out['%s/%s' % (name, step)] = cuda_activities(lambda: _run(eng, step))
    del eng
    torch.cuda.empty_cache()
    return out


def main(out=OUT):
    import torch
    torch.cuda.set_device(0)
    seqs = {}
    for cfg in CONFIGS:
        seqs.update(record_config(cfg))
    missing = [k for k, v in seqs.items() if v is None]
    if missing:
        raise SystemExit('torch.profiler recorded no CUDA activity for %s' % missing)
    with open(out, 'w') as f:
        json.dump(seqs, f, indent=0, sort_keys=True)
        f.write('\n')
    print('wrote %s: %d cases, %d activities' % (out, len(seqs), sum(len(v) for v in seqs.values())))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
