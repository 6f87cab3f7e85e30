"""The engine launches exactly the recorded kernel sequence (tests/golden/engine_kernels.json).

Each case is one eager step (engine.profile(1): one stream, launch order) of MADNet or DispNet at a size and mode listed
in tests/golden/make_engine_kernels.py.  Kernel names carry their template arguments, so the sequence pins which kernel
and which tile variant every convolution, correlation and elementwise pass dispatches to.  A change to the
dispatch, to the plan of a layer or to which tensors have 16-bit planes (and so need a split pass) changes it.
"""
import importlib.util
import json
import os

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_engine_kernels', os.path.join(HERE, 'golden', 'make_engine_kernels.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)
GOLDEN = json.load(open(mk.OUT))


@pytest.mark.parametrize('cfg', mk.CONFIGS, ids=[c[0] for c in mk.CONFIGS])
def test_engine_kernel_sequence(cfg):
    got = mk.record_config(cfg)
    if all(v is None for v in got.values()):
        pytest.skip('torch.profiler recorded no CUDA kernel events on this machine: the kernel sequence cannot be observed')
    for case, seq in got.items():
        want = GOLDEN[case]
        assert seq is not None, case
        if seq != want:
            i = next((k for k, (a, b) in enumerate(zip(seq, want)) if a != b), min(len(seq), len(want)))
            raise AssertionError('%s: %d launches vs %d recorded; first difference at %d: %r vs %r'
                                 % (case, len(seq), len(want), i, seq[i] if i < len(seq) else None,
                                    want[i] if i < len(want) else None))
    print('%s: %d steps match the recorded kernel sequence' % (cfg[0], len(got)))
