"""tests/golden/reference_demo_cli.json: the argparse actions of the reference's Demo/Live_Adaptation_Demo.py.

Captured as make_reference_golden.driver_cli captures the drivers: the script runs as __main__ under the eager TF shim and
stops at parse_args.  `pyzed` (the ZED SDK) is replaced by a stub module so that the reference's grabber registers its
ZED_Mini camera.  The reference path is read ONLY here, never by a test.

    python tests/golden/make_demo_golden.py
"""
import importlib.util
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))


def _stub_pyzed():
    class _Any(object):
        def __getattr__(self, name):
            return _Any()

        def __call__(self, *a, **k):
            return _Any()
    pyzed = types.ModuleType('pyzed'); pyzed.__path__ = []
    sl = types.ModuleType('pyzed.sl')
    for name in ('RESOLUTION', 'ERROR_CODE', 'VIEW', 'InitParameters', 'Camera', 'RuntimeParameters', 'Mat'):
        setattr(sl, name, _Any())
    pyzed.sl = sl
    sys.modules['pyzed'] = pyzed
    sys.modules['pyzed.sl'] = sl


def main():
    spec = importlib.util.spec_from_file_location('make_reference_golden', os.path.join(HERE, 'make_reference_golden.py'))
    mrg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mrg)
    _stub_pyzed()
    sys.path.insert(0, os.path.join(mrg.REF, 'Demo'))
    try:
        acts = mrg.driver_cli(os.path.join('Demo', 'Live_Adaptation_Demo.py'))
    finally:
        sys.path.remove(os.path.join(mrg.REF, 'Demo'))
    out_path = os.path.join(HERE, 'reference_demo_cli.json')
    json.dump({'source': 'CVLAB-Unibo/Real-time-self-adaptive-deep-stereo: Demo/Live_Adaptation_Demo.py (argparse actions)',
               'actions': acts}, open(out_path, 'w'), indent=1)
    print('wrote', out_path)


if __name__ == '__main__':
    main()
