import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (select with -m gpu)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


@pytest.fixture
def emulated(monkeypatch):
    """swap the C ABI for its torch-on-CPU emulation (tests/emu_lib.py): the product's HOST code then runs without a GPU."""
    import emu_lib
    from thinktwice_b200 import lib
    emu = emu_lib.Emu()
    p = emu_lib.make_p()
    monkeypatch.setattr(lib, 'load', lambda: emu)
    monkeypatch.setattr(lib, 'require_cuda', lambda dev: None)
    monkeypatch.setattr(lib, '_p', p)
    monkeypatch.setattr(lib, '_stream', lambda: None)
    monkeypatch.setattr(lib, 'F16sIO', emu_lib.IO)
    monkeypatch.setattr(lib, 'ref', lambda s: s)
    import thinktwice_b200.engine as engine
    import thinktwice_b200.lss as lss
    import thinktwice_b200.lidarnet as lidarnet
    import thinktwice_b200.thinktwice_decoder as dec
    import thinktwice_b200.encoder_decoder_framework as fw
    import thinktwice_b200.preprocess as pre
    for mod in (engine, lss, lidarnet, dec, fw, pre):
        monkeypatch.setattr(mod, '_p', p, raising=False)
        monkeypatch.setattr(mod, '_stream', lib._stream, raising=False)
    return emu
