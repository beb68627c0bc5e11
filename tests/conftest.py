import os
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    config.addinivalue_line('markers', 'multigpu: needs >= 2 CUDA devices')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        n = 0
    for item in items:
        if 'gpu' in item.keywords and n == 0:
            item.add_marker(pytest.mark.skip(reason='no CUDA device'))
        if 'multigpu' in item.keywords and n < 2:
            item.add_marker(pytest.mark.skip(reason='needs >= 2 CUDA devices'))


def free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


@pytest.fixture
def master_port():
    return free_port()
