"""pytest configuration: markers, repo-root import path, golden-vector loader."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    # GPU tests are skipped (not failed) when no device is visible, so `pytest tests/` works anywhere;
    # the drivers select with -m gpu / -m "not gpu".
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """Reader for the shards tests/golden/<name>.<k>.npz written by tests/golden/make_golden.py (Bag.save)."""

    def __init__(self, name):
        self.meta, self._shard = {}, {}
        k = 0
        while os.path.exists(path := os.path.join(ROOT, "tests", "golden", f"{name}.{k}.npz")):
            z = np.load(path)
            meta = json.loads(bytes(z["__meta__"]).decode())
            self.meta.update(meta)
            self._shard.update(dict.fromkeys(meta, z))
            k += 1
        assert self.meta, f"no golden shards {name}.*.npz"

    def names(self, op=None):
        return [k for k, v in self.meta.items() if op is None or v["op"] == op]

    def case(self, name):
        import torch

        m, z = self.meta[name], self._shard[name]
        ins = {k: torch.from_numpy(z[h].copy()) for k, h in m["inputs"].items()}
        outs = {k: torch.from_numpy(z[h].copy()) for k, h in m["outputs"].items()}
        return m["op"], dict(m["kwargs"]), ins, outs


_CACHE = {}


def golden(name):
    if name not in _CACHE:
        _CACHE[name] = Golden(name)
    return _CACHE[name]


@pytest.fixture(autouse=True)
def _default_kernel_switches():
    """Tests flip kernel-selection switches (kornia_b200.config); every test starts from, and leaves, the defaults."""
    yield
    mod = sys.modules.get("kornia_b200.config")
    if mod is not None:
        mod.reset()
