import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    # `-m gpu` tests must never silently pass on a box without a GPU
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        skip = pytest.mark.skip(reason="no CUDA device")
        for it in items:
            if "gpu" in it.keywords:
                it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return load


@pytest.fixture(scope="session")
def tiny_triples():
    def read(fn):
        out = []
        with open(os.path.join(GOLDEN, fn)) as f:
            for line in f:
                a, b, w = line.strip().split(" ")
                out.append([a, b, float(w)])
        return out
    return read("tiny_train.txt"), read("tiny_test.txt")


@pytest.fixture(scope="session")
def orc():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def built_lib():
    from selfrec_b200 import build
    build.build()
    from selfrec_b200 import _lib
    return _lib.load()


class TinyConf:
    """Minimal ModelConf stand-in (same __getitem__/contain contract)."""

    def __init__(self, model, extra=None, **over):
        self.config = {
            "training.set": "./dataset/tiny/train.txt", "test.set": "./dataset/tiny/test.txt",
            "model": {"name": model, "type": "graph"}, "item.ranking.topN": [5, 10], "embedding.size": 64,
            "max.epoch": 1, "batch.size": 128, "learning.rate": 0.001, "reg.lambda": 0.0001, "output": "./results/",
        }
        self.config.update(over)
        if extra is not None:
            self.config[model] = extra

    def __getitem__(self, k):
        return self.config[k]

    def contain(self, k):
        return k in self.config


@pytest.fixture()
def tiny_conf():
    return TinyConf


@pytest.fixture()
def in_tmp_cwd(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    return tmp_path
