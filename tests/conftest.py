import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "whisper-timestamped_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _build_everything():
    """libwts.so and the oracle's C restatement must exist (and be current) BEFORE collection: test modules import
    the package, which loads the library.  nvcc cross-compiles on a CPU-only box; a no-op when nothing changed."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("wts_build", os.path.join(ROOT, "whisper-timestamped_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()
    import oracle
    oracle.build()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")
    _build_everything()


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a box without CUDA, so a plain `pytest tests` is green there."""
    import pytest
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (run on an H100: pytest -m gpu)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
