import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_sessionstart(session):
    # the CPU oracle is ATen: on many-core hosts more threads than the small test problems can feed is slower
    import torch
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: select with `-m gpu`)")
    config.addinivalue_line("markers", "reference: needs the reference tree at /root/reference (absent on the GPU box)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests are skipped (not failed) on a host without a CUDA device or without the built library, so a plain `pytest tests`
    works on CPU-only CI; `-m gpu` selects them on an H100."""
    import torch
    lib = os.path.join(ROOT, "fastspeech2_b200", "libfs2b200.so")
    why = None
    if not torch.cuda.is_available():
        why = "no CUDA device"
    elif not os.path.exists(lib):
        why = "libfs2b200.so not built"
    if why:
        skip = pytest.mark.skip(reason=why)
        for it in items:
            if "gpu" in it.keywords:
                it.add_marker(skip)


@pytest.fixture(scope="session")
def scratch(tmp_path_factory):
    return str(tmp_path_factory.mktemp("fs2cfg"))


@pytest.fixture(scope="session")
def lj_configs(scratch):
    from fastspeech2_b200 import configs
    return configs.make_configs("LJSpeech", scratch)


@pytest.fixture(scope="session")
def libri_configs(scratch):
    from fastspeech2_b200 import configs
    return configs.make_configs("LibriTTS", scratch)


@pytest.fixture(scope="session")
def parity_log():
    """Append max-abs errors to gpurun_out/parity_report.jsonl (when that directory exists) so the margins are on record."""
    import json
    path = os.path.join(ROOT, "gpurun_out", "parity_report.jsonl")

    def log(test, **vals):
        if os.path.isdir(os.path.dirname(path)):
            with open(path, "a") as f:
                f.write(json.dumps({"test": test, **{k: (float(v) if hasattr(v, "__float__") else v) for k, v in vals.items()}}) + "\n")
    return log
