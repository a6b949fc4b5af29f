import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run on a GPU machine with -m gpu)")


def has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """A plain `pytest` on a machine without a GPU skips the tests marked `gpu` instead of failing in them (the product has no CPU
    fallback, so they cannot pass there); `-m gpu` on a GPU machine runs them."""
    if has_gpu():
        return
    skip = pytest.mark.skip(reason="needs an H100 (no CUDA device here)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def tmp_models(tmp_path_factory):
    """Synthetic model files shared by the tests."""
    from katago_b200 import modelgen
    d = tmp_path_factory.mktemp("models")
    out = {}
    for cfg, seed in (("tiny_reg", 3), ("tiny_nbt", 4), ("mid_nbt", 5)):
        out[cfg] = modelgen.write_model(str(d / f"{cfg}.bin"), cfg, seed=seed)
    out["tiny_nbt_gz"] = modelgen.write_model(str(d / "tiny_nbt2.bin.gz"), "tiny_nbt", seed=4)
    out["tiny_relu_v8"] = modelgen.write_model(str(d / "tiny_v8.bin"), "tiny_reg", seed=6, version=8, activation="ACTIVATION_RELU")
    return out
