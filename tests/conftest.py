import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); select with -m gpu")


@pytest.fixture(scope="session")
def repo_root():
    return ROOT


def c3lier(lora_module):
    """Context helper: extend DEFAULT_TARGET_REPLACE in place like the trainers do (train_lora_xl.py:50-52)."""

    class _Ctx:
        def __enter__(self_inner):
            self_inner.saved = list(lora_module.DEFAULT_TARGET_REPLACE)
            lora_module.DEFAULT_TARGET_REPLACE += lora_module.UNET_TARGET_REPLACE_MODULE_CONV

        def __exit__(self_inner, *a):
            del lora_module.DEFAULT_TARGET_REPLACE[len(self_inner.saved):]

    return _Ctx()
