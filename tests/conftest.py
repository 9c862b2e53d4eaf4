import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")
os.environ.setdefault("HF_HUB_OFFLINE", "1")
os.environ.setdefault("TOKENIZERS_PARALLELISM", "false")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    import warnings

    warnings.filterwarnings("ignore")
    try:
        import transformers

        transformers.logging.set_verbosity_error()
    except Exception:
        pass


@pytest.fixture(scope="session")
def gold_dir():
    return GOLD


@pytest.fixture(scope="session")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test running without a CUDA device")
    return torch.device("cuda:0")
