import base64
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "calfkit-sdk_b200"), ROOT, os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def golden(name: str):
    with open(os.path.join(ROOT, "tests", "golden", name), encoding="utf-8") as f:
        return json.load(f)["cases"]


def as_bytes(x) -> bytes:
    """Inverse of make_golden.s(): text, or {"b64": ...} for inputs that are not valid UTF-8."""
    if isinstance(x, dict):
        return base64.b64decode(x["b64"])
    return x.encode("utf-8")


@pytest.fixture(scope="session")
def has_cuda() -> bool:
    import torch
    return torch.cuda.is_available()
