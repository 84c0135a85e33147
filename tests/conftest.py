"""pytest configuration: `gpu` marker + shared helpers.

`-m "not gpu"` runs here (CPU only): oracle vs golden vectors, host logic, C-ABI symbol export.
`-m gpu` runs on the H100 box: parity of the CUDA path (through the C-ABI) against the oracle.
"""

from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = ROOT / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box)")


def load_golden(name: str):
    return np.load(GOLDEN / name, allow_pickle=False)


def golden_json(npz, key: str):
    return json.loads(bytes(npz[key]).decode())


def pytest_terminal_summary(terminalreporter):
    """Says which decoder the decode tests exercised: where NVDEC is not usable they ran on the host path and csrc/nvdec.cpp did not."""
    rt = sys.modules.get("cosmos_curate_b200.runtime")
    if rt is not None and False in rt._NVDEC_OK.values():
        terminalreporter.write_line("decode tests ran on the HOST decode path (libavcodec): NVDEC is not usable from this process, csrc/nvdec.cpp was NOT exercised")


@pytest.fixture(scope="session")
def golden_dir() -> Path:
    return GOLDEN
