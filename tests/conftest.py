import os
import sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    import __graft_entry__ as g
    return g.load_oracle()


@pytest.fixture(scope="session")
def pkg():
    import __graft_entry__ as g
    return g.load_package()


@pytest.fixture(scope="session")
def icl_gray():
    """640x480 ICL-NUIM office frame (reference images/input.png, cv2.COLOR_BGR2GRAY), committed as a fixture."""
    import cv2
    img = cv2.imread(os.path.join(GOLDEN, "icl_office_gray.png"), cv2.IMREAD_GRAYSCALE)
    assert img is not None and img.shape == (480, 640)
    return img


@pytest.fixture(scope="session")
def synth():
    import synth as s
    return s
