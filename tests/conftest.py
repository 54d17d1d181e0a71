import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from tests import oracle_binding
    return oracle_binding


@pytest.fixture(scope="session")
def bunny_scene():
    """S-bunny (synthetic P3 scene): tris, nodes, eye, cam"""
    from ezrt_b200 import scenes
    return scenes.s_bunny()


@pytest.fixture(scope="session")
def grid_scene():
    """3x2 blob grid (~32k triangles) with lights: a mid-size scene with varied Disney materials"""
    from ezrt_b200 import scenes
    return scenes.s_grid(3, 2, 2)


@pytest.fixture(scope="session")
def small_hdr():
    from ezrt_b200 import api, scenes
    hdr = scenes.synth_hdr(128, 64)
    return hdr, api.hdr_cache(hdr)
