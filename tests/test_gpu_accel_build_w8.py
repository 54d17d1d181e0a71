"""The binary SAH tree the 8-wide form is collapsed from: built down to W8_BINARY_LEAF_TRIS = 1 triangle per leaf (w8_node.h),
the GPU builder (accel_build.cu) produces the host builder's tree (host_scene.cpp ezrt_build_accel) node for node on S-1M, the
size at which scene creation picks the 8-wide form (tests/test_gpu_accel_build.py checks leaf size 4 there)."""
import pytest

from ezrt_b200 import scenes
from tests.test_gpu_accel_build import _same_tree

pytestmark = pytest.mark.gpu


def test_s1m_single_triangle_leaves():
    tris = scenes.s_1m_bunny()[0]
    nn, ms_d, ms_h = _same_tree(tris, leaf_n=1)
    assert nn == 2 * tris.shape[0] - 1   # one triangle per leaf: a full binary tree
    print("S-1M binary SAH tree, 1 triangle per leaf: %d nodes; device %.1f ms, host %.1f ms" % (nn, ms_d, ms_h))
