"""The vertex de-duplication behind the indexed triangle records of the 8-wide traversal (scene_prep.cu, ezrt_prep_vertex_ids), restated
in numpy: the device's algorithm step by step (a stable radix sort of the positions by z, then by x:y; run heads; an exclusive scan
of the first occurrences) against a direct definition (vertices = distinct (x, y, z) bit patterns, numbered by first occurrence),
on bit patterns built to trip it: +0 / -0, NaNs with equal and with different payloads, degenerate triangles whose vertices repeat.
Then the layout rule of ezrt_scene_create at its boundary.  tests/test_gpu_tri_layout.py checks the device's result through
renders and ray queries."""
import numpy as np
import pytest


def device_vertex_ids(pos):
    """pos: [m, 3] uint32 bit patterns of the positions j = 3 i + k.  Returns (vid [m], vert_src [V]) as the kernels compute them."""
    m = len(pos)
    idx1 = np.argsort(pos[:, 2], kind="stable")                                   # sort 1: by z
    key_xy = (pos[idx1, 0].astype(np.uint64) << np.uint64(32)) | pos[idx1, 1].astype(np.uint64)
    idx2 = idx1[np.argsort(key_xy, kind="stable")]                                # sort 2: by x:y, stable
    s = pos[idx2]
    head = np.ones(m, np.uint32)
    head[1:] = (s[1:] != s[:-1]).any(1)
    first = np.zeros(m, np.uint32)
    first[idx2[head == 1]] = 1
    num = np.cumsum(first) - first                                                # exclusive scan
    run = np.cumsum(head)                                                         # inclusive scan, 1-based runs
    run_vid = np.zeros(int(run[-1]), np.uint32)
    vert_src = np.zeros(int(first.sum()), np.uint32)
    hp = np.flatnonzero(head)
    run_vid[run[hp] - 1] = num[idx2[hp]]
    vert_src[num[idx2[hp]]] = idx2[hp]
    vid = np.zeros(m, np.uint32)
    vid[idx2] = run_vid[run - 1]
    return vid, vert_src


def direct_vertex_ids(pos):
    ids, vid, src = {}, np.zeros(len(pos), np.uint32), []
    for j, p in enumerate(map(tuple, pos)):
        if p not in ids:
            ids[p] = len(ids)
            src.append(j)
        vid[j] = ids[p]
    return vid, np.array(src, np.uint32)


def use_indexed(n_triangles, n_vertices):
    """capi.cu: the indexed layout for a W8 scene iff 32 T + 16 V < 64 T bytes."""
    return 32 * n_triangles + 16 * n_vertices < 64 * n_triangles


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _check(pos):
    vid, src = device_vertex_ids(pos)
    rvid, rsrc = direct_vertex_ids(pos)
    np.testing.assert_array_equal(vid, rvid)
    np.testing.assert_array_equal(src, rsrc)
    np.testing.assert_array_equal(pos[src][vid], pos)        # the records reproduce every position bit for bit
    return vid, src


def test_first_occurrence_order():
    rng = np.random.default_rng(1)
    grid = _bits(rng.integers(-3, 4, (4000, 3)) * 0.25)        # few distinct values: many repeats in random order
    vid, src = _check(grid)
    assert vid[0] == 0 and (np.diff(src) > 0).all()
    assert (np.maximum.accumulate(vid)[1:] - np.maximum.accumulate(vid)[:-1] <= 1).all()   # a new vertex gets the next id
    assert len(src) < len(grid) // 10


def test_signed_zeros_and_nan_payloads_stay_distinct():
    qnan, nan2, nan3 = np.uint32(0x7fc00000), np.uint32(0x7fc00001), np.uint32(0xffc00000)
    z, nz = np.uint32(0), np.uint32(0x80000000)
    one = _bits(1.0)
    pos = np.array([[z, z, z], [nz, z, z], [z, nz, z], [z, z, nz], [z, z, z], [nz, z, z],
                    [qnan, one, one], [nan2, one, one], [nan3, one, one], [qnan, one, one], [one, one, qnan], [one, one, nan2]], np.uint32)
    vid, src = _check(pos)
    assert vid.tolist() == [0, 1, 2, 3, 0, 1, 4, 5, 6, 4, 7, 8]


def test_degenerate_triangles_with_repeated_vertices():
    rng = np.random.default_rng(2)
    p = _bits(rng.normal(size=(300, 3)))
    tri = p[rng.integers(0, 300, (500, 3))]                     # random triangles over 300 points: repeats inside triangles
    tri[:50, 1] = tri[:50, 0]                                   # two equal vertices
    tri[50:80, 1:] = tri[50:80, :1]                             # all three equal
    vid, _ = _check(tri.reshape(-1, 3))
    v = vid.reshape(-1, 3)
    assert (v[:50, 0] == v[:50, 1]).all() and (v[50:80] == v[50:80, :1]).all()


@pytest.mark.parametrize("n", [1, 2, 65536, 999860])
def test_layout_rule_boundary(n):
    assert use_indexed(n, 2 * n - 1)
    assert not use_indexed(n, 2 * n)                            # 32 T + 32 T = 64 T: equal size keeps the flat record
    assert not use_indexed(n, 3 * n)                            # a triangle soup


def test_s1m_scene_is_indexed():
    """bench.py's 1 M-triangle scene shares its vertices: about 0.5 distinct positions per triangle."""
    from ezrt_b200 import scenes
    tris = scenes.s_1m_bunny()[0]
    pos = np.ascontiguousarray(tris[:, :9]).view(np.uint32).reshape(-1, 3)
    v = len(np.unique(pos, axis=0))
    assert use_indexed(len(tris), v) and v < 0.6 * len(tris)
