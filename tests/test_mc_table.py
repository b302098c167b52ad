"""CPU: the marching-cubes table of the TSDF extraction (tools/gen_mc_table.py -> csrc/mc_table.cuh)."""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("gen_mc_table", os.path.join(ROOT, "tools", "gen_mc_table.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
TABLE = gen.table()


def _point(e):
    """Midpoint of edge e."""
    a, b = gen.EDGES[e]
    return (np.array(gen.corner_offset(a), float) + np.array(gen.corner_offset(b), float)) / 2


def _crossing(code):
    return {e for e in range(12) if ((code >> gen.EDGES[e][0]) ^ (code >> gen.EDGES[e][1])) & 1}


def test_committed_header_matches_generator():
    with open(gen.HEADER) as f:
        assert f.read() == gen.render_header(), "csrc/mc_table.cuh is stale: run python tools/gen_mc_table.py"


def test_empty_codes():
    assert TABLE[0] == [] and TABLE[255] == []


@pytest.mark.parametrize("code", range(256))
def test_vertices_are_exactly_the_crossing_edges(code):
    used = {e for tri in TABLE[code] for e in tri}
    assert used == _crossing(code)
    for tri in TABLE[code]:
        assert len(set(tri)) == 3


@pytest.mark.parametrize("code", range(256))
def test_face_boundaries_follow_the_face_rule(code):
    """The triangles' boundary edges that lie on a cube face are exactly the segments the face rule draws from that face's four
    signs; interior edges appear in exactly two triangles with opposite directions."""
    neg = {c for c in range(8) if (code >> c) & 1}
    directed = {}
    for tri in TABLE[code]:
        for i in range(3):
            d = (tri[i], tri[(i + 1) % 3])
            directed[d] = directed.get(d, 0) + 1
    boundary = {d for d in directed if (d[1], d[0]) not in directed}
    interior = {d for d in directed if (d[1], d[0]) in directed}
    assert all(n == 1 for n in directed.values())
    expected = set()
    for cyc in gen.FACES:
        signs = [c in neg for c in cyc]
        face_edges = {gen.EDGE_OF[frozenset((cyc[i], cyc[(i + 1) % 4]))] for i in range(4)}
        n_neg = sum(signs)
        segs = set(map(frozenset, gen.face_segments(cyc, neg)))
        # the rule restated from the signs alone: one segment per negative run; diagonal pairs are cut off one by one
        crossing = [e for e in face_edges if e in _crossing(code)]
        assert len(crossing) == (0 if n_neg in (0, 4) else (4 if (n_neg == 2 and signs[0] == signs[2]) else 2))
        if n_neg == 2 and signs[0] == signs[2]:
            want = set()
            for i in range(4):
                if signs[i]:
                    want.add(frozenset((gen.EDGE_OF[frozenset((cyc[i - 1], cyc[i]))], gen.EDGE_OF[frozenset((cyc[i], cyc[(i + 1) % 4]))])))
            assert segs == want
        elif crossing:
            assert segs == {frozenset(crossing)}
        else:
            assert not segs
        expected |= segs
        # no interior (fan) edge may lie across a face as well as a segment of it
        for d in interior:
            assert frozenset(d) not in segs
    assert set(map(frozenset, boundary)) == expected
    assert len(boundary) == len(expected)


@pytest.mark.parametrize("code", range(1, 255))
def test_normals_point_towards_positive_corners(code):
    """With vertices at the edge midpoints, the component of a triangle's normal along its vertices' edges (taken from the
    negative to the positive corner, summed over the three vertices) is never negative -- a fan triangle can stand exactly
    perpendicular to that sum -- and is positive summed over the code's triangles."""
    total = 0.0
    for tri in TABLE[code]:
        p = [_point(e) for e in tri]
        n = np.cross(p[1] - p[0], p[2] - p[0])
        assert np.linalg.norm(n) > 0
        s = 0.0
        for e in tri:
            a, b = gen.EDGES[e]
            neg_c, pos_c = (a, b) if (code >> a) & 1 else (b, a)
            s += n @ (np.array(gen.corner_offset(pos_c), float) - np.array(gen.corner_offset(neg_c), float))
        assert s >= 0, (code, tri)
        total += s
    assert total > 0
