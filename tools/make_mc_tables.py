"""Derive the marching-cubes triangle table of scsfm/mc_tables.py and print it (python tools/make_mc_tables.py).

Corners and edges are numbered as scsfm/mc_tables.py states (Lorensen and Cline's numbering); bit c of a cell's
configuration is set when corner c is inside (tsdf < 0).
For every configuration the surface's intersection with each face is a set of directed segments between the crossings of
that face's edges: seen from outside the cell, walking the face's corners counter-clockwise, an edge entering the inside
is joined to the next edge leaving it.  On a face with two diagonal inside corners this cuts each inside corner off on its
own, the same choice from both cells that share the face, so the welded mesh has no cracks.  The segments chain into closed
loops; each loop is fanned into triangles from the first crossing whose fan puts no triangle flat in a cell face (such a
triangle would also come, reversed, from the neighbour sharing that face), and the triangles face away from the inside.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sc-sfmlearner-release_b200"))
from scsfm.mc_tables import CORNERS, EDGES  # noqa: E402


def _faces():
    """The six faces as corner cycles, counter-clockwise seen from outside the cell."""
    out = []
    for axis in range(3):
        for side in (0, 1):
            cs = [c for c in range(8) if CORNERS[c][axis] == side]
            ctr = np.mean([CORNERS[c] for c in cs], axis=0)
            n = np.zeros(3)
            n[axis] = 1 if side else -1
            a, b = [i for i in range(3) if i != axis]
            ang = {c: np.arctan2(CORNERS[c][b] - ctr[b], CORNERS[c][a] - ctr[a]) for c in cs}
            cyc = sorted(cs, key=lambda c: ang[c])
            e1 = np.subtract(CORNERS[cyc[1]], CORNERS[cyc[0]])
            e2 = np.subtract(CORNERS[cyc[2]], CORNERS[cyc[1]])
            if np.dot(np.cross(e1, e2), n) < 0:
                cyc = cyc[::-1]
            out.append(cyc)
    return out


def _edge(a, b):
    return EDGES.index((a, b)) if (a, b) in EDGES else EDGES.index((b, a))


def triangles(config):
    inside = [(config >> c) & 1 for c in range(8)]
    nxt = {}
    for cyc in _faces():
        for i in range(4):
            c0, c1 = cyc[i], cyc[(i + 1) % 4]
            if inside[c0] or not inside[c1]:
                continue                       # not an edge entering the inside
            j = i + 1
            while inside[cyc[(j + 1) % 4]]:
                j += 1
            nxt[_edge(c0, c1)] = _edge(cyc[j % 4], cyc[(j + 1) % 4])
    tris = []
    while nxt:
        start = min(nxt)
        loop = [start]
        e = nxt.pop(start)
        while e != start:
            loop.append(e)
            e = nxt.pop(e)
        tris += _triangulate(loop)
    return tris


def _flat(tri):
    """True when the triangle's three crossings lie on one face of the cell (it would lie in that face)."""
    return any(set(tri) <= f for f in _FACE_EDGES)


def _triangulate(loop):
    """Triangles of a loop of crossings, in the loop's orientation: the fan from the first crossing (in loop order, starting
    at the smallest edge number) whose fan has no triangle flat in a cell face.  A flat triangle would also be emitted,
    reversed, by the neighbour sharing that face, leaving a doubled face in the welded mesh."""
    n = len(loop)
    for r in range(n):
        rot = loop[r:] + loop[:r]
        fan = [(rot[0], rot[i], rot[i + 1]) for i in range(1, n - 1)]
        if not any(_flat(t) for t in fan):
            return fan
    raise AssertionError("no fan of loop %s avoids the cell faces" % (loop,))


_FACE_EDGES = [{_edge(cyc[i], cyc[(i + 1) % 4]) for i in range(4)} for cyc in _faces()]


def table():
    return [triangles(m) for m in range(256)]


def rows():
    """The table as scsfm/mc_tables.py stores it: 256 rows of 16 edge numbers, the triangles' then -1."""
    return tuple(tuple([e for tri in t for e in tri] + [-1] * (16 - 3 * len(t))) for t in table())


def main():
    print("TRI_TABLE = (")
    for r in rows():
        print("    (%s)," % ", ".join(str(v) for v in r))
    print(")")


if __name__ == "__main__":
    main()
