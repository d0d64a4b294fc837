"""Generate the marching-cubes triangle table of patchmatchnet_b200/csrc/pm_mesh_math.cuh.

    python tools/mc_table.py            # prints the C initialiser

Corner c of a cube sits at (c & 1 ^ (c >> 1 & 1), c >> 1 & 1, c >> 2) -- the classic numbering 0 (0,0,0), 1 (1,0,0),
2 (1,1,0), 3 (0,1,0), 4..7 the same at z = 1 -- and the twelve edges are 0-1, 1-2, 2-3, 3-0, 4-5, 5-6, 6-7, 7-4, 0-4, 1-5,
2-6, 3-7.  Case bit c is set when corner c is negative.

Rule: on every face, walked counter-clockwise as seen from outside the cube, each edge that enters a negative corner is joined
to the next edge that leaves one.  On a face with two negative corners on a diagonal this keeps the negative corners apart,
and the rule does not depend on the side the face is seen from, so the two cubes that share a face cut it alike and the
mesh has no cracks.  The joins chain into closed loops (each sign-change edge is entered once and left once); every loop is
fanned from its first edge.  Walking a loop keeps the negative corners on the right as seen from outside, so the right-hand
normal of each triangle points from the negative to the positive side.
"""
from __future__ import annotations

import numpy as np

CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
# faces as corner cycles, counter-clockwise seen from outside (right-hand normal outwards)
FACES = [(0, 3, 2, 1), (4, 5, 6, 7), (0, 1, 5, 4), (3, 7, 6, 2), (0, 4, 7, 3), (1, 2, 6, 5)]


def _edge(a: int, b: int) -> int:
    return EDGES.index((a, b)) if (a, b) in EDGES else EDGES.index((b, a))


def case_triangles(case: int):
    neg = [(case >> c) & 1 for c in range(8)]
    nxt = {}
    for face in FACES:
        cyc = [(face[i], face[(i + 1) % 4]) for i in range(4)]
        for i, (a, b) in enumerate(cyc):
            if neg[a] or not neg[b]:
                continue  # not an edge entering a negative corner
            for k in range(1, 4):
                c, d = cyc[(i + k) % 4]
                if neg[c] and not neg[d]:
                    nxt[_edge(a, b)] = _edge(c, d)
                    break
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start
        loop = _fan_start(loop)
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def _faces_of(e: int):
    a, b = EDGES[e]
    return {f for f, face in enumerate(FACES) if a in face and b in face}


def _fan_start(loop):
    """The loop rotated so that no diagonal of its fan joins two edges of one face (such a diagonal would lie in the face
    that the neighbouring cube cuts too)."""
    k = len(loop)
    for r in range(k):
        rot = loop[r:] + loop[:r]
        if all(not (_faces_of(rot[0]) & _faces_of(rot[i])) for i in range(2, k - 1)):
            return rot
    raise AssertionError(f"no fan apex for loop {loop}")


def table():
    rows = [case_triangles(c) for c in range(256)]
    width = 3 * max(len(r) for r in rows) + 1
    out = np.full((256, width), -1, dtype=np.int8)
    for c, r in enumerate(rows):
        flat = [e for t in r for e in t]
        out[c, : len(flat)] = flat
    return out


def _check_orientation(tab) -> None:
    """Every triangle's right-hand normal (vertices at the edge midpoints) agrees with the negative-to-positive direction of
    its three edges."""
    mid = [(np.array(CORNERS[a], float) + np.array(CORNERS[b], float)) / 2 for a, b in EDGES]
    for case in range(1, 255):
        neg = [(case >> c) & 1 for c in range(8)]
        row = [e for e in tab[case] if e >= 0]
        for t in range(0, len(row), 3):
            p = [mid[e] for e in row[t:t + 3]]
            n = np.cross(p[1] - p[0], p[2] - p[0])
            g = np.zeros(3)
            for e in row[t:t + 3]:
                a, b = EDGES[e]
                g += (np.array(CORNERS[b], float) - np.array(CORNERS[a], float)) * (1.0 if neg[a] else -1.0)
            assert np.dot(n, g) > 0, (case, row[t:t + 3])


def c_initialiser(tab) -> str:
    lines = []
    for c in range(256):
        lines.append("    {" + ", ".join("%d" % v for v in tab[c]) + "},")
    return "\n".join(lines)


if __name__ == "__main__":
    t = table()
    _check_orientation(t)
    print(f"// [256][{t.shape[1]}]")
    print(c_initialiser(t))
