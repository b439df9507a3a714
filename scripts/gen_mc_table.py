"""Generates xrnerf_b200/csrc/mc_table.cuh, the marching-cubes triangulation table of xrb_mc_count / xrb_mc_emit (csrc/mesh.cu).

    python scripts/gen_mc_table.py            # rewrite the header
    python scripts/gen_mc_table.py --check    # exit 1 if the committed header differs from what this script emits

Cell corners: corner c sits at (c & 1, c >> 1 & 1, c >> 2 & 1). Edges: edge e runs along axis a = e / 4 from the corner whose bit a is 0; its
other two axes, in increasing order, take the bits of k = e % 4 (low bit first). The case index has bit c set iff corner c is inside.

Each case is built from the cube's faces, one face at a time, so that the two cells sharing a face draw the same segments on it:
  - a face with two crossing edges gets one segment between them;
  - a face with four (its two inside corners diagonal) gets two segments, each cutting off one inside corner: inside corners are kept apart.
Each segment is oriented so that, walking it, the inside region of the face lies to the right when seen from outside the cube; the segments
then link into closed loops that run counter-clockwise around the outward (inside -> outside) normal. Each loop is triangulated with its
orientation (the fan from its first edge unless a diagonal of the fan would lie on a cube face, see triangulate()), so every triangle's
right-hand normal points out of the inside region. Sharing the face rule with the neighbour makes the mesh closed: every edge of the mesh
lies in exactly two triangles, once in each direction.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'xrnerf_b200', 'csrc', 'mc_table.cuh')


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.float64)


def edge_corners(e):
    """(start corner, end corner) of edge e"""
    a, k = e // 4, e % 4
    others = [b for b in range(3) if b != a]
    c0 = ((k & 1) << others[0]) | (((k >> 1) & 1) << others[1])
    return c0, c0 | (1 << a)


def edge_mid(e):
    c0, c1 = edge_corners(e)
    return 0.5 * (corner_pos(c0) + corner_pos(c1))


def face_segments(case, fa, side):
    """segments (edge_from, edge_to) that case draws on the face {bit fa == side}, oriented as the module docstring says"""
    inside = lambda c: (case >> c) & 1
    corners = [c for c in range(8) if ((c >> fa) & 1) == side]
    edges = [e for e in range(12) if e // 4 != fa and ((edge_corners(e)[0] >> fa) & 1) == side]
    crossing = [e for e in edges if inside(edge_corners(e)[0]) != inside(edge_corners(e)[1])]
    n_face = np.zeros(3); n_face[fa] = 1.0 if side else -1.0
    if len(crossing) == 0:
        return []
    if len(crossing) == 2:
        cin = [corner_pos(c) for c in corners if inside(c)]
        cout = [corner_pos(c) for c in corners if not inside(c)]
        pairs = [(crossing, np.mean(cout, 0) - np.mean(cin, 0))]
    else:   # four crossing edges: each inside corner is cut off on its own
        assert len(crossing) == 4
        centre = np.mean([corner_pos(c) for c in corners], 0)
        pairs = [([e for e in crossing if c in edge_corners(e)], centre - corner_pos(c)) for c in corners if inside(c)]
    segs = []
    for (a, b), n_out in pairs:
        d = np.cross(n_out, n_face)               # the walking direction: inside on the right seen from outside the cube
        s = float(np.dot(edge_mid(b) - edge_mid(a), d))
        assert s != 0.0
        segs.append((a, b) if s > 0 else (b, a))
    return segs


def case_triangles(case):
    """triangles of one case, as edge triples, in table order"""
    nxt = {}
    for fa in range(3):
        for side in (0, 1):
            for a, b in face_segments(case, fa, side):
                assert a not in nxt
                nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values())   # every crossing edge starts one segment and ends one
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop = [start]
        while nxt[loop[-1]] != start:
            loop.append(nxt[loop[-1]])
        seen.update(loop)
        tris += triangulate(loop)
    return tris


def shares_face(a, b):
    """do the distinct cube edges a and b lie on a common face?"""
    ca, cb = edge_corners(a), edge_corners(b)
    return any(len({(c >> ax) & 1 for c in ca + cb}) == 1 for ax in range(3))


def triangulations(poly):
    """every triangulation of the polygon poly (edge ids in loop order) with the loop's orientation; the first is the fan from poly[0]"""
    if len(poly) == 3:
        yield [tuple(poly)]
        return
    for k in range(2, len(poly)):                  # the triangle on the side (poly[0], poly[1]) has its third corner at poly[k]
        left, right = poly[1:k + 1], [poly[0]] + poly[k:]
        for tl in (triangulations(left) if len(left) >= 3 else [[]]):
            for tr in (triangulations(right) if len(right) >= 3 else [[]]):
                yield [(poly[0], poly[1], poly[k])] + tl + tr


def triangulate(loop):
    """The first triangulation of the loop none of whose diagonals joins two edges on one face. Such a diagonal is the one a triangle can share
    with the neighbouring cell: a loop that passes a four-crossing face twice has two vertices on that face that no segment joins, and the
    neighbour may join them with a diagonal too, putting that edge in four triangles."""
    sides = {frozenset((loop[i], loop[(i + 1) % len(loop)])) for i in range(len(loop))}
    for tris in triangulations(loop):
        diags = {frozenset(p) for t in tris for p in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0]))} - sides
        if not any(shares_face(*d) for d in diags):
            return tris
    raise AssertionError(f'no triangulation of loop {loop} keeps its diagonals off the faces')


def build_table():
    """(counts uint8[256], tris int8[256, max_tris, 3] padded with -1)"""
    per_case = [case_triangles(c) for c in range(256)]
    max_tris = max(len(t) for t in per_case)
    counts = np.array([len(t) for t in per_case], np.uint8)
    tris = np.full((256, max_tris, 3), -1, np.int8)
    for c, t in enumerate(per_case):
        if t:
            tris[c, :len(t)] = t
    return counts, tris


def render_header():
    counts, tris = build_table()
    max_tris = tris.shape[1]
    lines = ['// Generated by scripts/gen_mc_table.py; do not edit. The script\'s docstring gives the corner and edge numbering and the face rule.',
             '#pragma once',
             '#include <stdint.h>',
             '',
             'namespace xrb {',
             '',
             '// device arrays: read through the L1 by the threads whose cell has triangles (most cells of a lattice have none)',
             f'constexpr int MC_MAX_TRIS = {max_tris};   // most triangles of any case',
             '// triangles of case c',
             '__device__ const uint8_t MC_TRI_COUNT[256] = {']
    for r in range(0, 256, 32):
        lines.append('    ' + ', '.join(str(int(v)) for v in counts[r:r + 32]) + ',')
    lines += ['};',
              '// edge e (0..11) of corner k of triangle t of case c, at [c][3 t + k]; 15 pads',
              f'__device__ const uint8_t MC_TRI_EDGES[256][{3 * max_tris}] = {{']
    for c in range(256):
        flat = [int(v) if v >= 0 else 15 for v in tris[c].reshape(-1)]
        lines.append('    {' + ', '.join(str(v) for v in flat) + '},')
    lines += ['};', '', '}  // namespace xrb', '']
    return '\n'.join(lines)


if __name__ == '__main__':
    text = render_header()
    if '--check' in sys.argv:
        same = os.path.exists(HEADER) and open(HEADER).read() == text
        print('mc_table.cuh is up to date' if same else 'mc_table.cuh differs from the generator')
        sys.exit(0 if same else 1)
    with open(HEADER, 'w') as fh:
        fh.write(text)
    print(HEADER)
