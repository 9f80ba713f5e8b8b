#!/usr/bin/env python
"""Generate the marching-cubes case tables used by dg-mesh_b200/csrc/mc.cu (and by the numpy oracle).

The reference takes its marching cubes from the third-party `diso` package (DiffMC), which is
neither vendored nor installable offline (SURVEY.md 8(c)), so its 256-case table cannot be
consulted.  Instead of typing a table from memory, the cases are DERIVED here:

  * corners v = x + 2y + 4z, bit v of the case index set when phi(corner) < iso ("inside");
  * 12 edges e = 4*axis + combo, combo = the two other coordinates of the edge's lower corner;
  * on every cube face the intersected edges are paired into segments; an ambiguous face (two
    diagonal corners inside) always SEPARATES the inside corners -- a rule that only looks at
    the face's four signs, so the two cubes sharing the face agree and the surface is watertight;
  * segments are chained into closed loops (every intersected edge lies on exactly two faces)
    and each loop is fan-triangulated, oriented so the normal points from inside to outside.

Output: dg-mesh_b200/csrc/mc_tables.h with  MC_NTRI[256]  and  MC_TRI[256][MC_MAX_TRI*3]
(edge ids, -1 padded), and the dual-marching-cubes patches of the same loops: DMC_PATCH[256][4][7] (each
patch's edges in increasing id, -1 padded) and DMC_PATCH_OF_EDGE[256][12] (-1 for an edge the level set does
not cut).  `python tools/gen_mc_tables.py --check` verifies the committed header.
"""
import itertools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "dg-mesh_b200", "csrc", "mc_tables.h")


def corner_xyz(v):
    return np.array([v & 1, (v >> 1) & 1, (v >> 2) & 1])


def edge_corners(e):
    """edge e = 4*axis + combo -> (lower corner, upper corner)."""
    axis, combo = divmod(e, 4)
    others = [a for a in range(3) if a != axis]
    c = [0, 0, 0]
    c[others[0]] = combo & 1
    c[others[1]] = (combo >> 1) & 1
    lo = c[0] + 2 * c[1] + 4 * c[2]
    return lo, lo + (1 << axis)


EDGES = [edge_corners(e) for e in range(12)]
EDGE_OF = {frozenset(p): e for e, p in enumerate(EDGES)}


def faces():
    """Each face: its 4 corners in cyclic order."""
    out = []
    for axis in range(3):
        o = [a for a in range(3) if a != axis]
        for side in (0, 1):
            cyc = []
            for (p, q) in ((0, 0), (1, 0), (1, 1), (0, 1)):
                c = [0, 0, 0]
                c[axis] = side
                c[o[0]], c[o[1]] = p, q
                cyc.append(c[0] + 2 * c[1] + 4 * c[2])
            out.append(cyc)
    return out


FACES = faces()


def case_loops(case):
    """The closed loops of intersected edges of a case, each oriented so that its normal points from inside to
    outside.  A loop is one surface patch of the cell: the triangles of case_triangles and the patches of dual
    marching cubes are both built from these loops."""
    inside = [(case >> v) & 1 for v in range(8)]
    segs = []
    for cyc in FACES:
        s = [inside[v] for v in cyc]
        cut = [i for i in range(4) if s[i] != s[(i + 1) % 4]]          # face edge i joins cyc[i], cyc[i+1]
        fe = [EDGE_OF[frozenset((cyc[i], cyc[(i + 1) % 4]))] for i in range(4)]
        if len(cut) == 2:
            segs.append((fe[cut[0]], fe[cut[1]]))
        elif len(cut) == 4:
            # ambiguous: cut off each inside corner separately -> pair the two edges at that corner
            for i in range(4):
                if s[i]:
                    segs.append((fe[(i - 1) % 4], fe[i]))
    # chain segments into loops
    adj = {}
    for a, b in segs:
        adj.setdefault(a, []).append(b)
        adj.setdefault(b, []).append(a)
    assert all(len(v) == 2 for v in adj.values()), (case, adj)
    loops, seen = [], set()
    for start in sorted(adj):
        if start in seen:
            continue
        loop, prev, cur = [start], None, start
        seen.add(start)
        while True:
            nxt = [n for n in adj[cur] if n != prev] or adj[cur]
            n = nxt[0]
            if n == start:
                break
            if n in seen:                      # two-edge degenerate loop cannot happen on a cube
                raise AssertionError((case, loop))
            loop.append(n)
            seen.add(n)
            prev, cur = cur, n
        loops.append(loop)
    out = []
    mid = lambda e: (corner_xyz(EDGES[e][0]) + corner_xyz(EDGES[e][1])) / 2.0  # noqa: E731
    for loop in loops:
        pts = np.array([mid(e) for e in loop])
        nrm = np.zeros(3)
        for i in range(len(loop)):             # Newell normal of the loop
            p, q = pts[i], pts[(i + 1) % len(loop)]
            nrm += np.cross(p, q)
        d = np.zeros(3)                        # inside -> outside direction along the loop's edges
        for e in loop:
            a, b = EDGES[e]
            ia, ib = inside[a], inside[b]
            d += (corner_xyz(b) - corner_xyz(a)) * (1 if ia else -1) if ia != ib else 0
        if np.dot(nrm, d) < 0:
            loop = loop[::-1]
        out.append(loop)
    return out


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def case_patches(case):
    """Dual marching cubes: the patches of a case, one per loop, each as its edges in increasing edge id (the
    order in which a dual vertex sums its crossings)."""
    return [sorted(loop) for loop in case_loops(case)]


def build():
    table = [case_triangles(c) for c in range(256)]
    mx = max(len(t) for t in table)
    return table, mx


def patch_tables():
    """(patch[256, DMC_MAX_PATCH, DMC_MAX_PATCH_EDGES], patch_of_edge[256, 12]), -1 padded."""
    pt = [case_patches(c) for c in range(256)]
    mp, me = max(len(p) for p in pt), max(len(q) for p in pt for q in p)
    assert (mp, me) == (4, 7), (mp, me)
    patch = -np.ones((256, mp, me), np.int64)
    pof = -np.ones((256, 12), np.int64)
    for c, ps in enumerate(pt):
        for i, q in enumerate(ps):
            patch[c, i, :len(q)] = q
            pof[c, q] = i
    return patch, pof


def render_patches():
    patch, pof = patch_tables()
    lines = ["// Dual marching cubes: patch p of a case is one loop above, as its edges in increasing id.",
             f"#define DMC_MAX_PATCH {patch.shape[1]}", f"#define DMC_MAX_PATCH_EDGES {patch.shape[2]}",
             f"static const signed char DMC_PATCH[256][{patch.shape[1]}][{patch.shape[2]}] = {{"]
    for c in range(256):
        lines.append("    {" + ", ".join("{" + ", ".join(f"{v:2d}" for v in q) + "}" for q in patch[c]) + "},")
    lines += ["};", "static const signed char DMC_PATCH_OF_EDGE[256][12] = {"]
    for c in range(256):
        lines.append("    {" + ", ".join(f"{v:2d}" for v in pof[c]) + "},")
    lines.append("};")
    return "\n".join(lines) + "\n"


def render(table, mx):
    lines = ["// mc_tables.h -- GENERATED by tools/gen_mc_tables.py (do not edit).",
             "// Corner v = x + 2y + 4z; bit v of the case index is set when phi(corner) < iso.",
             "// Edge e = 4*axis + combo joins corner lo(e) and lo(e) + (1 << axis).",
             "#pragma once", f"#define MC_MAX_TRI {mx}",
             "static const unsigned char MC_EDGE_LO[12] = {" + ", ".join(str(EDGES[e][0]) for e in range(12)) + "};",
             "static const unsigned char MC_NTRI[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(table[c])) for c in range(r, r + 32)) + ",")
    lines.append("};")
    lines.append(f"static const signed char MC_TRI[256][{mx * 3}] = {{")
    for c in range(256):
        flat = [e for t in table[c] for e in t]
        flat += [-1] * (mx * 3 - len(flat))
        lines.append("    {" + ", ".join(f"{v:2d}" for v in flat) + "},")
    lines.append("};")
    return "\n".join(lines) + "\n" + render_patches()


def tables_for_python():
    """(ntri[256], tri[256, MC_MAX_TRI*3], edge_lo[12]) for the numpy oracle."""
    table, mx = build()
    tri = -np.ones((256, mx * 3), np.int64)
    for c, t in enumerate(table):
        flat = [e for x in t for e in x]
        tri[c, :len(flat)] = flat
    return np.array([len(t) for t in table]), tri, np.array([EDGES[e][0] for e in range(12)])


def dmc_tables_for_python():
    """(patch[256, 4, 7], patch_of_edge[256, 12], edge_lo[12]) for the dual-marching-cubes reference."""
    patch, pof = patch_tables()
    return patch, pof, np.array([EDGES[e][0] for e in range(12)])


if __name__ == "__main__":
    table, mx = build()
    txt = render(table, mx)
    if "--check" in sys.argv:
        ok = os.path.exists(OUT) and open(OUT).read() == txt
        print("mc_tables.h up to date" if ok else "mc_tables.h STALE")
        sys.exit(0 if ok else 1)
    open(OUT, "w").write(txt)
    print(f"wrote {OUT}: max {mx} triangles per cell, {sum(len(t) for t in table)} triangles over 256 cases")
