"""Exact, vectorised numpy restatement of dual marching cubes (csrc/dmc.cu) and of its backward.

A cell's patches come from tools/gen_mc_tables.py (each patch's edges in increasing id).  Every edge crossing is
computed as mc_reference computes its vertex, t = (iso - p0) / (p1 - p0), pos = n, pos[axis] += t, in fp32; a
patch's dual vertex is the fp32 sum of its crossings in increasing edge id, / k (its edge count), / (G - 1), so
vertices compare bit for bit.  Only patches with an interior edge get a vertex.  Each sign-changing interior edge
gives the quad of the four cells around it, c, c + e_b, c + e_b + e_c, c + e_c ((a, b, c) cyclic, c the lowest
cell), reversed when the edge's lower node is outside; triangles (q0, q1, q2), (q0, q2, q3).  Runs at G = 288 in
seconds."""
import os
import sys

import numpy as np

_TOOLS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
if _TOOLS not in sys.path:
    sys.path.insert(0, _TOOLS)
from gen_mc_tables import dmc_tables_for_python  # noqa: E402

_tables = None


def tables():
    global _tables
    if _tables is None:
        patch, pof, edge_lo = dmc_tables_for_python()
        pmask = np.zeros((256, 4), np.int64)            # 12-bit edge mask of every patch
        for p in range(4):
            pmask[:, p] = ((pof == p).astype(np.int64) << np.arange(12)).sum(1)
        _tables = patch, pof, edge_lo, pmask
    return _tables


def _others(a):
    return [x for x in range(3) if x != a]


class DMCRef:
    """verts [V,3] fp32, faces [2Q,3] and quads [Q,4] int64 (rows of verts); each vertex's cell [V] (flat index
    into the [G,G,G] grid) and patch [V]."""

    def __init__(self, G, iso, verts, faces, quads, cell, patch):
        self.G, self.iso, self.verts, self.faces, self.quads = G, iso, verts, faces, quads
        self.cell, self.patch = cell, patch


def cell_cases(inside):
    G = inside.shape[0]
    cs = np.zeros((G - 1,) * 3, np.int64)
    for c in range(8):
        sl = tuple(slice((c >> b) & 1, G - 1 + ((c >> b) & 1)) for b in (0, 1, 2))
        cs |= inside[sl].astype(np.int64) << c
    return cs


def interior_edges(cells, G):
    """[n, 12] bool: edge e of each cell (coordinates [n, 3]) is interior."""
    out = np.zeros((len(cells), 12), bool)
    for e in range(12):
        a, combo = divmod(e, 4)
        o = _others(a)
        ok = np.ones(len(cells), bool)
        for bit, ax in ((combo & 1, o[0]), (combo >> 1, o[1])):
            x = cells[:, ax] + bit
            ok &= (x >= 1) & (x <= G - 2)
        out[:, e] = ok
    return out


def needed_patches(cs, cells, G):
    """[n, 4] bool: patch p of each cell has a dual vertex."""
    _, _, _, pmask = tables()
    im = (interior_edges(cells, G).astype(np.int64) << np.arange(12)).sum(1)
    return (pmask[cs] & im[:, None]) != 0


def dmc_reference(phi, iso=0.0):
    patch_t, pof, edge_lo, pmask = tables()
    phi = np.ascontiguousarray(phi, np.float32)
    G = phi.shape[0]
    iso = np.float32(iso)
    inside = phi < iso
    cs_all = cell_cases(inside)
    surf = (cs_all != 0) & (cs_all != 255)
    cells = np.stack(np.nonzero(surf), 1)                    # C order: increasing flat index
    cs = cs_all[surf]
    need = needed_patches(cs, cells, G)
    # crossings of the 12 edges of every surface cell (uncut edges are never read)
    s = np.zeros((len(cells), 4, 3), np.float32)
    for e in range(12):
        a = e >> 2
        lo = int(edge_lo[e])
        n = cells + np.array([lo & 1, (lo >> 1) & 1, lo >> 2])
        m = n.copy()
        m[:, a] += 1
        pe = pof[cs, e]
        cut = pe >= 0
        p0, p1 = phi[tuple(n[cut].T)], phi[tuple(m[cut].T)]
        t = (iso - p0) / (p1 - p0)
        pos = n[cut].astype(np.float32)
        pos[:, a] += t
        rows = np.nonzero(cut)[0]
        s[rows, pe[cut]] += pos                             # one crossing per (cell, patch) per edge: no collision
    k = np.stack([np.bitwise_count(pmask[cs, p]) for p in range(4)], 1).astype(np.float32)
    ci, pi = np.nonzero(need)                               # cell-major, increasing patch
    verts = (s[ci, pi] / k[ci, pi][:, None]) / np.float32(G - 1)
    cell_flat = np.ravel_multi_index(cells.T, (G, G, G))
    first = np.concatenate([[0], np.cumsum(need.sum(1))[:-1]]).astype(np.int64)
    need_bits = (need.astype(np.int64) << np.arange(4)).sum(1)

    def vertex(cellc, e):
        """Vertex of the patch containing local edge e of cells [n, 3]."""
        idx = np.searchsorted(cell_flat, np.ravel_multi_index(cellc.T, (G, G, G)))
        c = cs[idx]
        p = pof[c, e]
        assert (p >= 0).all()
        nb = need_bits[idx]
        assert ((nb >> p) & 1).all(), "quad corner without a vertex"
        return first[idx] + np.bitwise_count(nb & ((1 << p) - 1)).astype(np.int64)

    quads = []
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[a], hi[a] = slice(0, G - 1), slice(1, G)
        cross = inside[tuple(lo)] != inside[tuple(hi)]
        n = np.stack(np.nonzero(cross), 1)
        ok = (n[:, b] >= 1) & (n[:, b] <= G - 2) & (n[:, c] >= 1) & (n[:, c] <= G - 2)
        n = n[ok]
        lo_in = inside[tuple(n.T)]
        eb, ec = np.eye(3, dtype=np.int64)[b], np.eye(3, dtype=np.int64)[c]
        c0 = n - eb - ec
        o0, o1 = _others(a)
        corners = []
        for db, dc in ((0, 0), (1, 0), (1, 1), (0, 1)):
            rel = {b: 1 - db, c: 1 - dc}
            e = 4 * a + rel[o0] + 2 * rel[o1]
            corners.append(vertex(c0 + db * eb + dc * ec, e))
        q = np.stack(corners, 1)
        q = np.where(lo_in[:, None], q, q[:, [0, 3, 2, 1]])
        quads.append(q)
    quads = np.concatenate(quads) if quads else np.zeros((0, 4), np.int64)
    faces = np.concatenate([quads[:, [0, 1, 2]], quads[:, [0, 2, 3]]])
    return DMCRef(G, float(iso), verts.astype(np.float32), faces, quads, cell_flat[ci], pi)


def grad_reference(ref, phi, dverts):
    """(dL/dphi, sum |contribution|), both fp64 [G,G,G], for dL/dverts [V,3] w.r.t. the normalised vertices, in
    ref's vertex order: every crossing of a k-edge patch moves its vertex by d t / (k (G - 1)) along its edge."""
    _, pof, edge_lo, pmask = tables()
    G, n = ref.G, ref.G ** 3
    p = np.asarray(phi, np.float32).astype(np.float64).ravel()
    cells = np.stack(np.unravel_index(ref.cell, (G, G, G)), 1)
    ph = np.asarray(phi, np.float32)
    cs = cell_cases(ph < np.float32(ref.iso))[tuple(cells.T)]
    dv = np.asarray(dverts, np.float64)
    k = np.bitwise_count(pmask[cs, ref.patch]).astype(np.float64)
    dphi, absum = np.zeros(n), np.zeros(n)
    for e in range(12):
        sel = pof[cs, e] == ref.patch
        if not sel.any():
            continue
        a, lo = e >> 2, int(edge_lo[e])
        n0 = cells[sel] + np.array([lo & 1, (lo >> 1) & 1, lo >> 2])
        i0 = np.ravel_multi_index(n0.T, (G, G, G))
        i1 = i0 + [G * G, G, 1][a]
        p0, p1 = p[i0], p[i1]
        d = p1 - p0
        t, u = (ref.iso - p0) / d, (p1 - ref.iso) / d
        g = dv[sel, a] / (G - 1) / k[sel]
        c0, c1 = -g * u / d, -g * t / d
        dphi += np.bincount(i0, c0, n) + np.bincount(i1, c1, n)
        absum += np.bincount(i0, np.abs(c0), n) + np.bincount(i1, np.abs(c1), n)
    return dphi.reshape(G, G, G), absum.reshape(G, G, G)


def _lexmin_cycle(q):
    """Rotate each oriented cycle [Q,4] to its lexicographically smallest rotation."""
    best = q
    rows = np.arange(len(q))
    for r in (1, 2, 3):
        cand = np.roll(q, -r, axis=1)
        diff = cand != best
        first = diff.argmax(1)
        less = diff.any(1) & (cand[rows, first] < best[rows, first])
        best = np.where(less[:, None], cand, best)
    return best


def assert_same_quads(va, qa, vb, qb):
    """The same multiset of oriented quads, each as the 4-cycle of its vertices' fp32 bit patterns (the vertex
    multisets are compared by mc_reference.assert_same_mesh)."""
    va, vb = np.ascontiguousarray(va, np.float32), np.ascontiguousarray(vb, np.float32)
    qa, qb = np.asarray(qa, np.int64), np.asarray(qb, np.int64)
    assert qa.shape == qb.shape, (qa.shape, qb.shape)
    if len(qa) == 0:
        return
    bits = np.concatenate([va, vb]).view(np.uint32).astype(np.int64)
    order = np.lexsort(bits.T[::-1])
    sb = bits[order]
    new = np.ones(len(sb), bool)
    new[1:] = (sb[1:] != sb[:-1]).any(1)
    cid = np.empty(len(sb), np.int64)
    cid[order] = np.cumsum(new) - 1
    ta, tb = _lexmin_cycle(cid[:len(va)][qa]), _lexmin_cycle(cid[len(va):][qb])
    ta, tb = ta[np.lexsort(ta.T[::-1])], tb[np.lexsort(tb.T[::-1])]
    bad = int((ta != tb).any(1).sum())
    assert bad == 0, f"quad multisets differ in {bad} of {len(qa)} sorted positions"


def dmc_loop_reference(phi, iso=0.0):
    """A per-cell loop restatement (small grids only): (verts [V,3] fp32, quads [Q,4])."""
    patch_t, pof, edge_lo, _ = tables()
    phi = np.asarray(phi, np.float32)
    G = phi.shape[0]
    iso = np.float32(iso)
    vid = {}
    verts = []
    for i in range(G - 1):
        for j in range(G - 1):
            for k in range(G - 1):
                cs = 0
                for c in range(8):
                    if phi[i + (c & 1), j + ((c >> 1) & 1), k + (c >> 2)] < iso:
                        cs |= 1 << c
                for p in range(4):
                    edges = [int(e) for e in patch_t[cs, p] if e >= 0]
                    if not edges:
                        continue
                    acc = np.zeros(3, np.float32)
                    interior = False
                    for e in edges:
                        a, lo = e >> 2, int(edge_lo[e])
                        n = [i + (lo & 1), j + ((lo >> 1) & 1), k + (lo >> 2)]
                        m = list(n)
                        m[a] += 1
                        p0, p1 = phi[tuple(n)], phi[tuple(m)]
                        t = (iso - p0) / (p1 - p0)
                        pos = np.array(n, np.float32)
                        pos[a] = pos[a] + t
                        acc = acc + pos
                        interior |= all(1 <= n[o] <= G - 2 for o in _others(a))
                    if interior:
                        vid[(i, j, k, p)] = len(verts)
                        verts.append(acc / np.float32(len(edges)) / np.float32(G - 1))
    quads = []
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        for n in np.ndindex(G, G, G):
            if n[a] > G - 2 or not (1 <= n[b] <= G - 2 and 1 <= n[c] <= G - 2):
                continue
            m = list(n)
            m[a] += 1
            s0, s1 = phi[n] < iso, phi[tuple(m)] < iso
            if s0 == s1:
                continue
            ring = []
            for db, dc in ((1, 1), (0, 1), (0, 0), (1, 0)):   # cells n - e_b - e_c, n - e_c, n, n - e_b
                cell = list(n)
                cell[b] -= db
                cell[c] -= dc
                cs = 0
                for cc in range(8):
                    if phi[cell[0] + (cc & 1), cell[1] + ((cc >> 1) & 1), cell[2] + (cc >> 2)] < iso:
                        cs |= 1 << cc
                rel = [0, 0, 0]
                rel[b], rel[c] = db, dc
                o0, o1 = _others(a)
                e = 4 * a + rel[o0] + 2 * rel[o1]
                ring.append(vid[(cell[0], cell[1], cell[2], int(pof[cs, e]))])
            quads.append(ring if s0 else [ring[0], ring[3], ring[2], ring[1]])
    return np.array(verts, np.float32).reshape(-1, 3), np.array(quads, np.int64).reshape(-1, 4)
