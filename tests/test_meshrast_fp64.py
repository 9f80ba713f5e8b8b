"""Mesh rasterisation (csrc/meshrast.cu through meshrast.py) against the fast float64 restatement of
tests/meshrast_fp64.py, at the sizes DG-Mesh trains at (marching-cubes meshes of 1e4-1e5 triangles, 800x800) and on
the edge cases of the contract (clipping, near / far, degenerate and back-facing triangles, open and non-manifold
meshes, image sizes that are not multiples of the resolve kernel's 32x8 block, 1-pixel images).

Comparison rule.  Every discrete decision -- the triangle id of a pixel, the edge and coverage branch of an
antialias pair -- that float64 takes with a margin above its fp32 tolerance must match the kernel exactly; where
the margin is smaller the kernel's choice must be one float64 admits within the tolerance, and such pixels / pairs
are counted and asserted few.  The continuous outputs are then compared with the oracle evaluated ON THE KERNEL'S
OWN DECISIONS: its ids go to meshrast_fp64.rast, and its per-pair choices -- read from one antialias call on a
one-hot image of the pixels' (x mod 4, y mod 4) classes -- go to meshrast_fp64.antialias.

The CPU tests pin the fast restatement to the loop one of oracle/meshrast_oracle.py and to central differences."""
import math

import pytest
import torch

import meshrast_fp64 as fp
import util
from oracle import meshrast_oracle as orc
from test_meshrast import _random_scene, clip_from_world, icosphere

# Values and attribute / colour gradients: within 1e-4 of the largest float64 value (util.rel_err's scale), plus,
# per element, the first-order bound of the rounding error the kernel's own fp32 arithmetic can make there
# (meshrast_fp64.rast_rounding / wgt_rounding: every rounding of mr_project, edge_fn, mr_bary and aa_pair, in their
# order, times the output's sensitivity to it).  That bound exceeds 1e-4 only on slivers and near-degenerate
# triangles; it carries no safety factor.  The worst ratio of error to allowance is reported per scene and output.
VALUE_TOL = 1e-4
# Vertex-position gradients are fp32 atomic sums over every pixel and pair that touches the vertex.  The error of
# each vertex is held to POS_BUDGET times the sum of the |per-pixel / per-pair contributions| float64 finds for it,
# plus SPREAD_SAFETY times how much those contributions move when the pixel centres / scanlines move by the fp32
# edge tolerance (meshrast_fp64.rounding_spread): a pixel centre a 1e-3 px from an edge has b_k ~ 1e-3, which fp32
# gets to ~1e-4, so its contribution to the opposite vertex (proportional to b_k) is off by ~10 % in any fp32
# evaluation.  Measured on an H100: the worst vertex over the scenes below uses 0.77 of this budget (a G = 288
# marching-cubes mesh at 800x800); with a factor 2 instead of 4 the worst used 0.92.
POS_BUDGET = 1e-3
SPREAD_SAFETY = 4.0
# Pixels / pairs whose decision float64 cannot make with margin, as a fraction of the covered pixels / pairs (plus
# a few, for the 1-pixel-wide images).  The denser the edges, the more: a G = 288 marching-cubes mesh puts up to
# 3.2 % of its pixels within tolerance of an edge at 800x800, an 81 920-face sphere 0.6 %.
MARGIN_FRACTION = 0.06
MARGIN_SLACK = 8


# ------------------------------------------------------------------------------------------------ scenes
def _pose(verts, rot, shift):
    c, s = math.cos(rot), math.sin(rot)
    R = torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float64)
    return (verts.double() @ R.T + torch.tensor(shift, dtype=torch.float64)).float()


def _clip(verts, W, H, **kw):
    return clip_from_world(verts.double(), W, H, **kw).float()


def scene_mixed(W, H, seed=0):
    verts, tri, _ = _random_scene(seed, W, H)
    return _clip(verts, W, H), tri


def scene_occlusion(W, H):
    """Two spheres overlapping in depth, and two large triangles that cross each other: their depth order flips
    inside a pixel row."""
    v1, t1 = icosphere(2, 0.7)
    v2, t2 = icosphere(2, 0.6)
    v1 = v1 + torch.tensor([-0.25, 0.05, 0.0])
    v2 = v2 + torch.tensor([0.3, -0.1, 0.35])
    xa = torch.tensor([[-1.2, -0.9, -0.6], [1.1, -0.7, 0.6], [0.0, 0.9, 0.0]])
    xb = torch.tensor([[-1.1, -0.8, 0.55], [1.2, -0.95, -0.5], [0.1, 0.95, 0.05]])
    verts = torch.cat([v1, v2, xa, xb])
    n1, n2 = v1.shape[0], v2.shape[0]
    tri = torch.cat([t1, t2 + n1, torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32) + n1 + n2])
    return _clip(verts, W, H), tri


def scene_ties(W, H):
    """A sphere whose faces are all duplicated (same vertices, higher ids), plus one face duplicated through its own
    copies of the vertices: the lower id must win every tie."""
    v, t = icosphere(2, 0.8)
    v = v + torch.tensor([0.0123, -0.0071, 0.0])              # no vertex on a pixel centre
    tri = torch.cat([t, t, t[:1]])
    verts = torch.cat([v, v[t[0].long()]])
    tri[-1] = torch.arange(v.shape[0], v.shape[0] + 3, dtype=torch.int32)
    return _clip(verts, W, H), tri


def scene_clip(W, H):
    """A sphere crossing the viewport's left border; a triangle with vertices far outside the viewport at small
    positive w (x/w, y/w of -1000 to 1300: pixel coordinates hundreds of image widths away, which the kernel's
    float-to-int bounding box and the tolerances at that magnitude must handle); a triangle with one vertex behind the eye (w <= 0, dropped whole) sharing an edge with a drawn one,
    so that the drawn one's antialias silhouette test meets an opposite vertex behind the eye; triangles reaching
    beyond the far and the near plane."""
    v, t = icosphere(2, 0.7)
    pos = _clip(v + torch.tensor([-1.45, 0.2, 0.0]), W, H)
    extra = torch.tensor([
        [-2.0e-3, -1.5e-3, 1.99e-6, 2.0e-6], [3.0e-3, -1.0e-3, 2.4875e-6, 2.5e-6], [0.0, 4.0e-3, 2.985e-6, 3.0e-6],  # w small
        [0.2, 0.1, 0.5, 1.0], [0.7, 0.2, 0.5, 1.0], [0.45, 0.6, 0.5, 1.0], [0.5, 0.0, 0.2, -0.5],       # drawn + w<0
        [-0.6, -0.6, 0.5, 1.0], [0.1, -0.55, 1.6, 1.0], [-0.3, -0.1, 0.4, 1.0],                         # beyond far
        [-0.7, 0.3, -1.5, 1.0], [-0.2, 0.35, 0.2, 1.0], [-0.5, 0.8, -0.3, 1.0],                         # beyond near
        [0.6, -0.9, -0.2, 0.0], [0.9, -0.5, 0.1, 1.0], [0.5, -0.4, 0.1, 1.0],                           # w == 0
    ], dtype=torch.float32)
    n = pos.shape[0]
    tri = torch.cat([t, torch.tensor([[0, 1, 2], [3, 4, 5], [4, 3, 6], [7, 8, 9], [10, 11, 12], [13, 14, 15]],
                                     dtype=torch.int32) + n])
    return torch.cat([pos, extra]), tri


def scene_degenerate(W, H):
    """Mixed winding (every third face of a sphere flipped), back-facing faces, zero-area triangles (collinear and
    repeated vertices)."""
    v, t = icosphere(2, 0.8)
    v = v + torch.tensor([0.0123, -0.0071, 0.0])              # no vertex on a pixel centre
    t = t.clone()
    t[::3] = t[::3][:, [0, 2, 1]]
    n = v.shape[0]
    flat = torch.tensor([[-0.9, -0.9, 0.5], [-0.5, -0.5, 0.5], [-0.1, -0.1, 0.5]])     # collinear
    verts = torch.cat([v, flat])
    tri = torch.cat([t, torch.tensor([[n, n + 1, n + 2], [n, n, n + 1], [0, 1, 1]], dtype=torch.int32)])
    return _clip(verts, W, H), tri


def scene_topology(W, H):
    """An open mesh (a sphere cut in half: boundary edges) and a fin: an edge shared by three triangles."""
    v, t = icosphere(2, 0.8)
    v = v + torch.tensor([-0.0093, 0.0117, 0.0])              # no vertex on a pixel centre
    keep = v[t.long()].mean(1)[:, 2] < 0.15
    t = t[keep]
    n = v.shape[0]
    fin = torch.tensor([[0.3, -0.3, -0.5], [0.3, 0.4, -0.5], [0.9, 0.0, -0.6], [-0.2, 0.1, -0.7], [0.5, 0.05, 0.1]])
    verts = torch.cat([v, fin])
    tri = torch.cat([t, torch.tensor([[n, n + 1, n + 2], [n + 1, n, n + 3], [n, n + 1, n + 4]], dtype=torch.int32)])
    return _clip(verts, W, H), tri


SMALL_SCENES = {"mixed": scene_mixed, "occlusion": scene_occlusion, "ties": scene_ties, "clip": scene_clip,
                "degenerate": scene_degenerate, "topology": scene_topology}
SMALL_SIZES = [(33, 41), (37, 1), (1, 37), (64, 48)]


def _attr(V, C, seed):
    g = torch.Generator().manual_seed(seed)
    return 0.05 + 0.9 * torch.rand(V, C, generator=g)


# ------------------------------------------------------------------------------------------------ CPU: oracle pins
@pytest.mark.parametrize("name", sorted(SMALL_SCENES))
@pytest.mark.parametrize("W,H", SMALL_SIZES)
def test_fast_oracle_equals_loop_oracle_cpu(name, W, H):
    pos, tri = SMALL_SCENES[name](W, H)
    pos = pos.double()
    ids_l = orc.rasterize_ids(pos, tri.long(), H, W)
    fr = fp.rasterize(pos, tri, H, W)
    assert torch.equal(fr["ids"], ids_l)
    rast_l = orc.rast_from_ids(pos, tri.long(), ids_l)
    rast_f, _, _ = fp.rast(pos, tri, ids_l)
    assert torch.equal(rast_f[..., 3], rast_l[..., 3])
    assert float((rast_f - rast_l).abs().max()) <= 1e-12
    for C in (1, 3, 4, 7):
        attr = _attr(pos.shape[0], C, C).double()
        ci_l = orc.interpolate(attr, rast_l, tri.long())
        ci_f = fp.interpolate(attr, rast_f, tri)
        assert float((ci_f - ci_l).abs().max()) <= 1e-12
    opp = orc.edge_opposites(tri, pos.shape[0])
    assert torch.equal(fp.edge_opposites(tri, pos.shape[0]), opp)
    pairs = fp.aa_pairs(ids_l, rast_l[..., 2], pos, tri, opp, W, H)
    for C, bg in ((1, 0.0), (3, 0.0), (3, 1.0)):
        col = orc.interpolate(_attr(pos.shape[0], C, 7).double(), rast_l, tri.long())
        col = torch.where((ids_l >= 0)[..., None], col, torch.full_like(col, bg))
        out_l = orc.antialias(col, rast_l, pos, tri.long(), opp)
        out_f, _, _, _ = fp.antialias(col, pos, tri, pairs, W, H)
        assert float((out_f - out_l).abs().max()) <= 1e-12, (C, bg)


def test_fast_oracle_sees_every_edge_case_cpu():
    """The edge-case scenes contain what they are meant to: a dropped w <= 0 triangle, pixels rejected beyond near
    and far, lost zero-area triangles, exact ties won by the lower id, a non-manifold edge paired by face order."""
    W, H = 64, 48
    pos, tri = scene_clip(W, H)
    fr = fp.rasterize(pos.double(), tri, H, W)
    F = tri.shape[0]
    ids = fr["ids"]
    assert bool((ids == F - 6).any()) and bool((ids == F - 5).any()) and not bool((ids == F - 4).any())
    assert bool((ids == F - 3).any()) and bool((ids == F - 2).any()) and not bool((ids == F - 1).any())
    g = fr["geometry"]
    assert not bool(g["drawn"][F - 4]) and not bool(g["drawn"][F - 1])
    far = fp.project(pos.double(), W, H)[tri[F - 6].long(), :2]
    assert float(far.abs().max(1).values.min()) > 100 * max(W, H)               # hundreds of image widths away
    # the beyond-far / beyond-near triangles lose part of their bbox interior to the z/w test
    for f in (F - 3, F - 2):
        s = fp.project(pos.double(), W, H)[tri[f].long()]
        zs = s[:, 2]
        assert float(zs.max()) > 1 or float(zs.min()) < -1
    pos, tri = scene_ties(W, H)
    fr = fp.rasterize(pos.double(), tri, H, W)
    n = (tri.shape[0] - 1) // 2
    assert int((fr["ids"] >= 0).sum()) > 0 and not bool((fr["ids"] >= n).any())
    pos, tri = scene_topology(W, H)
    opp = fp.edge_opposites(tri, pos.shape[0])
    V = pos.shape[0]
    F = tri.shape[0]
    assert int(opp[F - 3, 0]) == V - 2 and int(opp[F - 2, 0]) == V - 3 and int(opp[F - 1, 0]) == -1
    assert bool((opp[:F - 3] < 0).any())                                        # boundary edges of the open mesh


def test_fast_oracle_gradient_is_the_derivative_of_its_forward_cpu():
    """Autograd through the fast restatement (pos.grad, and the per-pixel / per-pair copies summed per vertex)
    equals central differences of its own forward, with a step far below the next pixel-centre crossing."""
    W, H = 33, 41
    verts, tri = icosphere(1, 1.0)
    opp = fp.edge_opposites(tri, verts.shape[0])
    g = torch.Generator().manual_seed(0)
    attr = torch.rand(verts.shape[0], 3, generator=g, dtype=torch.float64)
    wimg = torch.randn(H, W, 3, generator=g, dtype=torch.float64)

    def f(shift, keep=None):
        pos = clip_from_world(verts.double() + shift, W, H)
        ids = fp.rasterize(pos.detach(), tri, H, W)["ids"]
        r, P, pf = fp.rast(pos, tri, ids)
        pairs = fp.aa_pairs(ids, r[..., 2].detach(), pos.detach(), tri, opp, W, H)
        out, Pv, vid, _ = fp.antialias(fp.interpolate(attr, r, tri), pos, tri, pairs, W, H)
        if keep is not None:
            keep.update(pos=pos, P=P, pf=pf, Pv=Pv, vid=vid)
        return (out * wimg).sum()

    sh = torch.tensor([0.013, -0.007, 0.02], dtype=torch.float64, requires_grad=True)
    keep = {}
    loss = f(sh, keep)
    keep["pos"].retain_grad()
    loss.backward()
    tot, ab = fp.vertex_budget(verts.shape[0], [(keep["P"].grad, keep["pf"]), (keep["Pv"].grad, keep["vid"])])
    assert float((tot - keep["pos"].grad).abs().max()) <= 1e-9 * float(ab.max())
    assert float(keep["Pv"].grad.abs().sum()) > 0
    eps = 1e-7
    for k in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[k] = eps
        fd = float((f(sh.detach() + e) - f(sh.detach() - e)) / (2 * eps))
        assert abs(fd - float(sh.grad[k])) < 1e-4 * max(1.0, abs(fd)), (k, fd, float(sh.grad[k]))


def test_fast_oracle_margins_cpu():
    """A pixel centre exactly on an edge shared by two triangles is a margin pixel and one far from every edge is
    not; an exact copy of the winner ties without doubt (fp32 computes the same depth for both and the lower id
    wins), a copy moved in depth by far less than the depth tolerance does not."""
    W, H = 8, 8
    px = torch.tensor([[1.0, 1.0], [7.0, 1.0], [7.0, 7.0], [1.0, 7.0]], dtype=torch.float64)
    pos = torch.stack([px[:, 0] / W * 2 - 1, px[:, 1] / H * 2 - 1, torch.zeros(4, dtype=torch.float64),
                       torch.ones(4, dtype=torch.float64)], -1)
    tri = torch.tensor([[0, 1, 2], [0, 2, 3]])               # the shared diagonal runs through (3.5, 3.5)
    fr = fp.rasterize(pos, tri, H, W)
    assert bool(fr["certain"][2, 5]) and int(fr["ids"][2, 5]) == 0
    assert not bool(fr["certain"][3, 3]) and int(fr["ids"][3, 3]) == 0
    assert float(fr["edge_px"][3, 3]) == 0.0
    fr = fp.rasterize(pos, torch.tensor([[0, 1, 2], [0, 1, 2]]), H, W)
    assert int(fr["ids"][2, 5]) == 0 and bool(fr["certain"][2, 5])
    pos2 = torch.cat([pos, pos[:1] + torch.tensor([0.0, 0.0, 1e-12, 0.0], dtype=torch.float64)])
    fr = fp.rasterize(pos2, torch.tensor([[0, 1, 2], [4, 1, 2]]), H, W)
    assert int(fr["ids"][2, 5]) in (0, 1) and not bool(fr["certain"][2, 5])


def _bary_fp32(pos32, tri, ids):
    """mr_project + mr_bary in float32, operation by operation (an fp32 evaluation like the kernel's, without its
    fused multiply-adds): (u, v, z/w) [H,W,3] on the given ids."""
    H, W = ids.shape
    flat = ids.reshape(-1)
    p = torch.nonzero(flat >= 0).flatten()
    P = pos32.float()[tri.long()[flat[p]]]
    px = (p % W).float() + 0.5
    py = torch.div(p, W, rounding_mode="floor").float() + 0.5
    iw = 1.0 / P[..., 3]
    sx = (P[..., 0] * iw * 0.5 + 0.5) * W
    sy = (P[..., 1] * iw * 0.5 + 0.5) * H
    zv = P[..., 2] * iw
    e = fp._edge
    inv = 1.0 / e(sx[:, 0], sy[:, 0], sx[:, 1], sy[:, 1], sx[:, 2], sy[:, 2])
    b0 = e(sx[:, 1], sy[:, 1], sx[:, 2], sy[:, 2], px, py) * inv
    b1 = e(sx[:, 2], sy[:, 2], sx[:, 0], sy[:, 0], px, py) * inv
    b2 = 1.0 - b0 - b1
    q0, q1, q2 = b0 * iw[:, 0], b1 * iw[:, 1], b2 * iw[:, 2]
    d = 1.0 / (q0 + q1 + q2)
    out = torch.zeros(H * W, 3)
    out[p] = torch.stack([q0 * d, q1 * d, b0 * zv[:, 0] + b1 * zv[:, 1] + b2 * zv[:, 2]], 1)
    return out.view(H, W, 3)


def test_rounding_bound_covers_fp32_and_sees_a_sub_pixel_shift_cpu():
    """The value allowance (VALUE_TOL of the scale plus meshrast_fp64.rast_rounding) holds an fp32 evaluation of
    the barycentrics on an 81 920-face sphere at 800x800, and is tight enough that sampling 1/1024 px off the pixel
    centre -- with every triangle id unchanged -- breaks it."""
    W = H = 800
    verts, tri = icosphere(6, 0.8)
    pos32 = _clip(_pose(verts, 0.37, (0.0131, -0.0213, 0.3)), W, H)
    pos = pos32.double()
    ids = fp.rasterize(pos, tri, H, W)["ids"]
    r64, _, _ = fp.rast(pos, tri, ids)
    rb = fp.rast_rounding(pos, tri, ids)
    allow = VALUE_TOL + rb
    err32 = (_bary_fp32(pos32, tri, ids).double() - r64[..., :3]).abs()
    assert float((err32 / allow).max()) <= 1.0
    assert float((err32 / rb.clamp_min(1e-300))[ids >= 0].max()) <= 1.0      # the bound alone holds fp32
    n = int((ids >= 0).sum())
    s = torch.full((n,), 1.0 / 1024, dtype=torch.float64)
    shifted, _, _ = fp.rast(pos, tri, ids, (s, s))
    assert float(((shifted[..., :3] - r64[..., :3]).abs() / allow).max()) > 1.0


# ------------------------------------------------------------------------------------------------ GPU
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")


def _report(**kw):
    print("meshrast_fp64 " + " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in kw.items()))


def _close(name, got, ref, extra=None):
    """|got - ref| <= VALUE_TOL max|ref| + extra (extra: a per-element conditioning bound, default 0); returns the
    worst ratio of error to allowance."""
    got, ref = got.double(), ref.double().to(got.device)
    err = (got - ref).abs()
    allow = VALUE_TOL * float(ref.abs().max()) + (0.0 if extra is None else extra)
    ratio = float((err / allow).max()) if err.numel() else 0.0
    assert ratio <= 1.0, (name, ratio, util.rel_err(got, ref))
    return ratio


def _neighbour_max(x):
    """max over each pixel and its four neighbours of x [H,W]."""
    m = x.clone()
    m[1:] = torch.maximum(m[1:], x[:-1])
    m[:-1] = torch.maximum(m[:-1], x[1:])
    m[:, 1:] = torch.maximum(m[:, 1:], x[:, :-1])
    m[:, :-1] = torch.maximum(m[:, :-1], x[:, 1:])
    return m


def _applied(pairs, k, branch):
    use = k >= 0
    dst = torch.where(branch[use], pairs["p_out"][use], pairs["p_in"][use])
    src = torch.where(branch[use], pairs["p_in"][use], pairs["p_out"][use])
    return dst, src


def _aa_allowance(pairs, k, branch, col, ecol, bw, H, W):
    """[H,W,C] fp32 error bound of the antialiased image: out[dst] = col[dst] + wgt (col[src] - col[dst]) with
    wgt <= 1/2 carries the colour errors ecol of both pixels and the weight's rounding bound bw times the colour
    difference."""
    dst, src = _applied(pairs, k, branch)
    cf, ef = col.reshape(H * W, -1), ecol.reshape(H * W, -1)
    e = ef.clone()
    e.index_add_(0, dst, 0.5 * (ef[src] + ef[dst]) + bw[:, None] * (cf[src] - cf[dst]).abs())
    return e.view(H, W, -1)


def _aa_grad_allowance(pairs, k, branch, gout, bw, H, W):
    """[H,W,C] fp32 error bound of dL/dcolour through antialias: each applied pair moves |dL/dout[dst]| times its
    weight between its two pixels, and the weight is off by up to its rounding bound bw."""
    dst, src = _applied(pairs, k, branch)
    gf = gout.reshape(H * W, -1).abs()
    e = torch.zeros_like(gf)
    e.index_add_(0, dst, bw[:, None] * gf[dst])
    e.index_add_(0, src, bw[:, None] * gf[dst])
    return e.view(H, W, -1)


def _interp_allowance(attr, t, ids, rb):
    """[H,W,C] fp32 error bound of interpolate from the rounding bounds rb of the rast's u, v: the output moves by
    |a0 - a2| du + |a1 - a2| dv (its own rounding is far below VALUE_TOL)."""
    f = ids.clamp_min(0)
    a0, a1, a2 = (attr.double()[t.long()[f, j]] for j in range(3))
    e = (a0 - a2).abs() * rb[..., 0:1] + (a1 - a2).abs() * rb[..., 1:2]
    return torch.where((ids >= 0)[..., None], e, torch.zeros_like(e))


def _per_vertex(V, t, ids, x):
    """Sum of x [H,W,C] over the covered pixels into each of their triangle's three vertices."""
    flat = ids.reshape(-1)
    hit = torch.nonzero(flat >= 0).flatten()
    xs = x.reshape(flat.numel(), -1)[hit]
    out = torch.zeros(V, xs.shape[1], dtype=torch.float64, device=x.device)
    for j in range(3):
        out.index_add_(0, t.long()[flat[hit], j], xs)
    return out


def _decisions(label, pos, tri, H, W, rast_k, opp, probe):
    """The kernel's ids and antialias choices against float64's; returns (pairs, k, branch) for the value pass."""
    ids_k = rast_k[..., 3].long() - 1
    fr = fp.rasterize(pos, tri, H, W)
    covered = int((fr["ids"] >= 0).sum())
    certain = fr["certain"]
    wrong = certain & (ids_k != fr["ids"])
    assert not bool(wrong.any()), (label, "ids differ at pixels float64 decides with margin", int(wrong.sum()),
                                   torch.nonzero(wrong)[:5].tolist())
    adm = fp.admissible(fr, ids_k, H, W)
    assert bool(adm.all()), (label, "inadmissible ids", int((~adm).sum()), torch.nonzero(~adm)[:5].tolist())
    n_margin = int((~certain).sum())
    assert n_margin <= MARGIN_FRACTION * covered + MARGIN_SLACK, (label, n_margin, covered)
    pairs = fp.aa_pairs(ids_k, rast_k[..., 2], pos, tri, opp, W, H)
    to_out, wgt, both = fp.read_choices(probe, pairs, W)
    assert not bool(both.any()), (label, "a pair wrote both of its pixels")
    k, branch, matched = fp.match_choices(pairs, to_out, wgt)
    assert bool(matched.all()), (label, "kernel coverage matches no admissible edge", int((~matched).sum()))
    cp = pairs["certain"]
    same = (k == pairs["k"]) & ((k < 0) | (branch == (torch.where(pairs["first_in"], pairs["alpha"].gather(
        1, pairs["k"].clamp_min(0)[:, None])[:, 0], 1 - pairs["alpha"].gather(1, pairs["k"].clamp_min(0)[:, None])[
        :, 0]) >= 0.5)))
    bad = cp & ~same
    assert not bool(bad.any()), (label, "antialias choice differs where float64 decides with margin", int(bad.sum()))
    npairs, ndoubt = int(pairs["p0"].numel()), int((~cp).sum())
    assert ndoubt <= MARGIN_FRACTION * npairs + MARGIN_SLACK, (label, ndoubt, npairs)
    _report(scene=label, W=W, H=H, covered=covered, margin_pixels=n_margin, pairs=npairs, margin_pairs=ndoubt,
            min_edge_px=float(torch.where(certain & (fr["ids"] >= 0), fr["edge_px"], math.inf).min()))
    return pairs, k, branch


def _kernel_side(pos32, tri, H, W, C=3, bg=None, seed=0):
    """Kernel rasterize -> interpolate -> (background) -> antialias, forward and backward for a random-weight image
    loss, and the antialias of the class image that reveals the per-pair choices."""
    import meshrast as dr
    dev = torch.device("cuda")
    V = pos32.shape[0]
    t = tri.to(dev).int()
    attr = _attr(V, C, seed).to(dev)
    wimg = torch.randn(H, W, C, generator=torch.Generator().manual_seed(seed + 1)).to(dev)
    pos_k = pos32.to(dev).clone().requires_grad_(True)
    attr_k = attr.clone().requires_grad_(True)
    rast_k = dr.rasterize(None, pos_k[None], t, resolution=[H, W])[0]
    col_k = dr.interpolate(attr_k[None], rast_k, t)[0][0]
    if bg is not None:
        col_k = torch.where(rast_k[0, ..., 3:] > 0, col_k, torch.full_like(col_k, bg))
    col_k.retain_grad()
    opp = dr.edge_opposites(t, V)
    out_k = dr.antialias(col_k[None], rast_k, pos_k[None], t, topology_hash=opp)[0]
    (out_k * wimg).sum().backward()
    probe = dr.antialias(fp.class_colors(H, W, dev)[None], rast_k.detach(), pos_k.detach()[None], t,
                         topology_hash=opp)[0]
    return dict(rast=rast_k[0].detach(), opp=opp, probe=probe, col=col_k.detach(), out=out_k.detach(),
                d_pos=pos_k.grad, d_attr=attr_k.grad, d_col=col_k.grad, attr=attr, wimg=wimg)


def _check_scene(label, pos32, tri, H, W, C=3, bg=None, seed=0, ks=None):
    """The kernel side against float64 on the kernel's decisions (`ks`: a recorded kernel side)."""
    ks = _kernel_side(pos32, tri, H, W, C, bg, seed) if ks is None else ks
    dev = ks["rast"].device
    V = pos32.shape[0]
    t = tri.to(dev).int()
    rast_k, opp, probe, attr, wimg = ks["rast"], ks["opp"], ks["probe"], ks["attr"], ks["wimg"]
    col_k, out_k = ks["col"], ks["out"]
    assert torch.equal(opp.long(), fp.edge_opposites(t, V)), (label, "edge_opposites")
    # ---- decisions
    pos = pos32.to(dev).double()
    pairs, k, branch = _decisions(label, pos, t, H, W, rast_k, opp, probe)
    ids_k = rast_k[..., 3].long() - 1
    # ---- float64 on the kernel's decisions
    pos_o = pos.clone().requires_grad_(True)
    attr_o = attr.double().requires_grad_(True)
    r_o, P, pf = fp.rast(pos_o, t, ids_k)
    col_o = fp.interpolate(attr_o, r_o, t)
    if bg is not None:
        col_o = torch.where((ids_k >= 0)[..., None], col_o, torch.full_like(col_o, bg))
    col_o.retain_grad()
    r_o.retain_grad()
    off = torch.zeros(int((k >= 0).sum()), dtype=torch.float64, device=dev, requires_grad=True)
    out_o, Pv, vid, use = fp.antialias(col_o, pos_o, t, pairs, W, H, k=k, branch=branch, alpha_offset=off)
    (out_o * wimg.double()).sum().backward()
    # ---- values: 1e-4 of the largest value plus the first-order bound of the kernel's own fp32 rounding
    rb = fp.rast_rounding(pos, t, ids_k)
    bw = fp.wgt_rounding(pos, t, pairs, k, branch, W, H)
    worst = {}
    worst["uv"] = _close(label + " u,v", rast_k[..., :2], r_o[..., :2].detach(), rb[..., :2])
    worst["zw"] = _close(label + " z/w", rast_k[..., 2], r_o[..., 2].detach(), rb[..., 2])
    ecol = _interp_allowance(attr, t, ids_k, rb)
    worst["interp"] = _close(label + " interpolate", col_k, col_o.detach(), ecol)
    worst["antialias"] = _close(label + " antialias", out_k, out_o.detach(),
                                _aa_allowance(pairs, k, branch, col_o.detach(), ecol, bw, H, W))
    # ---- gradients
    # d/d colour: the antialias weights are off by up to bw; d/d attr = sum over pixels of dL/dcolour * (u, v,
    # 1 - u - v), whose barycentrics are off by up to rb
    e_col = _aa_grad_allowance(pairs, k, branch, wimg.double(), bw, H, W)
    worst["d_color"] = _close(label + " d/d color", ks["d_col"], col_o.grad, e_col)
    battr = _per_vertex(V, t, ids_k, col_o.grad.abs() * (rb[..., 0:1] + rb[..., 1:2]) + e_col)
    worst["d_attr"] = _close(label + " d/d attr", ks["d_attr"], attr_o.grad, battr)
    tot, ab = fp.vertex_budget(V, [(P.grad, pf), (Pv.grad, vid)])
    assert float((tot - pos_o.grad).abs().max()) <= 1e-9 * float(ab.max()) + 1e-30
    spread = fp.rounding_spread(pos, t, ids_k, pairs, k, branch, W, H, r_o.grad[..., :2], off.grad)
    err = (ks["d_pos"].double() - pos_o.grad).abs()
    allow = POS_BUDGET * ab + SPREAD_SAFETY * spread + 1e-7 * float(ab.max())
    worst["d_pos_budget"] = float((err / allow).max())
    worst["d_pos_maxnorm"] = util.rel_err(ks["d_pos"], pos_o.grad)
    _report(scene=label, C=C, bg=-1.0 if bg is None else float(bg), **worst)
    assert worst["d_pos_budget"] <= 1.0, (label, "d/d pos", worst)
    return worst


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("name", sorted(SMALL_SCENES))
@pytest.mark.parametrize("W,H", SMALL_SIZES)
def test_cuda_edge_case_scenes_match_float64(name, W, H):
    pos, tri = SMALL_SCENES[name](W, H)
    _check_scene(f"{name}", pos, tri, H, W)


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("C", [1, 3, 4, 7])
def test_cuda_interpolate_channels_match_float64(C):
    pos, tri = scene_occlusion(64, 48)
    _check_scene(f"occlusion_C{C}", pos, tri, 48, 64, C=C, seed=C)


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("C,bg", [(1, 0.0), (1, 1.0), (3, 0.0), (3, 1.0)])
def test_cuda_antialias_background_matches_float64(C, bg):
    pos, tri = scene_mixed(64, 48, seed=1)
    _check_scene(f"mixed_C{C}_bg{bg}", pos, tri, 48, 64, C=C, bg=bg, seed=3)


@pytest.mark.gpu
@needs_cuda
def test_cuda_exact_depth_ties_go_to_the_lower_id():
    import meshrast as dr
    W, H = 96, 80
    pos, tri = scene_ties(W, H)
    n = (tri.shape[0] - 1) // 2
    rast = dr.rasterize(None, pos.cuda()[None], tri.cuda(), resolution=[H, W])[0][0]
    ids = rast[..., 3].long() - 1
    assert int((ids >= 0).sum()) > 0
    assert not bool((ids >= n).any()), "a duplicate (higher id) won a tie"
    base = dr.rasterize(None, pos.cuda()[None], tri[:n].cuda(), resolution=[H, W])[0][0]
    assert torch.equal(rast, base)                               # bit for bit the picture without the duplicates
    _check_scene("ties", pos, tri, H, W)


def _sdf_mesh(G):
    """A marching-cubes mesh (diso.DiffMC) of the union of a sphere and a tilted torus: slivers and
    near-degenerate triangles where the two surfaces meet."""
    from diso import DiffMC
    x = torch.linspace(0, 1, G, device="cuda")
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    sphere = ((X - 0.42) ** 2 + (Y - 0.5) ** 2 + (Z - 0.5) ** 2).sqrt() - 0.3
    c, s = math.cos(0.6), math.sin(0.6)
    tx, ty, tz = X - 0.62, (Y - 0.5) * c - (Z - 0.5) * s, (Y - 0.5) * s + (Z - 0.5) * c
    torus = ((tx ** 2 + ty ** 2).sqrt() - 0.22) ** 2 + tz ** 2
    torus = torus.sqrt() - 0.07
    verts, faces = DiffMC().cuda()(torch.minimum(sphere, torus), deform=None, isovalue=0.0)
    return ((verts.detach() * 2 - 1) * 0.9).float().cpu(), faces.int().cpu()


def _ico6():
    return icosphere(6, 0.8)


BIG = [("ico6", 800, 800, 0.0, (0.0, 0.0, 0.0)), ("ico6", 800, 800, 0.37, (0.0131, -0.0213, 0.3)),
       ("ico6", 800, 800, 1.1, (0.05, 0.0207, 0.1)), ("mc128", 800, 800, 0.3, (0.0, 0.0, 0.0)),
       ("mc288", 800, 800, 0.0, (0.0, 0.0, 0.0)), ("mc288", 800, 800, 2.2, (0.0093, 0.017, -0.4)),
       ("mc288", 1920, 1080, 0.7, (0.0, 0.0, 1.0))]


@pytest.mark.gpu
@needs_cuda
@pytest.mark.parametrize("mesh,W,H,rot,shift", BIG)
def test_cuda_marching_cubes_scale_matches_float64(mesh, W, H, rot, shift):
    verts, tri = _ico6() if mesh == "ico6" else _sdf_mesh(int(mesh[2:]))
    assert tri.shape[0] > 2e4
    pos = _clip(_pose(verts, rot, shift), W, H)
    _check_scene(f"{mesh}_{W}x{H}_r{rot}", pos, tri, H, W)


def _fan_and_sphere():
    """A fan of 40 triangles on one edge (either orientation), and the same faces shuffled into a 2e4-face sphere."""
    g = torch.Generator().manual_seed(5)
    fan = torch.stack([torch.zeros(40, dtype=torch.int32), torch.ones(40, dtype=torch.int32),
                       torch.arange(2, 42, dtype=torch.int32)], 1)
    flip = torch.rand(40, generator=g) < 0.5
    fan[flip] = fan[flip][:, [1, 0, 2]]
    v, t = icosphere(5, 1.0)
    big = torch.cat([t + 42, fan])[torch.randperm(t.shape[0] + 40, generator=g)]
    pos, top = scene_topology(33, 41)
    return [(fan, 42), (big, v.shape[0] + 42), (top, pos.shape[0])]


def test_edge_opposites_pairs_the_first_two_users_cpu():
    """meshrast.edge_opposites pairs every edge's first two users in face order, as meshrast_oracle.edge_opposites
    does, on non-manifold edges of up to 40 users.  A check of the contract: the sorts of the current torch keep
    equal keys in order with or without stable=True, so this passes either way and does not single out that flag."""
    import meshrast as dr
    for tri, V in _fan_and_sphere():
        ref = orc.edge_opposites(tri, V) if tri.shape[0] < 500 else fp.edge_opposites(tri, V)
        assert torch.equal(dr.edge_opposites(tri, V).long(), ref)


@pytest.mark.gpu
@needs_cuda
def test_cuda_edge_opposites_pairs_the_first_two_users():
    """The same contract check on CUDA tensors (again passing with or without stable=True on the current torch)."""
    import meshrast as dr
    for tri, V in _fan_and_sphere():
        ref = orc.edge_opposites(tri, V) if tri.shape[0] < 500 else fp.edge_opposites(tri, V)
        assert torch.equal(dr.edge_opposites(tri.cuda(), V).cpu().long(), ref)


@pytest.mark.gpu
@needs_cuda
def test_cuda_renderer_mask_and_mesh_loss_match_float64():
    """utils.renderer.render_mask + render_mesh (white background) on a marching-cubes mesh at 800x800 and a
    mask-plus-mesh-image L1 loss: the vertex and vertex-colour gradients against float64 on the kernel's decisions
    (its ids, antialias choices, background mask and the signs of the L1 terms)."""
    import importlib
    import meshrast as dr
    rend = importlib.import_module("utils.renderer")
    verts, tri = _sdf_mesh(128)
    dev = torch.device("cuda")
    H = W = 800
    V = verts.shape[0]
    col = _attr(V, 3, 9).to(dev)
    focal = W / (2 * math.tan(0.6911 / 2))
    K = torch.tensor([[focal, 0, W / 2 + 0.37], [0, focal, H / 2 - 0.21], [0, 0, 1.0]])
    c2w = torch.eye(4)
    c2w[2, 3] = 4.0
    pose = torch.inverse(c2w)
    g = torch.Generator().manual_seed(11)
    gt_m = torch.rand(H, W, 1, generator=g).to(dev)
    gt_i = torch.rand(3, H, W, generator=g).to(dev)
    t = tri.to(dev)
    vk = verts.to(dev).requires_grad_(True)
    ck = col.clone().requires_grad_(True)
    mask = rend.render_mask(None, vk, t, pose, K, resolution=[H, W])
    img = rend.render_mesh(None, vk, t, ck, pose, K, resolution=[H, W], whitebackground=True)
    loss = (mask[..., :1] - gt_m).abs().mean() * 100 + (img - gt_i).abs().mean()
    loss.backward()
    # the clip-space positions and the rasterisation the renderer made
    mtx = (rend.K_to_projection(K, H, W) @ pose).to(dev)
    pos32 = rend.transform_pos(mtx, vk.detach())[0]
    rast_k = dr.rasterize(None, pos32[None], t, resolution=[H, W])[0]
    opp = dr.edge_opposites(t, V)
    probe = dr.antialias(fp.class_colors(H, W, dev)[None], rast_k, pos32[None], t, topology_hash=opp)[0]
    rast_k = rast_k[0]
    pos = pos32.double()
    pairs, k, branch = _decisions("renderer_mc128", pos, t, H, W, rast_k, opp, probe)
    ids_k = rast_k[..., 3].long() - 1
    pos_o = pos.clone().requires_grad_(True)
    co = col.double().requires_grad_(True)
    r_o, P, pf = fp.rast(pos_o, t, ids_k)
    r_o.retain_grad()
    off = torch.zeros(int((k >= 0).sum()), dtype=torch.float64, device=dev, requires_grad=True)
    ones = fp.interpolate(torch.ones(V, 3, dtype=torch.float64, device=dev), r_o, t)
    m_o, Pv1, vid1, _ = fp.antialias(ones, pos_o, t, pairs, W, H, k=k, branch=branch, alpha_offset=off)
    m_o = torch.flip(m_o, dims=[0])
    c_o = fp.interpolate(co, r_o, t)
    c_o.retain_grad()
    i_o, Pv2, vid2, _ = fp.antialias(c_o, pos_o, t, pairs, W, H, k=k, branch=branch, alpha_offset=off)
    i_o.retain_grad()
    i_aa = i_o
    i_o = torch.flip(i_o, dims=[0])
    keep = mask.detach().bool()
    i_o = torch.where(keep, i_o, torch.ones_like(i_o)).permute(2, 0, 1)
    inner = keep.permute(2, 0, 1)
    assert float(img.detach()[inner].min()) > 0.0 and float(img.detach()[inner].max()) < 1.0   # clamp inactive
    sm = torch.sign(mask.detach()[..., :1] - gt_m).double()
    si = torch.sign(img.detach() - gt_i).double()
    loss_o = (sm * (m_o[..., :1] - gt_m)).mean() * 100 + (si * (i_o - gt_i)).mean()
    loss_o.backward()
    rb = fp.rast_rounding(pos, t, ids_k)
    bw = fp.wgt_rounding(pos, t, pairs, k, branch, W, H)
    eaa = _aa_allowance(pairs, k, branch, ones.detach(), torch.zeros_like(ones), bw, H, W)
    d_mask = _close("renderer mask", mask.detach(), m_o.detach(), torch.flip(eaa, dims=[0]))
    e_col = _aa_grad_allowance(pairs, k, branch, i_aa.grad, bw, H, W) + c_o.grad.abs() * (rb[..., 0:1] + rb[..., 1:2])
    d_col = _close("renderer d/d vertex colour", ck.grad, co.grad, _per_vertex(V, t, ids_k, e_col))
    tot, ab = fp.vertex_budget(V, [(P.grad, pf), (Pv1.grad, vid1), (Pv2.grad, vid2)])
    m3 = mtx.double()[:, :3]
    gv_o = pos_o.grad @ m3
    spread = fp.rounding_spread(pos, t, ids_k, pairs, k, branch, W, H, r_o.grad[..., :2], off.grad)
    ab_v = (ab + SPREAD_SAFETY / POS_BUDGET * spread) @ m3.abs()
    err = (vk.grad.double() - gv_o).abs()
    ratio = float((err / (POS_BUDGET * ab_v + 1e-7 * float(ab_v.max()))).max())
    _report(scene="renderer_mc128", mask=d_mask, d_color=d_col, d_verts_budget=ratio,
            d_verts_maxnorm=util.rel_err(vk.grad, gv_o))
    assert ratio <= 1.0
