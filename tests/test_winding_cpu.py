"""Winding number without a GPU: the float64 oracle (tests/winding_oracle.py) pinned by hand on a cube, a regular
tetrahedron, an open hemisphere, duplicated and degenerate faces; the order-1 moments, their merge and the
far-field term against the exact sum; the host-side argument and workspace checks of dgpm_winding with its ctypes
signature; and the ValueErrors that need no device."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import winding_oracle as wo


def _cube(flip=False):
    """The unit cube [0, 1]^3 as 12 triangles, counter-clockwise seen from outside (clockwise with flip)."""
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float64)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))])
    return v, (f[:, ::-1].copy() if flip else f)


def _tetrahedron():
    v = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64)
    f = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]])
    return v, f


def _hemisphere(n=24, m=8):
    """The upper unit hemisphere, pole at +z and its rim of n vertices in z = 0, counter-clockwise from outside."""
    v = [[0.0, 0.0, 1.0]]
    for k in range(1, m + 1):
        th = 0.5 * math.pi * k / m
        for j in range(n):
            ph = 2 * math.pi * j / n
            v.append([math.sin(th) * math.cos(ph), math.sin(th) * math.sin(ph), math.cos(th) if k < m else 0.0])
    ring = lambda k, j: 1 + (k - 1) * n + j % n    # noqa: E731
    f = [[0, ring(1, j), ring(1, j + 1)] for j in range(n)]
    for k in range(1, m):
        for j in range(n):
            f += [[ring(k, j), ring(k + 1, j), ring(k + 1, j + 1)], [ring(k, j), ring(k + 1, j + 1), ring(k, j + 1)]]
    return np.array(v), np.array(f)


def test_cube_inside_outside_and_each_face_from_the_centre():
    v, f = _cube()
    assert wo.polyhedron_volume(v, f) == pytest.approx(1.0)
    inside = np.array([[0.5, 0.5, 0.5], [0.1, 0.9, 0.3], [0.99, 0.01, 0.5]])
    outside = np.array([[1.5, 0.5, 0.5], [-0.1, 0.5, 0.5], [3, 4, 5], [0.5, 0.5, -1e-3], [-7, 2, 0.4]])
    assert np.abs(wo.winding(inside, v, f) - 1).max() < 1e-14
    assert np.abs(wo.winding(outside, v, f)).max() < 1e-14
    per_face = wo.solid_angles(np.array([[0.5, 0.5, 0.5]]), v, f)[0].numpy().reshape(6, 2).sum(1) / (4 * math.pi)
    assert np.abs(per_face - 1 / 6).max() < 1e-15
    vf, ff = _cube(flip=True)
    assert np.abs(wo.winding(inside, vf, ff) + 1).max() < 1e-14


def test_regular_tetrahedron():
    v, f = _tetrahedron()
    assert wo.polyhedron_volume(v, f) > 0
    c = np.zeros((1, 3))
    assert np.abs(wo.solid_angles(c, v, f)[0].numpy() / (4 * math.pi) - 0.25).max() < 1e-15
    g = np.random.default_rng(0)
    p = g.uniform(-1.5, 1.5, (2000, 3))
    # inside the tetrahedron: on the inner side of all four face planes
    a, b, cc = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = np.cross(b - a, cc - a)
    s = np.einsum("qfk,fk->qf", p[:, None] - a[None], n)
    far = np.abs(s).min(1) > 1e-3
    w = wo.winding(p, v, f)
    assert np.abs(w[far] - (s[far] < 0).all(1)).max() < 1e-12


def test_open_hemisphere_from_its_centre_is_one_half():
    v, f = _hemisphere()
    w = wo.winding(np.zeros((1, 3)), v, f)[0]
    assert abs(w - 0.5) < 1e-14


def test_duplicated_faces_double_and_degenerate_faces_add_nothing():
    v, f = _tetrahedron()
    p = np.random.default_rng(1).uniform(-2, 2, (500, 3))
    w = wo.winding(p, v, f)
    assert np.abs(wo.winding(p, v, np.concatenate([f, f])) - 2 * w).max() < 1e-14
    extra = np.array([[0, 0, 0], [1, 0, 0], [3, 0, 0], [2, 5, -1]], np.float64)
    v2 = np.concatenate([v, extra])
    deg = np.array([[4, 5, 6], [6, 5, 4], [7, 7, 7], [4, 4, 5]])
    om = wo.solid_angles(p, v2, deg).numpy()
    assert np.abs(om).max() < 1e-15                 # det is only rounding
    assert np.abs(wo.winding(p, v2, np.concatenate([f, deg])) - w).max() < 1e-15


def test_merged_moments_equal_the_moments_of_the_union():
    g = np.random.default_rng(2)
    v = g.normal(size=(60, 3))
    f = g.permutation(60).reshape(20, 3)
    p, N, M, r, A = wo.merge(wo.moments(v, f[:8]), wo.moments(v, f[8:]))
    p1, N1, M1, r1, A1 = wo.moments(v, f)
    assert np.abs(p - p1).max() < 1e-13 and np.abs(N - N1).max() < 1e-13 and np.abs(M - M1).max() < 1e-13
    assert A == pytest.approx(A1, rel=1e-14) and r >= r1


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_far_field_converges_as_r_over_d_squared(seed):
    """A cluster of 40 triangles of a sphere patch (radius r about p~): |far field - exact| relative to the
    zeroth-order scale A / (4 pi d^2) is at most (r / d)^2 over d = 2r ... 64r, and falls at least as fast."""
    g = np.random.default_rng(seed)
    d0 = g.normal(size=3)
    d0 /= np.linalg.norm(d0)
    pts = g.normal(size=(120, 3)) * 0.3 + d0
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    f = np.arange(120).reshape(40, 3)
    p, N, M, r, A = wo.moments(pts, f)
    ds, errs = 2.0 ** np.arange(1, 7), []
    for k in ds:
        dirs = g.normal(size=(64, 3))
        q = p + dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * k * r
        err = np.abs(wo.far_field(q, p, N, M) - wo.winding(q, pts, f)).max()
        errs.append(err * 4 * math.pi * (k * r) ** 2 / A)
    errs = np.array(errs)
    print("relative far-field error at d / r = 2..64:", " ".join(f"{e:.1e}" for e in errs))
    assert (errs <= (1 / ds) ** 2).all()
    assert (errs[1:] <= errs[:-1] * 0.25 * 1.5).all()


# ---- dgpm_winding host-side checks ---------------------------------------------------------------------------------
FAKE = 1 << 20
PTRS = ["verts", "faces", "points", "winding", "ws"]
SIZES = [dict(V=0), dict(V=-1), dict(F=0), dict(F=-3), dict(Q=-1), dict(V=1 << 30), dict(F=800_000_000),
         dict(Q=715_827_883)]
FNS = ["dgpm_winding", "dgpm_winding_workspace"]


def _header_params(fn):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "dgmesh_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+" + fn + r"\s*\(([^)]*)\)", txt).group(1)
    return [(re.split(r"[\s*]+", a.strip())[-1], a.strip()) for a in decl.split(",")]


def _call(fn, **over):
    import _dgm_lib
    lib = _dgm_lib.lib()
    args = {"V": 8, "F": 12, "Q": 5, "beta": 2.0, "ws_bytes": 1 << 40, "stream": None,
            "bytes": ctypes.pointer(ctypes.c_size_t())}
    args.update(over)
    rc = getattr(lib, fn)(*[args.get(name, FAKE) for name, _ in _header_params(fn)])
    return rc, lib.dgm_last_error()


ROWS = [(fn, s, b"bad size") for fn in FNS for s in SIZES]
ROWS += [("dgpm_winding", {p: None}, b"null pointer") for p in PTRS]
ROWS += [("dgpm_winding_workspace", {"bytes": None}, b"null pointer")]
ROWS += [("dgpm_winding", {"beta": b}, b"beta") for b in (0.0, -0.0, -1.0, -math.inf, math.nan, 1e-50)]
ROWS += [("dgpm_winding", {k: None for k in ks}, b"all NULL or none")
         for ks in (["dist2"], ["face"], ["bary"], ["dist2", "face"], ["face", "bary"], ["dist2", "bary"])]


@pytest.mark.parametrize("fn,over,text", ROWS, ids=[f"{f}-{','.join(f'{k}={v}' for k, v in o.items())}"
                                                    for f, o, _ in ROWS])
def test_bad_argument_is_refused_on_the_host(fn, over, text):
    rc, msg = _call(fn, **over)
    assert rc == -1 and text in msg and fn.encode() in msg, (rc, msg)


def test_infinite_beta_and_no_closest_points_pass_the_checks():
    """beta = +inf is the exact mode; dist2, face and bary may be NULL together (a short workspace then shows that
    every argument check passed without touching the device)."""
    for over in ({"beta": math.inf}, {"dist2": None, "face": None, "bary": None}, {"beta": 1e-30}):
        rc, msg = _call("dgpm_winding", ws_bytes=1, **over)
        assert rc == -2 and b"workspace too small" in msg, (over, rc, msg)


def test_the_size_limits_are_inclusive_below_two_to_the_31():
    n = ctypes.c_size_t()
    top = (2 ** 31 - 1) // 3
    for k in ("V", "F", "Q"):
        assert _call("dgpm_winding_workspace", **{k: top, "bytes": ctypes.byref(n)})[0] == 0, k
        assert _call("dgpm_winding_workspace", **{k: top + 1, "bytes": ctypes.byref(n)})[0] == -1, k


def test_no_query_succeeds_without_touching_anything():
    rc, _ = _call("dgpm_winding", Q=0, **{p: None for p in PTRS + ["dist2", "face", "bary"]}, ws_bytes=0)
    assert rc == 0


@pytest.mark.parametrize("V,F,Q", [(3, 1, 1), (8, 12, 5), (100_000, 200_000, 300_000), (5, 6_700_000, 1_000_000)])
def test_short_workspace_is_refused_on_the_host(V, F, Q):
    need = ctypes.c_size_t()
    rc, _ = _call("dgpm_winding_workspace", V=V, F=F, Q=Q, bytes=ctypes.byref(need))
    assert rc == 0 and need.value > 0
    rc, msg = _call("dgpm_winding", V=V, F=F, Q=Q, ws_bytes=need.value - 1)
    assert rc == -2 and b"workspace too small" in msg and b"dgpm_winding" in msg, (rc, msg)


def test_workspace_bytes_per_face_and_per_query():
    """dgpm_forward's workspace (94 bytes per face, 16 per query, CUB's sort storage) plus, per internal node
    (F / 4 of them), one 144-byte expansion record and one arrival counter: 37 more bytes per face."""
    fwd, wnd = ctypes.c_size_t(), ctypes.c_size_t()
    F, Q = 1_000_000, 10 ** 6
    for q in (1, Q):
        _call("dgpm_forward_workspace", F=F, Q=q, bytes=ctypes.byref(fwd))
        _call("dgpm_winding_workspace", F=F, Q=q, bytes=ctypes.byref(wnd))
        extra = wnd.value - fwd.value
        assert 37 * F - 1024 <= extra <= 37 * F + 1024, extra
    _call("dgpm_winding_workspace", F=F, Q=1, bytes=ctypes.byref(wnd))
    one = wnd.value
    _call("dgpm_winding_workspace", F=F, Q=Q, bytes=ctypes.byref(wnd))
    assert 131 * F <= one < 160 * F and 16 * Q - 1024 <= wnd.value - one < 20 * Q


@pytest.mark.parametrize("fn", FNS)
def test_ctypes_signature_matches_the_header(fn):
    import _dgm_lib
    res, argtypes = _dgm_lib.SIGNATURES[fn]
    params = _header_params(fn)
    assert res is ctypes.c_int and len(argtypes) == len(params)
    for (name, decl), t in zip(params, argtypes):
        if decl.startswith("size_t*"):
            assert t._type_ is ctypes.c_size_t, name
        elif "*" in decl:
            assert t is ctypes.c_void_p, name
        elif decl.startswith("size_t"):
            assert t is ctypes.c_size_t, name
        elif decl.startswith("float"):
            assert t is ctypes.c_float, name
        else:
            assert decl.startswith("int") and t is ctypes.c_int, name


# ---- ValueErrors that need no device -------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", ["winding_number", "signed_distance"])
def test_python_refusals(fn):
    import mesh_distance
    call = getattr(mesh_distance, fn)
    v, f = (torch.from_numpy(x) for x in _cube())
    p = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="CUDA"):
        call(p, v.float(), f)
    with pytest.raises(ValueError):
        call(np.zeros((4, 3), np.float32), v.float(), f)
    for beta in (0, 0.0, -1.0, math.nan, -math.inf, 1e-50, True, "2", None):
        with pytest.raises(ValueError, match="beta"):
            call(p, v.float(), f, beta=beta)


def test_mesh_metrics_refuses_a_bad_iou_point_count():
    from mesh_metrics import mesh_metrics
    v, f = (torch.from_numpy(x) for x in _cube())
    for n in (-1, 2.5, True, "10"):
        with pytest.raises(ValueError, match="iou_points"):
            mesh_metrics((v, f), (v, f), 100, iou_points=n)
