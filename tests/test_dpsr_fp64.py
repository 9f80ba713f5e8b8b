"""DPSR (csrc/dpsr.cu) against a float64 reference, with an error budget measured from fp32.

The reference is tests/ref_dpsr.py's algorithm run in float64 with autograd (_dpsr64). Its stencil takes the
discrete decisions (cell, wrapped upper index, node coordinates) in the same fp32 arithmetic as the kernel, so
points on nodes, in the last cell and at the clamp bounds land in the same cells with the same kink of |p - node|;
everything after that is float64. For every output -- the field, dV, dN and, for forward_signed, dthres -- the CUDA
path's util.rel_err against float64 must be at most max(K * e32, FLOOR) (K_NYQUIST on the Nyquist upstreams), where
e32 is the error of tests/ref_dpsr.py itself, run in fp32 on the GPU. On the oriented scenes the error must also
stay under the absolute ceiling CEIL, and the scene must stay well conditioned: the field is normalised by
|phi[0,0,0] - mean_p phi(p)|, and on unoriented normals that difference is ~1000x smaller than the field, which
loosens every fp32 comparison by as much.

The upstream gradients isolate the backward's paths: random; one-hot at (0,0,0), whose fv0 term cancels its direct
term exactly (out[0,0,0] is constant), so every gradient must be exactly 0; all ones, which leaves only the offset
and fv0 terms because the raw field has zero mean; one-hot at a voxel the last cell's wrapped corner reaches; and
(-1)^x r(y, z) and its y / z analogues, whose spectra lie in one Nyquist plane (index G/2), the spectral adjoint's
edge bins. Each runs for forward (mode 0) and forward_signed (mode 1).

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit), max over both modes, CUDA / fp32 restatement against
float64 (the file takes ~45 s there, 5 s for each G=288 scene):

    scene                          max|out|  field              random dV          random dN          others, dV and dN
    sphere-G8-out                     0.851  2.3e-07 / 2.5e-07  3.2e-07 / 1.9e-07  4.3e-07 / 2.6e-07  9.6e-06 / 2.5e-06
    ellipsoid-G32-out                 0.693  5.5e-07 / 5.0e-07  5.4e-07 / 5.1e-07  5.5e-07 / 3.5e-07  8.5e-04 / 5.2e-05
    torus-G48-nodes-out               0.906  5.3e-07 / 4.8e-07  4.1e-07 / 4.4e-07  4.6e-07 / 3.9e-07  2.8e-05 / 3.8e-05
    sphere-G96-last-crowd-in           1.18  4.1e-07 / 5.6e-07  7.2e-07 / 4.3e-07  9.0e-07 / 4.8e-07  1.7e-03 / 4.6e-03
    torus-G288-nodes-out               1.07  5.8e-07 / 5.9e-07  4.8e-07 / 1.4e+00  4.7e-07 / 1.1e-05  1.2e-03 / 1.5e+00
    ellipsoid-G288-last-crowd-out      2.12  3.7e-07 / 4.0e-07  1.4e-06 / 3.4e-03  1.4e-06 / 5.5e-07  3.1e-03 / 1.7e-01
    N1-G32                         1.07e+04  2.9e-04 / 4.5e-04  6.5e-04 / 8.6e-04  5.9e-04 / 9.0e-04  3.8e+08 / 3.6e+08
    N8-G48                              1.6  1.7e-07 / 1.7e-07  3.9e-07 / 9.3e-07  3.9e-07 / 8.1e-07  3.8e-06 / 1.8e-05

(the mirrored copy of each scene measured the same orders of magnitude).  At G=288 the fp32 restatement loses dV: it sums
the 24M-voxel reductions in fp32, where the kernels sum in fp64, so there the absolute ceiling CEIL is what binds.
The Nyquist upstreams are ill-conditioned (in float64 too their rounding error is ~100x that of the random one), and
there the CUDA path measured up to 47x the restatement's error, while the kernels' backward algebra, restated in
float64, agrees with autograd to 1e-13 on them: the excess is fp32 rounding of FFTs that round differently, hence
K_NYQUIST.
"""
import math

import numpy as np
import pytest
import torch

import ref_dpsr
import util
from oracle.oracle import _dpsr_stencil

K = 10.0         # the CUDA path may be this many times less accurate than the fp32 restatement (measured <= 3.2)
K_NYQUIST = 100.0  # ... and on the Nyquist upstreams (measured <= 47), see the module docstring
FLOOR = 2e-6     # ... or this far off where the restatement happens to be closer still
# absolute ceiling on the oriented scenes, per upstream gradient (the field: "-"; dthres: relative to sum |g|, one
# fp32 rounding): the paths they isolate differ in conditioning by three orders of magnitude.  out[0,0,0] is a
# constant, so its one-hot has exactly zero gradients.
CEIL = {"-": 2e-6, "random": 4e-6, "ones": 1e-4, "onehot-000": 0.0, "onehot-wrap": 4e-3, "nyquist-x": 1e-2,
        "nyquist-y": 1e-2, "nyquist-z": 1e-2, "dthres": 1e-7}
COND = 3.0       # max|out| of an oriented scene (|out[0,0,0]| is 0.5); unoriented normals give ~1000
ORDER_TOL = 1e-6  # two runs of the CUDA path differ only in the order of their atomic sums
THRES = 0.05


# ----------------------------------------------------------------------------------------------- float64 reference
def _stencil64(V, G):
    """Per-axis cell i0, wrapped upper index i1 and float64 weights w0 / w1 of the nodes i0 / i1 for float64 V [n,3].

    The discrete decisions -- the cell floor(p / fp32(1/G)), the wrapped ceil and the node coordinates
    fp32(fl * fp32(1/G)) -- are taken in fp32 with IEEE division, as csrc/dpsr.cu and oracle._dpsr_stencil take them,
    and the weights in float64 from there.  So a point on a node has |p - node| = 0 exactly here too, and the kink of
    |.| gets the same zero gradient; a plain float64 stencil would move such points to another cell or flip the kink's
    side."""
    cs32 = torch.tensor(1.0 / G, dtype=torch.float32, device=V.device)  # a device tensor: a true division on CUDA
    t = V.detach().float() / cs32
    fl, ce = torch.floor(t), torch.ceil(t)
    x0, x1 = (fl * cs32).double(), ((fl + 1) * cs32).double()
    cs = float(cs32)
    return fl.long(), ce.long() % G, (V - x1).abs() / cs, (V - x0).abs() / cs   # w0: distance to the opposite corner


def _dpsr64(V, N, G, sig):
    """tests/ref_dpsr.py's DPSR.forward (the reference's algorithm) in float64 on float64 V, N [n,3] -> [G,G,G], with
    the stencil of _stencil64."""
    i0, i1, w0, w1 = _stencil64(V, G)
    corners = []
    for a in (0, 1):
        for b in (0, 1):
            for c in (0, 1):
                ix, iy, iz = (i1 if a else i0)[:, 0], (i1 if b else i0)[:, 1], (i1 if c else i0)[:, 2]
                w = (w1 if a else w0)[:, 0] * (w1 if b else w0)[:, 1] * (w1 if c else w0)[:, 2]
                corners.append(((ix * G + iy) * G + iz, w))
    ras = torch.zeros(3, G * G * G, dtype=V.dtype, device=V.device)
    for idx, w in corners:
        ras = ras.index_add(1, idx, (w[:, None] * N).t())
    ras_s = torch.fft.rfftn(ras.view(3, G, G, G), dim=(1, 2, 3))
    fx = torch.fft.fftfreq(G, d=1 / G, device=V.device, dtype=V.dtype)
    fz = torch.fft.rfftfreq(G, d=1 / G, device=V.device, dtype=V.dtype)
    om = torch.stack(torch.meshgrid(fx, fx, fz, indexing="ij"), -1)
    filt = torch.exp(-0.5 * ((sig * 2 * torch.sqrt((om ** 2).sum(-1)) / G) ** 2))
    omega = om * (2 * math.pi)
    Nf = ras_s * filt[None]
    div = sum((-1j * omega[..., c]) * Nf[c] for c in range(3))
    lap = -(omega ** 2).sum(-1)
    keep = torch.ones_like(lap)
    keep[0, 0, 0] = 0
    phi = torch.fft.irfftn(div / (lap + 1e-6) * keep, s=(G, G, G), dim=(0, 1, 2))
    flat = phi.reshape(-1)
    phi = phi - sum(flat[idx] * w for idx, w in corners).mean()
    return -phi / phi[0, 0, 0].abs() * 0.5


def _reference(V, N, G, sig):
    """fp32: tests/ref_dpsr.py itself (the reference's own expressions); float64: _dpsr64."""
    if V.dtype == torch.float32:
        return ref_dpsr.DPSR(res=(G, G, G), sig=sig)(V[None], N[None])[0]
    return _dpsr64(V, N, G, sig)


# ----------------------------------------------------------------------------------------------- scenes
def _surface(kind, n, g):
    """n points on a closed surface inside (0,1)^3 and its unit outward normals, float64."""
    f64 = torch.float64
    if kind == "sphere":
        d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=f64), dim=1)
        return 0.5 + 0.3 * d, d
    if kind == "ellipsoid":
        c, a = torch.tensor([0.45, 0.55, 0.5], dtype=f64), torch.tensor([0.32, 0.2, 0.26], dtype=f64)
        d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=f64), dim=1)
        return c + a * d, torch.nn.functional.normalize(d / a, dim=1)
    assert kind == "torus"  # genus 1: the field has a hole
    u, v = (2 * math.pi * torch.rand(2, n, generator=g, dtype=f64)).unbind(0)
    nrm = torch.stack([v.cos() * u.cos(), v.cos() * u.sin(), v.sin()], 1)
    ring = torch.stack([u.cos(), u.sin(), torch.zeros_like(u)], 1)
    return 0.5 + 0.26 * ring + 0.1 * nrm, nrm


def _scene(kind, n, G, inward, nodes=False, last=False, crowd=False, seed=0):
    """fp32 V, N [n', 3] on an oriented surface.  Normals as DG-Mesh passes them (get_normal + d_normal): scaled by
    0.5..1.5, perturbed, 3 % exactly zero.  nodes: a quarter of the points snapped to fp32(k * fp32(1/G)) on all three
    axes.  last: 64 more points in the last cell, whose upper corner wraps to index 0, a quarter of them exactly at
    the clamp bound 1 - 1e-6 on every axis and 8 at 1e-6.  crowd: 300 more points in one cell, 100 of them exact
    duplicates of a surface point."""
    g = torch.Generator().manual_seed(seed)
    P, nrm = _surface(kind, n, g)
    nrm = nrm * (0.5 + torch.rand(n, 1, generator=g, dtype=torch.float64))
    nrm = nrm + 0.1 * torch.randn(n, 3, generator=g, dtype=torch.float64)
    nrm[torch.rand(n, generator=g) < 0.03] = 0
    V, N = P.float().clamp(1e-6, 1 - 1e-6), (-nrm if inward else nrm).float()
    cs = torch.tensor(1.0 / G, dtype=torch.float32)
    if nodes:
        V[: n // 4] = torch.round(V[: n // 4] / cs) * cs
    Vs, Ns = [V], [N]
    if last:
        e = 1 - cs * torch.rand(64, 3, generator=g)
        e[:32, 0] = 1 - 1e-6
        e[:16] = 1 - 1e-6
        e[56:] = 1e-6
        Vs.append(e.clamp(1e-6, 1 - 1e-6))
        Ns.append(0.2 * torch.randn(64, 3, generator=g))
    if crowd:
        e = torch.floor(V[7] / cs) * cs + cs * torch.rand(300, 3, generator=g)
        e[:100] = V[7]
        Vs.append(e)
        Ns.append(N[7] * (0.5 + torch.rand(300, 1, generator=g)))
    return torch.cat(Vs).contiguous(), torch.cat(Ns).contiguous()


def _few(n, G, flip, seed=0):
    """n unoriented points; from n = 8 on, one on a node, two at the clamp bounds, one in the last cell and a zero
    normal."""
    g = torch.Generator().manual_seed(seed)
    V = 0.1 + 0.8 * torch.rand(n, 3, generator=g)
    N = torch.randn(n, 3, generator=g) * (0.5 + torch.rand(n, 1, generator=g))
    if n >= 8:
        cs = torch.tensor(1.0 / G, dtype=torch.float32)
        V[0] = torch.tensor([G // 3, G // 2, G - 5], dtype=torch.float32) * cs
        V[1], V[2] = 1 - 1e-6, 1e-6
        V[3] = 1 - cs * torch.rand(3, generator=g)
        N[4] = 0
    return V, (-N if flip else N)


# id -> (G, sig, scene builder, oriented)
ORIENTED = [
    ("sphere-G8", 8, 2.0, dict(kind="sphere", n=2000)),
    ("ellipsoid-G32", 32, 3.0, dict(kind="ellipsoid", n=20_000)),
    ("torus-G48-nodes", 48, 2.0, dict(kind="torus", n=20_000, nodes=True)),
    ("sphere-G96-last-crowd", 96, 3.0, dict(kind="sphere", n=50_000, last=True, crowd=True)),
    ("torus-G288-nodes", 288, 3.0, dict(kind="torus", n=200_000, nodes=True)),   # DG-Mesh: 288^3, ~200k, sig 3
    ("ellipsoid-G288-last-crowd", 288, 2.0, dict(kind="ellipsoid", n=200_000, last=True, crowd=True)),
]
FEW = [("N1-G32", 32, 3.0, 1), ("N8-G48", 48, 2.0, 8)]

CASES = {}
for _id, _G, _sig, _kw in ORIENTED:
    for _inward in (False, True):
        CASES[f"{_id}-{'in' if _inward else 'out'}"] = (
            _G, _sig, (lambda G=_G, kw=_kw, inward=_inward: _scene(G=G, inward=inward, **kw)), True)
for _id, _G, _sig, _n in FEW:
    for _flip in (False, True):
        CASES[f"{_id}{'-flipped' if _flip else ''}"] = (
            _G, _sig, (lambda G=_G, n=_n, flip=_flip: _few(n, G, flip)), False)


def _upstreams(G, seed=11):
    """name -> dL/dout [G,G,G] fp32 (CPU), built one at a time; the float64 reference gets the same values."""
    g = torch.Generator().manual_seed(seed)
    alt = (-1.0) ** torch.arange(G, dtype=torch.float32)

    def onehot(ix):
        t = torch.zeros(G, G, G)
        t[ix] = 1
        return t

    yield "random", torch.randn(G, G, G, generator=g)
    yield "onehot-000", onehot((0, 0, 0))
    yield "ones", torch.ones(G, G, G)
    yield "onehot-wrap", onehot((G - 1, 0, G - 1))     # a corner the last cell's wrapped stencil reaches
    r = torch.randn(3, G, G, generator=g)
    yield "nyquist-x", alt[:, None, None] * r[0][None]
    yield "nyquist-y", alt[None, :, None] * r[1][:, None, :]
    yield "nyquist-z", alt[None, None, :] * r[2][:, :, None]


# ----------------------------------------------------------------------------------------------- the three paths
def _cuda(V, N, G, sig, mode, dev="cuda"):
    from nvdiffrast_utils.dpsr import DPSR
    v, n = V.to(dev).clone().requires_grad_(True), N.to(dev).clone().requires_grad_(True)
    m = DPSR(res=(G, G, G), sig=sig)
    if mode == 0:
        return m(v[None], n[None])[0], [v, n]
    th = torch.full((1,), THRES, device=dev, requires_grad=True)
    return m.forward_signed(v[None], n[None], th), [v, n, th]


def _ref(V, N, G, sig, mode, dtype, dev):
    """the restatement; mode 1 adds mesh_renderer's glue psr * sign(psr[0,0,0]) - thres (utils/renderer.py)."""
    v = V.to(dev, dtype).clone().requires_grad_(True)
    n = N.to(dev, dtype).clone().requires_grad_(True)
    psr = _reference(v, n, G, sig)
    if mode == 0:
        return psr, [v, n]
    th = torch.full((1,), THRES, dtype=dtype, device=dev, requires_grad=True)
    sign = -1 if psr[0, 0, 0].detach() < 0 else 1
    return psr * sign - th, [v, n, th]


def _grads(out, leaves, g):
    for x in leaves:
        x.grad = None
    out.backward(g.to(out.device, out.dtype), retain_graph=True)
    return [x.grad.detach().clone() for x in leaves]


NAMES = ("dV", "dN", "dthres")


def _compare(V, N, G, sig):
    """rows (mode, upstream, output, CUDA error, fp32 error) against float64, and max|out| of the float64 field.
    dthres = -sum g is 0 for the Nyquist upstreams, so its error is taken relative to sum |g| instead."""
    rows, peak = [], 0.0
    for mode in (0, 1):
        c = _cuda(V, N, G, sig, mode)
        r32 = _ref(V, N, G, sig, mode, torch.float32, "cuda")
        r64 = _ref(V, N, G, sig, mode, torch.float64, "cuda")
        if mode == 0:
            peak = float(r64[0].detach().abs().max())
        rows.append((mode, "-", "out", util.rel_err(c[0], r64[0]), util.rel_err(r32[0], r64[0])))
        for name, g in _upstreams(G):
            gc, g32, g64 = (_grads(*x, g) for x in (c, r32, r64))
            for k in range(len(gc)):
                if k < 2:
                    e, e32 = util.rel_err(gc[k], g64[k]), util.rel_err(g32[k], g64[k])
                else:
                    assert gc[2].shape == (1,)
                    s = float(g.double().abs().sum())
                    e, e32 = (float((x.double() - g64[2]).abs().max()) / s for x in (gc[2], g32[2]))
                rows.append((mode, name, NAMES[k], e, e32))
        del c, r32, r64
    return rows, peak


def _table(rows):
    return "\n".join(f"mode {m} {u:12s} {o:7s} cuda {e:.2e}  fp32 {e32:.2e}" for m, u, o, e, e32 in rows)


# ----------------------------------------------------------------------------------------------- CPU: the reference
def test_float64_reference_reproduces_golden_cpu():
    """The fp32 restatement reproduces the reference's stored field and gradients, and the float64 reference agrees
    with them to the golden's own fp32 rounding."""
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "dpsr_g32.npz"))
    for dtype, tol in ((torch.float32, 1e-5), (torch.float64, 2e-6)):
        V = torch.from_numpy(z["V"]).to(dtype).requires_grad_(True)
        N = torch.from_numpy(z["N"]).to(dtype).requires_grad_(True)
        phi = _reference(V, N, 32, float(z["sig"]))
        assert phi.dtype == dtype
        (phi * torch.from_numpy(z["gout"]).to(dtype)).sum().backward()
        errs = [util.rel_err(a, z[k]) for a, k in ((phi.detach(), "phi"), (V.grad, "dV"), (N.grad, "dN"))]
        assert max(errs) < tol, (dtype, errs)


@pytest.mark.parametrize("G", [8, 48, 96, 288])
def test_float64_stencil_takes_the_fp32_decisions_cpu(G):
    """The float64 stencil puts every point in the cell the fp32 oracle (and csrc/dpsr.cu) puts it in, with the same
    wrapped upper index, and gives the weights the fp32 ones round from; a weight is exactly zero, and its kink
    gradient zero, exactly where the fp32 one is: points on nodes of all three axes, at the clamp bounds, in the
    last cell and anywhere."""
    g = torch.Generator().manual_seed(G)
    cs = torch.tensor(1.0 / G, dtype=torch.float32)
    V = torch.cat([torch.arange(G, dtype=torch.float32)[:, None].expand(G, 3) * cs,            # every node
                   torch.randint(0, G, (200, 3), generator=g).float() * cs,
                   torch.tensor([[1 - 1e-6] * 3, [1e-6] * 3, [1e-6, 0.5, 1 - 1e-6]]),
                   1 - cs * torch.rand(50, 3, generator=g),
                   torch.rand(500, 3, generator=g)]).clamp(1e-6, 1 - 1e-6)
    i0, i1, w0, w1 = _dpsr_stencil(V.numpy(), G)
    assert (i1 == 0).any() and (w1 == 0).any()
    v = V.double().requires_grad_(True)
    j0, j1, u0, u1 = _stencil64(v, G)
    assert u0.dtype == torch.float64
    assert np.array_equal(j0.numpy(), i0) and np.array_equal(j1.numpy(), i1)
    for u, w in ((u0, w0), (u1, w1)):
        assert np.array_equal(u.detach().numpy() == 0, w == 0)
        assert np.abs(u.detach().numpy() - w).max() < 1e-6
        (d,) = torch.autograd.grad(u.sum(), v)
        assert np.array_equal(d.numpy() == 0, w == 0)


@pytest.mark.parametrize("mode", [0, 1])
def test_float64_gradients_match_central_differences_cpu(mode):
    """dV, dN (and dthres) of the float64 reference are the derivatives of its own forward, for points kept 0.1 cell
    away from cell boundaries so that a step of h does not cross a kink."""
    G, n, h = 8, 12, 1e-6
    g = torch.Generator().manual_seed(5)
    cell = torch.randint(1, G - 1, (n, 3), generator=g).double()
    V = ((cell + 0.1 + 0.8 * torch.rand(n, 3, generator=g, dtype=torch.float64)) / G).float().double()
    N = torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.7
    up = torch.randn(G, G, G, generator=g, dtype=torch.float64)

    def loss(v, nn_, th):
        psr = _dpsr64(v, nn_, G, 2.0)
        out = psr if mode == 0 else psr * (-1 if psr[0, 0, 0].detach() < 0 else 1) - th
        return (out * up).sum()

    leaves = [V.clone().requires_grad_(True), N.clone().requires_grad_(True),
              torch.full((1,), THRES, dtype=torch.float64, requires_grad=True)]
    grads = torch.autograd.grad(loss(*leaves), leaves, allow_unused=True)
    for k, (x, ad) in enumerate(zip(leaves, grads)):
        if ad is None:
            assert mode == 0 and k == 2
            continue
        fd = torch.zeros_like(x)
        for i in range(x.numel()):
            xs = [y.detach().clone() for y in leaves]
            xs[k].view(-1)[i] += h
            lp = loss(*xs)
            xs[k].view(-1)[i] -= 2 * h
            fd.view(-1)[i] = (lp - loss(*xs)) / (2 * h)
        assert util.rel_err(ad, fd) < 1e-6, (NAMES[k], util.rel_err(ad, fd))


@pytest.mark.parametrize("case", [k for k, v in CASES.items() if v[3]])
def test_scenes_are_well_conditioned_cpu(case):
    """The oriented scenes keep max|out| near 0.5 (checked here at G <= 96, and at the full grid on the GPU)."""
    G, sig, build, _ = CASES[case]
    V, N = build()
    G = min(G, 96)
    out = _dpsr64(V.double(), N.double(), G, sig)
    assert float(out[0, 0, 0].abs()) == pytest.approx(0.5)
    assert float(out.abs().max()) < COND


# ----------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_cuda_dpsr_within_fp32_budget_of_float64(case):
    G, sig, build, oriented = CASES[case]
    V, N = build()
    rows, peak = _compare(V, N, G, sig)
    print(f"\n{case}: max|out| {peak:.3f}\n{_table(rows)}")
    bad = [r for r in rows if r[3] > max((K_NYQUIST if r[1].startswith("nyquist") else K) * r[4], FLOOR)
           or (oriented and r[3] > CEIL["dthres" if r[2] == "dthres" else r[1]])]
    assert not bad, f"{case}: over budget\n{_table(bad)}"
    if oriented:
        assert peak < COND, peak


def _run_cuda(V, N, G, sig, mode, g):
    out, leaves = _cuda(V, N, G, sig, mode)
    return [out.detach().clone()] + _grads(out, leaves, g)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_cuda_dpsr_on_a_side_stream(mode):
    """The same inputs give the same field and gradients on the default stream and on a side stream whose inputs
    are written after a delay on that stream: the library enqueues everything on the caller's stream."""
    G, sig = 48, 2.0
    V, N = _scene("torus", 20_000, G, False, nodes=True)
    g = next(_upstreams(G))[1].cuda()
    base = _run_cuda(V, N, G, sig, mode, g)
    Vd, Nd = V.cuda(), N.cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        side = _run_cuda(Vd * 1, Nd * 1, G, sig, mode, g)
    torch.cuda.current_stream().wait_stream(s)
    for a, b in zip(side, base):
        assert util.rel_err(a, b) < ORDER_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_cuda_dpsr_repeated_backward(mode):
    """Two backward passes of one forward give the same gradients: the backward reads the forward's workspace
    (phi_raw, offset, fv0) and must not overwrite it."""
    G, sig = 48, 2.0
    V, N = _scene("ellipsoid", 20_000, G, True, last=True)
    out, leaves = _cuda(V, N, G, sig, mode)
    for name, g in _upstreams(G):
        first = _grads(out, leaves, g)
        second = _grads(out, leaves, g)
        for a, b in zip(first, second):
            assert util.rel_err(a, b) < ORDER_TOL, name


@pytest.mark.gpu
def test_cuda_dpsr_two_grids_interleaved():
    """Two DPSR modules with different G: forwards interleaved, backwards in reverse order, each equal to the same
    grid run on its own (the cuFFT plans are cached per grid)."""
    V, N = _scene("sphere", 20_000, 48, False, nodes=True)
    alone = {G: _run_cuda(V, N, G, 3.0, 0, next(_upstreams(G))[1].cuda()) for G in (32, 48)}
    runs = {G: _cuda(V, N, G, 3.0, 0) for G in (32, 48)}
    for G in (48, 32):
        out, leaves = runs[G]
        got = [out.detach()] + _grads(out, leaves, next(_upstreams(G))[1].cuda())
        for a, b in zip(got, alone[G]):
            assert util.rel_err(a, b) < ORDER_TOL, G
