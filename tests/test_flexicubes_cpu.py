"""FlexiCubes without a GPU: the float64 oracle (tests/flexicubes_oracle.py) against dual marching cubes' exact
reference with neutral weights, its gradients against central differences, closed training-mode meshes, and the
host refusals of the C-ABI and of FlexiCubes."""
import numpy as np
import pytest
import torch

from dmc_reference import dmc_reference
from flexicubes_oracle import flexicubes
from test_dmc_cpu import FIELDS, D, _err, _lib, torus
from test_mc_reference import smooth_noise, sphere


@pytest.mark.parametrize("name,phi,iso", FIELDS, ids=[f[0] for f in FIELDS])
def test_oracle_neutral_equals_dual_marching_cubes(name, phi, iso):
    ref = dmc_reference(phi, iso)
    for training in (False, True):
        o = flexicubes(torch.from_numpy(phi), iso=iso, training=training)
        V = len(ref.verts)
        assert np.allclose(o.verts[:V].numpy(), ref.verts, rtol=0, atol=4e-7), name
        if not training:
            assert np.array_equal(o.faces, ref.faces.reshape(2, -1, 3).transpose(1, 0, 2).reshape(-1, 3))
        else:
            assert o.verts.shape == (V + len(ref.quads), 3) and o.faces.shape == (4 * len(ref.quads), 3)


def _inputs(G, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    c = (G - 1,) * 3
    return dict(deform=0.3 * torch.tanh(torch.randn(G, G, G, 3, generator=g, dtype=dtype)),
                beta=torch.randn(*c, 12, generator=g, dtype=dtype), alpha=torch.randn(*c, 8, generator=g, dtype=dtype),
                gamma_f=torch.randn(*c, generator=g, dtype=dtype))


def _loss(o):
    w = torch.tensor([3.1, -2.3, 4.7], dtype=torch.float64)
    return torch.sin(o.verts * w + 0.3).sum() + torch.sin(5.0 * o.L_dev + 0.2).sum()


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("normalize", [True, False])
def test_oracle_gradients_central_differences(training, normalize):
    G, iso = 12, 0.05
    phi = torch.from_numpy(smooth_noise(G, 4)).double()
    ins = _inputs(G, 1)
    dmc = dmc_reference(phi.float().numpy(), iso)
    names = ["phi"] + list(ins)
    leaves = {"phi": phi.clone().requires_grad_(True), **{n: t.clone().requires_grad_(True) for n, t in ins.items()}}

    def run(vals):
        return _loss(flexicubes(vals["phi"], vals["deform"], vals["beta"], vals["alpha"], vals["gamma_f"], iso,
                                training, normalize, dmc=dmc))

    run(leaves).backward()
    g = torch.Generator().manual_seed(2)
    for n in names:
        if n == "gamma_f" and not training:
            assert leaves[n].grad is None or not leaves[n].grad.any()
            continue
        grad = leaves[n].grad
        assert grad is not None and grad.abs().sum() > 0, n
        for _ in range(3):
            dirn = torch.randn(leaves[n].shape, generator=g, dtype=torch.float64)
            if n == "phi":   # keep every sign: the topology is fixed under the perturbation
                dirn = dirn * (phi.abs() > 1e-3)
            eps = 1e-6
            vals = {m: t.detach() for m, t in leaves.items()}
            hi = run({**vals, n: vals[n] + eps * dirn})
            lo = run({**vals, n: vals[n] - eps * dirn})
            fd, an = float((hi - lo) / (2 * eps)), float((grad * dirn).sum())
            assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (n, fd, an)


def _closed(faces, nv):
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    return np.array_equal(np.sort(d[:, 0] * nv + d[:, 1]), np.sort(d[:, 1] * nv + d[:, 0]))


@pytest.mark.parametrize("kind", ["sphere", "torus"])
def test_training_mesh_is_closed(kind):
    G = 24
    phi = sphere(G) if kind == "sphere" else torus(G)
    ins = _inputs(G, 3)
    for training in (False, True):
        o = flexicubes(torch.from_numpy(phi), **ins, training=training)
        assert len(o.faces) > 100 and _closed(o.faces, len(o.verts)), (kind, training)
        used = np.zeros(len(o.verts), bool)
        used[o.faces.ravel()] = True
        assert used.all()


# ----------------------------------------------------------------------------- C-ABI and Python refusals
def test_abi_signatures():
    import _dgm_lib
    lib = _lib()
    for name in ("dgfc_emit", "dgfc_backward_workspace_size", "dgfc_backward"):
        restype, args = _dgm_lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args, name


def test_abi_refusals():
    import _dgm_lib
    lib = _lib()
    n = _dgm_lib.c_size_t()
    W = 1 << 40

    def emit(G=64, phi=D, training=0, ws_bytes=W, verts=D, ldev=D, vcap=16, faces=D, quads=D, qcap=16):
        return lib.dgfc_emit(G, phi, 0.0, None, None, None, None, training, 1, D, ws_bytes, verts, D, ldev, D, vcap,
                             faces, quads, qcap, None)

    for G in (1, 801):
        _err(lib, emit(G=G), b"dgfc_emit", b"G")
    _err(lib, emit(phi=None), b"null grid")
    for vcap, qcap in ((1 << 28) + 1, 16), (-1, 16), (16, 1 << 30), (16, -1):
        _err(lib, emit(vcap=vcap, qcap=qcap), b"capacity")
    _err(lib, emit(training=1, qcap=1 << 29), b"capacity")            # V + Q and 4 Q must fit int32
    _err(lib, emit(ldev=None), b"null output")
    _err(lib, emit(quads=None), b"null output")
    lib.dgdmc_workspace_size(64, n)
    assert emit(ws_bytes=n.value - 1) == -2 and b"workspace too small" in lib.dgm_last_error()

    for G, V, Q, tr in ((1, 0, 0, 0), (801, 0, 0, 0), (8, 4 * 7 ** 3 + 1, 0, 0), (8, -1, 0, 0),
                        (8, 4, 3 * 64 * 7 + 1, 0), (800, (1 << 28) + 1, 0, 0)):
        _err(lib, lib.dgfc_backward_workspace_size(G, V, Q, tr, n), b"dgfc_backward_workspace_size")
    _err(lib, lib.dgfc_backward_workspace_size(8, 4, 4, 0, None), b"null")
    lib.dgfc_backward_workspace_size(8, 5, 5, 1, n)

    def bwd(G=8, V=5, Q=5, phi=D, deform=None, alpha=None, gamma=None, training=1, verts=D, vsrc=D, quads=D,
            ws_bytes=W, dphi=D, ddeform=None, dalpha=None, dgamma=None):
        return lib.dgfc_backward(G, V, Q, phi, 0.0, deform, alpha, None, gamma, training, 1, verts, vsrc, quads, D,
                                 None, D, ws_bytes, dphi, ddeform, dalpha, None, dgamma, None)

    _err(lib, bwd(V=-1), b"V or Q out of range")
    _err(lib, bwd(phi=None), b"null grid")
    _err(lib, bwd(dphi=None), b"dL_dphi")
    _err(lib, bwd(ddeform=D), b"dL_ddeform without deform")
    _err(lib, bwd(dalpha=D), b"null weight")
    _err(lib, bwd(dgamma=D), b"null weight")
    _err(lib, bwd(gamma=D, dgamma=D, training=0), b"training mode")
    _err(lib, bwd(vsrc=None), b"null")
    _err(lib, bwd(verts=None), b"null")
    _err(lib, bwd(quads=None), b"null")
    assert bwd(ws_bytes=n.value - 1) == -2 and b"workspace too small" in lib.dgm_last_error()


def test_python_refusals():
    from flexicubes import FlexiCubes
    m = FlexiCubes()
    g = torch.zeros(8, 8, 8)
    with pytest.raises(ValueError, match="CUDA"):
        m(g)
    with pytest.raises(ValueError, match="cubic"):
        m(torch.zeros(8, 8, 7))
    with pytest.raises(ValueError, match="float32"):
        m(g.double())
    with pytest.raises(ValueError, match="G <= 800"):
        m(torch.zeros(1, 1, 1))
    for name, shape in (("deform", (8, 8, 8, 2)), ("beta", (7, 7, 7, 8)), ("alpha", (7, 7, 7, 12)),
                        ("gamma_f", (8, 8, 8))):
        with pytest.raises(ValueError, match=name):
            m(g, **{name: torch.zeros(shape)})
        with pytest.raises(ValueError, match=name):
            good = {"deform": (8, 8, 8, 3), "beta": (7, 7, 7, 12), "alpha": (7, 7, 7, 8), "gamma_f": (7, 7, 7)}
            m(g, **{name: torch.zeros(good[name], dtype=torch.float64)})
