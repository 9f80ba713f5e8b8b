"""FlexiCubes on the GPU against DiffDMC (neutral weights) and against the float64 oracle (tests/flexicubes_oracle.py).

Vertices are matched to the oracle's by (cell, patch): the GPU's vertex order is DiffDMC's, so a neutral call, whose
vertices equal dmc_reference's bit for bit, gives the permutation; a training-mode call gives the quad order.
Bounds (worst measured on an H100 in DESIGN.md §4): vertices and L_dev 1e-5 of the grid extent, gradients 1e-3 of
the largest oracle gradient of each input, with the L_dev entries that lie at |d_e - mean| = 0 to float32 rounding
left out of the gradient comparison."""
import numpy as np
import pytest
import torch

from dmc_reference import dmc_reference
from flexicubes_oracle import flexicubes as oracle
from mc_reference import LOSS_P, LOSS_W
from test_dmc_cpu import torus
from test_mc_reference import noise, smooth_noise, sphere

pytestmark = pytest.mark.gpu

NAMES = ("phi", "deform", "beta", "alpha", "gamma_f")
TOL_V, TOL_L, TOL_G = 1e-5, 1e-5, 1e-3


def _field(kind, G):
    return {"sphere": lambda: sphere(G), "torus": lambda: torus(G), "noise": lambda: noise(G, 3),
            "smooth": lambda: smooth_noise(G, 5)}[kind]()


def _inputs(G, seed):
    g = torch.Generator().manual_seed(seed)
    c = (G - 1,) * 3
    return {"deform": 0.3 * torch.tanh(torch.randn(G, G, G, 3, generator=g)), "beta": torch.randn(*c, 12, generator=g),
            "alpha": torch.randn(*c, 8, generator=g), "gamma_f": torch.randn(*c, generator=g)}


def _loss(verts, L_dev, lw=None):
    """An order-independent smooth loss; lw [len(L_dev)] weighs the L_dev terms (1 when None)."""
    w = torch.tensor(LOSS_W, dtype=torch.float64, device=verts.device)
    p = torch.tensor(LOSS_P, dtype=torch.float64, device=verts.device)
    ld = torch.sin(5.0 * L_dev.double() + 0.2)
    return torch.sin(verts.double() * w + p).sum() + (ld if lw is None else ld * lw.to(ld.device)).sum()


def _gpu(phi, ins=None, iso=0.0, training=False, normalize=True, grad=True, lw=None):
    from flexicubes import FlexiCubes
    leaves = {"phi": torch.from_numpy(np.ascontiguousarray(phi)).cuda()}
    leaves.update({n: t.cuda() for n, t in (ins or {}).items()})
    for t in leaves.values():
        t.requires_grad_(grad)
    v, f, L = FlexiCubes()(leaves["phi"], leaves.get("deform"), leaves.get("beta"), leaves.get("alpha"),
                           leaves.get("gamma_f"), isovalue=iso, training=training, normalize=normalize)
    assert f.dtype == torch.int64 and v.dtype == torch.float32
    grads = {}
    if grad:
        _loss(v, L, None if lw is None else lw(L)).backward()
        grads = {n: (None if t.grad is None else t.grad.cpu().double()) for n, t in leaves.items()}
    return v.detach().cpu(), f.cpu().numpy(), L.detach().cpu(), grads


def _perm(v_neutral, ref_verts):
    """GPU row -> dmc_reference row, from bit-identical neutral vertices (which must be distinct)."""
    a = np.ascontiguousarray(v_neutral, np.float32).view(np.uint32).astype(np.int64)
    b = np.ascontiguousarray(ref_verts, np.float32).view(np.uint32).astype(np.int64)
    assert a.shape == b.shape
    oa, ob = np.lexsort(a.T[::-1]), np.lexsort(b.T[::-1])
    assert np.array_equal(a[oa], b[ob]), "neutral vertices differ from dmc_reference's"
    assert (np.diff(b[ob], axis=0) != 0).any(1).all(), "duplicate vertices: no unique (cell, patch) match"
    perm = np.empty(len(a), np.int64)
    perm[oa] = ob
    return perm


@pytest.mark.parametrize("G", [32, 64, 288])
@pytest.mark.parametrize("kind", ["sphere", "torus", "noise"])
def test_neutral_equals_diffdmc(kind, G):
    from diso import DiffDMC
    phi = _field(kind, G)
    p = torch.from_numpy(phi).cuda().requires_grad_(True)
    vd, fd = DiffDMC()(p)
    w, ph = torch.tensor(LOSS_W, device="cuda"), torch.tensor(LOSS_P, device="cuda")
    torch.sin(vd.double() * w + ph).sum().backward()
    from flexicubes import FlexiCubes
    q = torch.from_numpy(phi).cuda().requires_grad_(True)
    v, f, L = FlexiCubes()(q)
    torch.sin(v.double() * w + ph).sum().backward()
    assert torch.equal(v.view(torch.int32), vd.view(torch.int32)) and torch.equal(f, fd)
    err = float((q.grad - p.grad).abs().max() / p.grad.abs().max())
    print(f"neutral {kind} G={G}: V={len(v)}, dphi rel err vs DiffDMC {err:.2e}")
    assert err <= 1e-5


def _compare(phi, ins, training, iso=0.0, normalize=True, grad=True):
    G = phi.shape[0]
    ref = dmc_reference(phi, iso)
    V = len(ref.verts)
    from diso import DiffDMC
    with torch.no_grad():   # FlexiCubes' vertex order is DiffDMC's, whose vertices are dmc_reference's at any iso
        vn, _ = DiffDMC()(torch.from_numpy(phi).cuda(), isovalue=iso)
    perm = _perm(vn.cpu().numpy(), ref.verts)
    o = oracle(*(t.double() for t in [torch.from_numpy(phi)] + [ins[n] for n in ("deform", "beta", "alpha", "gamma_f")]),
               iso, training, normalize, dmc=ref)
    ko = np.concatenate([[0], np.cumsum(o.k)])
    idx = np.concatenate([np.arange(ko[r], ko[r + 1]) for r in perm]) if V else np.zeros(0, np.int64)
    # |d_e - mean| is not differentiable at 0: entries within 1e-6 of the grid extent of it are left out of the
    # gradient comparison, where float32 and float64 may take different sides
    keep = (o.L_dev > 1e-6 * (1.0 if normalize else G - 1.0)).double()
    v, f, L, grads = _gpu(phi, ins, iso, training, normalize, grad, lw=lambda L: keep[idx])
    leaves = {"phi": torch.from_numpy(phi).double().requires_grad_(grad)}
    leaves.update({n: t.double().requires_grad_(grad) for n, t in ins.items()})
    o = oracle(leaves["phi"], leaves["deform"], leaves["beta"], leaves["alpha"], leaves["gamma_f"], iso, training,
               normalize, dmc=ref)
    scale = 1.0 if normalize else G - 1.0
    # vertices and quads in the oracle's rows
    if training:
        Q = len(ref.quads)
        gq = perm[f.reshape(-1, 4, 3)[:, :, 0]]                            # quad q's corners, in oracle rows
        key = {tuple(r): i for i, r in enumerate(ref.quads.tolist())}
        qmap = np.array([key[tuple(r)] for r in gq.tolist()], np.int64)
        full = np.concatenate([perm, V + qmap])
        assert np.array_equal(full[f], o.faces.reshape(-1, 4, 3)[qmap].reshape(-1, 3))
    else:
        full = perm
        _, ft, _, _ = _gpu(phi, iso=iso, training=True, grad=False)
        gq = perm[ft.reshape(-1, 4, 3)[:, :, 0]]
        key = {tuple(r): i for i, r in enumerate(ref.quads.tolist())}
        qmap = np.array([key[tuple(r)] for r in gq.tolist()], np.int64)
        got = full[f].reshape(-1, 2, 3)
        want = o.faces.reshape(-1, 2, 3)[qmap]
        bad = (got != want).any((1, 2)) & ~o.near_tie[qmap]
        assert not bad.any(), f"{int(bad.sum())} quads split differently"
    assert v.shape == o.verts.shape
    e_v = float((v.double() - o.verts.detach()[full]).abs().max()) / scale if len(v) else 0.0
    e_l = float((L.double() - o.L_dev.detach()[idx]).abs().max()) / scale if len(L) else 0.0
    errs = {}
    if grad:
        _loss(o.verts, o.L_dev, keep).backward()
        for n in ("phi",) + tuple(ins):
            r = leaves[n].grad
            if n == "gamma_f" and not training:
                assert grads[n] is None or not grads[n].any()
                continue
            errs[n] = float((grads[n] - r).abs().max() / r.abs().max())
    print(f"G={G} training={training}: V={V}, vertex err {e_v:.2e}, L_dev err {e_l:.2e}, grad rel err "
          + ", ".join(f"{n} {e:.2e}" for n, e in errs.items()))
    assert e_v <= TOL_V and e_l <= TOL_L
    for n, e in errs.items():
        assert e <= TOL_G, (n, e)


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("kind,G", [("sphere", 32), ("torus", 48), ("smooth", 64)])
def test_random_weights_against_oracle(kind, G, training):
    _compare(_field(kind, G), _inputs(G, G), training)


@pytest.mark.parametrize("training", [False, True])
def test_random_weights_at_an_isovalue_without_normalisation(training):
    _compare(smooth_noise(40, 7), _inputs(40, 2), training, iso=0.1, normalize=False)


@pytest.mark.parametrize("training", [False, True])
def test_smooth_field_forward_at_training_size(training):
    G = 288
    phi = smooth_noise(G, 11)
    _compare(phi, _inputs(G, 9), training, grad=False)


@pytest.mark.parametrize("training", [False, True])
def test_backward_is_deterministic(training):
    G = 288
    phi = smooth_noise(G, 11)
    ins = _inputs(G, 4)
    a = _gpu(phi, ins, training=training)[3]
    b = _gpu(phi, ins, training=training)[3]
    for n in NAMES:
        if a[n] is None:
            assert b[n] is None and n == "gamma_f" and not training
            continue
        assert torch.equal(a[n].float().view(torch.int32), b[n].float().view(torch.int32)), n


@pytest.mark.parametrize("training", [False, True])
def test_adam_steps_reduce_chamfer(training):
    from flexicubes import FlexiCubes
    from metrics.pytorch_structural_losses.nn_distance import nn_distance
    G = 32
    torch.manual_seed(0)
    phi = torch.from_numpy(sphere(G, 0.5)).cuda().requires_grad_(True)
    params = [phi] + [t.cuda().mul_(0.0).requires_grad_(True) for t in _inputs(G, 1).values()]
    d = torch.nn.functional.normalize(torch.randn(4000, 3), dim=1)
    target = (0.5 + d * torch.tensor([0.32, 0.22, 0.27])).cuda()[None]      # an ellipsoid in [0,1]^3
    opt = torch.optim.Adam(params, lr=1e-2)
    losses = []
    for _ in range(30):
        v, f, L = FlexiCubes()(params[0], params[1], params[2], params[3], params[4], training=training)
        d1, d2 = nn_distance(v[None], target)
        loss = d1.mean() + d2.mean() + 0.1 * L.mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(d1.mean() + d2.mean()))
    print(f"training={training}: chamfer {losses[0]:.3e} -> {losses[-1]:.3e}")
    assert losses[-1] < 0.8 * losses[0]
