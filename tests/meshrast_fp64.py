"""TEST INFRASTRUCTURE: a fast float64 restatement of the mesh rasterisation contract (csrc/meshrast.cu), for
images and meshes of the size DG-Mesh renders (800x800, 1e4-1e5 marching-cubes triangles).

oracle/meshrast_oracle.py states the same contract with loops (one full-image pass per triangle, one Python
iteration per antialias pixel pair); it stays the readable reference and tests/test_meshrast_fp64.py pins these
functions to it.  Here:

  * `rasterize` walks every triangle's own bounding box (the kernel's bbox formula), all triangles of similar bbox
    size at once, and resolves the nearest (z/w, id) per pixel by sorting.  Besides the ids it returns, for every
    pixel, whether float64 decides it with a MARGIN: the kernel evaluates the same decisions in fp32, so a pixel
    centre closer than `tau` px to an edge of a competing triangle, or two depths closer than `tau_z`, may go either
    way.  `admissible` checks that a kernel's choice is one of the ways float64 allows within those tolerances.
  * `rast` evaluates (u, v, z/w) on given ids (the kernel's), differentiable w.r.t. pos through per-pixel copies of
    the three clip-space vertices, so that each pixel's own contribution to a vertex gradient can be read.
  * `aa_pairs` finds the pixel pairs with different ids by array ops and evaluates the three candidate edges of
    each; `antialias` applies the first valid one (or the edge a kernel chose, `k=` / `branch=`), differentiable w.r.t.
    colour and pos the same way.

Tolerances come from fp32 rounding: a pixel-space coordinate s = (x / w * 0.5 + 0.5) W is rounded a few times at
its own magnitude, so a vertex is off by ~3 u with u = 2^-24 max(|s|, W, H) (unit roundoff at the coordinate
magnitude), and an edge function's products at the bbox extent e add 2^-23 e per unit edge length.  TAU_SAFETY
multiplies that estimate."""
import torch

U32 = 2.0 ** -24          # fp32 unit roundoff
TAU_SAFETY = 4.0          # estimate -> tolerance


def _edge(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def project(pos, W, H):
    """[V,4] clip -> [V,4] (px, py, z/w, 1/w), 1/w = -1 where w <= 0 (the kernel's 'behind the eye' mark)."""
    pos = pos.double()
    w = pos[:, 3]
    iw = torch.where(w > 0, 1.0 / torch.where(w > 0, w, torch.ones_like(w)), torch.full_like(w, -1.0))
    return torch.stack([(pos[:, 0] * iw * 0.5 + 0.5) * W, (pos[:, 1] * iw * 0.5 + 0.5) * H, pos[:, 2] * iw, iw], -1)


def _tri_geometry(s, tri, W, H):
    """Per-triangle quantities of the coverage test: vertices, doubled signed area, edge lengths (edge k joins
    vertices k+1 and k+2, i.e. it is the one b_k measures the distance to), bbox, drawn flag and tolerances."""
    a, b, c = s[tri[:, 0]], s[tri[:, 1]], s[tri[:, 2]]
    area = _edge(a[:, 0], a[:, 1], b[:, 0], b[:, 1], c[:, 0], c[:, 1])
    drawn = (a[:, 3] > 0) & (b[:, 3] > 0) & (c[:, 3] > 0) & (area != 0) & torch.isfinite(area)
    X = torch.stack([a[:, 0], b[:, 0], c[:, 0]], 1)
    Y = torch.stack([a[:, 1], b[:, 1], c[:, 1]], 1)
    big = float(max(W, H) + 2)
    x0 = torch.floor((X.min(1).values - 0.5).clamp(-2, big)).long().clamp_min(0)
    x1 = torch.ceil((X.max(1).values - 0.5).clamp(-2, big)).long().clamp_max(W - 1)
    y0 = torch.floor((Y.min(1).values - 0.5).clamp(-2, big)).long().clamp_min(0)
    y1 = torch.ceil((Y.max(1).values - 0.5).clamp(-2, big)).long().clamp_max(H - 1)
    drawn &= (x1 >= x0) & (y1 >= y0)
    L = torch.stack([torch.hypot(c[:, 0] - b[:, 0], c[:, 1] - b[:, 1]), torch.hypot(a[:, 0] - c[:, 0], a[:, 1] - c[:, 1]),
                     torch.hypot(b[:, 0] - a[:, 0], b[:, 1] - a[:, 1])], 1)
    mag = torch.maximum(X.abs().max(1).values, Y.abs().max(1).values).clamp_min(float(max(W, H)))
    mag = torch.where(torch.isfinite(mag), mag, torch.full_like(mag, float("inf")))
    ext = torch.maximum(X.max(1).values - X.min(1).values, Y.max(1).values - Y.min(1).values)
    # distance error of edge k at a pixel centre: both end points (3 u each) and the two products (2^-23 e);
    # b2 = 1 - b0 - b1 inherits the errors of b0 and b1, i.e. (L0 + L1) / L2 times theirs
    base = TAU_SAFETY * (6.0 * U32 * mag + 2.0 * U32 * ext)
    Ls = L.clamp_min(1e-300)
    tau = base[:, None] * torch.stack([torch.ones_like(area), torch.ones_like(area), 1.0 + (L[:, 0] + L[:, 1]) / Ls[:, 2]], 1)
    # the sign of the area itself is in doubt for a triangle flatter than its tolerance: every decision is
    height = area.abs() / Ls.max(1).values
    flat = height <= base
    return dict(a=a, b=b, c=c, area=area, drawn=drawn, x0=x0, x1=x1, y0=y0, y1=y1, L=L, tau=tau, flat=flat,
                base=base, kmax=L.argmax(1), zspread=torch.stack([a[:, 2], b[:, 2], c[:, 2]], 1))


def _eval_at(g, t, px, py):
    """Coverage / depth of triangles t at pixel centres (px, py), all float64 and elementwise."""
    a, b, c, area = g["a"][t], g["b"][t], g["c"][t], g["area"][t]
    b0 = _edge(b[:, 0], b[:, 1], c[:, 0], c[:, 1], px, py) / area
    b1 = _edge(c[:, 0], c[:, 1], a[:, 0], a[:, 1], px, py) / area
    b2 = 1 - b0 - b1
    zw = b0 * a[:, 2] + b1 * b[:, 2] + b2 * c[:, 2]
    covers = (b0 >= 0) & (b1 >= 0) & (b2 >= 0)
    # signed distance to each edge line, in px (positive inside): b_k times the height onto edge k
    d = torch.stack([b0, b1, b2], 1) * (area.abs()[:, None] / g["L"][t].clamp_min(1e-300))
    r = (d / g["tau"][t]).min(1).values          # >= 1: surely inside, <= -1: surely outside
    # a flat triangle may cover, in fp32, only points within its height (<= base) of its longest edge's line
    flat = g["flat"][t]
    V = torch.stack([a, b, c], 1)
    km = g["kmax"][t]
    A = V.gather(1, ((km + 1) % 3)[:, None, None].expand(-1, 1, 4))[:, 0]
    B = V.gather(1, ((km + 2) % 3)[:, None, None].expand(-1, 1, 4))[:, 0]
    dl = _edge(A[:, 0], A[:, 1], B[:, 0], B[:, 1], px, py).abs() / g["L"][t].max(1).values.clamp_min(1e-300)
    near_line = dl <= 2 * g["base"][t] + g["tau"][t].max(1).values
    r = torch.where(flat, torch.where(near_line, torch.zeros_like(r), torch.full_like(r, -float("inf"))), r)
    # depth error: each b_k is off by tau_k / height_k, times the depth spread, plus the fp32 sums and key
    zs = g["zspread"][t]
    spread = zs.max(1).values - zs.min(1).values
    dbk = (g["tau"][t] * g["L"][t] / area.abs()[:, None]).sum(1)
    tau_z = TAU_SAFETY * (dbk * spread + 8 * U32 * (1 + zw.abs()))
    tau_z = torch.where(flat, torch.full_like(tau_z, float("inf")), tau_z)
    inz = (zw >= -1) & (zw <= 1)
    zdoubt = ((zw - 1).abs() <= tau_z) | ((zw + 1).abs() <= tau_z)
    return dict(covers=covers, zw=zw, r=r, d=d.abs().min(1).values, tau_z=tau_z, inz=inz, zdoubt=zdoubt, db=dbk)


def _candidates(g, W, H, max_elems=1 << 22):
    """Every (triangle, pixel) pair of the drawn triangles' bounding boxes, bucketed by power-of-two bbox size."""
    dev = g["area"].device
    idx = torch.nonzero(g["drawn"]).flatten()
    bw = (g["x1"] - g["x0"] + 1)[idx]
    bh = (g["y1"] - g["y0"] + 1)[idx]
    pw = torch.pow(2, torch.ceil(torch.log2(bw.double())).long())
    ph = torch.pow(2, torch.ceil(torch.log2(bh.double())).long())
    key = pw * (1 << 20) + ph
    T, P = [], []
    for k in torch.unique(key).tolist():
        sel = idx[key == k]
        BW, BH = k >> 20, k & ((1 << 20) - 1)
        step = max(1, max_elems // (BW * BH))
        oy, ox = torch.meshgrid(torch.arange(BH, device=dev), torch.arange(BW, device=dev), indexing="ij")
        oy, ox = oy.reshape(-1), ox.reshape(-1)
        for i in range(0, sel.numel(), step):
            t = sel[i:i + step]
            x = g["x0"][t][:, None] + ox[None]
            y = g["y0"][t][:, None] + oy[None]
            ok = (x <= g["x1"][t][:, None]) & (y <= g["y1"][t][:, None])
            tt = t[:, None].expand_as(x)[ok]
            T.append(tt)
            P.append(y[ok] * W + x[ok])
    if not T:
        return torch.zeros(0, dtype=torch.long, device=dev), torch.zeros(0, dtype=torch.long, device=dev)
    return torch.cat(T), torch.cat(P)


def rasterize(pos, tri, H, W):
    """Float64 ids [H,W] (-1: none; nearest z/w, ties to the lower id) with, per pixel:
      certain   -- float64 decides the pixel with margin: no triangle that could win it has its coverage or near /
                   far test within tolerance, and the runner-up is more than the depth tolerances behind;
      edge_px   -- distance (px) from the centre to the nearest edge of a triangle that could win it;
      depth_gap -- z/w gap from the winner to the runner-up (inf: no runner-up).
    Also `sure_zw` / `sure_tz`: the nearest depth (and its tolerance) among the triangles that surely cover the
    pixel, which `admissible` needs."""
    tri = tri.long().to(pos.device)
    s = project(pos, W, H)
    g = _tri_geometry(s, tri, W, H)
    T, P = _candidates(g, W, H)
    px = (P % W).double() + 0.5
    py = torch.div(P, W, rounding_mode="floor").double() + 0.5
    e = _eval_at(g, T, px, py)
    n = H * W
    dev = pos.device
    hit = e["covers"] & e["inz"]
    # nearest (zw, id) per pixel: stable sorts, least significant key first (T is ascending within a bucket only)
    o = torch.nonzero(hit).flatten()
    o = o[torch.sort(T[o], stable=True).indices]
    o = o[torch.sort(e["zw"][o], stable=True).indices]
    o = o[torch.sort(P[o], stable=True).indices]
    Ps = P[o]
    first = torch.ones_like(Ps, dtype=torch.bool)
    first[1:] = Ps[1:] != Ps[:-1]
    ids = torch.full((n,), -1, dtype=torch.long, device=dev)
    zwin = torch.full((n,), float("inf"), dtype=torch.float64, device=dev)
    tzwin = torch.zeros((n,), dtype=torch.float64, device=dev)
    ids[Ps[first]] = T[o[first]]
    zwin[Ps[first]] = e["zw"][o[first]]
    tzwin[Ps[first]] = e["tau_z"][o[first]]
    # runner-up: the nearest other triangle that is not an exact copy of the winner (same pixel-space vertices in
    # the same order: fp32 computes the same depth for both, and the lower id wins the tie without doubt)
    pos_ = torch.arange(Ps.numel(), device=dev)
    wi = torch.cummax(torch.where(first, pos_, torch.zeros_like(pos_)), 0).values
    Ts, Tw = T[o], T[o[wi]]
    copy = torch.ones_like(first)
    for key in ("a", "b", "c"):
        copy &= (g[key][Ts] == g[key][Tw]).all(1)
    run = ~first & ~copy
    zrun = torch.full((n,), float("inf"), dtype=torch.float64, device=dev)
    tzrun = torch.zeros((n,), dtype=torch.float64, device=dev)
    zrun.scatter_reduce_(0, Ps[run], e["zw"][o[run]], reduce="amin")
    tzrun.scatter_reduce_(0, Ps[run], e["tau_z"][o[run]], reduce="amax")
    # doubt: a coverage or near/far decision within tolerance, of a triangle that could be nearest
    doubt = (e["r"].abs() < 1) | (e["covers"] & e["zdoubt"])
    could_win = e["zw"] <= zwin[P] + e["tau_z"] + tzwin[P]
    rel = doubt & could_win
    bad = torch.zeros((n,), dtype=torch.bool, device=dev)
    bad[P[rel]] = True
    bad |= (ids >= 0) & (zrun - zwin <= tzwin + tzrun)
    edge_px = torch.full((n,), float("inf"), dtype=torch.float64, device=dev)
    edge_px.scatter_reduce_(0, P[could_win], e["d"][could_win], reduce="amin")
    sure = (e["r"] >= 1) & e["inz"] & ~e["zdoubt"]
    sure_zw = torch.full((n,), float("inf"), dtype=torch.float64, device=dev)
    sure_zw.scatter_reduce_(0, P[sure], e["zw"][sure], reduce="amin")
    sure_tz = torch.zeros((n,), dtype=torch.float64, device=dev)
    sure_tz.scatter_reduce_(0, P[sure], e["tau_z"][sure], reduce="amax")
    sh = lambda t: t.view(H, W)  # noqa: E731
    return dict(ids=sh(ids), zw=sh(zwin), certain=sh(~bad), edge_px=sh(edge_px), depth_gap=sh(zrun - zwin),
                sure_zw=sh(sure_zw), sure_tz=sh(sure_tz), geometry=g)


def admissible(fr, ids_k, H, W):
    """[H,W] bool: the kernel's id per pixel is a choice float64 allows within tolerance -- its triangle is drawn,
    covers the centre and passes near / far to within tau, and is no more than the depth tolerances behind the
    nearest triangle that surely covers it; -1 only where no triangle surely covers the centre."""
    g = fr["geometry"]
    ids = ids_k.reshape(-1).to(g["area"].device).long()
    n = ids.numel()
    ok = torch.ones(n, dtype=torch.bool, device=ids.device)
    none = ids < 0
    ok[none] = ~torch.isfinite(fr["sure_zw"].reshape(-1)[none])
    p = torch.nonzero(~none).flatten()
    t = ids[p]
    px = (p % W).double() + 0.5
    py = torch.div(p, W, rounding_mode="floor").double() + 0.5
    e = _eval_at(g, t, px, py)
    z_ok = (e["zw"] >= -1 - e["tau_z"]) & (e["zw"] <= 1 + e["tau_z"])
    near_ok = e["zw"] <= fr["sure_zw"].reshape(-1)[p] + e["tau_z"] + fr["sure_tz"].reshape(-1)[p]
    ok[p] = g["drawn"][t] & (e["r"] > -1) & z_ok & near_ok
    return ok.view(H, W)


def _first_order_rounding(outs, vals):
    """First-order bound of the rounding error of an fp32 formula restated in float64: each intermediate r that fp32
    rounds (listed in `vals`, elementwise like the outputs) is off by at most u |r|, which moves an output o by at most
    |do/dr| u |r|; the bound of o is the sum over r.  (A fused multiply-add rounds once where the bound counts two
    roundings, so the bound holds whether or not the compiler contracts.)"""
    res = []
    for o in outs:
        gs = torch.autograd.grad(o.sum(), vals, retain_graph=True, allow_unused=True)
        b = torch.zeros_like(o.detach())
        for gr, r in zip(gs, vals):
            if gr is not None:
                b = b + gr.abs() * r.detach().abs()
        res.append(U32 * b)
    return res


def _project_rounded(Pv, W, H, rd):
    """mr_project of clip-space rows Pv [N,4] (exact fp32 values), every fp32 rounding marked with rd."""
    x, y, z, w = Pv.unbind(-1)
    iw = rd(1.0 / w)
    sx = rd(rd(rd(x * iw) * 0.5 + 0.5) * W)
    sy = rd(rd(rd(y * iw) * 0.5 + 0.5) * H)
    return sx, sy, rd(z * iw), iw


def rast_rounding(pos, tri, ids):
    """[H,W,3] first-order bound of the fp32 rounding error of (u, v, z/w) as mr_resolve_kernel computes them on
    the given ids (mr_project, edge_fn and mr_bary in their order of operations) -- the error the kernel's values
    can have from fp32 alone, without any of the margin tolerances."""
    H, W = ids.shape
    dev = pos.device
    tri = tri.long().to(dev)
    flat = ids.reshape(-1).to(dev).long()
    p = torch.nonzero(flat >= 0).flatten()
    out = torch.zeros(H * W, 3, dtype=torch.float64, device=dev)
    if p.numel() == 0:
        return out.view(H, W, 3)
    with torch.enable_grad():
        P = pos.detach().double()[tri[flat[p]]].requires_grad_(True)
        vals = []

        def rd(v):
            vals.append(v)
            return v

        px = (p % W).double() + 0.5
        py = torch.div(p, W, rounding_mode="floor").double() + 0.5
        a, b, c = (_project_rounded(P[:, i], W, H, rd) for i in range(3))

        def edge(A, B, qx, qy):
            return rd(rd(rd(B[0] - A[0]) * rd(qy - A[1])) - rd(rd(B[1] - A[1]) * rd(qx - A[0])))

        inv = rd(1.0 / edge(a, b, c[0], c[1]))
        b0 = rd(edge(b, c, px, py) * inv)
        b1 = rd(edge(c, a, px, py) * inv)
        b2 = rd(rd(1.0 - b0) - b1)
        q0, q1, q2 = rd(b0 * a[3]), rd(b1 * b[3]), rd(b2 * c[3])
        d = rd(1.0 / rd(rd(q0 + q1) + q2))
        u, v = rd(q0 * d), rd(q1 * d)
        zw = rd(rd(rd(b0 * a[2]) + rd(b1 * b[2])) + rd(b2 * c[2]))
        bu, bv, bz = _first_order_rounding([u, v, zw], vals)
    out[p] = torch.stack([bu, bv, bz], 1)
    return out.view(H, W, 3)


def wgt_rounding(pos, tri, pairs, k, branch, W, H):
    """[applied pairs] first-order bound of the fp32 rounding error of each applied pair's weight |cov - 0.5| as
    aa_pair computes it (projection, crossing, alpha, cov) for edge k with coverage branch `branch`."""
    dev = pos.device
    use = k >= 0
    if not bool(use.any()):
        return torch.zeros(0, dtype=torch.float64, device=dev)
    tri = tri.long().to(dev)
    f, kc = pairs["f"][use], k[use]
    ia = tri[f].gather(1, kc[:, None])[:, 0]
    ib = tri[f].gather(1, ((kc + 1) % 3)[:, None])[:, 0]
    with torch.enable_grad():
        Pa = pos.detach().double()[ia].requires_grad_(True)
        Pb = pos.detach().double()[ib].requires_grad_(True)
        vals = []

        def rd(v):
            vals.append(v)
            return v

        va, vb = _project_rounded(Pa, W, H, rd), _project_rounded(Pb, W, H, rd)
        hor = pairs["dir"][use] == 0
        at, as_ = torch.where(hor, va[0], va[1]), torch.where(hor, va[1], va[0])
        bt, bs = torch.where(hor, vb[0], vb[1]), torch.where(hor, vb[1], vb[0])
        sc, c0 = pairs["sc"][use], pairs["c0"][use]
        tt = rd(rd(sc - as_) / rd(bs - as_))
        alpha = rd(rd(at + rd(tt * rd(bt - at))) - c0)
        cov = torch.where(pairs["first_in"][use], alpha, rd(1.0 - alpha))
        wgt = rd(torch.where(branch[use], cov - 0.5, 0.5 - cov))
        (bw,) = _first_order_rounding([wgt], vals)
    return bw


def rast(pos, tri, ids, shift=None):
    """(u, v, z/w, id + 1) [H,W,4] on the given ids, and the per-pixel vertex copies [N,3,4] (N = covered pixels,
    in row-major order; they retain their .grad when `pos` requires grad): pos.grad collects their sum, and each
    copy's .grad is that pixel's own contribution.  Same formulas as meshrast_oracle.rast_from_ids.
    `shift` ([N] x, [N] y, px): sample each covered pixel that far from its centre instead."""
    H, W = ids.shape
    dev = pos.device
    tri = tri.long().to(dev)
    flat = ids.reshape(-1).to(dev)
    p = torch.nonzero(flat >= 0).flatten()
    f = flat[p]
    P = pos.double()[tri[f]]                                             # [N,3,4]
    if P.requires_grad:
        P.retain_grad()
    px = (p % W).double() + 0.5
    py = torch.div(p, W, rounding_mode="floor").double() + 0.5
    if shift is not None:
        px, py = px + shift[0], py + shift[1]
    iw = 1.0 / P[..., 3]
    sx = (P[..., 0] * iw * 0.5 + 0.5) * W
    sy = (P[..., 1] * iw * 0.5 + 0.5) * H
    zv = P[..., 2] * iw
    area = _edge(sx[:, 0], sy[:, 0], sx[:, 1], sy[:, 1], sx[:, 2], sy[:, 2])
    b0 = _edge(sx[:, 1], sy[:, 1], sx[:, 2], sy[:, 2], px, py) / area
    b1 = _edge(sx[:, 2], sy[:, 2], sx[:, 0], sy[:, 0], px, py) / area
    b2 = 1 - b0 - b1
    q0, q1, q2 = b0 * iw[:, 0], b1 * iw[:, 1], b2 * iw[:, 2]
    d = q0 + q1 + q2
    vals = torch.stack([q0 / d, q1 / d, b0 * zv[:, 0] + b1 * zv[:, 1] + b2 * zv[:, 2]], -1)
    out = torch.zeros((H * W, 3), dtype=torch.float64, device=dev).index_put((p,), vals)
    out = torch.cat([out, (flat + 1).double()[:, None]], 1).view(H, W, 4)
    return out, P, tri[f]


def interpolate(attr, rast_, tri):
    """Same as meshrast_oracle.interpolate (already vectorised)."""
    ids = rast_[..., 3].long() - 1
    hit = (ids >= 0)[..., None]
    f = ids.clamp_min(0)
    tri = tri.long().to(attr.device)
    a0, a1, a2 = (attr[tri[f, k]] for k in range(3))
    u, v = rast_[..., 0:1], rast_[..., 1:2]
    out = u * a0 + v * a1 + (1 - u - v) * a2
    return torch.where(hit, out, torch.zeros_like(out))


def aa_pairs(ids, zw, pos, tri, opp, W, H):
    """Every horizontally / vertically adjacent pixel pair with different ids, in the kernel's order of candidate
    pairs (pixel-major, horizontal before vertical), with the decisions of its three candidate edges evaluated in
    float64 and their margins:
      p0, p1, dir, first_in, f, p_in, p_out, c0, sc              -- the pair and its axis
      valid [P,3]    -- edge k passes the silhouette test, crosses the scanline and gives alpha in [0, 1]
      maybe [P,3]    -- edge k could pass all three within tolerance (fp32 may take it)
      doubt [P,3]    -- one of edge k's decisions is within tolerance
      alpha [P,3], tau_a [P,3]  -- the crossing's coverage and its tolerance
      k              -- first valid edge (-1: none); `certain`: every decision up to it has margin, and so does the
                        cov >= 0.5 branch of the chosen edge.
    `ids` / `zw` are the rast's (the kernel's, on the GPU: which pixels pair up and which side is nearer are
    decisions the kernel has already made)."""
    dev = pos.device
    tri = tri.long().to(dev)
    opp = opp.long().to(dev)
    idf = ids.reshape(-1).to(dev).long()
    zf = zw.reshape(-1).to(dev).double()
    P0, P1, D = [], [], []
    n = H * W
    pix = torch.arange(n, device=dev)
    x, y = pix % W, torch.div(pix, W, rounding_mode="floor")
    for d, (dx, dy) in enumerate(((1, 0), (0, 1))):
        ok = (x + dx < W) & (y + dy < H)
        p0 = pix[ok]
        p1 = p0 + dx + dy * W
        diff = idf[p0] != idf[p1]
        P0.append(p0[diff])
        P1.append(p1[diff])
        D.append(torch.full_like(p0[diff], d))
    p0, p1, dr = torch.cat(P0), torch.cat(P1), torch.cat(D)
    order = torch.argsort(p0 * 2 + dr)
    p0, p1, dr = p0[order], p1[order], dr[order]
    f0, f1 = idf[p0], idf[p1]
    first_in = (f1 < 0) | ((f0 >= 0) & (zf[p0] <= zf[p1]))
    f = torch.where(first_in, f0, f1)
    s = project(pos, W, H)
    wv = pos.double()[:, 3]
    v = s[tri[f]]                                                    # [P,3,4]
    area = _edge(v[:, 0, 0], v[:, 0, 1], v[:, 1, 0], v[:, 1, 1], v[:, 2, 0], v[:, 2, 1])
    xs, ys = (p0 % W).double(), torch.div(p0, W, rounding_mode="floor").double()
    hor = dr == 0
    c0 = torch.where(hor, xs, ys) + 0.5
    sc = torch.where(hor, ys, xs) + 0.5
    mag = v[..., :2].abs().amax((1, 2)).clamp_min(float(max(W, H)))
    tau = TAU_SAFETY * 6.0 * U32 * mag                               # pixel-space position tolerance
    Lmax = torch.stack([torch.hypot(v[:, (k + 1) % 3, 0] - v[:, k, 0], v[:, (k + 1) % 3, 1] - v[:, k, 1])
                        for k in range(3)], 1).max(1).values
    area_doubt = area.abs() / Lmax <= tau
    valid, maybe, doubt, alpha, tau_a = [], [], [], [], []
    for k in range(3):
        va, vb = v[:, k], v[:, (k + 1) % 3]
        o = opp[f, k]
        has_o = o >= 0
        oc = o.clamp_min(0)
        so = s[oc]
        o_front = has_o & (wv[oc] > 0)
        an = _edge(vb[:, 0], vb[:, 1], va[:, 0], va[:, 1], so[:, 0], so[:, 1])
        L = torch.hypot(vb[:, 0] - va[:, 0], vb[:, 1] - va[:, 1]).clamp_min(1e-300)
        interior = o_front & (area * an > 0)
        sil_doubt = o_front & ((an.abs() / L <= tau) | area_doubt)
        at, as_ = torch.where(hor, va[:, 0], va[:, 1]), torch.where(hor, va[:, 1], va[:, 0])
        bt, bs = torch.where(hor, vb[:, 0], vb[:, 1]), torch.where(hor, vb[:, 1], vb[:, 0])
        da, db = as_ - sc, bs - sc
        cross_ok = ((da > 0) != (db > 0)) & (bs != as_)
        cross_doubt = (da.abs() <= tau) | (db.abs() <= tau)
        den = torch.where(bs != as_, bs - as_, torch.ones_like(bs))
        tt = (sc - as_) / den
        al = at + tt * (bt - at) - c0
        ta = tau * (1 + 2 * (bt - at).abs() / den.abs())
        in01 = (al >= 0) & (al <= 1)
        a_doubt = (al.abs() <= ta) | ((al - 1).abs() <= ta)
        valid.append(~interior & cross_ok & in01)
        maybe.append((~interior | sil_doubt) & (cross_ok | cross_doubt) & (al >= -ta) & (al <= 1 + ta))
        doubt.append(sil_doubt | cross_doubt | (cross_ok & a_doubt))
        alpha.append(al)
        tau_a.append(ta)
    valid, maybe, doubt = torch.stack(valid, 1), torch.stack(maybe, 1), torch.stack(doubt, 1)
    alpha, tau_a = torch.stack(alpha, 1), torch.stack(tau_a, 1)
    kk = torch.arange(3, device=dev)[None]
    k = torch.where(valid.any(1), torch.argmax(valid.int(), 1), torch.full_like(f, -1))
    upto = kk <= torch.where(k >= 0, k, torch.full_like(k, 2))[:, None]
    certain = ~(doubt & upto).any(1)
    kc = k.clamp_min(0)
    a_k = alpha.gather(1, kc[:, None])[:, 0]
    cov = torch.where(first_in, a_k, 1 - a_k)
    certain &= ~((k >= 0) & ((cov - 0.5).abs() <= tau_a.gather(1, kc[:, None])[:, 0]))
    return dict(p0=p0, p1=p1, dir=dr, first_in=first_in, f=f, p_in=torch.where(first_in, p0, p1),
                p_out=torch.where(first_in, p1, p0), c0=c0, sc=sc, valid=valid, maybe=maybe, doubt=doubt,
                alpha=alpha, tau_a=tau_a, k=k, certain=certain)


def antialias(color, pos, tri, pairs, W, H, k=None, branch=None, shift=None, alpha_offset=None):
    """Antialiased [H,W,C] from the pairs of `aa_pairs`, applying edge `k` per pair (default: the float64 choice;
    -1: none) with the coverage branch `branch` (True: cov >= 0.5, the outer pixel changes; default: float64's).
    Differentiable w.r.t. color and, through per-pair copies [P,2,4] of the edge's clip-space end points (which
    retain their .grad), w.r.t. pos.  Returns (out, copies, their vertex ids [P,2], the applied pair mask).
    `shift` ([applied pairs] px): move each applied pair's scanline that far; `alpha_offset` ([applied pairs], zero):
    added to alpha, so that its .grad is dL/dalpha per pair."""
    dev = color.device
    tri = tri.long().to(dev)
    C = color.shape[-1]
    k = pairs["k"] if k is None else k
    use = k >= 0
    f, kc = pairs["f"][use], k[use]
    ia = tri[f].gather(1, kc[:, None])[:, 0]
    ib = tri[f].gather(1, ((kc + 1) % 3)[:, None])[:, 0]
    vid = torch.stack([ia, ib], 1)
    Pv = pos.double()[vid]                                             # [P,2,4]
    if Pv.requires_grad:
        Pv.retain_grad()
    iw = 1.0 / Pv[..., 3]
    sx = (Pv[..., 0] * iw * 0.5 + 0.5) * W
    sy = (Pv[..., 1] * iw * 0.5 + 0.5) * H
    hor = pairs["dir"][use] == 0
    at, as_ = torch.where(hor, sx[:, 0], sy[:, 0]), torch.where(hor, sy[:, 0], sx[:, 0])
    bt, bs = torch.where(hor, sx[:, 1], sy[:, 1]), torch.where(hor, sy[:, 1], sx[:, 1])
    sc, c0 = pairs["sc"][use], pairs["c0"][use]
    if shift is not None:
        sc = sc + shift
    alpha = at + (sc - as_) / (bs - as_) * (bt - at) - c0
    if alpha_offset is not None:
        alpha = alpha + alpha_offset
    fi = pairs["first_in"][use]
    cov = torch.where(fi, alpha, 1 - alpha)
    br = (cov.detach() >= 0.5) if branch is None else branch[use]
    p_in, p_out = pairs["p_in"][use], pairs["p_out"][use]
    dst = torch.where(br, p_out, p_in)
    src = torch.where(br, p_in, p_out)
    wgt = torch.where(br, cov - 0.5, 0.5 - cov)
    cf = color.reshape(H * W, C)
    add = wgt[:, None] * (cf[src] - cf[dst])
    out = cf.index_add(0, dst, add).view(H, W, C)
    return out, Pv, vid, use


def class_colors(H, W, device):
    """[H,W,16] one-hot colour of each pixel's (x mod 4, y mod 4) class: the four neighbours of a pixel fall in
    four classes other than its own, so antialiasing this image writes each pair's weight, alone, into the
    destination pixel's channel of the source's class."""
    y, x = torch.meshgrid(torch.arange(H, device=device), torch.arange(W, device=device), indexing="ij")
    return torch.nn.functional.one_hot((y % 4) * 4 + (x % 4), 16).float()


def read_choices(probe, pairs, W):
    """From the antialiased `class_colors` image: per pair, the destination the kernel wrote (True: p_out,
    False: p_in; only meaningful where wgt > 0) and the weight wgt = |cov - 0.5| it applied (0: nothing)."""
    flat = probe.reshape(-1, 16).double()
    cls = lambda p: (torch.div(p, W, rounding_mode="floor") % 4) * 4 + (p % W % 4)  # noqa: E731
    p_in, p_out = pairs["p_in"], pairs["p_out"]
    w_out = flat[p_out, cls(p_in)]          # inner colour arrived in the outer pixel
    w_in = flat[p_in, cls(p_out)]           # outer colour arrived in the inner pixel
    return w_out > 0, torch.maximum(w_out, w_in), (w_out > 0) & (w_in > 0)


def match_choices(pairs, to_out, wgt):
    """The kernel's edge per pair, from its (destination, weight): the first edge that fp32 may take whose float64
    alpha gives the kernel's coverage within tolerance.  Returns (k [-1: none], branch, matched [bool])."""
    used = wgt > 0
    cov_k = torch.where(to_out, 0.5 + wgt, 0.5 - wgt)
    alpha_k = torch.where(pairs["first_in"], cov_k, 1 - cov_k)
    close = (pairs["alpha"] - alpha_k[:, None]).abs() <= pairs["tau_a"] + 4 * U32
    cand = pairs["maybe"] & close
    k = torch.where(used & cand.any(1), torch.argmax(cand.int(), 1), torch.full_like(pairs["k"], -1))
    return k, to_out, ~used | cand.any(1)


def rounding_spread(pos, tri, ids, pairs, k, branch, W, H, g_uv, g_alpha):
    """Per vertex, how far fp32 rounding can move the per-pixel and per-pair contributions to dL/dpos.  A pixel's
    contribution is a function of its barycentrics, which fp32 gets only to within the edge tolerance tau: near an
    edge b_k is small and so is its own error-free value, so rounding changes the contribution by a large fraction
    of itself.  That change is measured, not estimated: the float64 contribution is re-evaluated at the pixel
    centre moved by +-tau in x and in y (and each antialias scanline by +-tau), and the largest change per vertex
    summed.  g_uv [H,W,2]: dL/d(u, v); g_alpha [applied pairs]: dL/dalpha (both held fixed)."""
    dev = pos.device
    V = pos.shape[0]
    g = _tri_geometry(project(pos, W, H), tri.long().to(dev), W, H)
    flat = ids.reshape(-1).to(dev).long()
    p = torch.nonzero(flat >= 0).flatten()
    tau_p = g["tau"][flat[p]].max(1).values
    gu, gv = g_uv.reshape(-1, 2)[p].unbind(1)

    def raster(shift):
        pl = pos.detach().double().requires_grad_(True)
        r, P, pf = rast(pl, tri, ids, shift)
        rr = r.reshape(-1, 4)[p]
        (rr[:, 0] * gu + rr[:, 1] * gv).sum().backward()
        return P.grad, pf

    c0, pf = raster(None)
    spread = torch.zeros(V, 4, dtype=torch.float64, device=dev)
    dev_r = torch.zeros_like(c0)
    z = torch.zeros_like(tau_p)
    for sh in ((tau_p, z), (-tau_p, z), (z, tau_p), (z, -tau_p)):
        dev_r = torch.maximum(dev_r, (raster(sh)[0] - c0).abs())
    spread.index_add_(0, pf.reshape(-1), dev_r.reshape(-1, 4))
    use = k >= 0
    if bool(use.any()):
        ta = pairs["tau_a"].gather(1, k.clamp_min(0)[:, None])[:, 0][use]
        mag = torch.ones(int(use.sum()), dtype=torch.float64, device=dev)

        def aa(shift):
            pl = pos.detach().double().requires_grad_(True)
            col = torch.zeros(H, W, 1, dtype=torch.float64, device=dev)
            _, Pv, vid, _ = antialias(col, pl, tri, pairs, W, H, k=k, branch=branch, shift=shift)
            # alpha of each applied pair, recomputed from the copies, times its fixed dL/dalpha
            sx = (Pv[..., 0] / Pv[..., 3] * 0.5 + 0.5) * W
            sy = (Pv[..., 1] / Pv[..., 3] * 0.5 + 0.5) * H
            hor = pairs["dir"][use] == 0
            at, as_ = torch.where(hor, sx[:, 0], sy[:, 0]), torch.where(hor, sy[:, 0], sx[:, 0])
            bt, bs = torch.where(hor, sx[:, 1], sy[:, 1]), torch.where(hor, sy[:, 1], sx[:, 1])
            sc = pairs["sc"][use] + (0 if shift is None else shift)
            alpha = at + (sc - as_) / (bs - as_) * (bt - at)
            (alpha * g_alpha).sum().backward()
            return Pv.grad, vid

        a0, vid = aa(None)
        dev_a = torch.maximum((aa(ta * mag)[0] - a0).abs(), (aa(-ta * mag)[0] - a0).abs())
        spread.index_add_(0, vid.reshape(-1), dev_a.reshape(-1, 4))
    return spread


def vertex_budget(V, grads_and_ids):
    """Per-vertex (signed sum, sum of |.|) of per-pixel / per-pair contributions [N,m,4] with vertex ids [N,m]."""
    dev = grads_and_ids[0][0].device
    tot = torch.zeros(V, 4, dtype=torch.float64, device=dev)
    ab = torch.zeros(V, 4, dtype=torch.float64, device=dev)
    for g, ids in grads_and_ids:
        tot.index_add_(0, ids.reshape(-1), g.reshape(-1, 4))
        ab.index_add_(0, ids.reshape(-1), g.abs().reshape(-1, 4))
    return tot, ab


def edge_opposites(tri, V):
    """The pairing rule of meshrast_oracle.edge_opposites (first two users of an edge, in face order), by a
    stable sort of the 3F undirected edge keys."""
    t = tri.long()
    F = t.shape[0]
    a, b = t, t[:, [1, 2, 0]]
    key = (torch.minimum(a, b) * int(V) + torch.maximum(a, b)).reshape(-1)
    order = torch.sort(key, stable=True).indices
    ks = key[order]
    opp = torch.full((3 * F,), -1, dtype=torch.long, device=t.device)
    if F == 0:
        return opp.view(0, 3)
    start = torch.ones_like(ks, dtype=torch.bool)
    start[1:] = ks[1:] != ks[:-1]
    pair = start[:-1] & ~start[1:]
    i, j = order[:-1][pair], order[1:][pair]
    third = t[:, [2, 0, 1]].reshape(-1)
    opp[i] = third[j]
    opp[j] = third[i]
    return opp.view(F, 3)
