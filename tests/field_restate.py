"""Field mode restated in plain numpy float32 (not a test module; imported by test_field_on_host.py and
test_gpu_field_exact.py).

numpy's float32 operations round to nearest, one operation at a time, as the device does with -fmad=false, so every
function below returns the device's bits:
- the lattice: near_layout (device_funcs.cuh) for the NN field's radius, which build_map_on_device (engine.cu) picks:
  the likelihood radius rpad, or with the KD-tree raycaster max(rpad, r2_pad) (r1_pad under MCL3DL_NNF_KD_R2=0);
- the node volume of field_nodes_kernel: node (i, j, k) sits at origin + float(i) * edge (float ops), and holds
  min(sqrt(d2), clamp) when the float flann::L2_Simple minimum d2 over all map points is below r2 = float(clamp^2),
  clamp otherwise (clamp = the field's radius);
- field_expand_kernel's corner layout and field_dist's lookup;
- lik_kernel_field's test of one distance: d < match_dist_min and lik_term.
"""
import numpy as np

F = np.float32
KD_R2 = "kd"      # KD-tree raycaster, the field also covers its second search (the default)
KD_R1 = "kd_r1"   # KD-tree raycaster with MCL3DL_NNF_KD_R2=0
DDA = "dda"
LIK = "lik"       # likelihood model only


def lik_rpad(R):
    """derive_lik: R * 1.0001f + 1e-6f."""
    return F(F(R) * F(1.0001)) + F(1e-6)


def kd_pads(map_grid=(0.1, 0.1, 0.1)):
    """fill_kd_scalars: (r1_pad, r2_pad)."""
    g = [F(v) for v in map_grid]
    gmin, gmax = min(g), max(g)
    r1 = F(np.sqrt(2.0) * float(gmax) / 2.0)
    r2 = F(float(F(gmin * F(2))) + np.sqrt(2.0) * float(gmax) / 2.0)
    return F(F(r1 * F(1.0001)) + F(1e-6)), F(F(r2 * F(1.0001)) + F(1e-6))


def field_radius(R, beam, map_grid=(0.1, 0.1, 0.1)):
    """The NN field's radius as build_map_on_device picks it; the field-mode clamp."""
    r = lik_rpad(R)
    if beam in (KD_R2, KD_R1):
        r1, r2 = kd_pads(map_grid)
        r = max(r, r2 if beam == KD_R2 else r1)
    return F(r)


def near_layout(r, k, sc_min, sc_max, max_bytes=1 << 40):
    """device_funcs.cuh near_layout: (cells per axis, origin float32[3], inv_cell, ef) or None."""
    ef = F(F(F(1.01) * F(r)) / F(k))
    for _ in range(40):
        org = np.array([F(F(sc_min[a]) - F(F(F(k) + F(0.5)) * ef)) for a in range(3)], F)
        dims = [np.floor((float(F(sc_max[a])) - float(org[a])) / float(ef)) + k + 2 for a in range(3)]
        if all(1.0 <= d <= 16384.0 * k for d in dims):
            pitch = np.floor((dims[0] + 31.0) / 32.0)
            if pitch * dims[1] * dims[2] * 4.0 <= max_bytes:
                return tuple(int(d) for d in dims), org, F(F(1) / ef), ef
        ef = F(ef * F(2))
    return None


def rescaled(xyz, dw):
    """The map points in the rescaled space: float(p * dist_weight) per axis."""
    return (np.asarray(xyz, F) * np.asarray(dw, F)).astype(F)


def lattice(xyz, dw, radius):
    """The field-mode lattice of a map: (node dims (nx+1, ny+1, nz+1), origin, edge, inv_e)."""
    sc = rescaled(xyz, dw)
    dims, org, inv_e, _ = near_layout(radius, 2, sc.min(axis=0), sc.max(axis=0))
    return tuple(d + 1 for d in dims), org, F(F(1) / inv_e), inv_e


def node_positions(org, edge, node_dims):
    """Node (i, j, k) at origin + float(i) * edge, per axis in float32; returned as float32[nz, ny, nx, 3]."""
    ax = [F(org[a]) + np.arange(node_dims[a], dtype=F) * F(edge) for a in range(3)]
    z, y, x = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return np.stack([x, y, z], axis=-1).astype(F)


def l2_simple(q, p):
    """flann::L2_Simple in float: fadd(fadd(dx^2, dy^2), dz^2) (broadcasting)."""
    dx, dy, dz = (q[..., a] - p[..., a] for a in range(3))
    return ((dx * dx + dy * dy) + dz * dz).astype(F)


def node_values(pts, org, edge, node_dims, clamp, k=8):
    """field_nodes_kernel's volume float32[nz, ny, nx] over the rescaled map points pts (float32[n, 3]): the exact float
    minimum over ALL points.  A cKDTree in double finds every point within 1e-5 (relative) of the nearest one, far more
    than the float evaluation can reorder (a few ulps); only those are evaluated in float."""
    from scipy.spatial import cKDTree
    clamp = F(clamp)
    r2 = F(float(clamp) * float(clamp))
    Q = node_positions(org, edge, node_dims).reshape(-1, 3)
    tree = cKDTree(pts.astype(np.float64))
    ub = float(clamp) * (1 + 1e-4) + 1e-6
    d, idx = tree.query(Q.astype(np.float64), k=k, distance_upper_bound=ub, workers=-1)
    reach = d[:, :1] * (1 + 1e-5) + 1e-7
    near = np.isfinite(d) & (d <= reach)
    best = np.full(len(Q), np.inf, F)
    rows = np.nonzero(near[:, 0])[0]
    safe = np.where(near, idx, 0)
    d2 = np.where(near[rows], l2_simple(Q[rows, None, :], pts[safe[rows]]), F(np.inf))
    best[rows] = d2.min(axis=1)
    # nodes whose k-th neighbour still lies within reach may have more candidates: all of them, one node at a time
    for r in np.nonzero(near[:, -1])[0]:
        c = tree.query_ball_point(Q[r].astype(np.float64), float(reach[r, 0]))
        best[r] = l2_simple(Q[r][None, :], pts[c]).min()
    out = np.where(best < r2, np.minimum(np.sqrt(best), clamp), clamp).astype(F)
    return out.reshape(node_dims[2], node_dims[1], node_dims[0])


def expand(V):
    """field_expand_kernel: cell (i, j, k) <- {d000, d100, d010, d110}, {d001, d101, d011, d111} with dABC the node
    (i + A, j + B, k + C); float32[nz, ny, nx, 8] over a node volume V[nz + 1, ny + 1, nx + 1]."""
    c = [V[z:z + V.shape[0] - 1, y:y + V.shape[1] - 1, x:x + V.shape[2] - 1]
         for z in (0, 1) for y in (0, 1) for x in (0, 1)]
    return np.ascontiguousarray(np.stack(c, axis=-1), F)


def float2int_rd(t):
    """cvt.rmi.s32.f32: floor, saturated to int32, NaN -> 0."""
    f = np.floor(np.asarray(t, np.float64))
    f = np.where(np.isnan(f), 0.0, np.clip(f, -2.0 ** 31, 2.0 ** 31 - 1))
    return f.astype(np.int64)


def field_dist(V, org, inv_e, clamp, q):
    """device_funcs.cuh field_dist at q (float32[n, 3], rescaled space) over the node volume V[nz + 1, ny + 1, nx + 1],
    with the corners read in field_expand_kernel's order."""
    with np.errstate(invalid="ignore", over="ignore"):   # (NaN / inf from queries outside: masked below)
        return _field_dist(V, org, inv_e, clamp, np.asarray(q, F))


def _field_dist(V, org, inv_e, clamp, q):
    t = ((q - np.asarray(org, F)).astype(F) * F(inv_e)).astype(F)
    ix = float2int_rd(t)
    n = np.array([V.shape[2] - 1, V.shape[1] - 1, V.shape[0] - 1])
    inside = ((ix >= 0) & (ix < n)).all(axis=1)
    i = np.where(inside[:, None], ix, 0)
    fr = (t - i.astype(F)).astype(F)
    fx, fy, fz = fr[:, 0], fr[:, 1], fr[:, 2]
    x, y, z = i[:, 0], i[:, 1], i[:, 2]
    a = [V[z, y, x], V[z, y, x + 1], V[z, y + 1, x], V[z, y + 1, x + 1]]
    b = [V[z + 1, y, x], V[z + 1, y, x + 1], V[z + 1, y + 1, x], V[z + 1, y + 1, x + 1]]

    def lerp(u, v, f):
        return (u + (f * (v - u)).astype(F)).astype(F)
    c00, c10 = lerp(a[0], a[1], fx), lerp(a[2], a[3], fx)
    c01, c11 = lerp(b[0], b[1], fx), lerp(b[2], b[3], fx)
    c0, c1 = lerp(c00, c10, fy), lerp(c01, c11, fy)
    return np.where(inside, lerp(c0, c1, fz), F(clamp)).astype(F)


def field_term(d, R, flat, w):
    """lik_kernel_field's test of one distance: (contribution, counted) = d < R and lik_term(d)."""
    d = np.asarray(d, F)
    dist = (F(R) - np.fmax(d, F(flat))).astype(F)
    counted = (d < F(R)) & ~(dist < F(0))
    return np.where(counted, (dist * F(w)).astype(F), F(0)).astype(F), counted


def one_eval_records(V, org, inv_e, clamp, q, R, flat, w):
    """The record of a particle whose one-point scan evaluates the field at q: (score_like, match_cnt)."""
    t, m = field_term(field_dist(V, org, inv_e, clamp, q), R, flat, w)
    return (F(0) + t).astype(F), m.astype(np.uint32)


def edge_axis_values(n, org, edge, inv_e, rng, sweep=8):
    """Coordinates along one axis (rescaled space) that put tx = (q - o) * inv_e at the lookup's edges, for a lattice
    of n cells: around nodes 0, 1, n // 2, n - 1 and n, the last coordinate whose tx lies below the node and the first
    one at or above it, each with `sweep` - 1 more coordinate ulps outwards; cell centres, random points, the last
    cell, below 0, past n, and magnitudes past int range."""
    o, e, ie = F(org), F(edge), F(inv_e)

    def tx(q):
        return F(F(q - o) * ie)

    def step(q, s):
        return np.nextafter(q, F(np.inf if s > 0 else -np.inf), dtype=F)
    vals = []
    for i in sorted({0, 1, n // 2, max(n - 1, 0), n}):
        q = F(o + F(F(i) * e))
        while tx(q) >= i:   # the last coordinate whose tx lies below the node, and the next one (tx >= the node)
            q = step(q, -1)
        while tx(step(q, 1)) < i:
            q = step(q, 1)
        lo, hi = q, step(q, 1)
        for s in range(sweep):
            vals += [lo, hi]
            lo, hi = step(lo, -1), step(hi, 1)
    vals += [F(o + F(F(i + 0.5) * e)) for i in (0, n // 3, n - 1)]
    vals += list((o + (rng.uniform(0, n, 16).astype(F) * e).astype(F)).astype(F))
    vals += [F(o - e), F(o + F(F(n + 1) * e)), F(o + F(F(n) * F(0.9999) * e))]
    big = F(3e9) * e
    vals += [F(o + big), F(o - big), F(1e30), F(-1e30)]
    return np.array(vals, F)


def edge_queries(node_dims, org, edge, inv_e, rng, n=20000):
    """Query points for the lookup: random combinations of the edge values of each axis (nodes, cell centres, face
    and edge midpoints and the outside come out of the mix)."""
    axes = [edge_axis_values(node_dims[a] - 1, org[a], edge, inv_e, rng) for a in range(3)]
    return np.stack([a[rng.integers(0, len(a), n)] for a in axes], axis=1).astype(F)
