"""Property tests: the repo-owned oracle equals the reference's own sources bit for bit on random small worlds — DDA
walks (every visited voxel), KD-tree walks (positions, sin_angle_), radius search, per-ray BeamStatus and per-particle
records.  The examples are a fixed, seeded draw over the same ranges (*_EXAMPLES below); what the reference build
returned for them is stored in tests/golden/reference_properties.npz (tests/golden/make_golden.py)."""
import numpy as np

from conftest import golden
from oracle import cpu_checker as cc
from test_oracle_golden import digest


def world(seed, n):
    rng = np.random.default_rng(seed)
    kind = seed % 3
    if kind == 0:      # scattered points
        pts = rng.uniform(-2, 2, (n, 3))
    elif kind == 1:    # lattice wall: exact ties and voxel-boundary coordinates
        g = np.arange(-1.0, 1.0, 0.1, dtype=np.float32)
        yy, zz = np.meshgrid(g, g)
        pts = np.stack([np.full(yy.size, 0.5), yy.ravel(), zz.ravel()], 1)[:max(n, 8)]
    else:              # two noisy planes
        a = np.c_[rng.uniform(-2, 2, n // 2), rng.uniform(-2, 2, n // 2), rng.normal(0, 0.01, n // 2)]
        b = np.c_[rng.normal(1.0, 0.01, n - n // 2), rng.uniform(-2, 2, n - n // 2), rng.uniform(-1, 2, n - n // 2)]
        pts = np.vstack([a, b])
    pts = np.vstack([pts, [[-2.55, -2.55, -2.55], [2.55, 2.55, 2.55]]]).astype(np.float32)
    lab = (rng.random(len(pts)) < 0.2).astype(np.uint32) * 2
    return cc.points(pts, lab), rng


def _examples(draw_seed, count, n_lo, n_hi, *choices):
    """`count` (seed, n, *choice) tuples: the corners of the ranges first, then uniform draws."""
    rng = np.random.default_rng(draw_seed)
    out = [(0, n_lo) + tuple(c[0] for c in choices), (10_000, n_hi) + tuple(c[-1] for c in choices)]
    while len(out) < count:
        out.append((int(rng.integers(0, 10_001)), int(rng.integers(n_lo, n_hi + 1)))
                   + tuple(c[int(rng.integers(0, len(c)))] for c in choices))
    return out


def _flat(parts):
    """One float32 vector of a list of walk outputs (every value is a float32 or a small integer)."""
    return np.concatenate([np.atleast_1d(np.asarray(p, dtype=np.float32)).ravel() for p in parts])


DDA_EXAMPLES = _examples(101, 60, 4, 120, [0.05, 0.1, 0.2, 0.37], [0.0, 0.1, 0.3])
KD_EXAMPLES = _examples(102, 60, 4, 120, [0.0, 0.17, 0.3])
RECORD_EXAMPLES = _examples(103, 25, 20, 400, [True, False], [(1, 1, 1), (1, 1, 5), (2, 1, 3)])


def dda_walks(chk, seed, n, grid, tol):
    m, rng = world(seed, n)
    ctor = [0.1, 0.1, 0.1, grid, 0.25 * np.pi / 180.0 if seed % 2 else 0.5, tol]
    parts = []
    for _ in range(4):
        b = rng.uniform(-2.6, 2.6, 3) if rng.random() < 0.8 else rng.uniform(-4, 4, 3)
        e = rng.uniform(-3, 3, 3)
        if seed % 5 == 0:
            e[2] = b[2]   # axis-aligned components: infinite t_delta path (raycast_using_dda.h:88-92)
        c, coll, cid = chk.dda_walk(m, ctor, b, e, stop_at_collision=bool(seed % 2))
        parts += [len(c), c, coll, cid]
    return _flat(parts)


def kd_walks(chk, seed, n, hit):
    """Stored as a digest (tests/test_oracle_golden.py: digest): the KD-caster walks are the bulk of the outputs."""
    m, rng = world(seed, n)
    ctor = [0.1, 0.1 if seed % 2 else 0.05, 0.1, hit]
    parts = []
    for _ in range(3):
        b, e = rng.uniform(-2, 2, 3), rng.uniform(-2, 2, 3)
        pos, coll, sa, cid = chk.kd_walk(m, ctor, b, e, stop_at_collision=False)
        # the colliding point may differ only between exactly equidistant map points; both pick the lowest index
        parts += [len(pos), pos, coll, sa, cid]
    return _flat(parts)


def records(chk, seed, n, use_dda, w):
    """(records, beam status, radius-search results) of one small world."""
    m, rng = world(seed, n)
    lik = cc.lik_params(dist_weight=w, match_dist_min=0.2 if seed % 2 else 0.35)
    braw = cc.beam_raw(num_points_default=6, use_raycast_using_dda=use_dda, dda_grid_size=0.2 if seed % 3 else 0.1,
                       filter_label_max=1 if seed % 4 == 0 else 0xFFFFFFFF, hit_range=0.3 if seed % 2 else 0.1,
                       add_penalty_short_only_mode=bool(seed % 3))
    a = chk.create(m, lik, braw, 20.0, 1.0)
    P = 5
    q = rng.normal(0, 1, (P, 4))
    poses = cc.poses(rng.uniform(-1.5, 1.5, (P, 3)), q)
    scan_l = cc.points(rng.uniform(-2, 2, (9, 3)))
    scan_b = cc.points(rng.uniform(-2, 2, (6, 3)), rng.integers(0, 2, 6))
    org = rng.uniform(-0.3, 0.3, (2, 3)).astype(np.float32)
    rec, st = a.measure(poses, scan_l, scan_b, org), a.beam_status(poses, scan_b, org)
    rs = []
    for _ in range(5):
        i, d2 = a.radius_search(rng.uniform(-2.5, 2.5, 3).astype(np.float32), 0.3)
        rs.append((float(i >= 0), np.float32(d2) if i >= 0 else 0.0))
    return rec, st, np.array(rs, dtype=np.float32)


def test_dda_walk_matches_reference(port):
    g = golden("reference_properties.npz")
    for i, ex in enumerate(DDA_EXAMPLES):
        assert np.array_equal(dda_walks(port, *ex), g["dda_%d" % i]), ex


def test_kd_walk_matches_reference(port):
    g = golden("reference_properties.npz")
    for i, ex in enumerate(KD_EXAMPLES):
        assert digest(kd_walks(port, *ex)) == str(g["kd_%d" % i]), ex


def test_records_match_reference(port):
    g = golden("reference_properties.npz")
    for i, ex in enumerate(RECORD_EXAMPLES):
        rec, st, rs = records(port, *ex)
        want = g["rec_%d" % i].view(cc.RESULT)
        for f in want.dtype.names:
            assert np.array_equal(want[f], rec[f]), (ex, f)
        assert np.array_equal(g["status_%d" % i], st), ex
        assert np.array_equal(g["radius_%d" % i], rs), ex
