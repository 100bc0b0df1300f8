"""Cloud accumulation restated in numpy float32 — TEST INFRASTRUCTURE ONLY.

What the node does to its incoming clouds (src/mcl_3dl.cpp:274-342), written independently of
mcl_3dl_b200/csrc/accum_funcs.cuh from the rule pinned in include/mcl3dl_b200.h:
  R = Eigen::Quaternion<float>(float(w), float(x), float(y), float(z)).toRotationMatrix() (raw, not normalised),
  t = float(translation), out_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i, one rounding per operation;
  accumCloud: every point, label = accumulation index; measure(): pcl::transformPointCloud, which leaves a point with a
  non-finite coordinate as it is unless every accumulated cloud was dense.
numpy float32 arrays round each elementwise operation on its own (no contraction), which is the rule.

Also builds PointCloud2 byte layouts for the tests (point_step, shuffled x / y / z offsets, row padding, organized
clouds, special values)."""
import numpy as np

from mcl_3dl_b200 import synth

F = np.float32


def xform(translation, rotation):
    """(R float32[3, 3], t float32[3]) from a double translation and a raw double quaternion (x y z w)."""
    x, y, z, w = (F(v) for v in rotation)
    two = F(2)
    tx, ty, tz = two * x, two * y, two * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = F(1)
    R = np.array([[one - (tyy + tzz), txy - twz, txz + twy],
                  [txy + twz, one - (txx + tzz), tyz - twx],
                  [txz - twy, tyz + twx, one - (txx + tyy)]], dtype=F)
    t = np.array([F(v) for v in translation], dtype=F)
    return R, t


def apply(R, t, xyz):
    """float32[n, 3] -> float32[n, 3]: ((R_i0 x + R_i1 y) + R_i2 z) + t_i."""
    xyz = np.asarray(xyz, F)
    with np.errstate(all="ignore"):
        cols = [((R[i, 0] * xyz[:, 0] + R[i, 1] * xyz[:, 1]) + R[i, 2] * xyz[:, 2]) + t[i] for i in range(3)]
    return np.stack(cols, axis=1).astype(F)


def second(R, t, xyz, dense):
    """pcl::transformPointCloud: not dense -> points with a non-finite coordinate pass unchanged."""
    xyz = np.asarray(xyz, F)
    out = apply(R, t, xyz)
    if not dense:
        keep = ~np.all(np.isfinite(xyz), axis=1)
        out[keep] = xyz[keep]
    return out


def read(data, width, height, point_step, row_step, offsets):
    """The raw x / y / z of a PointCloud2's bytes (uint8 array), row-major: float32[width * height, 3]."""
    data = np.asarray(data, np.uint8)
    r = np.repeat(np.arange(height, dtype=np.int64), width)
    c = np.tile(np.arange(width, dtype=np.int64), height)
    base = r * row_step + c * point_step
    out = np.empty((width * height, 3), F)
    for k, o in enumerate(offsets):
        idx = base[:, None] + o + np.arange(4)
        out[:, k] = data[idx].copy().view("<f4").reshape(-1)
    return out


def canon(pts):
    """The bytes of a POINT array with every NaN coordinate replaced by one NaN: which NaN an operation returns is not
    fixed across processors (x86 keeps an operand's payload and sign, the GPU returns its canonical NaN), and nothing
    downstream reads it."""
    p = np.array(pts, copy=True)
    for k in ("x", "y", "z"):
        p[k][np.isnan(p[k])] = np.float32(np.nan)
    return p.tobytes()


def to_points(xyz, label):
    p = np.zeros(len(xyz), synth.POINT)
    p["x"], p["y"], p["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    p["label"] = label
    return p


def pack_cloud(xyz, width, height, point_step, offsets, row_pad=0, filler=0xA5, rng=None):
    """A PointCloud2 data buffer (uint8) holding xyz (float32[width * height, 3]) at the given offsets; the other bytes
    of each point and the row padding get `filler` (or random bytes).  Returns (data, row_step)."""
    row_step = width * point_step + row_pad
    n = width * height
    size = height * row_step
    data = (rng.integers(0, 256, size, dtype=np.uint8) if rng is not None else np.full(size, filler, np.uint8))
    r = np.repeat(np.arange(height, dtype=np.int64), width)
    c = np.tile(np.arange(width, dtype=np.int64), height)
    base = r * row_step + c * point_step
    raw = np.ascontiguousarray(np.asarray(xyz, F).reshape(n, 3)).view(np.uint8).reshape(n, 3, 4)
    for k, o in enumerate(offsets):
        data[base[:, None] + o + np.arange(4)] = raw[:, k, :]
    return data, row_step


SPECIALS = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-45, -1e-45, 1.17e-38, 3e-39, 1e30, -1e30, 3.4e38], F)


def random_xyz(rng, n, scale=10.0, specials=0.0):
    xyz = (rng.standard_normal((n, 3)) * scale).astype(F)
    if specials > 0:
        m = rng.random((n, 3)) < specials
        xyz[m] = rng.choice(SPECIALS, int(m.sum()))
    return xyz


def random_quat(rng, unit=False):
    q = rng.standard_normal(4)
    if unit:
        q /= np.linalg.norm(q)
    else:
        q *= rng.uniform(0.5, 1.5)
    return tuple(float(v) for v in q)


def node_cloud(clouds, base_tf):
    """The cloud measure() hands the VoxelGrid: clouds = [(xyz_raw float32[n, 3], is_dense, (translation, rotation))],
    accumulated with labels 0, 1, .. and moved into base_link by base_tf."""
    acc, dense = [], True
    for k, (xyz, is_dense, tf) in enumerate(clouds):
        R, t = xform(*tf)
        acc.append(to_points(apply(R, t, xyz), k))
        dense = dense and bool(is_dense)
    pts = np.concatenate(acc)
    R, t = xform(*base_tf)
    xyz = second(R, t, np.stack([pts["x"], pts["y"], pts["z"]], axis=1), dense)
    return to_points(xyz, pts["label"])
