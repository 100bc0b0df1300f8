"""Numpy restatement of the map intake (mcl3dl_map_load / mcl3dl_map_update_set), written apart from the device code:
fromROSMsg into PointXYZIL (x / y / z / label as raw 32-bit words, intensity as a FLOAT32 word, absent fields 0), then
the VoxelGrid of tests/test_gpu_scan_exact.py (voxel_grid_ref) with the intensity centroid (float32 sums in input order
over float(cnt)), or, when the cloud passes unfiltered, its finite points in order."""
import numpy as np

from mcl_3dl_b200 import synth
from test_gpu_scan_exact import _sequential_sums, lattice_ref, voxel_grid_ref

F = np.float32
U = np.uint32


def _base(width, height, point_step, row_step):
    r = np.repeat(np.arange(height, dtype=np.int64), width)
    c = np.tile(np.arange(width, dtype=np.int64), height)
    return r * row_step + c * point_step


def pack_map(pts, intensity, width, height, point_step, offsets, io=-1, lo=-1, row_pad=0, rng=None, filler=0xA5):
    """A map PointCloud2's data (uint8) holding pts (POINT: x / y / z words and, at lo, the label) and, at io, the
    intensities; every other byte is `filler` (or random).  Returns (data, row_step)."""
    row_step = width * point_step + row_pad
    size = height * row_step
    data = rng.integers(0, 256, size, dtype=np.uint8) if rng is not None else np.full(size, filler, np.uint8)
    base = _base(width, height, point_step, row_step)
    words = np.ascontiguousarray(pts).view(U).reshape(-1, 4)
    cols = [(offsets[0], words[:, 0]), (offsets[1], words[:, 1]), (offsets[2], words[:, 2])]
    if lo >= 0:
        cols.append((lo, words[:, 3]))
    if io >= 0:
        cols.append((io, np.ascontiguousarray(intensity, F).view(U)))
    for o, w in cols:
        data[base[:, None] + o + np.arange(4)] = np.ascontiguousarray(w, "<u4").view(np.uint8).reshape(-1, 4)
    return data, row_step


def convert(data, width, height, point_step, row_step, offsets, io=-1, lo=-1):
    """fromROSMsg: (POINT array, float32 intensities) in row-major order, every word copied as it is."""
    base = _base(width, height, point_step, row_step)
    n = width * height

    def word(o):
        if o < 0:
            return np.zeros(n, U)
        return np.ascontiguousarray(data[base[:, None] + o + np.arange(4)]).view("<u4").reshape(-1)

    w = np.stack([word(offsets[0]), word(offsets[1]), word(offsets[2]), word(lo)], axis=1).astype(U)
    return np.ascontiguousarray(w).view(synth.POINT).reshape(-1), word(io).view(F)


def intake_ref(pts, intensity, leaf):
    """(points, intensities, downsampled) of the intake on a converted cloud."""
    xyz = np.stack([pts["x"], pts["y"], pts["z"]], axis=1).astype(F)
    fin = np.isfinite(xyz).all(axis=1)
    leaf = np.asarray(leaf, F)
    if (leaf > 0).all():
        ds = voxel_grid_ref(pts, leaf)
        if ds is not None:
            if len(ds) == 0:
                return ds, np.zeros(0, F), True
            inv, min_b, div = lattice_ref(leaf, xyz[fin].min(axis=0), xyz[fin].max(axis=0))
            ijk = np.floor(xyz[fin] * inv).astype(np.int64) - min_b
            key = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * (div[0] * div[1])
            order = np.argsort(key, kind="stable")
            ks = key[order]
            starts = np.flatnonzero(np.concatenate([[True], ks[1:] != ks[:-1]]))
            cnt = np.diff(np.concatenate([starts, [len(ks)]]))
            v = np.zeros((len(order), 3), F)
            v[:, 0] = np.asarray(intensity, F)[fin][order]
            s = _sequential_sums(v, starts, cnt)[:, 0] / cnt.astype(F)
            return ds, s.astype(F), True
    return pts[fin].copy(), np.asarray(intensity, F)[fin].copy(), False
