"""The map intake without a GPU.
  - host build == restatement: the map intake's functions of mcl_3dl_b200/csrc/accum_funcs.cuh, compiled for the host
    with scan_funcs.cuh's VoxelGrid (tests/hostsim/map_intake_hostsim.cpp, -ffp-contract=off), give
    tests/map_intake_restate.py's values bit for bit: the conversion at point_step 16 / 20 / 24 / 32 / 48, unaligned
    offsets, fields that end at point_step, absent fields, padded rows and organized clouds; NaN payloads, -0.0,
    subnormals and infinities copied word for word, and on the unfiltered path the finite points kept bit for bit;
    and the VoxelGrid's points and intensity centroids on every case of tests/test_gpu_scan_exact.py.
  - Engine.map_load / map_update_set hand the engine a view of the caller's own bytes and refuse views that overrun
    them, before the engine is called."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import accum_restate as A
import map_intake_restate as M
from mcl_3dl_b200 import engine, synth
from test_gpu_scan_exact import VOXEL_CASES, case_ref

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostsim", "map_intake_hostsim.cpp")
F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mapintake") / "libmapintakehs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, u32 = C.c_void_p, C.c_uint32
    L.hostsim_map_read.argtypes = [vp, u32, u32, u32, u32, vp, C.c_int32, C.c_int32, vp, vp]
    L.hostsim_map_read.restype = None
    L.hostsim_map_intake.argtypes = [vp, vp, C.c_size_t, vp, vp, vp, C.POINTER(C.c_int)]
    L.hostsim_map_intake.restype = C.c_long
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_read(L, data, width, height, point_step, row_step, offsets, io, lo):
    n = width * height
    out, inten = np.zeros(n, synth.POINT), np.zeros(n, F)
    L.hostsim_map_read(_p(data), width, height, row_step, point_step, _p(np.asarray(offsets, np.uint32)), io, lo, _p(out), _p(inten))
    return out, inten


def host_intake(L, pts, inten, leaf):
    out, oi = np.zeros(max(len(pts), 1), synth.POINT), np.zeros(max(len(pts), 1), F)
    ds = C.c_int(0)
    m = L.hostsim_map_intake(_p(pts), _p(np.ascontiguousarray(inten, F)), len(pts), _p(np.asarray(leaf, F)), _p(out), _p(oi),
                             C.byref(ds))
    return out[:m], oi[:m], bool(ds.value)


def _cloud(rng, n, specials=0.0):
    xyz = A.random_xyz(rng, n, specials=specials)
    pts = synth.make_points(xyz, rng.integers(0, 2 ** 32, n, dtype=np.uint64))
    inten = (rng.standard_normal(n) * 100).astype(F)
    if specials:
        m = rng.random(n) < specials
        inten[m] = rng.choice(A.SPECIALS, int(m.sum()))
    # NaN payloads and signs, as words
    k = min(n, 4)
    pts.view(np.uint32).reshape(-1, 4)[:k, 0] = [0x7FC00001, 0xFFC12345, 0x7F800001, 0x7FBFFFFF][:k]
    inten.view(np.uint32)[:k] = [0x7FC0BEEF, 0xFFFFFFFF, 0x80000000, 0x00000001][:k]
    return pts, inten


LAYOUTS = [  # (point_step, xyz offsets, intensity offset, label offset, row padding, height)
    (16, (0, 4, 8), 12, -1, 0, 1),         # xyzi
    (16, (0, 4, 8), -1, 12, 0, 1),         # xyzl
    (12, (0, 4, 8), -1, -1, 0, 1),         # xyz
    (20, (0, 4, 8), 12, 16, 0, 1),         # xyzil, label at the edge of point_step
    (32, (0, 4, 8), 16, 20, 0, 1),         # PointXYZIL's own layout (padding after z and after label)
    (24, (1, 5, 9), 13, 17, 3, 7),         # unaligned, padded rows, organized
    (48, (40, 8, 24), 44, 0, 5, 3),        # shuffled, intensity at the edge
    (32, (0, 4, 8), 16, -1, 0, 4),         # organized xyzi
]


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: "ps%d_io%d_lo%d_h%d" % (l[0], l[2], l[3], l[5]))
def test_conversion_host(hs, layout):
    ps, off, io, lo, pad, h = layout
    rng = np.random.default_rng(ps * 31 + io + 7 * lo + h)
    w = 257
    pts, inten = _cloud(rng, w * h, specials=0.1)
    data, rs = M.pack_map(pts, inten, w, h, ps, off, io, lo, row_pad=pad, rng=rng)
    want_p, want_i = M.convert(data, w, h, ps, rs, off, io, lo)
    got_p, got_i = host_read(hs, data, w, h, ps, rs, off, io, lo)
    assert got_p.tobytes() == want_p.tobytes() and got_i.tobytes() == want_i.tobytes()
    # the restatement reads back what was packed: words as they are, absent fields 0
    words = pts.view(np.uint32).reshape(-1, 4)
    gw = got_p.view(np.uint32).reshape(-1, 4)
    assert (gw[:, :3] == words[:, :3]).all()
    assert (gw[:, 3] == (words[:, 3] if lo >= 0 else 0)).all()
    assert (got_i.view(np.uint32) == (inten.view(np.uint32) if io >= 0 else 0)).all()


@pytest.mark.parametrize("leaf", [(0.0, 0.0, 0.0), (0.5, -1.0, 0.5), (np.nan, 1.0, 1.0)])
def test_unfiltered_keeps_finite_points_bit_for_bit(hs, leaf):
    """No leaf: the finite points in order, every word kept (-0.0, subnormals, 1e30-scale, NaN intensity payloads)."""
    rng = np.random.default_rng(5)
    pts, inten = _cloud(rng, 3000, specials=0.15)
    got = host_intake(hs, pts, inten, leaf)
    want = M.intake_ref(pts, inten, leaf)
    assert got[2] is False and want[2] is False
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    xyz = np.stack([pts["x"], pts["y"], pts["z"]], 1)
    fin = np.isfinite(xyz).all(1)
    assert 0 < len(got[0]) == fin.sum() < len(pts)
    assert (np.signbit(got[0]["x"]) & (got[0]["x"] == 0)).any()  # a -0.0 survived as -0.0
    assert np.isnan(got[1]).any()  # an intensity NaN on a finite point is kept


@pytest.mark.parametrize("name", VOXEL_CASES)
def test_voxel_intake_host(hs, name):
    """VoxelGrid points and intensity centroids on every voxel case (unfiltered ones: the finite points in order)."""
    raw, leaf, _ = case_ref(name)
    rng = np.random.default_rng(len(raw))
    inten = (rng.uniform(0, 255, len(raw))).astype(F)
    got = host_intake(hs, raw, inten, leaf)
    want = M.intake_ref(raw, inten, leaf)
    assert got[2] == want[2]
    assert got[0].tobytes() == want[0].tobytes()
    assert got[1].tobytes() == want[1].tobytes()


def test_intensity_centroid_is_an_ordered_float_sum(hs):
    """One voxel whose float sum depends on the order: 1e8 + 1 ... - 1e8 in input order."""
    pts = synth.make_points(np.full((5, 3), 0.05, F))
    inten = np.array([1e8, 1.0, 1.0, -1e8, 3.0], F)
    got = host_intake(hs, pts, inten, (0.1, 0.1, 0.1))
    s = F(0)
    for v in inten:
        s = F(s + v)
    assert got[1].tobytes() == np.array([s / F(5)], F).tobytes()


# ---------------------------------------------------------------- binding
class FakeLib:
    def __init__(self):
        self.calls = []

    def _rec(self, name):
        def f(*a):
            self.calls.append((name, a))
            return 0
        return f

    def __getattr__(self, name):
        if name.startswith("mcl3dl_"):
            return self._rec(name)
        raise AttributeError(name)


def _fake_engine():
    e = object.__new__(engine.Engine)
    e.L, e.h = FakeLib(), 1
    return e


def test_binding_hands_over_the_view_and_refuses_overruns():
    e = _fake_engine()
    pts = synth.make_points(np.arange(30, dtype=F).reshape(10, 3), np.arange(10))
    data, rs = M.pack_map(pts, np.arange(10, dtype=F), 5, 2, 32, (0, 4, 8), 16, 20, row_pad=4)
    assert rs == 164
    e.map_load(data, 5, 2, 32, rs, (0, 4, 8), (0.1, 0.1, 0.1), engine.LikParams(), None, intensity_offset=16, label_offset=20,
               stamp=9)
    name, a = e.L.calls[-1]
    assert name == "mcl3dl_map_load" and a[3] == 9
    m = a[1]._obj
    assert m.view.data == data.ctypes.data and (m.view.width, m.view.height, m.view.point_step, m.view.row_step) == (5, 2, 32, 164)
    assert (m.intensity_offset, m.label_offset) == (16, 20) and list(m.view.offset) == [0, 4, 8]
    e.map_update_set(data, 5, 2, 32, rs, (0, 4, 8), (0.1, 0.1, 0.1))
    name, a = e.L.calls[-1]
    assert name == "mcl3dl_map_update_set" and (a[1]._obj.intensity_offset, a[1]._obj.label_offset) == (-1, -1)
    n = len(e.L.calls)
    # the last row ends at its last point: one byte less than (h - 1) row_step + w point_step is an overrun
    short = data[:rs + 5 * 32 - 1].copy()
    for call in (lambda d: e.map_load(d, 5, 2, 32, rs, (0, 4, 8), (0.1,) * 3, engine.LikParams()),
                 lambda d: e.map_update_set(d, 5, 2, 32, rs, (0, 4, 8), (0.1,) * 3)):
        with pytest.raises(ValueError):
            call(short)
        with pytest.raises(ValueError):
            call(data[::2])  # not contiguous
        call(data[:rs + 5 * 32].copy())  # exactly the span
    with pytest.raises(ValueError):
        e.map_load(data, 5, 2, 32, rs, (0, 4), (0.1,) * 3, engine.LikParams())
    with pytest.raises(ValueError):
        e.map_update_set(data, 5, 2, 32, rs, (0, 4, 8), (0.1, 0.1))
    assert len(e.L.calls) == n + 2
    e.h = None
