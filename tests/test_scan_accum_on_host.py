"""Cloud accumulation without a GPU.
  - host build == restatement: the functions of mcl_3dl_b200/csrc/accum_funcs.cuh compiled for the host
    (tests/hostsim/scan_accum_hostsim.cpp, -ffp-contract=off) give tests/accum_restate.py's numpy float32 values bit for
    bit: the matrix from random and non-unit quaternions and large translations, the strided read at point_step
    12 / 16 / 32 / 48 with shuffled and unaligned offsets, padded rows and organized clouds, and both transforms with
    NaN, infinities, -0, subnormals and 1e30-scale coordinates, dense and not (a computed NaN's sign and payload are
    not compared: x86 and the GPU return different NaNs; a point the not-dense rule passes keeps every bit).
  - nvcc accepts the accumulation kernels for sm_90a with the product's flags.
  - Engine.scan_accumulate hands the engine a view of the caller's own bytes and refuses views that overrun them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import accum_restate as A
from mcl_3dl_b200 import engine, synth

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostsim", "scan_accum_hostsim.cpp")
F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("accumhost") / "libaccumhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, u32 = C.c_void_p, C.c_uint32
    L.hostsim_accum_xform.argtypes = [vp, vp, vp, vp]
    L.hostsim_accum_xform.restype = None
    L.hostsim_accum_read.argtypes = [vp, u32, u32, u32, u32, vp, vp]
    L.hostsim_accum_read.restype = None
    L.hostsim_accum_cloud.argtypes = [vp, u32, u32, u32, u32, vp, vp, vp, u32, vp]
    L.hostsim_accum_cloud.restype = None
    L.hostsim_accum_second.argtypes = [vp, C.c_size_t, vp, vp, C.c_int, vp]
    L.hostsim_accum_second.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _tf(tf):
    return np.array(tf[0], np.float64), np.array(tf[1], np.float64)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _transforms(rng, k):
    out = [((0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0)), ((1e6, -3e5, 12.5), (0.0, 0.0, 0.0, 1.0)),
           ((0.1, 0.2, 0.3), (0.0, 0.0, 0.0, 0.0)), ((-7.0, 3.0, 1.0), (0.3, -0.2, 0.9, 2.0))]
    for i in range(k):
        tr = tuple(float(v) for v in rng.standard_normal(3) * (10.0 ** rng.integers(0, 7)))
        out.append((tr, A.random_quat(rng, unit=bool(i % 2))))
    return out


def test_matrix_equals_restatement(hs):
    rng = np.random.default_rng(0)
    for tf in _transforms(rng, 200):
        t, q = _tf(tf)
        r, tt = np.zeros(9, F), np.zeros(3, F)
        hs.hostsim_accum_xform(_p(t), _p(q), _p(r), _p(tt))
        R, tw = A.xform(*tf)
        assert _bits(r) == _bits(R.reshape(9)) and _bits(tt) == _bits(tw), tf


LAYOUTS = [(12, (0, 4, 8)), (12, (8, 0, 4)), (16, (0, 4, 8)), (16, (4, 12, 0)), (16, (1, 5, 10)),
           (32, (16, 0, 8)), (32, (3, 17, 26)), (48, (40, 20, 0)), (48, (44, 2, 23))]


@pytest.mark.parametrize("point_step,offsets", LAYOUTS)
def test_strided_read_equals_restatement(hs, point_step, offsets):
    rng = np.random.default_rng(point_step + sum(offsets))
    for width, height, pad in ((1, 1, 0), (37, 1, 0), (13, 7, 5), (8, 16, 64), (200, 3, 3)):
        xyz = A.random_xyz(rng, width * height, specials=0.2)
        data, row_step = A.pack_cloud(xyz, width, height, point_step, offsets, pad, rng=rng)
        for shift in (0, 1):  # an unaligned data pointer takes the byte-wise loads
            buf = np.zeros(len(data) + shift, np.uint8)
            buf[shift:] = data
            got = np.zeros((width * height, 3), F)
            off = np.array(offsets, np.uint32)
            hs.hostsim_accum_read(C.c_void_p(buf.ctypes.data + shift), width, height, row_step, point_step, _p(off), _p(got))
            want = A.read(data, width, height, point_step, row_step, offsets)
            assert _bits(got) == _bits(want) == _bits(xyz), (width, height, pad, shift)


@pytest.mark.parametrize("point_step,offsets", LAYOUTS[::2])
def test_first_transform_equals_restatement(hs, point_step, offsets):
    rng = np.random.default_rng(100 + point_step)
    for k, tf in enumerate(_transforms(rng, 12)):
        width, height = int(rng.integers(1, 90)), int(rng.integers(1, 5))
        scale = 10.0 ** rng.integers(-3, 31) if k % 3 == 0 else 20.0
        xyz = A.random_xyz(rng, width * height, scale=min(scale, 1e30), specials=0.15)
        data, row_step = A.pack_cloud(xyz, width, height, point_step, offsets, int(rng.integers(0, 9)), rng=rng)
        t, q = _tf(tf)
        out = np.zeros(width * height, synth.POINT)
        off = np.array(offsets, np.uint32)
        hs.hostsim_accum_cloud(_p(data), width, height, row_step, point_step, _p(off), _p(t), _p(q), k, _p(out))
        R, tw = A.xform(*tf)
        want = A.to_points(A.apply(R, tw, xyz), k)  # every point, finite or not
        assert A.canon(out) == A.canon(want), (k, tf)


@pytest.mark.parametrize("dense", [True, False])
def test_second_transform_equals_restatement(hs, dense):
    rng = np.random.default_rng(7 + dense)
    for k, tf in enumerate(_transforms(rng, 20)):
        n = int(rng.integers(1, 400))
        xyz = A.random_xyz(rng, n, scale=10.0 ** rng.integers(-2, 30), specials=0.25)
        pts = A.to_points(xyz, rng.integers(0, 10, n))
        t, q = _tf(tf)
        out = np.zeros(n, synth.POINT)
        hs.hostsim_accum_second(_p(pts), n, _p(t), _p(q), 1 if dense else 0, _p(out))
        R, tw = A.xform(*tf)
        want = A.to_points(A.second(R, tw, xyz, dense), pts["label"])
        assert A.canon(out) == A.canon(want), (k, tf)
        if not dense:  # a point with a non-finite coordinate keeps its bits
            bad = ~np.all(np.isfinite(xyz), axis=1)
            assert out[bad].tobytes() == pts[bad].tobytes()


def test_accum_kernels_compile_for_sm_90a(tmp_path):
    """nvcc accepts the accumulation kernels (scan_kernels.cuh) for sm_90a with the product's flags (no GPU needed)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = tmp_path / "accum_check.cu"
    src.write_text('#include "%s"\n' % os.path.join(HERE, "..", "mcl_3dl_b200", "csrc", "scan_kernels.cuh"))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-fmad=false", "-std=c++17", "-c",
                        "-o", str(tmp_path / "accum.o"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run(["cuobjdump", "-sass", str(tmp_path / "accum.o")], capture_output=True, text=True)
    if r.returncode == 0:
        assert "accum_cloud_kernel" in r.stdout and "accum_transform_kernel" in r.stdout


class _FakeLib:
    def __init__(self):
        self.calls = []

    def mcl3dl_scan_accumulate(self, h, view, tf, n):
        v, t = view._obj, tf._obj  # the structures behind C.byref
        self.calls.append((v.data, v.width, v.height, v.point_step, v.row_step, tuple(v.offset), v.is_dense,
                           tuple(t.translation), tuple(t.rotation)))
        n._obj.value = len(self.calls)
        return 0


def test_binding_passes_the_callers_bytes_and_refuses_overruns():
    e = object.__new__(engine.Engine)
    e.L, e.h = _FakeLib(), 1
    # a structured array (x y z intensity at 16 B) and its raw bytes are the same view
    pts = np.zeros(12, np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("i", "<f4")]))
    assert e.scan_accumulate(pts, 4, 3, 16, 64, (0, 4, 8), True, (1, 2, 3), (0, 0, 0.5, 1)) == 1
    a = e.L.calls[-1]
    assert a[0] == pts.ctypes.data and a[1:7] == (4, 3, 16, 64, (0, 4, 8), 1)
    assert a[7] == (1.0, 2.0, 3.0) and a[8] == (0.0, 0.0, 0.5, 1.0)
    raw = pts.view(np.uint8)
    assert e.scan_accumulate(raw, 12, 1, 16, 192, (8, 4, 0), False) == 2
    assert e.L.calls[-1][0] == raw.ctypes.data and e.L.calls[-1][6] == 0
    # padded rows: the last row needs only width * point_step bytes
    buf = np.zeros(2 * 40 + 32, np.uint8)
    assert e.scan_accumulate(buf, 2, 3, 16, 40, (0, 4, 8)) == 3
    n = len(e.L.calls)
    with pytest.raises(ValueError):
        e.scan_accumulate(buf, 2, 3, 16, 41, (0, 4, 8))      # one byte past the end
    with pytest.raises(ValueError):
        e.scan_accumulate(raw, 13, 1, 16, 208, (0, 4, 8))    # one point too many
    with pytest.raises(ValueError):
        e.scan_accumulate(raw, 4, 4, 16, 64, (0, 4, 8))      # one row too many
    with pytest.raises(ValueError):
        e.scan_accumulate(raw[::2], 2, 1, 16, 32, (0, 4, 8))  # not contiguous
    with pytest.raises(ValueError):
        e.scan_accumulate(bytes(64), 1, 1, 16, 16, (0, 4, 8))  # not a numpy array
    with pytest.raises(ValueError):
        e.scan_accumulate(raw, 1, 1, 16, 16, (0, 4))          # two offsets
    assert len(e.L.calls) == n  # none of them reached the engine
    # an empty view spans no bytes: the engine's own check (INVALID_ARG) decides
    assert engine.cloud_span(0, 3, 16, 64) == 0 and engine.cloud_span(5, 0, 16, 80) == 0
    e.h = None
