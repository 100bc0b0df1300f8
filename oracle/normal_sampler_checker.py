"""ctypes binding of oracle/normal_sampler_api.h — TEST INFRASTRUCTURE ONLY.

The CPU checkers of the normal-weighted sampler (PointCloudSamplerWithNormal, selected by use_random_sampler_with_normal,
src/mcl_3dl.cpp:369-375), built by oracle/normal_sampler.mk:
  kind="port"       oracle/libmcl3dl_normal_oracle.so   (repo-owned restatement, always available)
  kind="reference"  oracle/_ref/libmcl3dl_normal_ref.so (the reference's own sampler, built where a checkout of the
                    reference exists)
  kind="parity"     oracle/_ref/normal_sampler_parity_test (the C++ adapter's sampleWithNormalPrepared with the reference
                    filter's statistics vs the port; H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import cpu_checker as cc
from mcl_3dl_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"port": ("libmcl3dl_normal_oracle.so", "normal-port"),
           "reference": (os.path.join("_ref", "libmcl3dl_normal_ref.so"), "normal-ref"),
           "parity": (os.path.join("_ref", "normal_sampler_parity_test"), "normal-parity")}
DEFAULT_PARAMS = (2.0, 5.0, 5.0, 0.4)  # perform_weighting_ratio, max_weight_ratio, max_weight, normal_search_range


def lib_path(kind):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "normal_sampler.mk"] + args + ref, capture_output=quiet, text=True)


def build(kind="port", quiet=True):
    """Compile if missing or stale.  "reference" and "parity" compile the reference's own code from its checkout;
    where there is none they only report whether an earlier build exists."""
    path = lib_path(kind)
    if kind != "port" and _make(["-s", "has-ref"]).returncode != 0:
        return os.path.exists(path)
    r = _make([TARGETS[kind][1]], quiet)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + (r.stdout or "") + (r.stderr or ""))
    return os.path.exists(path)


def available(kind):
    return os.path.exists(lib_path(kind))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class NormalSamplerChecker:
    """One loaded checker library ("port" or "reference")."""

    def __init__(self, kind="port"):
        path = lib_path(kind)
        if not os.path.exists(path):
            build(kind)
        self.lib = L = C.CDLL(path)
        self.kind = kind
        L.mcl3dl_cpu_ns_kind.restype = C.c_char_p
        assert L.mcl3dl_cpu_ns_kind().decode() == kind
        vp, sz = C.c_void_p, C.c_size_t
        L.mcl3dl_cpu_ns_sample.argtypes = [vp, sz, vp, vp, vp, sz, C.c_uint32, vp, C.POINTER(sz), vp]
        if kind == "port":
            L.mcl3dl_cpu_ns_normals.argtypes = [vp, sz, C.c_double, vp, vp]
            L.mcl3dl_cpu_ns_normals.restype = None
            L.mcl3dl_cpu_ns_weights.argtypes = [vp, sz, vp, C.c_double, vp]
            L.mcl3dl_cpu_ns_weights.restype = None
            L.mcl3dl_cpu_ns_select.argtypes = [vp, sz, sz, C.c_uint32, vp]
            L.mcl3dl_cpu_ns_select.restype = None
            L.mcl3dl_cpu_ns_eigen.argtypes = [vp, vp, vp]
            L.mcl3dl_cpu_ns_eigen.restype = None

    def sample(self, pts, cov3, mean_rot, num, seed, params=DEFAULT_PARAMS):
        """-> (points POINT[k] in output order, consts float64[4]: max_weight, fpc_local (port only))."""
        pts = np.ascontiguousarray(pts, dtype=synth.POINT)
        cov = np.ascontiguousarray(cov3, dtype=np.float32).reshape(9)
        rot = np.ascontiguousarray(mean_rot, dtype=np.float32).reshape(4)
        prm = np.ascontiguousarray(params, dtype=np.float64).reshape(4)
        out = np.zeros(max(1, min(num, len(pts))), synth.POINT)
        n_out = C.c_size_t(0)
        consts = np.zeros(4, np.float64)
        src = pts if len(pts) else np.zeros(1, synth.POINT)
        assert self.lib.mcl3dl_cpu_ns_sample(_ptr(src), len(pts), _ptr(cov), _ptr(rot), _ptr(prm), num, seed, _ptr(out),
                                             C.byref(n_out), _ptr(consts)) == 0
        return out[:n_out.value].copy(), consts

    def normals(self, pts, r):
        """-> (normals float32[n, 3], neighbour counts uint32[n]) by brute force (port)."""
        pts = np.ascontiguousarray(pts, dtype=synth.POINT)
        nrm = np.zeros((len(pts), 3), np.float32)
        cnt = np.zeros(len(pts), np.uint32)
        if len(pts):
            self.lib.mcl3dl_cpu_ns_normals(_ptr(pts), len(pts), r, _ptr(nrm), _ptr(cnt))
        return nrm, cnt

    def weights(self, normals, fpc, max_weight):
        """sample()'s double weights of given normals, with std::acos (port)."""
        nrm = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
        f = np.ascontiguousarray(fpc, dtype=np.float32).reshape(3)
        w = np.zeros(len(nrm), np.float64)
        if len(nrm):
            self.lib.mcl3dl_cpu_ns_weights(_ptr(nrm), len(nrm), _ptr(f), max_weight, _ptr(w))
        return w

    def eigen(self, cov3):
        """setParticleStatistics' eigendecomposition of |cov| (port): (values ascending, vectors as columns)."""
        cov = np.ascontiguousarray(cov3, dtype=np.float32).reshape(9)
        vals, vecs = np.zeros(3), np.zeros(9)
        self.lib.mcl3dl_cpu_ns_eigen(_ptr(cov), _ptr(vals), _ptr(vecs))
        return vals, vecs.reshape(3, 3)
