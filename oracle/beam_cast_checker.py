"""ctypes binding of oracle/beam_cast_api.h — TEST INFRASTRUCTURE ONLY.

The CPU checkers of the ray markers (src/mcl_3dl.cpp:464-628, mcl3dl_beam_cast), built by oracle/beam_cast.mk:
  kind="port"       oracle/libmcl3dl_beam_cast_oracle.so   (repo-owned restatement, always available)
  kind="reference"  oracle/_ref/libmcl3dl_beam_cast_ref.so (the node's marker loop on the reference's own beam model, built
                    where a checkout of the reference exists, as for cpu_checker's "reference")
  kind="parity"     oracle/_ref/beam_cast_parity_test      (that loop vs the C++ adapter's castBeams, and a node without its
                    CPU map index; one process, H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import cpu_checker as cc

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"port": ("libmcl3dl_beam_cast_oracle.so", "beam-cast-port"),
           "reference": (os.path.join("_ref", "libmcl3dl_beam_cast_ref.so"), "beam-cast-ref"),
           "parity": (os.path.join("_ref", "beam_cast_parity_test"), "beam-cast-parity")}
# mcl3dl_beam_ray (include/mcl3dl_b200.h)
BEAM_RAY = np.dtype([("begin", "<f4", 3), ("end", "<f4", 3), ("pos", "<f4", 3), ("status", "<u4")])


def lib_path(kind):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "beam_cast.mk"] + args + ref, capture_output=quiet, text=True)


def build(kind="port", quiet=True):
    """Compile if missing or stale.  "reference" and "parity" compile the reference's own sources from its checkout;
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


class BeamCastChecker:
    """One loaded checker library ("port" or "reference")."""

    def __init__(self, kind="port"):
        path = lib_path(kind)
        if not os.path.exists(path):
            build(kind)
        self.lib = L = C.CDLL(path)
        self.kind = kind
        L.mcl3dl_cpu_kind.restype = C.c_char_p
        assert L.mcl3dl_cpu_kind().decode() == kind
        L.mcl3dl_cpu_create.restype = C.c_void_p
        L.mcl3dl_cpu_create.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_float, C.c_float]
        L.mcl3dl_cpu_destroy.argtypes = [C.c_void_p]
        L.mcl3dl_cpu_beam_cast.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]

    def create(self, map_pts, lik=None, beam=None, chunk_length=20.0, max_search_radius=0.2):
        """lik: cc.lik_params(...), beam: cc.beam_raw(...) (None: the reference's defaults)."""
        return BeamCastMap(self, map_pts, lik, beam, chunk_length, max_search_radius)


class BeamCastMap:
    def __init__(self, checker, map_pts, lik, beam, chunk_length, max_search_radius):
        self.c = checker
        self.map_pts = np.ascontiguousarray(map_pts, dtype=cc.POINT)
        self.h = checker.lib.mcl3dl_cpu_create(cc._ptr(self.map_pts), len(self.map_pts),
                                               C.byref(lik) if lik is not None else None,
                                               C.byref(beam) if beam is not None else None, chunk_length, max_search_radius)
        if not self.h:
            raise RuntimeError("mcl3dl_cpu_create failed")

    def close(self):
        if self.h:
            self.c.lib.mcl3dl_cpu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def beam_cast(self, pose, pts, origins):
        """The node's marker loop from one pose: BEAM_RAY per scan point."""
        pose = np.ascontiguousarray(pose, dtype=cc.POSE).reshape(1)
        pts = np.ascontiguousarray(pts, dtype=cc.POINT)
        origins = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(pts), dtype=BEAM_RAY)
        rc = self.c.lib.mcl3dl_cpu_beam_cast(self.h, cc._ptr(pose), cc._ptr(pts), len(pts), cc._ptr(origins), len(origins),
                                             cc._ptr(out))
        if rc != 0:
            raise RuntimeError("mcl3dl_cpu_beam_cast rc=%d" % rc)
        return out
