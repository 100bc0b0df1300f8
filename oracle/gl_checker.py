"""ctypes binding of oracle/gl_api.h — TEST INFRASTRUCTURE ONLY.

The CPU checkers of global localisation (src/mcl_3dl.cpp:1039-1099 after its VoxelGrid) and of
pf::ParticleFilter::resizeParticle (pf.h:399-436), built by oracle/gl.mk:
  kind="port"       oracle/libmcl3dl_gl_oracle.so   (repo-owned restatement, always available)
  kind="reference"  oracle/_ref/libmcl3dl_gl_ref.so (the reference's own filter, Quat and State6DOF, built where a
                    checkout of the reference exists, as for cpu_checker's "reference")
  kind="parity"     oracle/_ref/global_localization_parity_test (the service body and the node's shrink on the
                    reference filter vs the C++ adapter's resident calls, one process; H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import cpu_checker as cc
from mcl_3dl_b200 import engine as E

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"port": ("libmcl3dl_gl_oracle.so", "gl-port"),
           "reference": (os.path.join("_ref", "libmcl3dl_gl_ref.so"), "gl-ref"),
           "parity": (os.path.join("_ref", "global_localization_parity_test"), "gl-parity")}


def lib_path(kind):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "gl.mk"] + args + ref, capture_output=quiet, text=True)


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


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class GlChecker:
    """One loaded checker library ("port" or "reference")."""

    def __init__(self, kind="port"):
        path = lib_path(kind)
        if not os.path.exists(path):
            build(kind)
        self.lib = L = C.CDLL(path)
        self.kind = kind
        L.mcl3dl_cpu_gl_kind.restype = C.c_char_p
        assert L.mcl3dl_cpu_gl_kind().decode() == kind
        L.mcl3dl_cpu_gl_seed.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.mcl3dl_cpu_pf_resize_6dof.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]

    def gl_seed(self, ds, grid=0.3, div_yaw=12, imu_quat=(0, 0, 0, 1), dist_weight=(1, 1, 1)):
        """The service body over the downsampled cloud ds -> (states, probs) as STATE / float32 arrays."""
        ds = np.ascontiguousarray(ds, dtype=cc.POINT)
        q = np.ascontiguousarray(imu_quat, dtype=np.float32)
        w = np.ascontiguousarray(dist_weight, dtype=np.float32)
        n = C.c_size_t(0)
        rc = self.lib.mcl3dl_cpu_gl_seed(_ptr(ds), len(ds), grid, div_yaw, _ptr(q), _ptr(w), None, None, 0, C.byref(n))
        if rc != 0:
            raise RuntimeError("mcl3dl_cpu_gl_seed rc=%d" % rc)
        states = np.zeros(n.value, dtype=E.STATE)
        probs = np.zeros(n.value, dtype=np.float32)
        if n.value:
            rc = self.lib.mcl3dl_cpu_gl_seed(_ptr(ds), len(ds), grid, div_yaw, _ptr(q), _ptr(w), _ptr(states), _ptr(probs),
                                             n.value, C.byref(n))
            if rc != 0:
                raise RuntimeError("mcl3dl_cpu_gl_seed rc=%d" % rc)
        return states, probs

    def resize(self, states, probs, num):
        """resizeParticle(num) of (states, probs) -> (states, probs) of num particles."""
        states = np.ascontiguousarray(states, dtype=E.STATE)
        probs = np.ascontiguousarray(probs, dtype=np.float32)
        out_s = np.zeros(num, dtype=E.STATE)
        out_p = np.zeros(num, dtype=np.float32)
        rc = self.lib.mcl3dl_cpu_pf_resize_6dof(_ptr(probs), _ptr(states), len(states), num, _ptr(out_s), _ptr(out_p))
        if rc != 0:
            raise RuntimeError("mcl3dl_cpu_pf_resize_6dof rc=%d" % rc)
        return out_s, out_p
