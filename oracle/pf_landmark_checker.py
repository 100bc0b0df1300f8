"""ctypes binding of oracle/pf_landmark_api.h — TEST INFRASTRUCTURE ONLY.

The CPU checkers of the node's landmark update (cbLandmark's pf_->measure, src/mcl_3dl.cpp:899-931), the odometry-error
reset (integ_reset_func, :190-195,653-658) and publishParticles' normalised poses (:1101-1125), built by
oracle/pf_landmark.mk:
  kind="port"       oracle/libmcl3dl_pf_landmark_oracle.so   (repo-owned restatement, always available)
  kind="reference"  oracle/_ref/libmcl3dl_pf_landmark_ref.so (the reference's own code, built where a checkout of the
                    reference exists)
  kind="parity"     oracle/_ref/landmark_parity_test (a resident cycle, cbLandmark, a pose-jump reset and the published
                    poses through the C++ adapter vs the reference filter; H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import cpu_checker as cc
from mcl_3dl_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"port": ("libmcl3dl_pf_landmark_oracle.so", "pf-landmark-port"),
           "reference": (os.path.join("_ref", "libmcl3dl_pf_landmark_ref.so"), "pf-landmark-ref"),
           "parity": (os.path.join("_ref", "landmark_parity_test"), "landmark-parity")}


def lib_path(kind):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "pf_landmark.mk"] + args + ref, capture_output=quiet, text=True)


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


def measured7(measured):
    """(x, y, z, qx, qy, qz, qw) float32 of one POSE (or of 7 numbers)."""
    m = np.asarray(measured)
    if m.dtype == synth.POSE:
        m = m.reshape(1)[0]
        return np.array([m["px"], m["py"], m["pz"], m["qx"], m["qy"], m["qz"], m["qw"]], np.float32)
    return np.ascontiguousarray(m, dtype=np.float32).reshape(7)


class PfLandmarkChecker:
    """One loaded checker library ("port" or "reference")."""

    def __init__(self, kind="port"):
        path = lib_path(kind)
        if not os.path.exists(path):
            build(kind)
        self.lib = L = C.CDLL(path)
        self.kind = kind
        L.mcl3dl_cpu_pf_landmark_kind.restype = C.c_char_p
        assert L.mcl3dl_cpu_pf_landmark_kind().decode() == kind
        vp = C.c_void_p
        L.mcl3dl_cpu_pf_landmark.argtypes = [vp, vp, C.c_size_t, vp, C.c_float, vp, vp, C.POINTER(C.c_int),
                                             C.POINTER(C.c_float), C.POINTER(C.c_float)]
        L.mcl3dl_cpu_pf_reset_odom_err.argtypes = [vp, C.c_size_t]
        L.mcl3dl_cpu_pf_poses.argtypes = [vp, C.c_size_t, vp]

    def landmark(self, states, probs, measured, nd_a, sigma_inv):
        """-> (probs after pf_->measure, likelihoods, kept, float sum, entropy)."""
        states = np.ascontiguousarray(states, dtype=synth.STATE)
        p = np.ascontiguousarray(probs, dtype=np.float32).copy()
        m = measured7(measured)
        si = np.ascontiguousarray(sigma_inv, dtype=np.float32).reshape(36)
        lik = np.zeros(len(states), np.float32)
        kept, s, ent = C.c_int(0), C.c_float(0), C.c_float(0)
        rc = self.lib.mcl3dl_cpu_pf_landmark(_ptr(states), _ptr(p), len(states), _ptr(m), nd_a, _ptr(si), _ptr(lik),
                                             C.byref(kept), C.byref(s), C.byref(ent))
        assert rc == 0, rc
        return p, lik, bool(kept.value), np.float32(s.value), np.float32(ent.value)

    def reset_odom_err(self, states):
        out = np.ascontiguousarray(states, dtype=synth.STATE).copy()
        assert self.lib.mcl3dl_cpu_pf_reset_odom_err(_ptr(out), len(out)) == 0
        return out

    def poses(self, states):
        states = np.ascontiguousarray(states, dtype=synth.STATE)
        out = np.zeros(len(states), synth.POSE)
        assert self.lib.mcl3dl_cpu_pf_poses(_ptr(states), len(states), _ptr(out)) == 0
        return out
