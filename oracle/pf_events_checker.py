"""ctypes binding of oracle/pf_events_api.h — TEST INFRASTRUCTURE ONLY.

The CPU checkers of the node's odometry-noise redraw (src/mcl_3dl.cpp:817-825), expansion resetting's noise
(pf::ParticleFilter::addNoiseUsingNoiseGenerator, pf.h:226-237) and the IMU gravity update
(ImuMeasurementModelGravity inside pf::ParticleFilter::measure), built by oracle/pf_events.mk:
  kind="port"       oracle/libmcl3dl_pf_events_oracle.so   (repo-owned restatement, always available)
  kind="reference"  oracle/_ref/libmcl3dl_pf_events_ref.so (the reference's own code on replayed draws, built where a
                    checkout of the reference exists)
  kind="parity"     oracle/_ref/pf_events_parity_test (resident cycles through the C++ adapter with IMU updates, the
                    redraw and expansion resetting vs the reference filter fed the same draws; H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import cpu_checker as cc
from mcl_3dl_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"port": ("libmcl3dl_pf_events_oracle.so", "pf-events-port"),
           "reference": (os.path.join("_ref", "libmcl3dl_pf_events_ref.so"), "pf-events-ref"),
           "parity": (os.path.join("_ref", "pf_events_parity_test"), "pf-events-parity")}


def lib_path(kind):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "pf_events.mk"] + args + ref, capture_output=quiet, text=True)


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


class PfEventsChecker:
    """One loaded checker library ("port" or "reference")."""

    def __init__(self, kind="port"):
        path = lib_path(kind)
        if not os.path.exists(path):
            build(kind)
        self.lib = L = C.CDLL(path)
        self.kind = kind
        L.mcl3dl_cpu_pf_events_kind.restype = C.c_char_p
        assert L.mcl3dl_cpu_pf_events_kind().decode() == kind
        d = C.c_double
        L.mcl3dl_cpu_pf_redraw.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, d, d, d, d]
        L.mcl3dl_cpu_pf_noise.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        L.mcl3dl_cpu_pf_imu.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, d, C.c_void_p,
                                        C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_float)]

    def redraw(self, states, z, lin_lin, lin_ang, ang_lin, ang_ang):
        """states after the node's redraw with the standard normals z [n, 4] (draw order ll, la, aa, al)."""
        out = np.ascontiguousarray(states, dtype=synth.STATE).copy()
        z = np.ascontiguousarray(z, dtype=np.float32)
        assert z.shape == (len(out), 4)
        rc = self.lib.mcl3dl_cpu_pf_redraw(_ptr(out), len(out), _ptr(z), lin_lin, lin_ang, ang_lin, ang_ang)
        assert rc == 0, rc
        return out

    def noise(self, states, org):
        """states after addNoiseUsingNoiseGenerator with the draws org [n, 6] (already times sigma)."""
        out = np.ascontiguousarray(states, dtype=synth.STATE).copy()
        org = np.ascontiguousarray(org, dtype=np.float32)
        assert org.shape == (len(out), 6)
        rc = self.lib.mcl3dl_cpu_pf_noise(_ptr(out), len(out), _ptr(org))
        assert rc == 0, rc
        return out

    def imu(self, states, probs, acc, acc_var):
        """-> (probs after pf_->measure, likelihoods, kept, float sum, entropy)."""
        states = np.ascontiguousarray(states, dtype=synth.STATE)
        p = np.ascontiguousarray(probs, dtype=np.float32).copy()
        a = np.ascontiguousarray(acc, dtype=np.float32)
        lik = np.zeros(len(states), np.float32)
        kept, s, ent = C.c_int(0), C.c_float(0), C.c_float(0)
        rc = self.lib.mcl3dl_cpu_pf_imu(_ptr(states), _ptr(p), len(states), _ptr(a), acc_var, _ptr(lik), C.byref(kept),
                                        C.byref(s), C.byref(ent))
        assert rc == 0, rc
        return p, lik, bool(kept.value), np.float32(s.value), np.float32(ent.value)
