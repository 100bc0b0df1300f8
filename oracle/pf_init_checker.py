"""ctypes binding of oracle/pf_init_api.h — TEST INFRASTRUCTURE ONLY.

The CPU checkers of the resident set's initial seed (pf::ParticleFilter::initUsingNoiseGenerator with the configured
start's DiagonalNoiseGenerator, src/mcl_3dl.cpp:1276, and cbPosition's MultivariateNoiseGenerator, :155-198), built by
oracle/pf_init.mk:
  kind="port"       oracle/libmcl3dl_pf_init_oracle.so   (repo-owned restatement, always available)
  kind="reference"  oracle/_ref/libmcl3dl_pf_init_ref.so (the reference's own code, built where a checkout of the
                    reference exists)
  kind="parity"     oracle/_ref/init_parity_test (the configured start, cbPosition and a predict / measure / resample
                    cycle through the C++ adapter vs the reference filter; H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import cpu_checker as cc
from mcl_3dl_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"port": ("libmcl3dl_pf_init_oracle.so", "pf-init-port"),
           "reference": (os.path.join("_ref", "libmcl3dl_pf_init_ref.so"), "pf-init-ref"),
           "parity": (os.path.join("_ref", "init_parity_test"), "init-parity")}


def lib_path(kind):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "pf_init.mk"] + args + ref, capture_output=quiet, text=True)


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


class PfInitChecker:
    """One loaded checker library ("port" or "reference")."""

    def __init__(self, kind="port"):
        path = lib_path(kind)
        if not os.path.exists(path):
            build(kind)
        self.lib = L = C.CDLL(path)
        self.kind = kind
        L.mcl3dl_cpu_pf_init_kind.restype = C.c_char_p
        assert L.mcl3dl_cpu_pf_init_kind().decode() == kind
        vp = C.c_void_p
        L.mcl3dl_cpu_pf_init_mean.argtypes = [vp, vp]
        L.mcl3dl_cpu_pf_init.argtypes = [C.c_size_t, C.c_int, vp, vp, vp, vp, vp, vp]
        L.mcl3dl_cpu_pf_init_transform.argtypes = [vp, vp]

    def mean(self, pose7):
        """NoiseGeneratorBase::setMean(State6DOF(pose)): (x y z roll pitch yaw) float32."""
        p = np.ascontiguousarray(pose7, dtype=np.float32).reshape(7)
        out = np.zeros(6, np.float32)
        assert self.lib.mcl3dl_cpu_pf_init_mean(_ptr(p), _ptr(out)) == 0
        return out

    def init(self, pose7, z, sigma=None, norm_transform=None):
        """-> (states, probs) of initUsingNoiseGenerator on len(z) particles with the standard normals z [n, 6]."""
        p = np.ascontiguousarray(pose7, dtype=np.float32).reshape(7)
        z = np.ascontiguousarray(z, dtype=np.float32).reshape(-1, 6)
        mv = norm_transform is not None
        sg = None if mv else np.ascontiguousarray(sigma, dtype=np.float32).reshape(6)
        t = np.ascontiguousarray(norm_transform, dtype=np.float32).reshape(36) if mv else None
        states = np.zeros(len(z), synth.STATE)
        probs = np.zeros(len(z), np.float32)
        rc = self.lib.mcl3dl_cpu_pf_init(len(z), int(mv), _ptr(p), _ptr(sg), _ptr(t), _ptr(z), _ptr(states), _ptr(probs))
        assert rc == 0, rc
        return states, probs

    def transform(self, covariance):
        """norm_transform_ [6, 6] of MultivariateNoiseGenerator<float>(mean, covariance) (reference tier only)."""
        cov = np.ascontiguousarray(covariance, dtype=np.float64).reshape(36)
        out = np.zeros(36, np.float32)
        rc = self.lib.mcl3dl_cpu_pf_init_transform(_ptr(cov), _ptr(out))
        assert rc == 0, rc
        return out.reshape(6, 6)
