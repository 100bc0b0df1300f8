"""Build hook of oracle/map_intake.mk — TEST INFRASTRUCTURE ONLY.

The adapter parity program of the map intake (include/mcl3dl_b200.h: mcl3dl_map_load):
  kind="parity"  oracle/_ref/map_intake_parity_test  (the node's map callbacks on its restated host path and through the
                 C++ adapter's intake methods, with the reference's own models; built where a checkout of the reference
                 exists, as for cpu_checker's "reference"; one process, H100)

Only tests/, __graft_entry__.build() and profiles/ may import this module.  The product package never does.
"""
import os
import subprocess

from oracle import cpu_checker as cc

HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = {"parity": (os.path.join("_ref", "map_intake_parity_test"), "map-intake-parity")}


def lib_path(kind="parity"):
    return os.path.join(HERE, TARGETS[kind][0])


def _make(args, quiet=True):
    ref = ["REFERENCE=" + cc.REFERENCE] if cc.REFERENCE else []
    return subprocess.run(["make", "-C", HERE, "-f", "map_intake.mk"] + args + ref, capture_output=quiet, text=True)


def build(kind="parity", quiet=True):
    """Compile if missing or stale from the reference's checkout; where there is none, only report whether an earlier
    build exists."""
    path = lib_path(kind)
    if _make(["-s", "has-ref"]).returncode != 0:
        return os.path.exists(path)
    r = _make([TARGETS[kind][1]], quiet)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + (r.stdout or "") + (r.stderr or ""))
    return os.path.exists(path)


def available(kind="parity"):
    return os.path.exists(lib_path(kind))
