"""Runs the prebuilt map-update parity program (oracle/_ref/map_update_parity_test) on the GPU.

Built by build() where a checkout of the reference exists (oracle/map_update.mk): measurement cycles of the reference
models and the host C++ adapter, then the node's map update timer (src/mcl_3dl.cpp:1350-1378, pc_map2_ aliasing
pc_map_) and more cycles.  They agree at every cycle, and the adapter took every update as an append.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "map_update_parity_test")


@pytest.mark.gpu
@pytest.mark.parametrize("n_particles,caster", [(300, "dda"), (64, "kd"), (600, "kd")])
def test_map_updates_through_the_adapter_match_reference_models(n_particles, caster):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/map_update_parity_test not built (needs a checkout of the reference at build time)")
    r = subprocess.run([BIN, str(n_particles), caster], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "MAP UPDATE PARITY OK" in r.stdout
    assert "3 appended, 1 staged whole" in r.stdout
