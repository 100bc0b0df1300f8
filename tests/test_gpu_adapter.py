"""Runs the prebuilt host-C++-adapter parity binary (oracle/_ref/adapter_parity_test) on the GPU.

The binary is compiled by build() where a checkout of the reference exists, from its own
sources + oracle/shim + mcl_3dl_b200/host/lidar_measurement_model_b200.h and drives both model sets the
way MCL3dlNode::measure does (src/mcl_3dl.cpp:376-426): setGlobalLocalizationStatus, filter,
pf.measure(lambda), resample — three cycles, plus the node's dynamic_pointer_cast and a non-particle pose.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "adapter_parity_test")


@pytest.mark.gpu
@pytest.mark.parametrize("n_particles,caster", [(300, "dda"), (64, "dda"), (2049, "dda"), (300, "kd"), (64, "kd")])
def test_cpp_adapter_matches_reference_models(n_particles, caster):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/adapter_parity_test not built (needs a checkout of the reference at build time)")
    r = subprocess.run([BIN, str(n_particles), caster], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "ADAPTER PARITY OK" in r.stdout
