"""CPU-only checks of the drop-in boundary: the C-ABI library builds, loads, exports every symbol that
include/mcl3dl_b200.h declares, derives the beam parameters like the reference, and fails loudly
(no CPU fallback) when there is no CUDA device.  No compute calls are made here."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "mcl3dl_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mcl3dl_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from mcl_3dl_b200 import engine
    L = engine.load_library()
    names = declared_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(L, n), n
    assert sorted(engine.EXPORTED_SYMBOLS) == names
    assert L.mcl3dl_abi_version() == 3
    assert L.mcl3dl_strerror(-2).decode().startswith("measure()")


def test_struct_layouts_match_header():
    import ctypes as C
    from mcl_3dl_b200 import engine, synth
    assert synth.POINT.itemsize == 16 and synth.POSE.itemsize == 32 and synth.RESULT.itemsize == 24
    assert C.sizeof(engine.LikParams) == 24
    assert C.sizeof(engine.BeamParams) == 80
    assert C.sizeof(engine.MapInfo) == 88


@pytest.mark.parametrize("kw", [
    dict(),
    dict(num_points_default=27, hit_range=0.0, add_penalty_short_only_mode=False, dda_grid_size=0.1),
    dict(map_grid=(0.05, 0.1, 0.2), num_points_default=1024, beam_likelihood_min=0.35, hit_range=1.0,
         filter_label_max=1, ang_total_ref=1.2),
    dict(use_raycast_using_dda=False, num_points_default=7),
])
def test_beam_params_derivation_matches_oracle(port, kw):
    """mcl3dl_beam_params_from_reference == refreshParameters (beam.cpp:58-80) as restated by the oracle
    (which tests/test_oracle_golden.py pins to the reference build)."""
    from mcl_3dl_b200 import engine
    from oracle import cpu_checker as cc
    mine = engine.beam_params_from_reference(**kw)
    m = port.create(cc.points([[0, 0, 0], [1, 1, 1]]), None, cc.beam_raw(**kw))
    assert mine.as_tuple() == m.beam_params().as_tuple()


def test_no_cpu_fallback_without_device():
    import torch
    from mcl_3dl_b200 import engine
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine((0,))
    assert ei.value.code == -4


def test_product_package_never_touches_the_oracle():
    """The product path must not import, link or load anything under oracle/."""
    pkg = os.path.join(ROOT, "mcl_3dl_b200")
    bad = re.compile(r'#\s*include\s*[<"][^>"]*oracle|^\s*(from|import)\s+oracle|libmcl3dl_oracle|libmcl3dl_ref|'
                     r'cpu_checker|dlopen\([^)]*oracle', re.M)
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert not bad.search(txt), os.path.join(dirpath, f)
    import subprocess
    out = subprocess.run(["ldd", os.path.join(pkg, "libmcl3dl_b200.so")], capture_output=True, text=True).stdout
    assert "oracle" not in out and "mcl3dl_ref" not in out


def test_bench_byte_model():
    import bench
    assert bench.bytes_per_eval_model() == (1200, 75)            # SURVEY 8d: 5*5*3 cells at w=(1,1,5)
    assert bench.bytes_per_eval_model(w=(1, 1, 1)) == (2000, 125)


def test_bound_measure_call_resolves_buffers_once():
    """Engine.bind_measure hands mcl3dl_measure the addresses of the caller's own arrays (no hidden copies) and
    refuses arrays that would need one."""
    import numpy as np

    from mcl_3dl_b200 import engine, synth

    class FakeLib:
        def __init__(self):
            self.calls = []

        def mcl3dl_measure(self, *a):
            self.calls.append(a)
            return 0

    e = object.__new__(engine.Engine)
    e.L, e.h = FakeLib(), 1
    s = synth.scene(500, 8, 16, 4, seed=1)
    out = np.zeros(8, dtype=synth.RESULT)
    call = e.bind_measure(s["particles"], s["lik"], s["beam"], s["origins"], out)
    assert call() is out and call() is out
    a = e.L.calls[1]
    assert (a[2], a[4], a[6], a[8]) == (8, 16, 4, len(s["origins"]))
    assert a[1].value == s["particles"].ctypes.data and a[3].value == s["lik"].ctypes.data
    assert a[5].value == s["beam"].ctypes.data and a[9].value == out.ctypes.data
    lik_only = e.bind_measure(s["particles"], s["lik"], np.zeros(0, synth.POINT), None, out)
    lik_only()
    assert e.L.calls[-1][5] is None and e.L.calls[-1][6] == 0 and e.L.calls[-1][8] == 0
    with pytest.raises(ValueError):
        e.bind_measure(s["particles"][::2], s["lik"], None, None, out[:4])      # not contiguous
    with pytest.raises(ValueError):
        e.bind_measure(s["particles"], np.zeros(4, np.float32), None, None, out)  # wrong dtype
    with pytest.raises(ValueError):
        e.bind_measure(s["particles"], s["lik"], None, None, out[:4])           # one record per particle
    e.h = None  # nothing to destroy


def test_kernels_match_the_last_gpu_validated_fingerprint():
    """Informational guard: profiles/sass_fingerprint.txt holds per-kernel SASS hashes of the build that last passed the
    GPU suite on an H100.  A kernel that differs has not been validated on hardware yet: re-run the GPU suite, then
    regenerate the file (python profiles/sass_fingerprint.py > profiles/sass_fingerprint.txt).  Reported as xfail, never
    as a failure."""
    import shutil
    import sys
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, os.path.join(ROOT, "profiles"))
    import sass_fingerprint as sf
    from mcl_3dl_b200 import engine
    engine.load_library()   # builds if stale
    want = dict(line.split() for line in open(os.path.join(ROOT, "profiles", "sass_fingerprint.txt"))
                if line.strip() and not line.startswith("#"))
    got = sf.fingerprints(sf.DEFAULT)
    changed = sorted(k for k in got if k in want and want[k] != got[k])
    added = sorted(k for k in got if k not in want)
    # kernels that did not exist then (prepared variants: exchange, resident particle set, ...) are not regressions
    if changed:
        pytest.xfail("kernels changed since the last GPU-validated build: %d changed, %d new (%s)"
                     % (len(changed), len(added), ", ".join(n[:40] for n in changed[:4])))
