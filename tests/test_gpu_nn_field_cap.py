"""MCL3DL_NNF_MAX_MB caps the NN field's directory + candidates.  The directory and the near bits are known before the
count pass, the candidates only after it: a cap between the two drops the field after the count pass, and the
CSR-window search serves the map as if the field had never been asked for (MCL3DL_NNF=0)."""
import numpy as np
import pytest

from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


def test_field_dropped_after_the_count_pass(eng_mod, monkeypatch):
    s = synth.scene(100_000, 600, 64, 0, seed=171)
    lik = eng_mod.LikParams()

    def engine_with(**env):
        for k in ("MCL3DL_NNF", "MCL3DL_NNF_MAX_MB"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = eng_mod.Engine((0,))  # (the switches are read when the engine is created)
        e.set_map(s["map"], lik, None)
        return e

    full = engine_with()
    info = full.nn_field_info()
    assert info["bytes"] > 0
    # bytes = directory (8 B per cell) + candidates (16 B each) + wide-cell table (16 B per cell, at most 2^18 cells)
    rest = info["bytes"] - 16 * info["candidates"]
    directory = rest // 3 if rest <= 3 << 21 else rest - (1 << 22)
    # the near bits are one bit per fine voxel (8 per cell) rounded up to 32-bit rows: below a quarter of the directory
    cap_mb = -(-(directory + directory // 4) // (1 << 20))
    assert cap_mb << 20 < directory + 16 * info["candidates"], "no cap separates the two checks on this map"

    capped = engine_with(MCL3DL_NNF_MAX_MB=str(cap_mb))
    plain = engine_with(MCL3DL_NNF="0")
    assert capped.nn_field_info()["bytes"] == 0 and plain.nn_field_info()["bytes"] == 0
    want = plain.measure(s["particles"], s["lik"]).copy()
    assert capped.measure(s["particles"], s["lik"]).tobytes() == want.tobytes()
    assert capped.map_info().device_bytes == plain.map_info().device_bytes
    # a second map on the same engine is built and dropped the same way
    capped.set_map(s["map"], lik, None)
    assert capped.nn_field_info()["bytes"] == 0
    assert capped.measure(s["particles"], s["lik"]).tobytes() == want.tobytes()
    # the uncapped engine finds the same matches (its kernel may sum the likelihood terms in another order)
    assert np.array_equal(full.measure(s["particles"], s["lik"])["match_cnt"], want["match_cnt"])
    assert want["match_cnt"].sum() > 0
    for e in (full, capped, plain):
        e.close()
