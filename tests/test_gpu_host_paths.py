"""The host-array entry points on a multi-device engine, on one GPU.

mcl3dl_create only range-checks device ids, so Engine((0, 0)) is two device contexts on the same H100, each with its own
stream, buffers and pinned block: the multi-device branches of mcl3dl_measure, mcl3dl_beam_status and
mcl3dl_measure_update (particles split into contiguous blocks, the weight total summed over the devices between two
host round trips) run without a second GPU.  Every case is held against Engine((0,)) on the same scene: each context
computes its block as a one-device engine computes that block, byte for byte.  The sizes straddle the engine's
zero-copy threshold (8192 particles per device: the kernels store records, posterior and summaries straight into the
pinned block), on the two-context and on the one-device engine, and the resident update takes the same rule.
"""
import numpy as np
import pytest

from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu

N_LIK, N_BEAM = 48, 8


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(scope="module")
def scene():
    return synth.scene(50_000, 16386, N_LIK, N_BEAM, seed=161)


@pytest.fixture(scope="module")
def engines(eng_mod, scene):
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=N_BEAM, dda_grid_size=0.2)
    one, two = eng_mod.Engine((0,)), eng_mod.Engine((0, 0))
    for e in (one, two):
        e.set_map(scene["map"], lik, beam)
    yield one, two
    one.close()
    two.close()


def by_shard(fn, P):
    """fn(lo, hi) for each non-empty block [P d / 2, P (d + 1) / 2) of the two contexts, concatenated."""
    return np.concatenate([fn(P * d // 2, P * (d + 1) // 2) for d in range(2) if P * (d + 1) // 2 > P * d // 2])


def prior_of(P, seed):
    return np.random.default_rng(seed).uniform(0.1, 1.0, P).astype(np.float32)


# per context: one empty block, both sides of the zero-copy threshold
@pytest.mark.parametrize("P", [1, 600, 16384, 16386])
def test_measure_and_beam_status(engines, scene, P):
    one, two = engines
    s = scene
    poses = s["particles"][:P]
    want = by_shard(lambda lo, hi: one.measure(poses[lo:hi], s["lik"], s["beam"], s["origins"]).copy(), P)
    assert two.measure(poses, s["lik"], s["beam"], s["origins"]).tobytes() == want.tobytes()
    want = by_shard(lambda lo, hi: one.beam_status(poses[lo:hi], s["beam"], s["origins"]), P)
    assert two.beam_status(poses, s["beam"], s["origins"]).tobytes() == want.tobytes()


@pytest.mark.parametrize("P,with_extra,want_records", [
    (1, False, True),          # one empty block
    (600, True, True),
    (600, False, False),
    (8192, False, True),       # one device: the kernels store posterior and summaries
    (8193, True, True),        # ... and above the threshold the D2H copies
    (16384, True, False),      # 8192 per context
    (16386, False, True),      # 8193 per context
])
def test_measure_update(engines, scene, P, with_extra, want_records):
    """Records byte-identical; posteriors, entropy and summary within the bars of the two-GPU test in test_gpu_parity.py
    (the total is summed in another order)."""
    one, two = engines
    s = scene
    poses = s["particles"][:P]
    prior = prior_of(P, P)
    extra = np.random.default_rng(P + 1).uniform(0.5, 1.0, P).astype(np.float32) if with_extra else None
    p1, s1, r1 = one.measure_update(poses, s["lik"], s["beam"], s["origins"], prior, extra, want_records=want_records)
    p2, s2, r2 = two.measure_update(poses, s["lik"], s["beam"], s["origins"], prior, extra, want_records=want_records)
    if want_records:
        assert r1.tobytes() == one.measure(poses, s["lik"], s["beam"], s["origins"]).tobytes()
        want = by_shard(lambda lo, hi: one.measure(poses[lo:hi], s["lik"], s["beam"], s["origins"]).copy(), P)
        assert r2.tobytes() == want.tobytes()
    else:
        assert r1 is None and r2 is None
    assert s1["kept"] == s2["kept"] == 1
    assert np.allclose(p1, p2, rtol=1e-6, atol=0) and abs(float(p1.sum(dtype=np.float64)) - 1.0) < 1e-4
    assert abs(s1["entropy"] - s2["entropy"]) < 1e-5 and s1["max_index"] == s2["max_index"]
    assert p1[s1["max_index"]] == p1.max() and p2[s2["max_index"]] == p2.max()
    assert s1["match_ratio_min"] == s2["match_ratio_min"] and s1["match_ratio_max"] == s2["match_ratio_max"]
    assert abs(s1["weight_sum"] - s2["weight_sum"]) <= 1e-6 * s1["weight_sum"]


@pytest.mark.parametrize("P", [1, 600])
def test_measure_update_restores_the_prior(engines, scene, P):
    """Nothing matches: both engines hand the prior back (kept == 0) with the same summary."""
    one, two = engines
    s = scene
    far = s["particles"][:P].copy()
    far["px"] += np.float32(1e4)
    prior = prior_of(P, 7)
    for e in (one, two):
        post, summ, _ = e.measure_update(far, s["lik"], s["beam"], s["origins"], prior)
        assert np.array_equal(post, prior)
        assert summ == {"weight_sum": 0.0, "match_ratio_min": 0.0, "match_ratio_max": 0.0, "entropy": 0.0, "kept": 0,
                        "max_index": 0}, summ


def states_of(poses):
    st = np.zeros(len(poses), dtype=synth.STATE)
    st["pos"] = np.stack([poses["px"], poses["py"], poses["pz"]], axis=1)
    st["rot"] = np.stack([poses[k] for k in ("qx", "qy", "qz", "qw")], axis=1)
    return st


@pytest.mark.parametrize("P", [8192, 8193])
def test_resident_update_on_both_sides_of_the_zero_copy_threshold(engines, scene, P):
    """The resident update equals mcl3dl_measure_update on the same poses and priors, bit for bit (no odometry term),
    whether the weight summaries come back as the kernels' own stores or as copies."""
    one, _ = engines
    s = scene
    poses = s["particles"][:P]
    prior = prior_of(P, 3 * P)
    want_post, want_summ, _ = one.measure_update(poses, s["lik"], s["beam"], s["origins"], prior)
    one.particles_set(states_of(poses), prior)
    summ = one.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.0)
    _, post = one.particles_get()
    assert summ["kept"] == 1 and summ == want_summ
    assert post.tobytes() == want_post.tobytes()


def test_kernel_launches_per_call(engines, scene):
    """Launches of one call, per device context with particles: mcl3dl_measure 2 (beam + likelihood kernel),
    mcl3dl_beam_status 1, mcl3dl_measure_update 4 (both models, weight_kernel, normalize_kernel; on several devices the
    normalise pass only runs when something is kept: 3), the resident update 5 (pose pack + 4)."""
    one, two = engines
    s = scene

    def launches(e, fn):
        n0 = e.kernel_launches()
        fn()
        return e.kernel_launches() - n0

    def calls(e, P):
        poses = s["particles"][:P]
        far = poses.copy()
        far["px"] += np.float32(1e4)
        prior = prior_of(P, 11)
        return [launches(e, lambda: e.measure(poses, s["lik"], s["beam"], s["origins"])),
                launches(e, lambda: e.beam_status(poses, s["beam"], s["origins"])),
                launches(e, lambda: e.measure_update(poses, s["lik"], s["beam"], s["origins"], prior)),
                launches(e, lambda: e.measure_update(far, s["lik"], s["beam"], s["origins"], prior))]

    assert calls(one, 600) == [2, 1, 4, 4]
    assert calls(two, 600) == [4, 2, 8, 6]
    assert calls(two, 1) == [2, 1, 4, 3]
    poses = s["particles"][:600]
    one.particles_set(states_of(poses), prior_of(600, 11))
    assert launches(one, lambda: one.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.0)) == 5
