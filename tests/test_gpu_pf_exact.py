"""The resident particle set (mcl3dl_particles_*) against the host restatement of its own per-particle functions, and
its sums against exact sums.

tests/hostsim/pf_hostsim.cpp compiles pf_funcs.cuh for the host; test_hostsim.py pins those functions bit for bit to
the oracle port, which test_oracle_golden.py pins to the reference build.  So every difference between a kernel and
the host restatement comes either from the kernel's own plumbing (indexing, grid-stride loops, folds, counters, stream
order) or from the seven libm functions the device evaluates with its own code.

libm.  Everything in pf_funcs.cuh is explicit round-to-nearest arithmetic except sinf, cosf, logf, expf, acosf, asinf
and atan2f.  Their maximum errors, in ulps of the result, are those of the CUDA Math API's table of single-precision
functions (CUDA C++ Programming Guide, "Mathematical Functions", without -use_fast_math): sinf 2, cosf 2, expf 2,
logf 1, acosf 2, asinf 2, atan2f 3; glibc's manual ("Known Maximum Errors in Math Functions", x86_64) lists at most 1
ulp for each of them.  A bar that involves one of them adds the two (LIBM below) and carries the difference through the
round-to-nearest operations that follow, each of which may then round the other way (one more ulp).  Below, u = 2^-24
and a relative ulp is at most 2^-23.

Exact sums.  Every float is an integer multiple of 2^-149, so exact_row_sums (test_gpu_lik_exact.py) returns Σ of a
column exactly.  The estimate and weight kernels add doubles with a fixed tree: a thread's grid-stride iterations in
order, 5 xor-shuffle levels, the 8 warps of the CTA in order (7 adds) and the CTAs' slots in order (slots - 1 adds).
So a term passes through at most D additions, and the double result is within γ_D Σ|terms| of the exact sum, γ_D =
D 2^-53 / (1 - D 2^-53) (Higham, Accuracy and Stability of Numerical Algorithms, Lemma 3.1).  (The host restatement
in tests/fake_engine.py adds in particle order, so there D = n.)  D is far below 2^29, so the double rounded to float equals float(exact) unless the exact value lies within the bound
of a float rounding boundary; each case asserts from exact arithmetic that it does not (to_f32), and the comparisons
are then equalities.  G = 4 sm_count 256 is the particle count above which a thread runs a second grid-stride
iteration: the estimate and weight kernels both launch min(ceil(n / 256), 4 sm_count) CTAs of 256 threads.

1. Predict (pf_predict_kernel) against hostsim_pf_predict: pos, odom_err_integ_lin/ang and noise_* bit for bit; rot
   bit for bit where yaw_diff == 0 (sinf(±0) and cosf(0) are exact).  Elsewhere |Δrot| <= PREDICT_ROT_BAR per
   component: sinf / cosf of the half angle differ by at most 3 ulp (<= 3 2^-23, the values are <= 1); the map from
   (sin, cos) through the normalisation, two Hamilton products with |rot| <= 1.02 and the final normalisation has
   Lipschitz constant <= 1.1, so that difference moves the result by <= 1.1 sqrt(2) 3 2^-23 < 5 2^-23; on top of that
   each side's own rounding against exact arithmetic is <= 21 u (6 u per normalisation, 4 u per product component)
   and the two sides may round apart: 5 2^-23 + 21 2^-23 = 26 2^-23.
2. Resample (pf_accum_kernel + pf_resample_kernel) against hostsim_pf_resample_philox with the same initial_frac,
   seed and call number.  An Engine numbers its resampling calls from 1; particles_set does not reset the count.
   Output probabilities, plain copies and past-the-end copies bit for bit (hostsim's src / dup say which outputs those
   are).  Duplicates: noise_* exactly 0; every component whose sigma is 0 bit for bit; pos, lin and ang within
   ulp(value) + ORG_REL |org|: org = rad cos(phi) sigma with rad = sqrt(-2 logf(u)): logf 2 ulp (halved by the square
   root, which adds 1), cosf / sinf 3, two products 1 each: ORG_REL = 7 2^-23.  rot within RESAMPLE_ROT_BAR: each of
   the six half-angle cos / sin differs by <= 3 2^-23 (plus ORG_REL |org| / 2 through its argument), a component of
   the noise quaternion is a sum of two triple products (<= 2 x 3 x 3 2^-23 = 18 2^-23) plus its own 5 roundings per
   side (5 2^-23 for both); the product with rot (|rot| <= 1.02, four components: x 2.1) and the normalisation add
   10 2^-23 of rounding for both sides: 2.1 x 23 + 10 < 60 2^-23.
3. Estimate (pf_est_* kernels) against exact sums of hostsim_pf_est_terms / hostsim_pf_cov_terms (the float terms the
   kernels add).  Without prev (bias 1) every term is exact device arithmetic: weight_sum_biased = float(exact Σw),
   the mean_biased position = float(exact ratio), the position block of cov (j, k < 3) = float(exact Σ term / exact Σp)
   around the centre float(exact ratio) (a ratio of two doubles each within γ_D of its sum is within the sum of their
   relative bounds plus 2^-52 of the exact ratio).  The mean rotation, pf_quat_from_front_up of double sums, is within
   1 ulp of that function applied to the exact sums (the generators keep every quaternion component well away from
   0, where the square roots would amplify).  The angle rows of cov: each particle's RPY goes through atan2f (4 ulp
   apart) or asinf (3), the centre's too (plus 16 u for a 1-ulp difference of its quaternion), the difference and the
   ±2π wrap may each round apart (2 ulp(d)); the bar is Σ p (Δd_j |d_k| + |d_j| Δd_k + Δd_j Δd_k) + 4 u Σ|term|
   (two roundings per side) over Σp, plus the tree bound and ulp(cov).  The generators keep every wrapped difference
   at least 1e-3 away from ±π and still cross the wrap with a yaw near π.  With prev, pf_bias passes through acosf and
   two expf; their propagated relative bound ε_i on each w_i (see bias_rel_bound) bounds weight_sum_biased and the
   means.  In one generator the positions are ±1e5 by parity, so the sums cancel: a thread's partial is ~10^5 times
   the mean, and rounding the running partials to float would move the mean by several ulps.  max_index and max_state
   exactly: the first index of the largest probability, with ties in two lanes of a
   warp, two warps of a CTA, CTA 0's second grid-stride iteration against a later CTA's first, all equal, at n - 1
   and all zero.
4. The weight fold (weight_kernel -> normalize_kernel -> make_summary) through measure_update and the resident update:
   with w_i = prior ((1 beam) like) in float and S = exact Σw, weight_sum = float(S) and every posterior =
   fdiv(w_i, float(S)) bit for bit; match_ratio_min / max exactly; max_index the first index of the largest posterior;
   entropy within Σ (2 p ulp(ln p) + ulp(p ln p)) (logf 1 + glibc 1, then the product) plus the tree bound and
   ulp(entropy).  With an odometry sigma > 0, pf_pack_kernel's factor goes through expf: w_i is within 6 2^-23
   relative (expf 3, three products 1 each), the posterior within 2 x 6 2^-23 + 3 2^-23 relative (w, S, the rounding
   of S and the division).  One case is built so that S rounds up to float: rounding the total toward zero cannot pass.
5. A cycle: four rounds of predict -> resident update -> resample -> estimate on one engine without reading back, and
   the same on a second engine with particles_get after every step, each step held to the bars above against the host
   operation applied to the state read back from the step before.  The two engines' final states are byte-identical.
"""
import ctypes as C
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from test_gpu_lik_exact import exact_row_sums, half_ulp
from test_hostsim import hostsim  # noqa: F401  (builds tests/hostsim/libhostsim.so)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_LIB = os.path.join(ROOT, "tests", "hostsim", "libhostsim.so")
LIBM = {"sinf": 2 + 1, "cosf": 2 + 1, "expf": 2 + 1, "logf": 1 + 1, "acosf": 2 + 1, "asinf": 2 + 1, "atan2f": 3 + 1}
R = 2.0 ** -23  # a relative ulp is at most this
U = 2.0 ** -24
PREDICT_ROT_BAR = 26 * R
ORG_REL = (LIBM["logf"] / 2 + 1 + LIBM["cosf"] + 2) * R
RESAMPLE_ROT_BAR = 60 * R
NON_STATE_FIELDS = ("pos", "noise_ll", "noise_la", "noise_al", "noise_aa", "odom_err_integ_lin", "odom_err_integ_ang")


# ------------------------------------------------------------------ fixtures and helpers
@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def hs():
    L = C.CDLL(HS_LIB)
    vp, sz, f = C.c_void_p, C.c_size_t, C.c_float
    L.hostsim_pf_predict.argtypes = [vp, vp, f, f, f, vp, sz]
    L.hostsim_pf_resample_philox.argtypes = [vp, vp, sz, f, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp, vp, vp]
    L.hostsim_pf_est_terms.argtypes = [vp, vp, sz, vp, f, f, vp, vp]
    L.hostsim_pf_est_finish.argtypes = [vp, vp, vp, vp, vp]
    L.hostsim_pf_est_finish.restype = None
    L.hostsim_pf_cov_terms.argtypes = [vp, vp, sz, vp, vp, vp, vp]
    return L


def G(sm):
    return 4 * sm * 256


def size(spec, sm):
    """(k, off) -> k G + off; an int stands for itself."""
    return spec if isinstance(spec, int) else spec[0] * G(sm) + spec[1]


def depth(n, sm, E):
    """The longest addition chain of the estimate / weight folds of n particles (n for a sequential restatement)."""
    if getattr(E, "SEQUENTIAL_SUMS", False):
        return n
    grid = min(-(-n // 256), 4 * sm)
    return -(-n // (grid * 256)) + 5 + 7 + grid - 1


def gamma(D):
    return Fraction(D, (1 << 53) - D)


def to_f32(x, err):
    """float32 nearest to the Fraction x, asserting that no value within err of x rounds differently."""
    err = max(Fraction(err), abs(x) / (1 << 52))
    f = np.float32(float(x))
    lo, hi = np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))
    F = Fraction(float(f))
    assert (Fraction(float(lo)) + F) / 2 + err < x < (F + Fraction(float(hi))) / 2 - err, (float(x), float(err))
    return f


def ratio_err(A, a_abs, B, b_abs, D):
    """Bound on |double(A_d / B_d) - A / B| for double sums A_d, B_d within γ_D of A, B (terms with Σ|.| = a_abs, b_abs)."""
    g = gamma(D)
    return (g * Fraction(a_abs) + abs(A / B) * g * Fraction(b_abs)) / abs(B) * Fraction(101, 100) + abs(A / B) / (1 << 52)


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def col_sums(T):
    """Exact column sums of a float32 matrix [n, k] and the float64 sums of |T| (slightly rounded up)."""
    return exact_row_sums(np.ascontiguousarray(T.T)), np.abs(T.astype(np.float64)).sum(0) * (1 + 1e-9)


def fresh(E):
    return E.Engine((0,))


# ------------------------------------------------------------------ 1. predict
def predict_states(n, seed, zero_yaw_noise=False):
    rng = np.random.default_rng(seed)
    st = np.zeros(n, dtype=synth.STATE)
    st["pos"] = rng.uniform(-20, 20, (n, 3))
    q = rng.normal(0, 1, (n, 4))
    st["rot"] = q / np.linalg.norm(q, axis=1, keepdims=True) * rng.uniform(0.98, 1.02, (n, 1))   # rot_ is not exactly unit
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        st[f] = rng.normal(0, 0.05, n)
    st["odom_err_integ_lin"] = rng.normal(0, 0.1, (n, 3))
    st["odom_err_integ_ang"] = rng.normal(0, 0.1, (n, 3))
    # signed zeros: the byte comparison sees their sign
    st["pos"][::7, 1] = -0.0
    st["pos"][3::7, 2] = 0.0
    st["odom_err_integ_lin"][::5, 2] = -0.0
    st["odom_err_integ_ang"][1::5, 0] = -0.0
    st["noise_al"][::6] = -0.0
    st["noise_ll"][2::6] = -0.0
    st["noise_la"][::4] = -0.0       # yaw_diff = ±0 on every 4th particle
    st["noise_aa"][::4] = 0.0
    if zero_yaw_noise:
        st["noise_la"] = 0.0
        st["noise_aa"] = 0.0
    return st


def cutoff_floats():
    """The two floats either side of getAxisAng's cut-off |w| >= 1 - 1e-6 (compared in double)."""
    f = np.float32(1.0 - 1e-6)
    below = f if float(f) < 1.0 - 1e-6 else np.nextafter(f, np.float32(0))
    return below, np.nextafter(below, np.float32(2))


def odometry(kind):
    """(prev, cur, time_diff, still): the odometry pair of a predict case."""
    ident = np.array([[0.0, 0.0, 0.0, 1.0]], np.float32)
    prev = synth.make_poses([[1.0, 2.0, 0.1]], synth.quat_from_rpy([[0.02, -0.01, 0.4]]))
    if kind == "still":
        return prev, prev.copy(), 0.1, True
    if kind == "dt0":
        cur = synth.make_poses([[1.3, 2.1, 0.1]], synth.quat_from_rpy([[0.01, 0.03, 0.7]]))
        return prev, cur, 0.0, False
    if kind in ("w_below", "w_above"):
        w = cutoff_floats()[0 if kind == "w_below" else 1]
        q = np.array([[0.0, 0.0, np.sqrt(np.float32(1) - w * w), w]], np.float32)
        return synth.make_poses([[0.0, 0.0, 0.0]], ident), synth.make_poses([[0.2, -0.1, 0.0]], q), 0.1, False
    turn = float(kind)
    cur = synth.make_poses([[1.2, 1.9, 0.1]], synth.quat_from_rpy([[0.01, 0.03, 0.4 + turn]]))
    return prev, cur, 0.1, False


def check_predict(got, want, st):
    """got / want: STATE arrays after the predict of st."""
    for f in NON_STATE_FIELDS:
        assert got[f].tobytes() == want[f].tobytes(), f
    exact = (st["noise_la"] == 0) & (st["noise_aa"] == 0)
    assert got["rot"][exact].tobytes() == want["rot"][exact].tobytes()
    d = np.abs(got["rot"].astype(np.float64) - want["rot"])
    assert d.max(initial=0.0) <= PREDICT_ROT_BAR, d.max()


def host_predict(st, prev, cur, dt):
    out = np.ascontiguousarray(st.copy())
    assert hs().hostsim_pf_predict(_ptr(prev), _ptr(cur), dt, 10.0, 7.0, _ptr(out), len(out)) == 0
    return out


def predict_case(E, sm, n, kind, zero_yaw_noise=False, seed=5):
    n = size(n, sm)
    st = predict_states(n, seed, zero_yaw_noise)
    prev, cur, dt, still = odometry(kind)
    e = fresh(E)
    e.particles_set(st, np.full(n, 1.0 / n, np.float32))
    e.particles_predict(prev, cur, dt, 10.0, 7.0)
    got, _ = e.particles_get()
    e.close()
    want = host_predict(st, prev, cur, dt)
    if still or zero_yaw_noise:
        assert got.tobytes() == want.tobytes()
    check_predict(got, want, st)
    return got, want


PREDICT_CASES = [(1, "0.3"), (255, "0.3"), (256, "-2.9"), (257, "0.3"), ((0, (1 << 20) + 3), "3.1"),
                 (4099, "0.0"), (4099, "3.1"), (4099, str(math.pi - 1e-3)), (4099, str(-(math.pi - 1e-3))),
                 (4099, "w_below"), (4099, "w_above"), (4099, "dt0"), (4099, "still")]


@pytest.mark.parametrize("n,kind", PREDICT_CASES)
def test_predict(eng_mod, sm, hostsim, n, kind):  # noqa: F811
    predict_case(eng_mod, sm, n, kind)


@pytest.mark.parametrize("kind", ["0.3", "3.1", "w_below"])
def test_predict_without_yaw_noise_is_bit_exact(eng_mod, sm, hostsim, kind):  # noqa: F811
    predict_case(eng_mod, sm, 4099, kind, zero_yaw_noise=True)


def test_predict_cutoff_floats_straddle_the_threshold():
    below, above = cutoff_floats()
    assert float(below) < 1.0 - 1e-6 <= float(above) and np.nextafter(below, np.float32(2)) == above


# ------------------------------------------------------------------ 2. resample
def resample_states(n, seed):
    """Distinct positions (x = i / 1024), so that a wrong pick moves a particle by >= 8 ulp of x."""
    rng = np.random.default_rng(seed)
    st = predict_states(n, seed)
    st["pos"][:, 0] = np.arange(n, dtype=np.float64) / 1024.0
    st["pos"][:, 1] = -(np.arange(n) % 1000) * 0.01
    st["pos"][:, 2] = rng.normal(0, 1, n)
    return st


def resample_probs(n, kind, seed):
    rng = np.random.default_rng(seed)
    p = (rng.uniform(0.2, 1.0, n) ** 2).astype(np.float32)
    if kind == "ties":       # zero weights and weights below half an ulp of the running sum: tie groups
        p[rng.uniform(size=n) < 0.2] = 0.0
        tiny = rng.uniform(size=n) < 0.2
        tiny[:n // 8] = False
        p[tiny] = np.float32(1e-12)
    if kind == "one":
        p[:] = 0.0
        p[rng.integers(0, n)] = 0.7
    p = (p / p.sum(dtype=np.float64)).astype(np.float32)
    if kind == "total3.7":
        p = (p * np.float32(3.7)).astype(np.float32)
    if kind == "total1e-30":
        p = (p * np.float32(1e-30)).astype(np.float32)
    return p


SIGMA_POS = np.array([0.05, 0.0, 0.02], np.float32)
SIGMA_RPY = np.array([0.02, 0.0, 0.05], np.float32)


def host_resample(st, prob, frac, seed, call, sp=SIGMA_POS, sr=SIGMA_RPY):
    n = len(st)
    st = np.ascontiguousarray(st)
    prob = np.ascontiguousarray(prob, np.float32)
    out, out_p = np.zeros(n, synth.STATE), np.zeros(n, np.float32)
    src, dup, org = np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros((n, 6), np.float32)
    assert hs().hostsim_pf_resample_philox(_ptr(prob), _ptr(st), n, frac, seed, call, _ptr(sp), _ptr(sr), _ptr(out), _ptr(out_p),
                                           _ptr(src), _ptr(dup), _ptr(org)) == 0
    return out, out_p, src, dup.astype(bool), org


def check_resample(got, got_p, want, want_p, dup, org, sp=SIGMA_POS, sr=SIGMA_RPY):
    assert got_p.tobytes() == want_p.tobytes()
    assert got[~dup].tobytes() == want[~dup].tobytes()                  # plain and past-the-end copies
    g, w, o = got[dup], want[dup], org[dup].astype(np.float64)
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        assert (g[f].view(np.uint32) == 0).all(), f                       # +0.0: fresh states
    sig = np.concatenate([sp, sr])
    for f, cols in (("pos", [0, 1, 2]), ("odom_err_integ_lin", [0, 1, 2]), ("odom_err_integ_ang", [3, 4, 5])):
        for a, k in enumerate(cols):
            if sig[k] == 0:
                assert g[f][:, a].tobytes() == w[f][:, a].tobytes(), (f, a)
            else:
                d = np.abs(g[f][:, a].astype(np.float64) - w[f][:, a])
                assert (d <= ulp(w[f][:, a]) + ORG_REL * np.abs(o[:, k])).all(), (f, a, d.max())
    d = np.abs(g["rot"].astype(np.float64) - w["rot"])
    assert d.max(initial=0.0) <= RESAMPLE_ROT_BAR, d.max()


def resample_case(E, sm, n, frac, seed, kind="random"):
    n = size(n, sm)
    st = resample_states(n, n + 17)
    prob = resample_probs(n, kind, n)
    e = fresh(E)
    e.particles_set(st, prob)
    e.particles_resample(SIGMA_POS, SIGMA_RPY, frac, seed)
    got, got_p = e.particles_get()
    e.close()
    want, want_p, src, dup, org = host_resample(st, prob, frac, seed, 1)
    if n > 64 and kind == "random":
        assert 0 < dup.sum() < n
    check_resample(got, got_p, want, want_p, dup, org)
    return src, dup


FRACS = [0.0, 0.37, 0.99999994]
SEEDS = [0, 0xDEADBEEF12345678, (1 << 32) + 1]
RESAMPLE_SIZES = [1, 2, 15, 16, 17, 1023, 1024, 1025, 4097, 65536, (0, (1 << 20) + 3)]


@pytest.mark.parametrize("i,n", list(enumerate(RESAMPLE_SIZES)))
def test_resample(eng_mod, sm, hostsim, i, n):  # noqa: F811
    resample_case(eng_mod, sm, n, FRACS[i % 3], SEEDS[i % 3])


@pytest.mark.parametrize("kind,n", [("ties", 4097), ("ties", 65536), ("total3.7", 1025), ("total1e-30", 4097), ("one", 1024),
                                    ("one", 17)])
def test_resample_weights(eng_mod, sm, hostsim, kind, n):  # noqa: F811
    src, dup = resample_case(eng_mod, sm, n, 0.37, SEEDS[1], kind)
    if kind == "one":
        assert len(set(src.tolist())) == 1
    if kind == "ties":
        prob = resample_probs(n, kind, n)
        acc = np.cumsum(prob, dtype=np.float32)
        tie = np.concatenate([[False], np.diff(acc) == 0])
        assert tie.sum() > n // 10 and not tie[src].any()               # ties go to the lowest index


def test_resample_past_the_end_sweep(eng_mod, sm, hostsim):  # noqa: F811
    """test_hostsim.py's 400 sets whose last picks round past the end, on one engine: call k uses counter k."""
    frac = np.float32(0.99999994)
    e = fresh(eng_mod)
    hits = 0
    for k, seed in enumerate(range(400)):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(2, 300))
        prob = rng.uniform(0.05, 1.0, n).astype(np.float32)
        st = resample_states(n, seed)
        e.particles_set(st, prob)
        e.particles_resample(SIGMA_POS, SIGMA_RPY, float(frac), seed)
        got, got_p = e.particles_get()
        want, want_p, src, dup, org = host_resample(st, prob, float(frac), seed, k + 1)
        acc = np.cumsum(prob, dtype=np.float32)
        pstep = np.float32(acc[-1] / np.float32(n))
        pscan = (pstep * np.arange(n, dtype=np.float32) + np.float32(frac * pstep)).astype(np.float32)
        hits += int((np.searchsorted(acc, pscan, side="left") >= n).any())
        check_resample(got, got_p, want, want_p, dup, org)
    e.close()
    assert hits > 20


def test_resample_three_calls(eng_mod, sm, hostsim):  # noqa: F811
    """Calls 1, 2, 3 on one engine with a particles_set between the second and the third (the count goes on)."""
    n = 3001
    e = fresh(eng_mod)
    st, prob = resample_states(n, 1), resample_probs(n, "random", 1)
    e.particles_set(st, prob)
    for call in (1, 2, 3):
        if call == 3:
            st, prob = resample_states(n, 2), resample_probs(n, "random", 2)
            e.particles_set(st, prob)
        e.particles_resample(SIGMA_POS, SIGMA_RPY, 0.37, SEEDS[1])
        got, got_p = e.particles_get()
        want, want_p, src, dup, org = host_resample(st, prob, 0.37, SEEDS[1], call)
        check_resample(got, got_p, want, want_p, dup, org)
        st, prob = got, got_p
    e.close()


# ------------------------------------------------------------------ 3. estimate
def estimate_inputs(n, ties, seed, sm, far=False):
    """far: x = ±1e5 by parity, so that the sums cancel and a thread's partial sum is ~10^5 times the mean: a float
    rounding of the running partials would then move the mean by many ulps."""
    rng = np.random.default_rng(seed)
    st = predict_states(n, seed)
    st["pos"] = rng.normal([3.0, -4.0, 0.5], [0.3, 0.2, 0.05], (n, 3))
    if far:
        st["pos"][:, 0] += np.where(np.arange(n) % 2 == 0, 1e5, -1e5)
    yaw = rng.normal(2.9, 0.2, n)
    st["rot"] = synth.quat_from_rpy(np.stack([rng.normal(0.05, 0.02, n), rng.normal(-0.04, 0.02, n), yaw], axis=1))
    st["rot"] *= (1.0 + rng.normal(0, 1e-3, (n, 1))).astype(np.float32)
    prob = rng.uniform(0.1, 0.6, n).astype(np.float32)
    prob /= prob.sum(dtype=np.float64).astype(np.float32) * np.float32(1.001)
    top = np.float32(prob.max() * np.float32(1.5))
    grid = min(-(-n // 256), 4 * sm)
    at = {"lanes": [17, 3], "warps": [200, 40], "ctas": [grid * 256 + 5, 256 + 5], "last": [n - 1]}.get(ties)
    if at:
        assert max(at) < n
        prob[at] = top
    if ties == "all_equal":
        prob[:] = np.float32(1.0 / n)
    if ties == "zero":
        prob[:] = 0.0
    want_max = min(at) if at else int(np.argmax(prob))
    return st, prob, want_max, (yaw > math.pi).any()


def bias_rel_bound(st, prev, var_dist, var_ang, bias):
    """Relative bound ε_i on |w_dev - w_host| / w for pf_bias with prev (acosf and two expf)."""
    q = np.array([prev["qx"][0], prev["qy"][0], prev["qz"][0], prev["qw"][0]], np.float64)
    inv = np.array([-q[0], -q[1], -q[2], q[3]]) / (q @ q)
    r = st["rot"].astype(np.float64)
    qw = r[:, 3] * inv[3] - r[:, 0] * inv[0] - r[:, 1] * inv[1] - r[:, 2] * inv[2]
    a2 = 2.0 * np.arccos(np.clip(np.abs(qw), 0, 1)) * 1.001 + 1e-30       # 2 acos (before the wrap), rounded up
    ang = np.minimum(a2, np.abs(a2 - 2 * math.pi) + 1e-6)
    d_ang = LIBM["acosf"] * R * a2 + 2 * ulp(a2) + ulp(ang)                # acosf, the double product's and the wrap's roundings
    sq2a = float(np.float32(var_ang * var_ang * 2.0))
    arg_a = ang * ang / sq2a
    rel_na = 2 * ang * d_ang / sq2a + 2 * R * arg_a + (LIBM["expf"] + 1) * R
    rel_nl = (LIBM["expf"] + 1) * R                                          # its argument is exact device arithmetic
    nlna = np.maximum(bias.astype(np.float64) - 1e-6, 0)
    rel_bias = (rel_nl + rel_na + R) * nlna / bias + R
    return (rel_bias + R) * 1.01                                              # and w = fmul(p, bias)


def estimate_case(E, sm, n, ties="none", with_prev=False, seed=6, far=False):
    L = hs()
    n = size(n, sm)
    st, prob, want_max, wraps = estimate_inputs(n, ties, seed, sm, far)
    prev = synth.make_poses([[3.1, -4.0, 0.5]], synth.quat_from_rpy([[0.0, 0.0, 2.95]])) if with_prev else None
    vd, va = 0.2, 0.25
    e = fresh(E)
    e.particles_set(st, prob)
    got = e.particles_estimate(prev, vd, va)
    e.close()
    assert got["max_index"] == want_max
    assert got["max_state"]["px"][0] == st["pos"][want_max, 0] and got["max_state"]["qw"][0] == st["rot"][want_max, 3]
    if ties == "zero":
        return got
    bias, T = np.zeros(n, np.float32), np.zeros((n, 20), np.float32)
    assert L.hostsim_pf_est_terms(_ptr(prob), _ptr(st), n, _ptr(prev), vd, va, _ptr(bias), _ptr(T)) == 0
    S, A = col_sums(T)
    D = depth(n, sm, E)
    g = gamma(D)
    mean = got["mean_biased"]
    v = np.array([float(s) for s in S])
    mpos, mrot, epos, erpy = (np.zeros(k, np.float32) for k in (3, 4, 3, 3))
    L.hostsim_pf_est_finish(_ptr(v), _ptr(mpos), _ptr(mrot), _ptr(epos), _ptr(erpy))
    if not with_prev:
        assert np.float32(got["weight_sum_biased"]) == to_f32(S[0], g * Fraction(A[0]))
        for a, f in enumerate(("px", "py", "pz")):
            assert mean[f][0] == to_f32(S[1 + a] / S[0], ratio_err(S[1 + a], A[1 + a], S[0], A[0], D)), f
        q = np.array([mean[f][0] for f in ("qx", "qy", "qz", "qw")], np.float32)
        assert np.abs(mrot).min() > 1e-3
        assert (np.abs(q.astype(np.float64) - mrot) <= ulp(mrot)).all(), (q, mrot)
    else:
        eps = bias_rel_bound(st, prev, vd, va, bias)
        w = T[:, 0].astype(np.float64)
        dS0 = float((eps * w).sum()) + float(g) * A[0]
        assert abs(got["weight_sum_biased"] - float(S[0])) <= dS0 + ulp(float(S[0])), (got["weight_sum_biased"], float(S[0]))
        for a, f in enumerate(("px", "py", "pz")):
            m = float(S[1 + a] / S[0])
            dA = float(((eps + R) * np.abs(T[:, 1 + a])).sum()) + float(g) * A[1 + a]
            assert abs(mean[f][0] - m) <= (dA + abs(m) * dS0) / float(S[0]) * 1.01 + ulp(m), f
        fr, up = np.array([float(S[4 + k]) for k in range(3)]), np.array([float(S[7 + k]) for k in range(3)])
        df = float(((eps + R) * np.abs(T[:, 4:7]).sum(1)).sum()) / np.linalg.norm(fr)
        du = float(((eps + R) * np.abs(T[:, 7:10]).sum(1)).sum()) / np.linalg.norm(up)
        sin_fu = np.linalg.norm(np.cross(fr, up)) / np.linalg.norm(fr) / np.linalg.norm(up)
        q = np.array([mean[f][0] for f in ("qx", "qy", "qz", "qw")], np.float64)
        assert (np.abs(q - mrot) <= 2 * (df + du) / sin_fu + ulp(mrot)).all()
    # the covariance around the centre float(exact Σ p pos / Σ p) (with bias 1, Σw = Σp)
    for a in range(3):
        assert epos[a] == to_f32(S[11 + a] / S[10], ratio_err(S[11 + a], A[11 + a], S[10], A[10], D))
    d, T2 = np.zeros((n, 6), np.float32), np.zeros((n, 22), np.float32)
    assert L.hostsim_pf_cov_terms(_ptr(prob), _ptr(st), n, _ptr(epos), _ptr(erpy), _ptr(d), _ptr(T2)) == 0
    assert np.abs(d[:, 3:]).max() < math.pi - 1e-3                         # no wrapped difference near ±π
    assert wraps or n < 100                                                 # while some yaws cross π
    Cs, CA = col_sums(T2)
    dd = np.zeros((n, 6))
    rpy = np.abs(d[:, 3:].astype(np.float64) + erpy) * 1.001 + 1e-30         # |rpy_i| (up to the wrap), rounded up
    rpy = np.minimum(rpy, math.pi)
    lib = np.array([LIBM["atan2f"], LIBM["asinf"], LIBM["atan2f"]])
    dd[:, 3:] = lib * ulp(rpy) + lib * ulp(np.abs(erpy)) + 16 * U + 2 * ulp(d[:, 3:])
    p = prob.astype(np.float64)
    ad = np.abs(d.astype(np.float64))
    cov = got["cov"]
    t = 1
    for j in range(6):
        for k in range(j, 6):
            ratio = Cs[t] / Cs[0]
            if k < 3:
                assert cov[j, k] == cov[k, j] == to_f32(ratio, ratio_err(Cs[t], CA[t], Cs[0], CA[0], D)), (j, k)
            else:
                dT = (p * (dd[:, j] * ad[:, k] + ad[:, j] * dd[:, k] + dd[:, j] * dd[:, k])).sum() * (1 + 4 * U) + 4 * U * CA[t]
                bar = (dT + float(g) * (CA[t] + dT)) / float(Cs[0]) * 1.01 + ulp(float(ratio))
                assert cov[j, k] == cov[k, j] and abs(cov[j, k] - float(ratio)) <= bar, (j, k, cov[j, k], float(ratio), bar)
            t += 1
    return got


ESTIMATE_CASES = [(1, "none", False), (255, "lanes", False), (256, "warps", True), (257, "last", False),
                  ((1, -1), "warps", False), ((1, 0), "all_equal", False), ((1, 1), "lanes", False), ((1, 1), "none", True),
                  ((3, 7), "ctas", True), ((3, 7), "ctas", False), ((0, 1 << 20), "ctas", False), (4099, "zero", False),
                  ((1, 1), "zero", False)]


@pytest.mark.parametrize("n,ties,with_prev", ESTIMATE_CASES)
def test_estimate(eng_mod, sm, hostsim, n, ties, with_prev):  # noqa: F811
    estimate_case(eng_mod, sm, n, ties, with_prev)


@pytest.mark.parametrize("n", [(3, 7), (0, 1 << 20)])
def test_estimate_cancelling_sums(eng_mod, sm, hostsim, n):  # noqa: F811
    estimate_case(eng_mod, sm, n, far=True)


# ------------------------------------------------------------------ 4. the weight fold
class FoldScene:
    def __init__(self, P, seed=141):
        self.s = synth.scene(30_000, 1024, 24, 0, seed=seed)
        base = self.s["particles"]
        self.poses = np.ascontiguousarray(np.resize(base, P))
        self.states = np.zeros(P, synth.STATE)
        self.states["pos"] = np.stack([self.poses[f] for f in ("px", "py", "pz")], axis=1)
        self.states["rot"] = np.stack([self.poses[f] for f in ("qx", "qy", "qz", "qw")], axis=1)
        rng = np.random.default_rng(seed)
        self.states["odom_err_integ_lin"] = rng.normal(0, 0.1, (P, 3))

    def engine(self, E):
        e = fresh(E)
        e.set_map(self.s["map"], E.LikParams(dist_weight=(1, 1, 5)))
        return e


def fold_prior(P, ties, sm, scene):
    rng = np.random.default_rng(P)
    prior = rng.uniform(0.1, 0.9, P).astype(np.float32)
    nblk = min(-(-P // 256), 4 * sm)
    at = {"lanes": [17, 3], "warps": [200, 40], "ctas": [nblk * 256 + 5, 256 + 5], "last": [P - 1]}.get(ties)
    if at:
        assert max(at) < P
        prior[at] = 1.0                                    # the tied particles share the best pose: the largest w
        for i in at:
            scene.poses[i] = scene.poses[scene.best]
            scene.states[i] = scene.states[scene.best]
    if ties == "all_equal":
        prior[:] = np.float32(0.5)
        scene.poses[:] = scene.poses[scene.best]
        scene.states[:] = scene.states[scene.best]
    if ties == "zero":
        prior[:] = 0.0
    return prior, (min(at) if at else None)


def host_weights(rec, prior, extra=None):
    lk = (np.float32(1.0) * rec["score_beam"]).astype(np.float32)
    lk = (lk * rec["score_like"]).astype(np.float32)
    if extra is not None:
        lk = (lk * extra).astype(np.float32)
    return (prior * lk).astype(np.float32)


def odom_factor(states, sigma):
    """pf_pack_kernel's NormalLikelihood(sigma)(|odom_err_integ_lin|) with a correctly rounded exp."""
    s = float(np.float32(sigma))
    a, sq2 = np.float32(1.0 / np.sqrt(2.0 * np.pi * s * s)), np.float32(s * s * 2.0)
    lin = states["odom_err_integ_lin"]
    x = np.sqrt((lin[:, 0] * lin[:, 0] + lin[:, 1] * lin[:, 1]).astype(np.float32) + lin[:, 2] * lin[:, 2]).astype(np.float32)
    return (a * np.exp((-x * x / sq2).astype(np.float32).astype(np.float64)).astype(np.float32)).astype(np.float32)


def check_fold(E, post, summ, rec, prior, n_lik, sm, want_max, extra=None):
    P = len(prior)
    w = host_weights(rec, prior, extra)
    q = rec["match_cnt"].astype(np.float32) / np.float32(n_lik)
    assert summ["match_ratio_min"] == min(np.float32(1), q.min()) and summ["match_ratio_max"] == max(np.float32(0), q.max())
    S = exact_row_sums(w[None])[0]
    D = depth(P, sm, E)
    if S == 0:
        assert summ["kept"] == 0 and summ["max_index"] == 0 and post.tobytes() == prior.tobytes()
        return None
    assert summ["kept"] == 1
    if extra is None:
        Sf = to_f32(S, gamma(D) * Fraction(float(np.abs(w.astype(np.float64)).sum())))
        assert np.float32(summ["weight_sum"]) == Sf
        want = (w / Sf).astype(np.float32)
        assert post.tobytes() == want.tobytes()
    else:
        eps = 6 * R
        Sd = float(S)
        assert abs(summ["weight_sum"] - Sd) <= eps * Sd * 1.01 + ulp(Sd)
        want = (w.astype(np.float64) / Sd)
        assert (np.abs(post - want) <= want * (2 * eps + 3 * R) * 1.01).all()
        want = want.astype(np.float32)
    top = np.flatnonzero(post == post.max())[0]
    assert summ["max_index"] == top == (want_max if want_max is not None else top)
    if want_max is None and extra is None:
        assert top == int(np.argmax(want))
    pv = want.astype(np.float64)
    nz = want > 0
    lnp = np.log(pv[nz]).astype(np.float32)                                # correctly rounded (to within 2^-29 ulp)
    terms = (want[nz] * lnp).astype(np.float32)
    Ex = exact_row_sums(terms[None])[0]
    bar = (LIBM["logf"] * pv[nz] * ulp(lnp) + ulp(terms)).sum() + float(gamma(D)) * np.abs(terms.astype(np.float64)).sum()
    if extra is not None:
        bar += (pv[nz] * (2 * eps + 3 * R) * (np.abs(lnp) + 1)).sum()
    assert abs(summ["entropy"] + float(Ex)) <= bar * 1.01 + ulp(float(Ex)), (summ["entropy"], -float(Ex), bar)
    return S


def fold_case(E, sm, P, ties, path, sigma=0.0, round_up=False):
    P = size(P, sm)
    sc = FoldScene(P)
    e = sc.engine(E)
    lik, org = sc.s["lik"], sc.s["origins"]
    base = e.measure(sc.s["particles"], lik, None, org)
    lk = host_weights(base, np.ones(len(base), np.float32))
    sc.best = int(np.argmax(lk))
    assert lk[sc.best] > 0
    prior, want_max = fold_prior(P, ties, sm, sc)
    if path == "measure_update":
        post, summ, rec = e.measure_update(sc.poses, lik, None, org, prior, want_records=True)
    else:
        rec = e.measure(sc.poses, lik, None, org)
        if round_up:   # move one prior so that the exact total lies 3/4 of the way up a float interval
            i = sc.best
            S = exact_row_sums(host_weights(rec, prior)[None])[0]
            lo = np.float32(float(S))
            lo = lo if Fraction(float(lo)) <= S else np.nextafter(lo, np.float32(0))
            target = Fraction(float(lo)) + 3 * half_ulp(Fraction(float(lo))) / 2
            lk = host_weights(rec[i:i + 1], np.ones(1, np.float32))[0]
            prior[i] = np.float32(float(prior[i]) + float(target - S) / float(lk))
        e.particles_set(sc.states, prior)
        summ = e.particles_measure_update(lik, None, org, sigma)
        _, post = e.particles_get()
    e.close()
    extra = odom_factor(sc.states, sigma) if sigma > 0 else None
    S = check_fold(E, post, summ, rec, prior, len(lik), sm, want_max, extra)
    if round_up:
        assert Fraction(float(np.float32(float(S)))) > S
    return S


FOLD_CASES = [(1, "none"), (8192, "lanes"), (8193, "warps"), ((1, -1), "last"), ((1, 1), "lanes"), ((3, 7), "ctas"),
              (8193, "all_equal"), (8192, "zero")]


@pytest.mark.parametrize("path", ["measure_update", "resident"])
@pytest.mark.parametrize("P,ties", FOLD_CASES)
def test_weight_fold(eng_mod, sm, P, ties, path):
    fold_case(eng_mod, sm, P, ties, path)


@pytest.mark.parametrize("P", [8192, (1, 1)])
def test_weight_fold_total_rounds_up(eng_mod, sm, P):
    fold_case(eng_mod, sm, P, "none", "resident", round_up=True)


@pytest.mark.parametrize("P", [8193, (1, 1)])
def test_weight_fold_with_odometry_factor(eng_mod, sm, P):
    fold_case(eng_mod, sm, P, "none", "resident", sigma=0.4)


# ------------------------------------------------------------------ 5. a cycle
def cycle_case(E, sm, n=20_000, rounds=4):
    sc = FoldScene(n, seed=151)
    lik, org = sc.s["lik"], sc.s["origins"]
    rng = np.random.default_rng(9)
    st = sc.states.copy()
    st["noise_ll"] = rng.normal(0, 0.05, n)
    st["noise_al"] = rng.normal(0, 0.05, n)
    st["noise_la"][::3] = rng.normal(0, 0.05, len(st[::3]))
    prior = np.full(n, 1.0 / n, np.float32)
    odo = [synth.make_poses([[0.1 * k, 0.02 * k, 0.0]], synth.quat_from_rpy([[0.0, 0.0, 0.05 * k]])) for k in range(rounds + 1)]
    ea, eb = sc.engine(E), sc.engine(E)
    for e in (ea, eb):
        e.particles_set(st, prior)
    cur_s, cur_p = st, prior
    for k in range(rounds):
        sd = 1000 + k
        ea.particles_predict(odo[k], odo[k + 1], 0.1, 10.0, 7.0)
        ea.particles_measure_update(lik, None, org, 0.0)
        ea.particles_resample(SIGMA_POS, SIGMA_RPY, 0.37, sd)
        est_a = ea.particles_estimate(None)
        # engine b, step by step
        eb.particles_predict(odo[k], odo[k + 1], 0.1, 10.0, 7.0)
        got, _ = eb.particles_get()
        check_predict(got, host_predict(cur_s, odo[k], odo[k + 1], 0.1), cur_s)
        cur_s = got
        rec = eb.measure(synth.make_poses(cur_s["pos"], cur_s["rot"]), lik, None, org)
        summ = eb.particles_measure_update(lik, None, org, 0.0)
        _, post = eb.particles_get()
        check_fold(E, post, summ, rec, cur_p, len(lik), sm, None)
        cur_p = post
        eb.particles_resample(SIGMA_POS, SIGMA_RPY, 0.37, sd)
        got, got_p = eb.particles_get()
        want, want_p, src, dup, org = host_resample(cur_s, cur_p, 0.37, sd, k + 1)
        check_resample(got, got_p, want, want_p, dup, org)
        cur_s, cur_p = got, got_p
        est_b = eb.particles_estimate(None)
        assert est_a["max_index"] == est_b["max_index"] == 0                # uniform probabilities after resampling
        for f in ("mean_biased", "max_state", "cov"):
            assert np.asarray(est_a[f]).tobytes() == np.asarray(est_b[f]).tobytes(), f
    sa, pa = ea.particles_get()
    sb, pb = eb.particles_get()
    ea.close()
    eb.close()
    assert sa.tobytes() == sb.tobytes() and pa.tobytes() == pb.tobytes()
    assert sa.tobytes() == cur_s.tobytes()


def test_cycle(eng_mod, sm, hostsim):  # noqa: F811
    cycle_case(eng_mod, sm)
