"""Every likelihood kernel path against the exact sum of the reference's per-point terms.

score_like is the one record field the kernels do not reproduce bit for bit: each kernel adds a particle's float
contributions in its own order.  test_gpu_parity.py holds it to LIK_RTOL against the oracle's serial float sum; this
file holds each kernel to the bar its own summation guarantees.

Terms.  T[p, j] is the reference's float contribution of particle p at scan point j, and M[p, j] whether it counts.
The oracle port measured with the one-point scan lik[j:j+1] returns score_like = 0 + T[p, j] and match_cnt = M[p, j]:
likelihood.cpp:105-136 transforms and searches every point on its own, so these are the reference's terms bit for bit.
S[p] is the exact sum of row p's counted terms (every float is an integer multiple of 2^-149, so the sum is an exact
integer sum).  test_per_point_terms_fold_to_the_oracle_score checks this machinery on the CPU: T folded in scan order
in float is the oracle's score bit for bit.

Bars.  On every path match_cnt[p] = sum_j M[p, j], and the beam fields, where a beam scan is given, equal the oracle's.
* lik_kernel_nf_pm (P >= 256 particles and nf_pm_shape ok): the kernel's own arithmetic, bit for bit.  k = fx_shift
  of nf_pm_shape(N, blocks, slots, 4, match_dist_min, match_weight), taken from the shape helper itself, with slots =
  sm_count x per_sm as engine.cu's launch_lik_nf has it (per_sm = 4, or min(4, MCL3DL_LIK_SHARE) when a beam scan
  runs alongside).  K = sum_j rint(float(T[p, j] * 2^k)) as an exact integer, and the score is float(K) * 2^-k with
  K rounded to float once.  Independently of the shape, nf_pm_shape's promise: the N roundings to 2^-k stay below
  E = 2^-30 * N * match_dist_min * |match_weight|, so |score - S| <= E + 1/2 ulp(|S| + E) (the final rounding to
  float, of a value within E of S).
* lik_kernel_nf and lik_kernel_wi: |score - S| <= gamma_D * sum_j |T[p, j]|, gamma_D = D u / (1 - D u), u = 2^-24.
  A lane adds its evals j = l, l + TPP, ... serially (ceil(N / TPP) additions), the xor-shuffle tree adds
  log2(min(TPP, 32)) levels, and particle_reduce adds the particle's TPP / 32 warps in order (TPP / 32 - 1 more).  So
  each term passes through at most D = ceil(N / TPP) + log2(min(TPP, 32)) + max(TPP / 32 - 1, 0) float additions;
  each rounds by a factor (1 + d), |d| <= u, and a product of D such factors is within gamma_D of 1 (Higham, Accuracy
  and Stability of Numerical Algorithms, Lemma 3.1).  D is the maximum over the lanes per particle the launchers can
  pick: 8 .. 256 for lik_kernel_nf (pick_tpp_nf), 32 .. 256 for lik_kernel_wi (pick_tpp).

Each case names the kernel launch_lik selects for it, from nf_pm_shape for the device's SM count rather than from
constants.  Where that is lik_kernel_nf_pm, the bit-exact bar also shows that it ran: a particle-major sum of the same
terms is not float(K) * 2^-k.
"""
import ctypes as C
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.path.join(ROOT, "tests", "hostsim", "nf_pm_hostsim.cpp")
UNIT = 4  # kNfU: the points of one warp trip
NF_MINB = 4  # MCL3DL_NF_MINB: the likelihood kernels' CTA slots per SM
TPP_NF = [8 << i for i in range(6)]  # pick_tpp_nf: 8 .. 256 lanes per particle
TPP_WI = [32 << i for i in range(4)]  # pick_tpp: 32 .. 256
MAX_STAGED_NF = 200 * 1024 // 2  # lik_kernel_nf stages scans of up to kMaxStagedBytes / 2
MAX_STAGED_WI = 160 * 1024  # lik_kernel_wi: kMaxStagedSorted
U = Fraction(1, 1 << 24)


def cc():
    from oracle import cpu_checker
    return cpu_checker


# ------------------------------------------------------------------ exact arithmetic
def exact_row_sums(A):
    """The exact sum of each row of a float32 matrix, as Fractions.  A float32 is m * 2^(e - 150) with an integer
    |m| < 2^24 (e = max(exponent field, 1)); the m of one row and exponent are summed exactly (< 2^53 in float64)."""
    P = A.shape[0]
    b = np.ascontiguousarray(A, np.float32).view(np.uint32)
    e = ((b >> 23) & 0xff).astype(np.int64)
    m = ((b & 0x7fffff) | np.where(e > 0, 0x800000, 0)).astype(np.float64)
    m[(b >> 31) != 0] *= -1.0
    e = np.maximum(e, 1)
    key = (np.arange(P, dtype=np.int64)[:, None] * 256 + e).ravel()
    acc = np.bincount(key, weights=m.ravel(), minlength=P * 256).reshape(P, 256)
    out = []
    for row in acc:
        nz = np.nonzero(row)[0]
        out.append(Fraction(sum(int(row[i]) << int(i - 1) for i in nz), 1 << 149))
    return out


def half_ulp(x):
    """Half a float32 ulp at |x| (x a non-negative Fraction)."""
    if x == 0:
        return Fraction(1, 1 << 150)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1  # now 2^e <= x < 2^(e + 1)
    return Fraction(2) ** (max(e - 23, -149) - 1)


def depth(N, tpps):
    return max(-(-N // t) + int(math.log2(min(t, 32))) + max(t // 32 - 1, 0) for t in tpps)


def fold_serial(T, M):
    """likelihood.cpp:128-133: score_like += term in scan order, in float."""
    s = np.zeros(T.shape[0], np.float32)
    for j in range(T.shape[1]):
        s = np.where(M[:, j], s + T[:, j], s).astype(np.float32)
    return s


def terms(cpu, poses, lik):
    """(T, M): the oracle's per-point contributions and matched flags (one-point scans)."""
    T = np.zeros((len(poses), len(lik)), np.float32)
    M = np.zeros((len(poses), len(lik)), bool)
    for j in range(len(lik)):
        r = cpu.measure(poses, lik[j:j + 1], None, None, n_threads=8)
        assert set(np.unique(r["match_cnt"])) <= {0, 1}
        T[:, j] = r["score_like"]
        M[:, j] = r["match_cnt"] == 1
    return T, M


# ------------------------------------------------------------------ CPU: the reference machinery
@pytest.mark.parametrize("w,flat", [(5.0, 0.05), (-3.0, 0.05), (2.0, 0.2), (1e-36, 0.0)])
def test_per_point_terms_fold_to_the_oracle_score(port, w, flat):
    s = synth.scene(50_000, 64, 96, 0, seed=201)
    cpu = port.create(s["map"], cc().lik_params(w, 0.2, flat, (1, 1, 5)), None, 20.0, 0.4)
    T, M = terms(cpu, s["particles"], s["lik"])
    full = cpu.measure(s["particles"], s["lik"], None, None, n_threads=8)
    assert M.sum() > 0 and np.array_equal(full["match_cnt"], M.sum(axis=1).astype(np.uint32))
    assert np.array_equal(fold_serial(T, M).view(np.uint32), full["score_like"].view(np.uint32))
    # the exact sums are exact: against Fraction sums of a few rows
    S = exact_row_sums(np.where(M, T, np.float32(0)))
    for p in range(0, 64, 13):
        assert S[p] == sum((Fraction(float(t)) for t in T[p][M[p]]), Fraction(0))


def test_exact_row_sums_of_extreme_floats():
    rng = np.random.default_rng(3)
    A = np.concatenate([rng.normal(0, 1, (4, 50)) * 10.0 ** rng.integers(-44, 38, (4, 50)),
                        np.array([[3e38, 3e38, -3e38, 1e-45, -1e-45, 5e-39, 0.0] + [0.0] * 43])]).astype(np.float32)
    for row, s in zip(A, exact_row_sums(A)):
        assert s == sum((Fraction(float(t)) for t in row), Fraction(0))
    assert half_ulp(Fraction(1)) == Fraction(1, 1 << 24) and half_ulp(Fraction(3, 4)) == Fraction(1, 1 << 25)


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def nfpm(tmp_path_factory):
    """nf_pm_shape of device_funcs.cuh, compiled for the host (tests/hostsim/nf_pm_hostsim.cpp)."""
    so = str(tmp_path_factory.mktemp("nfpm") / "libnfpm.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, HOSTSIM],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    L.hostsim_nf_pm_shape.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p]

    def shape(N, P, slots, r, w):
        s = np.zeros(6, np.int32)
        L.hostsim_nf_pm_shape(N, (P + 255) // 256, slots, UNIT, r, w, s.ctypes.data)
        return dict(zip(("slice", "n_slices", "fx_shift", "arr_bits", "cnt_bits", "ok"), (int(v) for v in s)))
    return shape


@pytest.fixture
def make_engine(eng_mod, monkeypatch):
    made = []

    def make(**env):
        for k in ("MCL3DL_NNF", "MCL3DL_LIK_SHARE", "MCL3DL_LIK_MODE"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = eng_mod.Engine((0,))
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


class Lik:
    """One likelihood parameter set, for the engine, the oracle and the bars (float32 values)."""

    def __init__(self, w=5.0, r=0.2, flat=0.05, dw=(1, 1, 5)):
        self.w, self.r, self.flat, self.dw = w, r, flat, dw

    def eng(self, eng_mod):
        return eng_mod.LikParams(match_weight=self.w, match_dist_min=self.r, match_dist_flat=self.flat, dist_weight=self.dw)

    def cpu(self):
        return cc().lik_params(self.w, self.r, self.flat, self.dw)


def expected_kernel(nfpm, sm, P, N, lik, nnf=True, per_sm=NF_MINB):
    """(kernel, shape) that launch_lik picks: lik_kernel_wi without the NN field; lik_kernel_nf_pm for P >= 256 when
    nf_pm_shape is ok; lik_kernel_nf otherwise."""
    if not nnf:
        return "lik_kernel_wi", None
    if P >= 256:
        sh = nfpm(N, P, sm * per_sm, lik.r, lik.w)
        if sh["ok"]:
            return "lik_kernel_nf_pm", sh
    return "lik_kernel_nf", None


def check_lik(got, T, M, lik, kernel, sh):
    """The bars of the module docstring for the records `got` of P = len(got) particles over N = T.shape[1] points."""
    P, N = T.shape
    assert len(got) == P
    assert np.array_equal(got["match_cnt"], M.sum(axis=1).astype(np.uint32))
    Tm = np.where(M, T, np.float32(0))
    S = exact_row_sums(Tm)
    score = got["score_like"]
    if kernel == "lik_kernel_nf_pm":
        k = sh["fx_shift"]
        K = np.rint(Tm * np.float32(2.0 ** k)).astype(np.int64).sum(axis=1)
        want = np.array(K, np.int64).astype(np.float32) * np.float32(2.0 ** -k)
        bad = np.nonzero(want.view(np.uint32) != score.view(np.uint32))[0]
        assert len(bad) == 0, (len(bad), bad[:4], score[bad[:4]], want[bad[:4]], k)
        E = Fraction(1, 1 << 30) * N * Fraction(float(np.float32(lik.r))) * abs(Fraction(float(np.float32(lik.w))))
        for p in range(P):
            assert abs(Fraction(float(score[p])) - S[p]) <= E + half_ulp(abs(S[p]) + E), p
    else:
        D = depth(N, TPP_WI if kernel == "lik_kernel_wi" else TPP_NF)
        g = D * U / (1 - D * U)
        A = exact_row_sums(np.abs(Tm))
        for p in range(P):
            assert abs(Fraction(float(score[p])) - S[p]) <= g * A[p], (p, float(score[p]), float(S[p]), D)


def check_beam(got, want):
    for f in ("score_beam", "n_short", "n_hit", "n_long"):
        assert np.array_equal(got[f], want[f]), f


class Scene:
    """A synth.scene with its oracle and per-point terms (computed on first use, for the full P x N)."""

    def __init__(self, s, lik=None, beam_raw=None):
        self.s = s
        self.lik = lik or Lik()
        self.port = cc().CpuChecker("port")
        self.cpu = self.port.create(s["map"], self.lik.cpu(), beam_raw, 20.0, 0.4)
        self._T = None

    @property
    def TM(self):
        if self._T is None:
            self._T = terms(self.cpu, self.s["particles"], self.s["lik"])
        return self._T


def measure_and_check(nfpm, sm, eng, sc, P, N, nnf=True):
    s = sc.s
    T, M = sc.TM
    kernel, sh = expected_kernel(nfpm, sm, P, N, sc.lik, nnf=nnf)
    got = eng.measure(s["particles"][:P], s["lik"][:N], None, None)
    check_lik(got, T[:P, :N], M[:P, :N], sc.lik, kernel, sh)
    assert M[:P, :N].sum() > 0
    return kernel


def set_map(eng_mod, eng, sc, n_beam=8, use_dda=True):
    eng.set_map(sc.s["map"], sc.lik.eng(eng_mod),
                eng_mod.beam_params_from_reference(num_points_default=n_beam, dda_grid_size=0.2,
                                                   use_raycast_using_dda=use_dda))


# ------------------------------------------------------------------ §3: each kernel selection branch
@pytest.fixture(scope="module")
def ok_edge(nfpm, sm_count):
    """The longest scan for which 1024 particles keep the point-major kernel."""
    n = max(N for N in range(1, 8193) if nfpm(N, 1024, sm_count * NF_MINB, 0.2, 5.0)["ok"])
    assert not nfpm(n + 1, 1024, sm_count * NF_MINB, 0.2, 5.0)["ok"]
    return n


@pytest.fixture(scope="module")
def scene_a(ok_edge):
    return Scene(synth.scene(50_000, 1024, ok_edge + 1, 0, seed=211))


@pytest.fixture(scope="module")
def scene_long():
    return Scene(synth.scene(50_000, 300, MAX_STAGED_WI // 16 + 60, 0, seed=212))


@pytest.mark.gpu
@pytest.mark.parametrize("P,N,kernel", [
    (255, 96, "lik_kernel_nf"),        # below the point-major threshold
    (256, 96, "lik_kernel_nf_pm"),     # one particle block
    (257, 97, "lik_kernel_nf_pm"),     # a ragged block (one live lane in block 2), N not a multiple of 4
    (1024, 1, "lik_kernel_nf_pm"),     # scans shorter than one warp trip
    (1024, 3, "lik_kernel_nf_pm"),
    (1024, 5, "lik_kernel_nf_pm"),
    (1024, "edge", "lik_kernel_nf_pm"),      # the longest scan with nf_pm_shape ok ...
    (1024, "edge+1", "lik_kernel_nf"),       # ... and one point more: the particle-major fallback with P >= 256
])
def test_selection_branches_nf(eng_mod, make_engine, nfpm, sm_count, scene_a, ok_edge, P, N, kernel):
    N = {"edge": ok_edge, "edge+1": ok_edge + 1}.get(N, N)
    eng = make_engine()
    set_map(eng_mod, eng, scene_a)
    assert measure_and_check(nfpm, sm_count, eng, scene_a, P, N) == kernel


@pytest.mark.gpu
def test_selection_long_scan_nf(eng_mod, make_engine, nfpm, sm_count, scene_long):
    """P >= 256 with a scan beyond lik_kernel_nf's shared-memory tile: lik_kernel_nf reading the scan from global."""
    N = MAX_STAGED_NF // 16 + 100
    eng = make_engine()
    set_map(eng_mod, eng, scene_long)
    assert measure_and_check(nfpm, sm_count, eng, scene_long, 300, N) == "lik_kernel_nf"


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["staged", "unstaged"])
def test_selection_without_nn_field(eng_mod, make_engine, nfpm, sm_count, scene_a, scene_long, which):
    """MCL3DL_NNF=0: lik_kernel_wi, with the scan in its shared-memory tile or (beyond the tile) read from global."""
    sc, P, N = (scene_a, 1000, 96) if which == "staged" else (scene_long, 300, len(scene_long.s["lik"]))
    assert (N * 16 <= MAX_STAGED_WI) == (which == "staged")
    eng = make_engine(MCL3DL_NNF="0")
    set_map(eng_mod, eng, sc)
    assert eng.nn_field_info()["bytes"] == 0
    assert measure_and_check(nfpm, sm_count, eng, sc, P, N, nnf=False) == "lik_kernel_wi"


@pytest.mark.gpu
def test_selection_overflow_cells(eng_mod, make_engine, nfpm, sm_count):
    """The dense unit-cube cloud of test_dense_cloud_overflows_the_window_table: lik_kernel_nf_pm<OVF = true>."""
    rng = np.random.default_rng(91)
    pts = rng.uniform(0.0, 1.0, (120_000, 3)).astype(np.float32)
    pts = np.vstack([pts, [[-0.5, -0.5, -0.5], [1.5, 1.5, 1.5]]]).astype(np.float32)
    P, n_lik = 300, 48
    s = {"map": synth.make_points(pts),
         "particles": synth.make_poses(rng.uniform(0.3, 0.7, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.3, (P, 3)))),
         "lik": synth.make_points(rng.uniform(-0.7, 0.7, (n_lik, 3)))}
    sc = Scene(s, Lik(dw=(1, 1, 1)))
    eng = make_engine()
    set_map(eng_mod, eng, sc)
    assert eng.nn_field_info()["overflow_cells"] > 0
    assert measure_and_check(nfpm, sm_count, eng, sc, P, n_lik) == "lik_kernel_nf_pm"


@pytest.mark.gpu
def test_selection_wide_cells(eng_mod, make_engine, nfpm, sm_count):
    """The sparse volume of test_wide_cells_of_the_nn_field (15..40 candidates in some voxels): lik_kernel_nf_pm over
    wide cells."""
    rng = np.random.default_rng(92)
    P, n_lik = 512, 64
    s = {"map": synth.make_points(rng.uniform(0.0, 1.0, (600, 3)).astype(np.float32)),
         "particles": synth.make_poses(rng.uniform(0.3, 0.7, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.3, (P, 3)))),
         "lik": synth.make_points(rng.uniform(-0.7, 0.7, (n_lik, 3)))}
    sc = Scene(s, Lik(dw=(1, 1, 1)))
    eng = make_engine()
    set_map(eng_mod, eng, sc)
    info = eng.nn_field_info()
    assert info["wide_cells"] > 0 and info["overflow_cells"] == 0
    assert measure_and_check(nfpm, sm_count, eng, sc, P, n_lik) == "lik_kernel_nf_pm"


@pytest.mark.gpu
def test_selection_concurrent_beam(eng_mod, make_engine, nfpm, sm_count):
    """A beam scan alongside with MCL3DL_LIK_SHARE=1: the point-major kernel takes one CTA slot per SM, so its shape
    (and fixed-point scale) is that of sm_count slots."""
    n_beam = 16
    s = synth.scene(50_000, 4097, 512, n_beam, seed=213)
    sc = Scene(s, beam_raw=cc().beam_raw(num_points_default=n_beam, dda_grid_size=0.2))
    eng = make_engine(MCL3DL_LIK_SHARE="1")
    set_map(eng_mod, eng, sc, n_beam)
    T, M = sc.TM
    kernel, sh = expected_kernel(nfpm, sm_count, 4097, 512, sc.lik, per_sm=1)
    assert kernel == "lik_kernel_nf_pm"
    assert sh != nfpm(512, 4097, sm_count * NF_MINB, sc.lik.r, sc.lik.w)  # the reduced slot count changes the shape
    got = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    check_lik(got, T, M, sc.lik, kernel, sh)
    check_beam(got, sc.cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"], n_threads=8))


# ------------------------------------------------------------------ §4: parameter and geometry edges
@pytest.fixture(scope="module")
def scene_edges():
    return synth.scene(50_000, 300, 96, 0, seed=221)


@pytest.mark.gpu
@pytest.mark.parametrize("w,flat", [
    (5.0, 0.05), (-3.0, 0.05), (0.0, 0.05), (1e-6, 0.05), (3e4, 0.05),
    (1e-36, 0.05),  # 2^fx_shift would leave float's range: the particle-major kernel, also for P >= 256
    (5.0, 0.2),     # match_dist_flat == match_dist_min: every match adds exactly 0 and still counts
    (5.0, 0.0), (-3.0, -0.1),
])
def test_parameter_edges(eng_mod, make_engine, nfpm, sm_count, scene_edges, w, flat):
    sc = Scene(scene_edges, Lik(w=w, flat=flat))
    eng = make_engine()
    set_map(eng_mod, eng, sc)
    for P in (300, 200):
        kernel = measure_and_check(nfpm, sm_count, eng, sc, P, 96)
        assert kernel == ("lik_kernel_nf_pm" if P >= 256 and w != 1e-36 else "lik_kernel_nf")


@pytest.mark.gpu
def test_set_params_on_the_point_major_path(eng_mod, make_engine, nfpm, sm_count, scene_edges):
    """match_weight 5 -> 3e4 -> -2 without restaging: the fixed-point scale follows the weight."""
    eng = make_engine()
    set_map(eng_mod, eng, Scene(scene_edges))
    for w in (5.0, 3e4, -2.0):
        sc = Scene(scene_edges, Lik(w=w))
        eng.set_params(sc.lik.eng(eng_mod), None)
        assert measure_and_check(nfpm, sm_count, eng, sc, 300, 96) == "lik_kernel_nf_pm"


def radius_scene():
    """Map points on a coarse dyadic lattice (x, y step 1 m, z step 1 m = 5 m scaled, so one map point within the
    radius of any query below), and scan points at -8 .. +8 ulps around match_dist_min from three of them along each
    axis, in the scaled metric of dist_weight = (1, 1, 5).  Particles: 100 identity poses at the origin, 200
    near-identity ones (1e-6 m, 1e-6 rad)."""
    r, dw = np.float32(0.2), np.array([1, 1, 5], np.float32)
    g = np.stack(np.meshgrid(np.arange(8), np.arange(8), np.arange(4), indexing="ij"), -1).reshape(-1, 3)
    mp = (g + np.array([0.5, 0.5, 0.25])).astype(np.float32)
    scan = []
    for c in np.array([[0.5, 0.5, 0.25], [3.5, 2.5, 1.25], [7.5, 7.5, 3.25]], np.float32):
        for a in range(3):
            for sgn in (1, -1):
                v = np.float32(c[a] + sgn * r / dw[a])
                for i in range(-8, 9):
                    q = c.copy()
                    q[a] = v
                    for _ in range(abs(i)):
                        q[a] = np.nextafter(q[a], np.float32(np.inf if i > 0 else -np.inf), dtype=np.float32)
                    scan.append(q)
    rng = np.random.default_rng(231)
    pos = np.zeros((300, 3))
    rpy = np.zeros((300, 3))
    pos[100:] = rng.normal(0, 1e-6, (200, 3))
    rpy[100:] = rng.normal(0, 1e-6, (200, 3))
    return {"map": synth.make_points(mp), "lik": synth.make_points(np.array(scan, np.float32)),
            "particles": synth.make_poses(pos, synth.quat_from_rpy(rpy))}


@pytest.mark.gpu
def test_queries_on_the_search_radius(eng_mod, make_engine, nfpm, sm_count):
    """d2 < r2 is strict, and the NN field's candidate lists must hold the map points at the radius.  match_weight 0.7
    has a full float mantissa, so the tiny terms of the points just inside the radius carry bits below the fixed-point
    step of lik_kernel_nf_pm and test its rounding (with weight 5 every term is a multiple of the step)."""
    s = radius_scene()
    sc = Scene(s, Lik(w=0.7))
    eng = make_engine()
    set_map(eng_mod, eng, sc)
    T, M = sc.TM
    sweeps = M[0].reshape(-1, 17)  # identity pose: the 17 offsets around each (centre, axis, sign)
    assert sweeps.any(axis=1).all() and not sweeps.all(axis=1).any()  # every sweep crosses the radius
    for P in (300, 200):
        measure_and_check(nfpm, sm_count, eng, sc, P, len(s["lik"]))


@pytest.mark.gpu
@pytest.mark.parametrize("use_dda", [True, False])
def test_map_far_from_the_origin(eng_mod, make_engine, nfpm, sm_count, use_dda):
    """Map and particles translated by ~(2345.6, -1234.5, 3.2), the scans still in the sensor frame: the NN-field
    lattice and the raycasters index large float coordinates."""
    n_beam = 16
    s = synth.scene(50_000, 300, 96, n_beam, seed=241)
    off = np.array([2345.6, -1234.5, 3.2], np.float32)
    for a, f in enumerate("xyz"):
        s["map"][f] += off[a]
        s["particles"]["p" + f] += off[a]
    sc = Scene(s, beam_raw=cc().beam_raw(num_points_default=n_beam, dda_grid_size=0.2, use_raycast_using_dda=use_dda))
    eng = make_engine()
    set_map(eng_mod, eng, sc, n_beam, use_dda=use_dda)
    T, M = sc.TM
    want = sc.cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"], n_threads=8)
    for P in (300, 200):
        kernel, sh = expected_kernel(nfpm, sm_count, P, 96, sc.lik)
        got = eng.measure(s["particles"][:P], s["lik"], s["beam"], s["origins"])
        check_lik(got, T[:P], M[:P], sc.lik, kernel, sh)
        check_beam(got, want[:P])
    assert M.sum() > 0 and want["n_hit"].sum() > 0
    assert np.array_equal(eng.beam_status(s["particles"], s["beam"], s["origins"]),
                          sc.cpu.beam_status(s["particles"], s["beam"], s["origins"]))


@pytest.mark.gpu
def test_accumulators_are_left_at_zero(eng_mod, make_engine):
    """Point-major launches of different shapes (P, N, slices, field widths; with and without a beam scan; through
    measure, measure_update and the resident set) one after another on one engine: each record is byte-identical to
    the same call on a fresh engine, so no launch leaves a particle's accumulator non-zero."""
    s = synth.scene(50_000, 4097, 600, 16, seed=251)
    sc = Scene(s)
    P, L, B, O = s["particles"], s["lik"], s["beam"], s["origins"]
    prior = np.full(300, 1.0 / 300, np.float32)
    states = np.zeros(700, synth.STATE)
    states["pos"] = np.stack([P["px"][:700], P["py"][:700], P["pz"][:700]], axis=1)
    states["rot"] = np.stack([P["qx"][:700], P["qy"][:700], P["qz"][:700], P["qw"][:700]], axis=1)

    def resident(e, lik, beam):
        e.particles_set(states, np.full(700, 1.0 / 700, np.float32))
        summ = e.particles_measure_update(lik, beam, O)
        return e.particles_get()[1].tobytes() + repr(sorted(summ.items())).encode()

    calls = [
        lambda e: e.measure(P[:1024], L[:512], B, O).tobytes(),
        lambda e: e.measure_update(P[:300], L[:97], None, None, prior, want_records=True)[2].tobytes(),
        lambda e: e.measure(P, L[:5], None, None).tobytes(),
        lambda e: resident(e, L[:200], B),
        lambda e: e.measure(P[:256], L[:96], None, None).tobytes(),
        lambda e: e.measure(P[:2000], L, B[:3], O).tobytes(),
        lambda e: e.measure(P[:1024], L[:512], B, O).tobytes(),
    ]
    shared = make_engine()
    set_map(eng_mod, shared, sc, 16)
    for i, call in enumerate(calls):
        fresh = make_engine()
        set_map(eng_mod, fresh, sc, 16)
        assert call(shared) == call(fresh), i
        fresh.close()
