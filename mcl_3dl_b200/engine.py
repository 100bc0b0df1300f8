"""ctypes binding of include/mcl3dl_b200.h (the C ABI of the CUDA engine).

`Engine` is the C-ABI handle (set_map / measure / measure_device / beam_status).  The reference is
compiled C++, so the host-side mirror of its plugin classes is C++ too:
mcl_3dl_b200/host/lidar_measurement_model_b200.h.  This module is what tests and bench.py call.

There is no fallback: if the CUDA library is missing or no device is usable, construction raises.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build
from .synth import POINT, POSE, RESULT, STATE

# mcl3dl_beam_ray: one ray of mcl3dl_beam_cast (40 bytes)
BEAM_RAY = np.dtype([("begin", "<f4", 3), ("end", "<f4", 3), ("pos", "<f4", 3), ("status", "<u4")])

ERR = {0: "ok", -1: "invalid argument", -2: "measure() before set_map()", -3: "CUDA runtime error",
       -4: "no usable CUDA device", -5: "grid exceeds 2^31-1 cells", -6: "search radius out of range"}


class EngineError(RuntimeError):
    def __init__(self, code, detail=""):
        self.code = code
        super().__init__("mcl3dl error %d (%s) %s" % (code, ERR.get(code, "?"), detail))


class LikParams(C.Structure):
    """mcl3dl_lik_params; defaults = include/mcl_3dl/parameters.h:74-76."""
    _fields_ = [("match_weight", C.c_float), ("match_dist_min", C.c_float), ("match_dist_flat", C.c_float),
                ("dist_weight", C.c_float * 3)]

    def __init__(self, match_weight=5.0, match_dist_min=0.2, match_dist_flat=0.05, dist_weight=(1.0, 1.0, 1.0)):
        super().__init__()
        self.match_weight, self.match_dist_min, self.match_dist_flat = match_weight, match_dist_min, match_dist_flat
        self.dist_weight[:] = dist_weight


class BeamParams(C.Structure):
    """mcl3dl_beam_params (derived; fill through beam_params_from_reference)."""
    _fields_ = [("map_grid_size", C.c_double * 3), ("dda_grid_size", C.c_double), ("ray_angle_half", C.c_double),
                ("hit_tolerance", C.c_double), ("hit_range_sq", C.c_float), ("sin_total_ref", C.c_float),
                ("beam_likelihood", C.c_float), ("beam_likelihood_min", C.c_float),
                ("filter_label_max", C.c_uint32), ("add_penalty_short_only_mode", C.c_int32),
                ("use_raycast_using_dda", C.c_int32), ("_reserved", C.c_int32)]

    def as_tuple(self):
        return (tuple(self.map_grid_size), self.dda_grid_size, self.ray_angle_half, self.hit_tolerance,
                self.hit_range_sq, self.sin_total_ref, self.beam_likelihood, self.beam_likelihood_min,
                self.filter_label_max, self.add_penalty_short_only_mode, self.use_raycast_using_dda)


class MapInfo(C.Structure):
    _fields_ = [("n_points", C.c_uint64), ("nn_dims", C.c_int32 * 3), ("nn_cell", C.c_float),
                ("nn_origin", C.c_float * 3), ("dda_dims", C.c_int32 * 3), ("dda_min", C.c_float * 3),
                ("dda_max", C.c_float * 3), ("device_bytes", C.c_uint64), ("build_ms", C.c_double)]


class MapWindowInfo(C.Structure):
    """mcl3dl_window_info (mcl3dl_map_window_info): whether the staged map is windowed, the staged window (raw box, lattice dimensions), the
    windows built since the map was staged and the stream time of the last one (header: rebuild_ms)."""
    _fields_ = [("windowed", C.c_int32), ("staged", C.c_int32), ("box_min", C.c_float * 3), ("box_max", C.c_float * 3),
                ("dims", C.c_int32 * 3), ("_pad", C.c_int32), ("rebuilds", C.c_uint64), ("rebuild_ms", C.c_double)]

    def as_dict(self):
        return {"windowed": bool(self.windowed), "staged": bool(self.staged), "box_min": tuple(self.box_min),
                "box_max": tuple(self.box_max), "dims": tuple(self.dims), "rebuilds": int(self.rebuilds),
                "rebuild_ms": float(self.rebuild_ms)}


class MapAppendInfo(C.Structure):
    _fields_ = [("n_before", C.c_uint64), ("n_appended", C.c_uint64), ("n_after", C.c_uint64), ("incremental", C.c_int32),
                ("cells_reselected", C.c_uint64), ("build_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class UpdateSummary(C.Structure):
    _fields_ = [("weight_sum", C.c_float), ("entropy", C.c_float), ("match_ratio_min", C.c_float),
                ("match_ratio_max", C.c_float), ("kept", C.c_int32), ("max_index", C.c_uint32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ScanParams(C.Structure):
    """mcl3dl_scan_params; defaults = parameters.h:67-77,95-103 and the node's downsample_x/y/z (parameters.cpp:85-87)."""
    _fields_ = [("downsample", C.c_float * 3),
                ("lik_clip_near", C.c_float), ("lik_clip_far", C.c_float), ("lik_clip_z_min", C.c_float), ("lik_clip_z_max", C.c_float),
                ("beam_clip_near", C.c_float), ("beam_clip_far", C.c_float), ("beam_clip_z_min", C.c_float), ("beam_clip_z_max", C.c_float),
                ("lik_num_points", C.c_uint32), ("beam_num_points", C.c_uint32), ("seed", C.c_uint64)]

    def __init__(self, downsample=(0.1, 0.1, 0.1), lik_clip=(0.5, 10.0, -2.0, 2.0), beam_clip=(0.5, 4.0, -2.0, 2.0),
                 lik_num_points=96, beam_num_points=3, seed=1):
        super().__init__()
        self.downsample[:] = downsample
        self.lik_clip_near, self.lik_clip_far, self.lik_clip_z_min, self.lik_clip_z_max = lik_clip
        self.beam_clip_near, self.beam_clip_far, self.beam_clip_z_min, self.beam_clip_z_max = beam_clip
        self.lik_num_points, self.beam_num_points, self.seed = lik_num_points, beam_num_points, seed


class ScanInfo(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("n_raw", "n_downsampled", "n_lik_clipped", "n_beam_clipped", "n_lik", "n_beam")]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class CloudView(C.Structure):
    """mcl3dl_cloud_view: a PointCloud2's data and layout (x, y, z FLOAT32, little-endian)."""
    _fields_ = [("data", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("point_step", C.c_uint32),
                ("row_step", C.c_uint32), ("offset", C.c_uint32 * 3), ("is_dense", C.c_int32)]


class Transform(C.Structure):
    """mcl3dl_transform: translation and RAW rotation (x y z w), doubles as a geometry_msgs/Transform carries them."""
    _fields_ = [("translation", C.c_double * 3), ("rotation", C.c_double * 4)]

    def __init__(self, translation=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0)):
        super().__init__()
        self.translation[:] = [float(v) for v in translation]
        self.rotation[:] = [float(v) for v in rotation]


class MapCloud(C.Structure):
    """mcl3dl_map_cloud: a map PointCloud2's view (x, y, z FLOAT32) and the byte offsets of its FLOAT32 "intensity" and
    UINT32 "label" fields (-1: absent)."""
    _fields_ = [("view", CloudView), ("intensity_offset", C.c_int32), ("label_offset", C.c_int32)]


class MapIntakeInfo(C.Structure):
    _fields_ = [("n_input", C.c_uint64), ("n_staged", C.c_uint64), ("downsampled", C.c_int32), ("device_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def cloud_span(width, height, point_step, row_step):
    """Bytes mcl3dl_scan_accumulate reads from a view's data: (height - 1) row_step + width point_step (0 when empty)."""
    if width * height == 0:
        return 0
    return (height - 1) * row_step + width * point_step


class NormalSamplerParams(C.Structure):
    """mcl3dl_normal_sampler_params (Engine.scan_sample_with_normal fills it)."""
    _fields_ = [("perform_weighting_ratio", C.c_double), ("max_weight_ratio", C.c_double), ("max_weight", C.c_double),
                ("normal_search_range", C.c_double), ("eigen_values", C.c_double * 3), ("eigen_vector", C.c_double * 3),
                ("mean_rot", C.c_float * 4), ("lik_num_points", C.c_uint32), ("beam_num_points", C.c_uint32),
                ("seed", C.c_uint64)]


class NormalSamplerInfo(C.Structure):
    _fields_ = [("n_lik", C.c_uint32), ("n_beam", C.c_uint32), ("n_normal", C.c_uint32 * 2), ("rounds", C.c_uint32 * 2),
                ("draws", C.c_uint64 * 2), ("max_weight", C.c_double), ("fpc_local", C.c_float * 3),
                ("weight_shift", C.c_int32)]

    def as_dict(self):
        return {"n_lik": int(self.n_lik), "n_beam": int(self.n_beam), "n_normal": [int(v) for v in self.n_normal],
                "rounds": [int(v) for v in self.rounds], "draws": [int(v) for v in self.draws],
                "max_weight": float(self.max_weight), "fpc_local": np.array(list(self.fpc_local), np.float32),
                "weight_shift": int(self.weight_shift)}


# PointCloudSamplerWithNormalParameters' defaults (parameters.h:50-56), the node's
NORMAL_SAMPLER_DEFAULTS = {"perform_weighting_ratio": 2.0, "max_weight_ratio": 5.0, "max_weight": 5.0,
                           "normal_search_range": 0.4}


class MatchParams(C.Structure):
    """mcl3dl_match_params (Engine.match_output fills it; its defaults are the node's)."""
    _fields_ = [("match_output_dist", C.c_double), ("unmatch_output_dist", C.c_double), ("chunk_length", C.c_float),
                ("max_search_radius", C.c_float)]


class GlobalLocalizationParams(C.Structure):
    """mcl3dl_global_localization_params (Engine.global_localization fills it; its defaults are the node's)."""
    _fields_ = [("grid", C.c_double), ("div_yaw", C.c_int32), ("imu_quat", C.c_float * 4), ("dist_weight", C.c_float * 3)]


class GlobalLocalizationInfo(C.Structure):
    _fields_ = [("n_input", C.c_uint64), ("n_downsampled", C.c_uint64), ("n_seeds", C.c_uint64), ("n_particles", C.c_uint64),
                ("probability", C.c_float), ("build_ms", C.c_double)]

    def as_dict(self):
        return {k: (float if k in ("probability", "build_ms") else int)(getattr(self, k)) for k, _ in self._fields_}


class LandmarkParams(C.Structure):
    """mcl3dl_landmark_params: the measured pose (mcl3dl_pose as 8 floats) and NormalLikelihoodNd<float, 6>'s a_ and
    sigma_inv_ (row-major)."""
    _fields_ = [("measured", C.c_float * 8), ("nd_a", C.c_float), ("sigma_inv", C.c_float * 36)]


def landmark_nd(covariance):
    """(nd_a, sigma_inv) of NormalLikelihoodNd<float, 6> for a 6x6 covariance given as cbLandmark reads it: the 36 values
    of the message's array taken column-major (so a non-symmetric covariance enters transposed), cast to float.  For
    callers without Eigen: the determinant and the inverse are numpy's (LAPACK LU in double on the float matrix), so
    these values are close to, but not, the bits Eigen's float LU gives; a node that wants the reference's values builds
    its own NormalLikelihoodNd and reads a_ and sigma_inv_ (mcl_3dl_b200/host/lidar_measurement_model_b200.h does)."""
    cov = np.asarray(covariance, dtype=np.float64).reshape(36)
    sigma = cov.reshape(6, 6, order="F").astype(np.float32)
    det = np.float32(np.linalg.det(sigma.astype(np.float64)))
    nd_a = np.float32(1.0 / ((2.0 * np.pi) ** 3 * np.float64(np.sqrt(det))))   # nd.h: std::sqrt of the float determinant
    sigma_inv = np.linalg.inv(sigma.astype(np.float64)).astype(np.float32)
    return nd_a, sigma_inv


class InitParams(C.Structure):
    """mcl3dl_init_params: the generator of the initial seed (diagonal sigma_ or multivariate norm_transform_, row-major)."""
    _fields_ = [("multivariate", C.c_int32), ("mean", C.c_float * 6), ("sigma", C.c_float * 6),
                ("norm_transform", C.c_float * 36)]


def noise_transform(covariance):
    """norm_transform_ of MultivariateNoiseGenerator<float> for cbPosition's covariance: the 36 values of the message's
    array read row-major (cov(i, j) = covariance[j + i * 6]), cast to float, only the lower triangle read, then
    V * sqrt(D) of the eigendecomposition, as float32 [6, 6].  For callers without Eigen: the eigendecomposition is
    numpy's (LAPACK in double on the float matrix), so these values are close to, but not, the bits Eigen's float
    SelfAdjointEigenSolver gives, and the order of the eigenvectors may differ; a node that wants the reference's values
    builds its own MultivariateNoiseGenerator and reads norm_transform_ (mcl_3dl_b200/host/lidar_measurement_model_b200.h
    does).  A negative eigenvalue gives NaN entries, which particles_init refuses."""
    cov = np.asarray(covariance, dtype=np.float64).reshape(6, 6).astype(np.float32).astype(np.float64)
    w, v = np.linalg.eigh(cov, UPLO="L")
    with np.errstate(invalid="ignore"):
        return (v * np.sqrt(w)).astype(np.float32)


class Estimate(C.Structure):
    """mcl3dl_estimate"""
    _fields_ = [("mean_biased", C.c_float * 8), ("max_state", C.c_float * 8), ("max_index", C.c_uint32),
                ("weight_sum_biased", C.c_float), ("cov", C.c_float * 36)]


class WorkStats(C.Structure):
    _fields_ = [("lik_index_rows", C.c_uint64), ("lik_points_scanned", C.c_uint64),
                ("beam_cells_stepped", C.c_uint64), ("beam_cells_occupied", C.c_uint64),
                ("beam_points_tested", C.c_uint64)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


EXPORTED_SYMBOLS = ["mcl3dl_measure_update", "mcl3dl_collect_stats", "mcl3dl_read_stats", "mcl3dl_abi_version", "mcl3dl_create", "mcl3dl_destroy", "mcl3dl_set_map", "mcl3dl_map_append", "mcl3dl_set_params",
                    "mcl3dl_measure", "mcl3dl_measure_device", "mcl3dl_beam_status",
                    "mcl3dl_beam_params_from_reference", "mcl3dl_get_map_info", "mcl3dl_last_timing",
                    "mcl3dl_kernel_launches", "mcl3dl_strerror", "mcl3dl_last_error_detail", "mcl3dl_near_field_info", "mcl3dl_nn_field_info", "mcl3dl_host_alloc", "mcl3dl_host_free", "mcl3dl_field_mode", "mcl3dl_field_nodes", "mcl3dl_field_upload", "mcl3dl_collect_timing",
                    "mcl3dl_exchange_create", "mcl3dl_exchange_open", "mcl3dl_measure_exchange_device", "mcl3dl_exchange_current",
                    "mcl3dl_particles_set", "mcl3dl_particles_get", "mcl3dl_particles_predict",
                    "mcl3dl_particles_measure_update", "mcl3dl_particles_resample", "mcl3dl_particles_estimate", "mcl3dl_scan_prepare", "mcl3dl_scan_get",
                    "mcl3dl_particles_measure_update_prepared", "mcl3dl_match_output",
                    "mcl3dl_particles_resize", "mcl3dl_global_localization",
                    "mcl3dl_particles_redraw_odom_noise", "mcl3dl_particles_noise", "mcl3dl_particles_imu_update",
                    "mcl3dl_particles_landmark_update", "mcl3dl_particles_reset_odom_err_integ", "mcl3dl_particles_get_poses",
                    "mcl3dl_particles_init", "mcl3dl_scan_sample_with_normal", "mcl3dl_scan_normals", "mcl3dl_beam_cast",
                    "mcl3dl_scan_accumulate", "mcl3dl_scan_accumulate_clear", "mcl3dl_scan_accumulated_get",
                    "mcl3dl_scan_prepare_accumulated", "mcl3dl_map_load", "mcl3dl_map_update_set",
                    "mcl3dl_map_update_commit", "mcl3dl_map_update_clear", "mcl3dl_map_get",
                    "mcl3dl_map_window_info"]

_LIBS = {}


def load_library(path=None):
    """Load (building if stale and nvcc is present) the in-tree CUDA library.  Raises if unavailable.
    `path` (or $MCL3DL_LIB) names an experiment variant built by build.build(out=...); libraries are cached per path."""
    path = path or os.environ.get("MCL3DL_LIB") or _build.LIB
    if path in _LIBS:
        return _LIBS[path]
    if path == _build.LIB and _build.stale():
        try:
            _build.build()
        except Exception:
            if not os.path.exists(path):
                raise
    L = C.CDLL(path)
    vp, sz = C.c_void_p, C.c_size_t
    L.mcl3dl_abi_version.restype = C.c_int
    L.mcl3dl_create.argtypes = [C.POINTER(vp), C.POINTER(C.c_int), C.c_int]
    L.mcl3dl_destroy.argtypes = [vp]
    L.mcl3dl_destroy.restype = None
    L.mcl3dl_set_map.argtypes = [vp, vp, sz, C.c_uint64, vp, vp]
    L.mcl3dl_map_append.argtypes = [vp, vp, sz, C.c_uint64, vp]
    L.mcl3dl_set_params.argtypes = [vp, vp, vp]
    L.mcl3dl_measure.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, vp]
    L.mcl3dl_measure_update.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp, vp, vp, vp]
    L.mcl3dl_measure_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp]
    L.mcl3dl_beam_status.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp]
    L.mcl3dl_beam_params_from_reference.argtypes = [vp, C.c_float, C.c_float, C.c_float, sz, C.c_float, C.c_float,
                                                    C.c_uint32, C.c_float, C.c_int, C.c_int, C.c_float, C.c_float]
    L.mcl3dl_beam_params_from_reference.restype = None
    L.mcl3dl_get_map_info.argtypes = [vp, vp]
    L.mcl3dl_map_window_info.argtypes = [vp, vp]
    L.mcl3dl_collect_stats.argtypes = [vp, C.c_int]
    L.mcl3dl_read_stats.argtypes = [vp, vp]
    L.mcl3dl_last_timing.argtypes = [vp] + [C.POINTER(C.c_double)] * 4
    L.mcl3dl_kernel_launches.argtypes = [vp]
    L.mcl3dl_kernel_launches.restype = C.c_uint64
    L.mcl3dl_strerror.argtypes = [C.c_int]
    L.mcl3dl_strerror.restype = C.c_char_p
    L.mcl3dl_last_error_detail.argtypes = [vp]
    L.mcl3dl_last_error_detail.restype = C.c_char_p
    L.mcl3dl_collect_timing.argtypes = [vp, C.c_int]
    L.mcl3dl_particles_set.argtypes = [vp, vp, vp, sz]
    L.mcl3dl_particles_get.argtypes = [vp, vp, vp, sz]
    L.mcl3dl_particles_predict.argtypes = [vp, vp, vp, C.c_float, C.c_float, C.c_float]
    L.mcl3dl_particles_measure_update.argtypes = [vp, vp, sz, vp, sz, vp, sz, C.c_float, vp]
    L.mcl3dl_particles_resample.argtypes = [vp, vp, vp, C.c_float, C.c_uint64]
    L.mcl3dl_particles_estimate.argtypes = [vp, vp, C.c_float, C.c_float, vp]
    L.mcl3dl_particles_resize.argtypes = [vp, sz]
    L.mcl3dl_global_localization.argtypes = [vp, vp, sz, vp, vp]
    L.mcl3dl_particles_redraw_odom_noise.argtypes = [vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_uint64]
    L.mcl3dl_particles_noise.argtypes = [vp, vp, vp, C.c_uint64]
    L.mcl3dl_particles_imu_update.argtypes = [vp, vp, C.c_double, vp]
    L.mcl3dl_particles_landmark_update.argtypes = [vp, vp, vp]
    L.mcl3dl_particles_reset_odom_err_integ.argtypes = [vp]
    L.mcl3dl_particles_get_poses.argtypes = [vp, vp, sz]
    L.mcl3dl_particles_init.argtypes = [vp, sz, vp, C.c_uint64]
    L.mcl3dl_scan_prepare.argtypes = [vp, vp, sz, vp, vp]
    L.mcl3dl_scan_get.argtypes = [vp, C.c_int, vp, sz, C.POINTER(sz)]
    L.mcl3dl_particles_measure_update_prepared.argtypes = [vp, vp, sz, C.c_float, vp]
    L.mcl3dl_scan_accumulate.argtypes = [vp, vp, vp, C.POINTER(C.c_uint32)]
    L.mcl3dl_scan_accumulate_clear.argtypes = [vp]
    L.mcl3dl_map_load.argtypes = [vp, vp, vp, C.c_uint64, vp, vp, vp]
    L.mcl3dl_map_update_set.argtypes = [vp, vp, vp, vp]
    L.mcl3dl_map_update_commit.argtypes = [vp, C.c_uint64, vp]
    L.mcl3dl_map_update_clear.argtypes = [vp]
    L.mcl3dl_map_get.argtypes = [vp, vp, vp, sz, C.POINTER(sz)]
    L.mcl3dl_scan_accumulated_get.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.mcl3dl_scan_prepare_accumulated.argtypes = [vp, vp, vp, vp]
    L.mcl3dl_scan_sample_with_normal.argtypes = [vp, vp, vp]
    L.mcl3dl_scan_normals.argtypes = [vp, C.c_int, vp, vp, vp, sz, C.POINTER(sz)]
    L.mcl3dl_match_output.argtypes = [vp, vp, vp, sz, vp, vp, C.POINTER(sz), vp, C.POINTER(sz)]
    L.mcl3dl_beam_cast.argtypes = [vp, vp, vp, sz, vp, sz, vp, sz, C.POINTER(sz)]
    L.mcl3dl_exchange_create.argtypes = [vp, sz, C.c_int, C.c_int, vp]
    L.mcl3dl_exchange_open.argtypes = [vp, vp]
    L.mcl3dl_measure_exchange_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, vp, C.POINTER(vp)]
    L.mcl3dl_exchange_current.argtypes = [vp, vp, C.POINTER(vp), C.POINTER(C.c_int)]
    L.mcl3dl_near_field_info.argtypes = [vp, C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]
    L.mcl3dl_nn_field_info.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.mcl3dl_field_mode.argtypes = [vp, C.c_int]
    L.mcl3dl_field_nodes.argtypes = [vp, vp, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.mcl3dl_field_upload.argtypes = [vp, vp, C.POINTER(C.c_int32)]
    L.mcl3dl_host_alloc.argtypes = [vp, sz, C.POINTER(vp)]
    L.mcl3dl_host_free.argtypes = [vp, vp]
    assert L.mcl3dl_abi_version() == 3
    _LIBS[path] = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else None


def beam_params_from_reference(map_grid=(0.1, 0.1, 0.1), num_points_default=3, beam_likelihood_min=0.2,
                               ang_total_ref=np.pi / 6.0, filter_label_max=0xFFFFFFFF, hit_range=0.3,
                               add_penalty_short_only_mode=True, ray_angle_half=0.25 * np.pi / 180.0,
                               dda_grid_size=0.2, use_raycast_using_dda=True):
    """LidarMeasurementModelBeamParameters (parameters.h:95-111) -> derived mcl3dl_beam_params.
    (use_raycast_using_dda defaults to True here; the reference's default is False = the KD-tree caster.)"""
    L = load_library()
    bp = BeamParams()
    L.mcl3dl_beam_params_from_reference(C.byref(bp), map_grid[0], map_grid[1], map_grid[2], num_points_default,
                                        beam_likelihood_min, ang_total_ref, filter_label_max, hit_range,
                                        1 if add_penalty_short_only_mode else 0, 1 if use_raycast_using_dda else 0,
                                        ray_angle_half, dda_grid_size)
    return bp


class Engine:
    """Handle on mcl3dl_engine.  devices: list of CUDA ordinals (map replicated, particles split)."""

    def __init__(self, devices=(0,), lib_path=None):
        self.L = load_library(lib_path)
        self.h = C.c_void_p()
        ids = (C.c_int * len(devices))(*devices)
        rc = self.L.mcl3dl_create(C.byref(self.h), ids, len(devices))
        if rc != 0:
            self.h = None
            raise EngineError(rc)
        self.devices = tuple(devices)

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self.L.mcl3dl_last_error_detail(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.mcl3dl_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_map(self, map_pts, lik=None, beam=None, stamp=None):
        """stamp: the cloud's header.stamp, the reference's rebuild trigger (same stamp, size and params = no-op).
        None: a fresh stamp per call (as the C++ adapter does), so that a different cloud is never mistaken for the old."""
        map_pts = np.ascontiguousarray(map_pts, dtype=POINT)
        if stamp is None:
            self._stamp = getattr(self, "_stamp", 0) + 1
            stamp = (1 << 40) + self._stamp
        self._check(self.L.mcl3dl_set_map(self.h, _ptr(map_pts), len(map_pts), stamp,
                                          C.byref(lik) if lik is not None else None,
                                          C.byref(beam) if beam is not None else None))

    def map_append(self, pts, stamp=None):
        """Append pts to the staged map (the node's map update; include/mcl3dl_b200.h: mcl3dl_map_append).  stamp as in
        set_map.  Returns {"n_before", "n_appended", "n_after", "incremental", "cells_reselected", "build_ms"}."""
        pts = np.ascontiguousarray(pts, dtype=POINT)
        if stamp is None:
            self._stamp = getattr(self, "_stamp", 0) + 1
            stamp = (1 << 40) + self._stamp
        info = MapAppendInfo()
        self._check(self.L.mcl3dl_map_append(self.h, _ptr(pts), len(pts), stamp, C.byref(info)))
        return info.as_dict()

    def set_params(self, lik=None, beam=None):
        self._check(self.L.mcl3dl_set_params(self.h, C.byref(lik) if lik is not None else None,
                                             C.byref(beam) if beam is not None else None))

    def map_info(self):
        mi = MapInfo()
        self._check(self.L.mcl3dl_get_map_info(self.h, C.byref(mi)))
        return mi

    def map_window_info(self):
        """The map window (include/mcl3dl_b200.h, "Map window"): {"windowed", "staged", "box_min", "box_max", "dims",
        "rebuilds", "rebuild_ms"}."""
        wi = MapWindowInfo()
        self._check(self.L.mcl3dl_map_window_info(self.h, C.byref(wi)))
        return wi.as_dict()

    def near_field_info(self):
        """[(k, bytes)] of the near-field screens of the staged map: [0] likelihood search, [1] KD-tree raycaster."""
        k = (C.c_int32 * 2)()
        b = (C.c_uint64 * 2)()
        self._check(self.L.mcl3dl_near_field_info(self.h, k, b))
        return [(int(k[0]), int(b[0])), (int(k[1]), int(b[1]))]

    def nn_field_info(self):
        """The NN field of the staged map: {"bytes", "candidates", "overflow_cells", "voxel_edge", "wide_cells"} (bytes 0:
        not staged)."""
        v = (C.c_uint64 * 5)()
        self._check(self.L.mcl3dl_nn_field_info(self.h, v))
        return {"bytes": int(v[0]), "candidates": int(v[1]), "overflow_cells": int(v[2]), "voxel_edge": v[3] * 1e-6,
                "wide_cells": int(v[4])}

    def field_mode(self, enable=True):
        """Opt-in, inexact: route the likelihood model through the trilinear distance volume (include/mcl3dl_b200.h)."""
        self._check(self.L.mcl3dl_field_mode(self.h, 1 if enable else 0))

    def field_nodes(self, download=True):
        """(nodes float32[nz, ny, nx] or None, origin[3], edge) of the field-mode lattice (rescaled space)."""
        dims, org, edge = (C.c_int32 * 3)(), (C.c_float * 3)(), C.c_float(0)
        self._check(self.L.mcl3dl_field_nodes(self.h, None, dims, org, C.byref(edge)))
        nodes = None
        if download:
            nodes = np.zeros((dims[2], dims[1], dims[0]), dtype=np.float32)
            self._check(self.L.mcl3dl_field_nodes(self.h, _ptr(nodes), dims, org, C.byref(edge)))
        return nodes, np.array(list(org), np.float32), float(edge.value), tuple(int(d) for d in dims)

    def field_upload(self, nodes):
        nodes = np.ascontiguousarray(nodes, dtype=np.float32)
        dims = (C.c_int32 * 3)(nodes.shape[2], nodes.shape[1], nodes.shape[0])
        self._check(self.L.mcl3dl_field_upload(self.h, _ptr(nodes), dims))

    def measure(self, poses, lik_pts=None, beam_pts=None, origins=None, out=None):
        poses = np.ascontiguousarray(poses, dtype=POSE)
        lik_pts = np.ascontiguousarray(lik_pts if lik_pts is not None else np.zeros(0, POINT), dtype=POINT)
        beam_pts = np.ascontiguousarray(beam_pts if beam_pts is not None else np.zeros(0, POINT), dtype=POINT)
        origins = np.ascontiguousarray(origins if origins is not None else np.zeros((0, 3)), dtype=np.float32)
        origins = origins.reshape(-1, 3)
        if out is None:
            out = np.zeros(len(poses), dtype=RESULT)
        self._check(self.L.mcl3dl_measure(self.h, _ptr(poses), len(poses), _ptr(lik_pts), len(lik_pts),
                                          _ptr(beam_pts), len(beam_pts), _ptr(origins), len(origins), _ptr(out)))
        return out

    def host_array(self, n, dtype):
        """A zeroed numpy array of n items in page-locked memory of this engine (mcl3dl_host_alloc): pose and record
        arrays passed to measure / bind_measure from such memory are transferred in place, without the staging memcpy.
        The memory is returned by host_free(array) or when the engine is closed - do not use the array after that."""
        dtype = np.dtype(dtype)
        nbytes = max(1, int(n) * dtype.itemsize)
        p = C.c_void_p()
        self._check(self.L.mcl3dl_host_alloc(self.h, nbytes, C.byref(p)))
        buf = (C.c_char * nbytes).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype, count=int(n))
        arr[...] = np.zeros((), dtype)
        return arr

    def host_free(self, arr):
        self._check(self.L.mcl3dl_host_free(self.h, arr.ctypes.data))

    def bind_measure(self, poses, lik_pts, beam_pts, origins, out):
        """A repeated update over the SAME host arrays (their contents may change between calls): resolves the buffer
        addresses once and returns a zero-argument callable that runs mcl3dl_measure on them.  What a C++ caller does
        anyway; it keeps ~20 us of numpy/ctypes argument marshalling out of every call.  The arrays must already have
        the ABI dtypes and be C-contiguous (no hidden copies, or the call would read stale copies)."""
        def chk(a, dt, name):
            if a is None:
                return np.zeros(0, dt)
            if a.dtype != dt or not a.flags["C_CONTIGUOUS"]:
                raise ValueError("%s must be a C-contiguous array of %s" % (name, dt))
            return a
        poses, lik_pts, beam_pts = chk(poses, POSE, "poses"), chk(lik_pts, POINT, "lik_pts"), chk(beam_pts, POINT, "beam_pts")
        origins = chk(origins if origins is None else origins.reshape(-1, 3), np.dtype(np.float32), "origins")
        out = chk(out, RESULT, "out")
        if len(out) != len(poses):
            raise ValueError("out must hold one record per particle")
        keep = (poses, lik_pts, beam_pts, origins, out)  # the closure keeps the buffers alive
        args = (self.h, _ptr(poses), len(poses), _ptr(lik_pts), len(lik_pts), _ptr(beam_pts), len(beam_pts), _ptr(origins),
                len(origins.reshape(-1, 3)), _ptr(out))
        fn = self.L.mcl3dl_measure

        def call():
            rc = fn(*args)
            if rc != 0:
                self._check(rc)
            return keep[4]
        return call

    def measure_update(self, poses, lik_pts, beam_pts, origins, prior, extra_likelihood=None, want_records=False):
        """Fused measurement + weight update (pf::ParticleFilter::measure with the node's lambda).
        Returns (posterior float32[P], summary dict, records or None)."""
        poses = np.ascontiguousarray(poses, dtype=POSE)
        lik_pts = np.ascontiguousarray(lik_pts if lik_pts is not None else np.zeros(0, POINT), dtype=POINT)
        beam_pts = np.ascontiguousarray(beam_pts if beam_pts is not None else np.zeros(0, POINT), dtype=POINT)
        origins = np.ascontiguousarray(origins if origins is not None else np.zeros((0, 3)), dtype=np.float32)
        origins = origins.reshape(-1, 3)
        prior = np.ascontiguousarray(prior, dtype=np.float32)
        extra = np.ascontiguousarray(extra_likelihood, dtype=np.float32) if extra_likelihood is not None else None
        post = np.zeros(len(poses), dtype=np.float32)
        rec = np.zeros(len(poses), dtype=RESULT) if want_records else None
        summ = UpdateSummary()
        self._check(self.L.mcl3dl_measure_update(self.h, _ptr(poses), len(poses), _ptr(lik_pts), len(lik_pts),
                                                 _ptr(beam_pts), len(beam_pts), _ptr(origins), len(origins),
                                                 _ptr(prior), _ptr(extra) if extra is not None else None,
                                                 _ptr(post), _ptr(rec) if rec is not None else None, C.byref(summ)))
        return post, summ.as_dict(), rec

    def measure_device(self, d_poses, n_particles, d_lik, n_lik, d_beam, n_beam, d_origins, n_origins, d_out,
                       stream=0):
        """All d_* are raw device addresses (ints, e.g. torch.Tensor.data_ptr()); async on `stream`."""
        self._check(self.L.mcl3dl_measure_device(self.h, d_poses, n_particles, d_lik, n_lik, d_beam, n_beam,
                                                 d_origins, n_origins, d_out, stream))

    def beam_status(self, poses, beam_pts, origins):
        poses = np.ascontiguousarray(poses, dtype=POSE)
        beam_pts = np.ascontiguousarray(beam_pts, dtype=POINT)
        origins = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
        st = np.zeros((len(poses), len(beam_pts)), dtype=np.uint8)
        self._check(self.L.mcl3dl_beam_status(self.h, _ptr(poses), len(poses), _ptr(beam_pts), len(beam_pts),
                                              _ptr(origins), len(origins), _ptr(st)))
        return st

    def beam_cast(self, pose, beam_pts=None, origins=((0.0, 0.0, 0.0),)):
        """The node's ray markers from one pose (include/mcl3dl_b200.h: mcl3dl_beam_cast) -> BEAM_RAY[n_rays] in scan
        order: begin, end, the deciding cast step's position (NaN for LONG) and the status.  beam_pts=None: the sampled
        beam scan of the last scan_prepare / scan_sample_with_normal."""
        pose = np.ascontiguousarray(pose, dtype=POSE).reshape(1)
        origins = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
        if beam_pts is not None:
            beam_pts = np.ascontiguousarray(beam_pts, dtype=POINT)
            cap = len(beam_pts)
        else:  # the prepared scan's size (no prepared scan: the call below reports the error)
            n_b = C.c_size_t(0)
            cap = n_b.value if self.L.mcl3dl_scan_get(self.h, 4, None, 0, C.byref(n_b)) == 0 else 0
        out = np.zeros(cap, dtype=BEAM_RAY)
        n = C.c_size_t(0)
        # (an empty host scan still needs a pointer: NULL selects the prepared scan)
        self._check(self.L.mcl3dl_beam_cast(self.h, _ptr(pose), beam_pts.ctypes.data if beam_pts is not None else None,
                                            len(beam_pts) if beam_pts is not None else 0, _ptr(origins), len(origins),
                                            _ptr(out), cap, C.byref(n)))
        return out[:n.value]

    def collect_stats(self, enable=True):
        self._check(self.L.mcl3dl_collect_stats(self.h, 1 if enable else 0))

    def read_stats(self):
        ws = WorkStats()
        self._check(self.L.mcl3dl_read_stats(self.h, C.byref(ws)))
        return ws.as_dict()

    # ---- resident particle set (scope row f3; see include/mcl3dl_b200.h)
    def particles_set(self, states, prob):
        states = np.ascontiguousarray(states, dtype=STATE)
        prob = np.ascontiguousarray(prob, dtype=np.float32)
        assert len(states) == len(prob)
        self._check(self.L.mcl3dl_particles_set(self.h, _ptr(states), _ptr(prob), len(states)))
        self._n_resident = len(states)

    def particles_init(self, n, mean6, seed, sigma=None, norm_transform=None):
        """pf_->initUsingNoiseGenerator on the device (include/mcl3dl_b200.h: mcl3dl_particles_init): creates or replaces
        the resident set with n particles.  mean6 = the generator's mean (x y z roll pitch yaw); exactly one of sigma (6,
        DiagonalNoiseGenerator) and norm_transform ([6, 6], MultivariateNoiseGenerator; noise_transform builds it from a
        covariance) is given."""
        assert (sigma is None) != (norm_transform is None)
        prm = InitParams()
        prm.multivariate = 0 if norm_transform is None else 1
        m = np.ascontiguousarray(mean6, dtype=np.float32)
        assert m.size == 6
        C.memmove(prm.mean, m.ctypes.data, 24)
        if sigma is not None:
            sg = np.ascontiguousarray(sigma, dtype=np.float32)
            assert sg.size == 6
            C.memmove(prm.sigma, sg.ctypes.data, 24)
        else:
            t = np.ascontiguousarray(norm_transform, dtype=np.float32)
            assert t.size == 36
            C.memmove(prm.norm_transform, t.ctypes.data, 144)
        self._check(self.L.mcl3dl_particles_init(self.h, n, C.byref(prm), seed))
        self._n_resident = int(n)

    def particles_get(self):
        states = np.zeros(self._n_resident, dtype=STATE)
        prob = np.zeros(self._n_resident, dtype=np.float32)
        self._check(self.L.mcl3dl_particles_get(self.h, _ptr(states), _ptr(prob), len(states)))
        return states, prob

    def particles_predict(self, odom_prev, odom_current, time_diff, tc_lin, tc_ang):
        a = np.ascontiguousarray(odom_prev, dtype=POSE).reshape(1)
        b = np.ascontiguousarray(odom_current, dtype=POSE).reshape(1)
        self._check(self.L.mcl3dl_particles_predict(self.h, _ptr(a), _ptr(b), time_diff, tc_lin, tc_ang))

    def particles_measure_update(self, lik_pts, beam_pts, origins, odom_err_integ_lin_sigma=0.0):
        lik_pts = np.ascontiguousarray(lik_pts if lik_pts is not None else np.zeros(0, POINT), dtype=POINT)
        beam_pts = np.ascontiguousarray(beam_pts if beam_pts is not None else np.zeros(0, POINT), dtype=POINT)
        origins = np.ascontiguousarray(origins if origins is not None else np.zeros((0, 3)), dtype=np.float32).reshape(-1, 3)
        summ = UpdateSummary()
        self._check(self.L.mcl3dl_particles_measure_update(self.h, _ptr(lik_pts), len(lik_pts), _ptr(beam_pts), len(beam_pts),
                                                           _ptr(origins), len(origins), odom_err_integ_lin_sigma,
                                                           C.byref(summ)))
        return summ.as_dict()

    def particles_resample(self, sigma_pos, sigma_rpy, initial_frac, seed):
        sp = np.ascontiguousarray(sigma_pos, dtype=np.float32)
        sr = np.ascontiguousarray(sigma_rpy, dtype=np.float32)
        self._check(self.L.mcl3dl_particles_resample(self.h, _ptr(sp), _ptr(sr), initial_frac, seed))

    def particles_redraw_odom_noise(self, lin_lin, lin_ang, ang_lin, ang_ang, seed):
        """The node's odometry-noise redraw on the resident set (include/mcl3dl_b200.h: mcl3dl_particles_redraw_odom_noise)."""
        self._check(self.L.mcl3dl_particles_redraw_odom_noise(self.h, lin_lin, lin_ang, ang_lin, ang_ang, seed))

    def particles_noise(self, sigma_pos, sigma_rpy, seed):
        """pf_->noise(State6DOF(sigma_pos, sigma_rpy)), expansion resetting, on the resident set
        (include/mcl3dl_b200.h: mcl3dl_particles_noise)."""
        sp = np.ascontiguousarray(sigma_pos, dtype=np.float32)
        sr = np.ascontiguousarray(sigma_rpy, dtype=np.float32)
        assert sp.size == 3 and sr.size == 3
        self._check(self.L.mcl3dl_particles_noise(self.h, _ptr(sp), _ptr(sr), seed))

    def particles_imu_update(self, acc_measure, acc_var):
        """The IMU gravity update on the resident set (include/mcl3dl_b200.h: mcl3dl_particles_imu_update); returns the
        update summary as a dict."""
        acc = np.ascontiguousarray(acc_measure, dtype=np.float32)
        assert acc.size == 3
        summ = UpdateSummary()
        self._check(self.L.mcl3dl_particles_imu_update(self.h, _ptr(acc), acc_var, C.byref(summ)))
        return summ.as_dict()

    def particles_landmark_update(self, measured, nd_a, sigma_inv):
        """cbLandmark's pf_->measure on the resident set (include/mcl3dl_b200.h: mcl3dl_particles_landmark_update).
        measured: one POSE (RAW rotation); nd_a, sigma_inv: NormalLikelihoodNd<float, 6>'s a_ and sigma_inv_ [6, 6]
        (landmark_nd builds them from a covariance).  Returns the update summary as a dict."""
        m = np.ascontiguousarray(measured, dtype=POSE).reshape(1)
        si = np.ascontiguousarray(sigma_inv, dtype=np.float32)
        assert si.size == 36
        prm = LandmarkParams()
        C.memmove(prm.measured, m.ctypes.data, 32)
        prm.nd_a = nd_a
        C.memmove(prm.sigma_inv, si.ctypes.data, 144)
        summ = UpdateSummary()
        self._check(self.L.mcl3dl_particles_landmark_update(self.h, C.byref(prm), C.byref(summ)))
        return summ.as_dict()

    def particles_reset_odom_err_integ(self):
        """The node's integ_reset_func on the resident set (include/mcl3dl_b200.h: mcl3dl_particles_reset_odom_err_integ)."""
        self._check(self.L.mcl3dl_particles_reset_odom_err_integ(self.h))

    def particles_get_poses(self):
        """publishParticles' poses: POSE [n] with normalised rotations (include/mcl3dl_b200.h: mcl3dl_particles_get_poses)."""
        out = np.zeros(self._n_resident, dtype=POSE)
        self._check(self.L.mcl3dl_particles_get_poses(self.h, _ptr(out), len(out)))
        return out

    def particles_resize(self, num):
        """pf_->resizeParticle(num) on the resident set (include/mcl3dl_b200.h: mcl3dl_particles_resize)."""
        self._check(self.L.mcl3dl_particles_resize(self.h, num))
        self._n_resident = int(num)

    def global_localization(self, pts=None, grid=0.3, div_yaw=12, imu_quat=(0.0, 0.0, 0.0, 1.0), dist_weight=(1.0, 1.0, 1.0)):
        """The node's global_localization service on the device (include/mcl3dl_b200.h: mcl3dl_global_localization): seeds
        the resident set from pts (POINT array) or, pts=None, from the staged map.  Returns the info as a dict; with no
        seed the resident set is left as it was."""
        gp = GlobalLocalizationParams(grid, div_yaw, (C.c_float * 4)(*imu_quat), (C.c_float * 3)(*dist_weight))
        info = GlobalLocalizationInfo()
        src, n = None, 0
        if pts is not None:  # a host cloud, possibly empty: never NULL, which would mean the staged map
            pts = np.ascontiguousarray(pts, dtype=POINT)
            n = len(pts)
            buf = pts if n else np.zeros(1, POINT)
            src = buf.ctypes.data_as(C.c_void_p)
        self._check(self.L.mcl3dl_global_localization(self.h, src, n, C.byref(gp), C.byref(info)))
        if info.n_particles:
            self._n_resident = int(info.n_particles)
        return info.as_dict()

    # ---- scan preprocessing on the device (scope row f4; include/mcl3dl_b200.h)
    def scan_prepare(self, raw_pts, params):
        raw_pts = np.ascontiguousarray(raw_pts, dtype=POINT)
        info = ScanInfo()
        self._check(self.L.mcl3dl_scan_prepare(self.h, _ptr(raw_pts), len(raw_pts), C.byref(params), C.byref(info)))
        return info.as_dict()

    def scan_get(self, which):
        """which: 0 downsampled, 1 / 2 clipped (likelihood / beam), 3 / 4 sampled scans."""
        n = C.c_size_t(0)
        self._check(self.L.mcl3dl_scan_get(self.h, which, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=POINT)
        if n.value:
            self._check(self.L.mcl3dl_scan_get(self.h, which, _ptr(out), len(out), C.byref(n)))
        return out

    # ---- cloud accumulation on the device (include/mcl3dl_b200.h: mcl3dl_scan_accumulate)
    def scan_accumulate(self, data, width, height, point_step, row_step, offsets, is_dense=True,
                        translation=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0)):
        """accumCloud on the device: one PointCloud2 (data: a C-contiguous numpy byte or structured array holding its
        bytes; offsets: the byte offsets of the FLOAT32 x, y, z) moved into the odom frame by (translation, RAW rotation x
        y z w) and appended with the next accumulation index as its label.  A view that would read past the end of data
        raises ValueError before the engine is called.  Returns the number of clouds accumulated."""
        if not isinstance(data, np.ndarray) or not data.flags.c_contiguous:
            raise ValueError("data must be a C-contiguous numpy array")
        span = cloud_span(int(width), int(height), int(point_step), int(row_step))
        if span > data.nbytes:
            raise ValueError("the view spans %d bytes, data holds %d" % (span, data.nbytes))
        offsets = [int(o) for o in offsets]
        if len(offsets) != 3:
            raise ValueError("offsets: the byte offsets of x, y, z")
        view = CloudView(data.ctypes.data_as(C.c_void_p) if data.nbytes else None, width, height, point_step, row_step,
                         (C.c_uint32 * 3)(*offsets), 1 if is_dense else 0)
        tf = Transform(translation, rotation)
        n = C.c_uint32(0)
        self._check(self.L.mcl3dl_scan_accumulate(self.h, C.byref(view), C.byref(tf), C.byref(n)))
        return int(n.value)

    def scan_accumulate_clear(self):
        """accumClear: empties the accumulation (the prepared scans stay)."""
        self._check(self.L.mcl3dl_scan_accumulate_clear(self.h))

    def scan_accumulated_get(self):
        """The accumulated points in the odom frame (POINT array; label = accumulation index)."""
        n = C.c_size_t(0)
        self._check(self.L.mcl3dl_scan_accumulated_get(self.h, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=POINT)
        if n.value:
            self._check(self.L.mcl3dl_scan_accumulated_get(self.h, _ptr(out), len(out), C.byref(n)))
        return out

    def scan_prepare_accumulated(self, params, translation=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0)):
        """measure() on the device: the accumulation moved into base_link by (translation, RAW rotation), then
        scan_prepare's pipeline (params: ScanParams).  Returns the scan info as a dict."""
        tf = Transform(translation, rotation)
        info = ScanInfo()
        self._check(self.L.mcl3dl_scan_prepare_accumulated(self.h, C.byref(tf), C.byref(params), C.byref(info)))
        return info.as_dict()

    # ---- map intake on the device (include/mcl3dl_b200.h: mcl3dl_map_load)
    @staticmethod
    def _map_cloud(data, width, height, point_step, row_step, offsets, intensity_offset, label_offset, is_dense):
        if not isinstance(data, np.ndarray) or not data.flags.c_contiguous:
            raise ValueError("data must be a C-contiguous numpy array")
        span = cloud_span(int(width), int(height), int(point_step), int(row_step))
        if span > data.nbytes:
            raise ValueError("the view spans %d bytes, data holds %d" % (span, data.nbytes))
        offsets = [int(o) for o in offsets]
        if len(offsets) != 3:
            raise ValueError("offsets: the byte offsets of x, y, z")
        io = -1 if intensity_offset is None else int(intensity_offset)
        lo = -1 if label_offset is None else int(label_offset)
        view = CloudView(data.ctypes.data_as(C.c_void_p) if data.nbytes else None, width, height, point_step, row_step,
                         (C.c_uint32 * 3)(*offsets), 1 if is_dense else 0)
        return MapCloud(view, io, lo)

    @staticmethod
    def _leaf(leaf):
        leaf = np.ascontiguousarray(leaf, dtype=np.float32)
        if leaf.shape != (3,):
            raise ValueError("leaf: three leaf sizes")
        return leaf

    def map_load(self, data, width, height, point_step, row_step, offsets, leaf, lik=None, beam=None, intensity_offset=None,
                 label_offset=None, is_dense=True, stamp=None):
        """loadMapCloud on the device: one map PointCloud2 (data: a C-contiguous numpy array holding its bytes; offsets:
        the byte offsets of the FLOAT32 x, y, z; intensity_offset / label_offset: the FLOAT32 intensity and UINT32 label
        fields, None when absent) converted, downsampled at leaf and staged as set_map stages a map (stamp as there).  A
        view that would read past the end of data raises ValueError before the engine is called.  Returns
        {"n_input", "n_staged", "downsampled", "device_ms"}."""
        m = self._map_cloud(data, width, height, point_step, row_step, offsets, intensity_offset, label_offset, is_dense)
        leaf = self._leaf(leaf)
        if stamp is None:
            self._stamp = getattr(self, "_stamp", 0) + 1
            stamp = (1 << 40) + self._stamp
        info = MapIntakeInfo()
        self._check(self.L.mcl3dl_map_load(self.h, C.byref(m), leaf.ctypes.data_as(C.c_void_p), stamp,
                                           C.byref(lik) if lik is not None else None,
                                           C.byref(beam) if beam is not None else None, C.byref(info)))
        return info.as_dict()

    def map_update_set(self, data, width, height, point_step, row_step, offsets, leaf, intensity_offset=None,
                       label_offset=None, is_dense=True):
        """cbMapcloudUpdate on the device: the patch converted and downsampled at leaf, pending until
        map_update_commit (it replaces a pending patch).  Arguments and the overrun check as map_load."""
        m = self._map_cloud(data, width, height, point_step, row_step, offsets, intensity_offset, label_offset, is_dense)
        leaf = self._leaf(leaf)
        info = MapIntakeInfo()
        self._check(self.L.mcl3dl_map_update_set(self.h, C.byref(m), leaf.ctypes.data_as(C.c_void_p), C.byref(info)))
        return info.as_dict()

    def map_update_commit(self, stamp=None):
        """The map update timer: the pending patch appended to the staged map (map_append's info dict)."""
        if stamp is None:
            self._stamp = getattr(self, "_stamp", 0) + 1
            stamp = (1 << 40) + self._stamp
        info = MapAppendInfo()
        self._check(self.L.mcl3dl_map_update_commit(self.h, stamp, C.byref(info)))
        return info.as_dict()

    def map_update_clear(self):
        """cbPosition's pc_update_.reset(): drops the pending patch."""
        self._check(self.L.mcl3dl_map_update_clear(self.h))

    def map_get(self):
        """The staged map: (POINT array, float32 intensities), in staged order."""
        n = C.c_size_t(0)
        self._check(self.L.mcl3dl_map_get(self.h, None, None, 0, C.byref(n)))
        pts = np.zeros(n.value, dtype=POINT)
        inten = np.zeros(n.value, dtype=np.float32)
        if n.value:
            self._check(self.L.mcl3dl_map_get(self.h, _ptr(pts), inten.ctypes.data_as(C.c_void_p), len(pts), C.byref(n)))
        return pts, inten

    def scan_sample_with_normal(self, mean_rot, pos_cov, params=None, lik_num_points=96, beam_num_points=3, seed=1):
        """The node's PointCloudSamplerWithNormal on the clipped clouds of the last scan_prepare; the new samples replace
        its sampled scans (include/mcl3dl_b200.h: mcl3dl_scan_sample_with_normal).  mean_rot: expectation().rot_ (x y z
        w, raw); pos_cov: the covariance (its 3 x 3 position block is used; 6 x 6 accepted); params: a dict over
        NORMAL_SAMPLER_DEFAULTS.  setParticleStatistics is restated with numpy: eigh of |pos_cov| in double (LAPACK, so the
        eigenvector's bits and sign may differ from Eigen's SelfAdjointEigenSolver; the C++ adapter uses Eigen).
        Returns the info as a dict."""
        prm = dict(NORMAL_SAMPLER_DEFAULTS, **(params or {}))
        cov = np.abs(np.asarray(pos_cov, dtype=np.float64)[:3, :3])
        w, v = np.linalg.eigh(cov)
        return self.scan_sample_with_normal_eigen(mean_rot, w, v[:, 2], prm, lik_num_points, beam_num_points, seed)

    def scan_sample_with_normal_eigen(self, mean_rot, eigen_values, eigen_vector, params=None, lik_num_points=96,
                                      beam_num_points=3, seed=1):
        """mcl3dl_scan_sample_with_normal with the eigendecomposition given (ascending eigenvalues, the eigenvector of
        the largest)."""
        prm = dict(NORMAL_SAMPLER_DEFAULTS, **(params or {}))
        sp = NormalSamplerParams()
        for k in NORMAL_SAMPLER_DEFAULTS:
            setattr(sp, k, float(prm[k]))
        sp.eigen_values[:] = [float(x) for x in eigen_values]
        sp.eigen_vector[:] = [float(x) for x in eigen_vector]
        sp.mean_rot[:] = [float(x) for x in np.asarray(mean_rot, np.float32).reshape(4)]
        sp.lik_num_points, sp.beam_num_points, sp.seed = lik_num_points, beam_num_points, seed
        info = NormalSamplerInfo()
        self._check(self.L.mcl3dl_scan_sample_with_normal(self.h, C.byref(sp), C.byref(info)))
        return info.as_dict()

    def scan_normals(self, which):
        """(normals float32[n, 3], neighbour counts uint32[n], fixed-point weights uint64[n]) of the clipped cloud of
        model `which` (0 likelihood, 1 beam) from the last scan_sample_with_normal."""
        n = C.c_size_t(0)
        self._check(self.L.mcl3dl_scan_normals(self.h, which, None, None, None, 0, C.byref(n)))
        nrm = np.zeros((n.value, 3), np.float32)
        nb = np.zeros(n.value, np.uint32)
        q = np.zeros(n.value, np.uint64)
        if n.value:
            self._check(self.L.mcl3dl_scan_normals(self.h, which, _ptr(nrm), _ptr(nb), _ptr(q), n.value, C.byref(n)))
        return nrm, nb, q

    def match_output(self, pose, pts=None, match_dist=0.1, unmatch_dist=0.5, chunk_length=20.0, max_search_radius=0.2):
        """The node's matched / unmatched clouds (include/mcl3dl_b200.h: mcl3dl_match_output) -> (matched, unmatched) as
        POINT arrays of the transformed points.  pts=None: the downsampled cloud of the last scan_prepare."""
        pose = np.ascontiguousarray(pose, dtype=POSE).reshape(1)
        mp = MatchParams(match_dist, unmatch_dist, chunk_length, max_search_radius)
        if pts is not None:
            pts = np.ascontiguousarray(pts, dtype=POINT)
            cap = len(pts)
        else:  # the prepared cloud's size (no prepared scan: the call below reports the error)
            n_ds = C.c_size_t(0)
            cap = n_ds.value if self.L.mcl3dl_scan_get(self.h, 0, None, 0, C.byref(n_ds)) == 0 else 0
        out = [np.zeros(cap, dtype=POINT), np.zeros(cap, dtype=POINT)]
        n = [C.c_size_t(0), C.c_size_t(0)]
        self._check(self.L.mcl3dl_match_output(self.h, _ptr(pose), _ptr(pts) if pts is not None else None,
                                               len(pts) if pts is not None else 0, C.byref(mp), _ptr(out[0]),
                                               C.byref(n[0]), _ptr(out[1]), C.byref(n[1])))
        return out[0][:n[0].value].copy(), out[1][:n[1].value].copy()

    def particles_measure_update_prepared(self, origins, odom_err_integ_lin_sigma=0.0):
        origins = np.ascontiguousarray(origins if origins is not None else np.zeros((0, 3)), dtype=np.float32).reshape(-1, 3)
        summ = UpdateSummary()
        self._check(self.L.mcl3dl_particles_measure_update_prepared(self.h, _ptr(origins), len(origins), odom_err_integ_lin_sigma,
                                                                    C.byref(summ)))
        return summ.as_dict()

    def particles_estimate(self, state_prev=None, bias_var_dist=1.0, bias_var_ang=1.0):
        """The node's pose estimate on the resident set: {"mean_biased": POSE[1], "max_state": POSE[1], "max_index",
        "weight_sum_biased", "cov": float32[6, 6]} (include/mcl3dl_b200.h: mcl3dl_particles_estimate)."""
        prev = np.ascontiguousarray(state_prev, dtype=POSE).reshape(1) if state_prev is not None else None
        e = Estimate()
        self._check(self.L.mcl3dl_particles_estimate(self.h, _ptr(prev) if prev is not None else None, bias_var_dist,
                                                     bias_var_ang, C.byref(e)))
        return {"mean_biased": np.frombuffer(bytes(e.mean_biased), dtype=POSE).copy(),
                "max_state": np.frombuffer(bytes(e.max_state), dtype=POSE).copy(), "max_index": int(e.max_index),
                "weight_sum_biased": float(e.weight_sum_biased), "cov": np.array(list(e.cov), np.float32).reshape(6, 6)}

    # ---- record exchange over peer memory (one process per GPU; see include/mcl3dl_b200.h)
    IPC_HANDLE_BYTES = 64

    def exchange_create(self, n_local, world, rank):
        """Allocates this rank's exchange buffer; returns its CUDA IPC handle (bytes) for the ranks to all-gather."""
        h = (C.c_ubyte * self.IPC_HANDLE_BYTES)()
        self._check(self.L.mcl3dl_exchange_create(self.h, n_local, world, rank, h))
        return bytes(h)

    def exchange_open(self, handles):
        """handles: the world ranks' ipc handles concatenated in rank order (bytes)."""
        buf = (C.c_ubyte * len(handles)).from_buffer_copy(handles)
        self._check(self.L.mcl3dl_exchange_open(self.h, buf))

    def measure_exchange_device(self, d_poses, n_local, d_lik, n_lik, d_beam, n_beam, d_origins, n_origins, stream=0):
        """This rank's shard + the record exchange folded into the kernels (raw device addresses, async on `stream`).
        Returns the device address that holds ALL ranks' records once the stream gets there (eager calls)."""
        d_all = C.c_void_p()
        self._check(self.L.mcl3dl_measure_exchange_device(self.h, d_poses, n_local, d_lik, n_lik, d_beam, n_beam,
                                                          d_origins, n_origins, stream, C.byref(d_all)))
        return d_all.value

    def exchange_current(self, stream=0):
        """(device address of the last completed gathered array, a peer timed out?) — synchronises `stream`."""
        d_all, f = C.c_void_p(), C.c_int(0)
        self._check(self.L.mcl3dl_exchange_current(self.h, stream, C.byref(d_all), C.byref(f)))
        return d_all.value, bool(f.value)

    def collect_timing(self, enable=True):
        """Record the per-call CUDA timing events read by last_timing() (off by default: ~28 us per update)."""
        self._check(self.L.mcl3dl_collect_timing(self.h, 1 if enable else 0))

    def last_timing(self):
        v = [C.c_double(0) for _ in range(4)]
        self.L.mcl3dl_last_timing(self.h, *[C.byref(x) for x in v])
        return {"h2d_ms": v[0].value, "lik_ms": v[1].value, "beam_ms": v[2].value, "d2h_ms": v[3].value}

    def kernel_launches(self):
        return int(self.L.mcl3dl_kernel_launches(self.h))
