/*
 * mcl3dl_b200.h — C ABI of the CUDA measurement-update engine for mcl_3dl (sm_90a, H100).
 *
 * This is the drop-in boundary: plain C, plain pointers and sizes, no STL, no torch
 * types, no exceptions.  Every entry point names the reference interface it replaces
 * (paths relative to the at-wat/mcl_3dl tree, v0.7.0).
 *
 * The engine is NOT thread-safe; the reference calls this path from the single
 * ros::spin() thread (src/mcl_3dl.cpp:1466) and so must the caller.
 *
 * There is no CPU fallback: if no CUDA device is usable every call fails with
 * MCL3DL_ERR_CUDA / MCL3DL_ERR_NO_DEVICE.
 */
#ifndef MCL3DL_B200_H
#define MCL3DL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MCL3DL_ABI_VERSION 3

/* ---- error codes (the reference has none: degenerate inputs yield (1,0); the only
 *      exception is ChunkedKdtree::radiusSearch's runtime_error, chunked_kdtree.h:224) */
enum
{
  MCL3DL_OK = 0,
  MCL3DL_ERR_INVALID_ARG = -1,  /* null pointer / bad size / label out of origins range */
  MCL3DL_ERR_NO_MAP = -2,       /* measure() before set_map() */
  MCL3DL_ERR_CUDA = -3,         /* a CUDA runtime call failed; see mcl3dl_last_error_detail */
  MCL3DL_ERR_NO_DEVICE = -4,    /* no usable sm_90 (H100) device */
  MCL3DL_ERR_TOO_LARGE = -5,    /* grid would exceed 2^31-1 cells (int point_total, raycast_using_dda.h:176) */
  MCL3DL_ERR_RADIUS = -6        /* match_dist_min > chunk length semantics (chunked_kdtree.h:224-225) */
};

/* One map / scan point.  Packed from mcl_3dl::PointXYZIL (include/mcl_3dl/point_types.h:40-55:
 * x,y,z at byte 0/4/8, label at byte 20 of a 32-byte struct) by the adapter. */
typedef struct
{
  float x, y, z;
  uint32_t label;
} mcl3dl_point;

/* One particle pose = State6DOF::pos_ / rot_ (include/mcl_3dl/state_6dof.h:55-56).
 * q is the RAW rot_; the engine normalises it exactly where the reference does
 * (State6DOF::transform, state_6dof.h:217) and uses it raw where the reference does
 * (beam origin, src/lidar_measurement_model_beam.cpp:145). */
typedef struct
{
  float px, py, pz, _pad;
  float qx, qy, qz, qw;
} mcl3dl_pose;

/* LidarMeasurementModelLikelihoodParameters (include/mcl_3dl/parameters.h:64-89) fields used by
 * LidarMeasurementModelLikelihood::measure (src/lidar_measurement_model_likelihood.cpp:105-139)
 * plus the kd-tree metric rescale (src/mcl_3dl.cpp:1270, Parameters::dist_weight_). */
typedef struct
{
  float match_weight;
  float match_dist_min;
  float match_dist_flat;
  float dist_weight[3]; /* (1,1,1) == no PointRepresentation rescale */
} mcl3dl_lik_params;

/* What LidarMeasurementModelBeam::refreshParameters (src/lidar_measurement_model_beam.cpp:58-80)
 * derives and hands to RaycastUsingDDA's constructor (raycast_using_dda.h:56-64).  The doubles are
 * doubles because the constructor takes doubles (the node passes floats promoted to double).
 * Fill it with mcl3dl_beam_params_from_reference() to get the exact same derivation. */
typedef struct
{
  double map_grid_size[3]; /* ctor args 1-3 -> min_dist_thr_sq_ (uses y twice, :59) */
  double dda_grid_size;    /* ctor arg 4 */
  double ray_angle_half;   /* ctor arg 5 */
  double hit_tolerance;    /* ctor arg 6 (= hit_range_) */
  float hit_range_sq;      /* hit_range_sq_ = pow(hit_range_,2) stored as float (:64) */
  float sin_total_ref;     /* sinf(ang_total_ref_) (:66) */
  float beam_likelihood;   /* pow(beam_likelihood_min_, 1/num_points_default) (:65) */
  float beam_likelihood_min;
  uint32_t filter_label_max;
  int32_t add_penalty_short_only_mode;
  int32_t use_raycast_using_dda; /* 1: RaycastUsingDDA; 0: RaycastUsingKDTree, the node's default (parameters.h:109).
                                  * The KD-tree caster is built from float(map_grid_size[]) and float(hit_tolerance)
                                  * (raycast_using_kdtree.h:48-55) and searches the likelihood grid, so lik params
                                  * must be given to mcl3dl_set_map as well. */
  int32_t _reserved;
} mcl3dl_beam_params;

/* Per-particle result record (24 B).
 *   likelihood model : LidarMeasurementResult{score_like, match_cnt / (float)n_lik}
 *   beam model       : LidarMeasurementResult{score_beam, 1.0f}
 * n_short/n_hit/n_long are the BeamStatus tallies (lidar_measurement_model_beam.h:64-70) over the
 * particle's rays; TOTAL_REFLECTION = n_beam - (n_short+n_hit+n_long).  They are the bit-exact
 * contract of the beam kernel. */
typedef struct
{
  float score_like;
  uint32_t match_cnt;
  float score_beam;
  uint32_t n_short;
  uint32_t n_hit;
  uint32_t n_long;
} mcl3dl_result;

/* Sizes / footprint of the staged map (for logging, tests and the roofline arithmetic). */
typedef struct
{
  uint64_t n_points;
  int32_t nn_dims[3];    /* likelihood search grid (rescaled space), cells per axis */
  float nn_cell;         /* cell edge in the rescaled space */
  float nn_origin[3];
  int32_t dda_dims[3];   /* RaycastUsingDDA::map_size_ */
  float dda_min[3];      /* min_p_ */
  float dda_max[3];      /* max_p_ */
  uint64_t device_bytes; /* per device */
  double build_ms;       /* device build time of the last set_map */
} mcl3dl_map_info;

/* Work counters accumulated over every measure call while collection is enabled (the reference logs
 * only a wall time, src/mcl_3dl.cpp:827-829; these feed the status path and the roofline arithmetic). */
typedef struct
{
  uint64_t lik_index_rows;      /* x-rows of the search grid whose two CSR bounds were read (8 B each) */
  uint64_t lik_points_scanned;  /* map points distance-tested (16 B each) */
  uint64_t beam_cells_stepped;  /* DDA cells visited (1 occupancy bit each) */
  uint64_t beam_cells_occupied; /* occupied cells whose point list was opened (8 B CSR each) */
  uint64_t beam_points_tested;  /* map points cone-tested (16 B each) */
} mcl3dl_work_stats;

typedef struct mcl3dl_engine mcl3dl_engine;

/* Create an engine on the given CUDA devices (n_devices >= 1; device_ids == NULL means 0..n-1).
 * Particles of one measure() call are split into n_devices contiguous blocks; the map is replicated. */
int mcl3dl_create(mcl3dl_engine** out, const int* device_ids, int n_devices);
void mcl3dl_destroy(mcl3dl_engine*);

/* The "setMap" event.  Replaces ChunkedKdtree::setInputCloud (include/mcl_3dl/chunked_kdtree.h:124-216)
 * and RaycastUsingDDA::updatePointCloud (raycast_using_dda.h:162-190): builds, on every device,
 * the exact-nearest-neighbour cell grid (likelihood) and the DDA occupancy bits + per-cell point
 * lists in map order (beam).  `stamp` is the cloud's header.stamp, the reference's rebuild trigger
 * (raycast_using_dda.h:168); calling again with the same stamp and n is a no-op.
 * Either params pointer may be NULL if that model is never used.  pts are only read during the call. */
int mcl3dl_set_map(mcl3dl_engine*, const mcl3dl_point* pts, size_t n, uint64_t stamp,
                   const mcl3dl_lik_params* lik, const mcl3dl_beam_params* beam);

typedef struct
{
  uint64_t n_before, n_appended, n_after;
  int32_t incremental;       /* 1: lattices unchanged, only reached NN-field cells re-selected; 0: full device rebuild */
  uint64_t cells_reselected; /* NN-field directory cells re-selected (all of them on the full path) */
  double build_ms;           /* device time of this append (max over devices) */
} mcl3dl_map_append_info;

/* The node's map update (cbMapUpdateTimer, src/mcl_3dl.cpp:1350-1378): pc_map2_ = pc_map_ + pc_update_ into the cloud
 * the index already holds, so every update appends to the staged map and nothing is removed or reordered.  After the
 * call the staged map is the previous map followed by pts[0..n) and `stamp` is its stamp; every later call gives the
 * records of a fresh engine that ran mcl3dl_set_map on the concatenated array.  The staged points stay on every device,
 * so only the n new points are uploaded.  When they lie inside the staged map's raw and rescaled bounding boxes every
 * lattice is unchanged: the grids are re-sorted on the device and the NN field re-selects only the directory cells the
 * new points can reach (incremental == 1; their new lists go after the live ones, the old ones become dead space).
 * Otherwise, or when the NN field's storage or MCL3DL_NNF_MAX_MB leaves no room, the map is rebuilt on the device from
 * the resident points (incremental == 0), which also compacts the field.
 * The resident particle set, the prepared scans, the exchange buffers and the scalar params are untouched; in field mode
 * the volume is restaged.  n == 0 only sets the stamp (incremental == 1, no cell re-selected).
 * NO_MAP before set_map; INVALID_ARG for a NULL engine or pts == NULL with n > 0; TOO_LARGE when the map would reach
 * 2^31 points (all checked before pts is read).  info may be NULL. */
int mcl3dl_map_append(mcl3dl_engine*, const mcl3dl_point* pts, size_t n, uint64_t stamp, mcl3dl_map_append_info* info);

/* Scalar parameters may change between updates without restaging the map
 * (refreshParameters(), lidar_measurement_model_likelihood.cpp:56-61 / _beam.cpp:58-80), as long as
 * match_dist_min, dist_weight and dda_grid_size are unchanged; otherwise returns INVALID_ARG. */
int mcl3dl_set_params(mcl3dl_engine*, const mcl3dl_lik_params* lik, const mcl3dl_beam_params* beam);

/* Page-locked host memory for the caller's pose and record arrays (optional).  mcl3dl_measure recognises arrays that lie
 * inside such a block: a pose array of >= 64 KB is DMA-ed from where it lies and the records are written where the caller
 * reads them (by the D2H copy, or by the kernels themselves for small updates) - the staging memcpy on both sides of the
 * call goes away (65 536 particles: 3.5 MB per update).  Any other host pointer keeps working through the engine's own
 * staging block.  No reference counterpart: pf::ParticleFilter keeps std::vector<Particle> (include/mcl_3dl/pf.h:395);
 * the adapter packs State6DOF into mcl3dl_pose anyway (host/lidar_measurement_model_b200.h) and can pack into this.
 * mcl3dl_host_free waits for the engine's streams; blocks still allocated at mcl3dl_destroy are freed there. */
int mcl3dl_host_alloc(mcl3dl_engine*, size_t bytes, void** out);
int mcl3dl_host_free(mcl3dl_engine*, void* block);

/* One measurement update for P particles: replaces the P x {beam, likelihood} calls
 *   lm.second->measure(kdtree_, pc_locals[name], origins, s)     (src/mcl_3dl.cpp:409-415)
 * that pf::ParticleFilter::measure makes one particle at a time (include/mcl_3dl/pf.h:256-260).
 * All pointers are HOST pointers; the call is synchronous and `out[0..P)` is valid on return.
 *   n_lik  == 0 -> score_like = 1, match_cnt = 0   (likelihood.cpp:111-114, quality 0)
 *   n_beam == 0 -> score_beam = 1, counts 0        (beam.cpp:130-133)
 *   beam_pts[i].label indexes origins (beam.cpp:142); out of range -> MCL3DL_ERR_INVALID_ARG. */
int mcl3dl_measure(mcl3dl_engine*, const mcl3dl_pose* poses, size_t n_particles,
                   const mcl3dl_point* lik_pts, size_t n_lik,
                   const mcl3dl_point* beam_pts, size_t n_beam,
                   const float* origins_xyz, size_t n_origins,
                   mcl3dl_result* out);

/* Same computation with every buffer already resident on engine device 0 (DEVICE pointers) and
 * the kernels enqueued on the caller's CUDA stream (a cudaStream_t cast to void*, NULL = legacy
 * default stream); asynchronous.  Used by the bench's device-resident arm and by callers that
 * all-gather the records with NCCL before reading them.  Single-device engines only.  d_origins_xyz holds
 * n_origins packed xyz triplets; beam labels are NOT range-checked here (the buffers live on the device), and the
 * engine's scratch buffers make concurrent calls on different streams unsupported. */
int mcl3dl_measure_device(mcl3dl_engine*, const mcl3dl_pose* d_poses, size_t n_particles,
                          const mcl3dl_point* d_lik_pts, size_t n_lik,
                          const mcl3dl_point* d_beam_pts, size_t n_beam,
                          const float* d_origins_xyz, size_t n_origins,
                          mcl3dl_result* d_out, void* cuda_stream);

/* Batched LidarMeasurementModelBeam::getBeamStatus (src/lidar_measurement_model_beam.cpp:157-192; the
 * node calls it for the mean pose's rays to colour its rviz markers, src/mcl_3dl.cpp:471-478).
 * status is row-major [n_particles][n_beam]: 0 SHORT, 1 HIT, 2 LONG, 3 TOTAL_REFLECTION (HOST buffers). */
int mcl3dl_beam_status(mcl3dl_engine*, const mcl3dl_pose* poses, size_t n_particles,
                       const mcl3dl_point* beam_pts, size_t n_beam,
                       const float* origins_xyz, size_t n_origins, uint8_t* status);

/* The node's rviz ray markers (src/mcl_3dl.cpp:464-628): every ray of one beam scan cast from ONE pose, the pose
 * estimate e after e.rot_.normalize(), through LidarMeasurementModelBeam::getBeamStatus with the staged caster.  One
 * record per ray, in scan order; begin / end / status are the bits the beam kernels compute for that pose.
 *   pos: CastResult::pos_ of the cast step that decided the status, what the node draws as the collision marker:
 *        DDA the deciding cell's centre fromIndex(current_index_) (raycast_using_dda.h:219-223, double, stored as float),
 *        KD the marching position pos_ of the deciding step (raycast_using_kdtree.h:67-109).  NaN for LONG.
 * beam_pts == NULL: the sampled beam scan the last mcl3dl_scan_prepare left on the device (or the last
 * mcl3dl_scan_sample_with_normal after it); single-device engines only, n_beam is ignored.  Host scans on a multi-device
 * engine run on device 0.  Synchronous.  Errors, all found before anything is written:
 *   INVALID_ARG: a null engine, pose or n_out; out == NULL with rays to write; capacity below the ray count; a label
 *                >= n_origins; a map staged without beam params, or the KD caster without lik params; beam_pts == NULL
 *                without a prepared scan or on a multi-device engine;
 *   NO_MAP:      before set_map.
 * An empty scan returns OK with *n_out = 0. */
typedef struct
{
  float begin[3];  /* e.pos_ + e.rot_ * origins[label], raw rot_ (mcl_3dl.cpp:475, beam.cpp:145) */
  float end[3];    /* the scan point transformed by the pose (State6DOF::transform, normalised rot_) */
  float pos[3];    /* CastResult::pos_ of the deciding cast step; NaN for LONG */
  uint32_t status; /* 0 SHORT, 1 HIT, 2 LONG, 3 TOTAL_REFLECTION (the codes of mcl3dl_beam_status) */
} mcl3dl_beam_ray;
int mcl3dl_beam_cast(mcl3dl_engine*, const mcl3dl_pose* pose, const mcl3dl_point* beam_pts, size_t n_beam,
                     const float* origins_xyz, size_t n_origins, mcl3dl_beam_ray* out, size_t capacity, size_t* n_out);

/* Summary of one fused weight update (row f2 of the scope table). */
typedef struct
{
  float weight_sum;      /* sum of prior * likelihood before normalisation (include/mcl_3dl/pf.h:255-260) */
  float entropy;         /* -sum p ln p over p > 0 (pf.h:263-272); 0 when !kept */
  float match_ratio_min; /* min / max over particles of the likelihood model's quality, started at 1 / 0 as the */
  float match_ratio_max; /*   node does (src/mcl_3dl.cpp:398-399,416-419) */
  int32_t kept;          /* 1: weights replaced; 0: every weight was zero, the prior is returned (pf.h:274-278) */
  uint32_t max_index;    /* particle with the largest posterior (first one on ties), pf::ParticleFilter::max */
} mcl3dl_update_summary;

/* mcl3dl_measure + the weight update that pf::ParticleFilter::measure performs with the node's lambda
 * (src/mcl_3dl.cpp:402-426, include/mcl_3dl/pf.h:252-279), fused on the device:
 *   likelihood_i = ((1 * score_beam_i) * score_like_i) [* extra_likelihood_i]     (map-key order, float)
 *   w_i = prior_i * likelihood_i;  posterior_i = w_i / sum(w)  if sum(w) > 0,  else posterior = prior
 * Only 4 bytes per particle come back (instead of the 24-byte records, which are optional: records may be NULL).
 * extra_likelihood (may be NULL) carries per-particle factors the host owns, e.g. the odometry-error term
 * (src/mcl_3dl.cpp:422-424).  The sum is accumulated in double with a fixed reduction tree (the reference
 * accumulates sequentially in float), so posteriors agree with the reference to ~1e-5 relative, not bitwise. */
int mcl3dl_measure_update(mcl3dl_engine*, const mcl3dl_pose* poses, size_t n_particles,
                          const mcl3dl_point* lik_pts, size_t n_lik,
                          const mcl3dl_point* beam_pts, size_t n_beam,
                          const float* origins_xyz, size_t n_origins,
                          const float* prior, const float* extra_likelihood,
                          float* posterior, mcl3dl_result* records, mcl3dl_update_summary* summary);

/* Derive mcl3dl_beam_params exactly as LidarMeasurementModelBeam::refreshParameters does from
 * LidarMeasurementModelBeamParameters (include/mcl_3dl/parameters.h:91-132). */
void mcl3dl_beam_params_from_reference(mcl3dl_beam_params* out,
                                       float map_grid_x, float map_grid_y, float map_grid_z,
                                       size_t num_points_default, float beam_likelihood_min,
                                       float ang_total_ref, uint32_t filter_label_max, float hit_range,
                                       int add_penalty_short_only_mode, int use_raycast_using_dda,
                                       float ray_angle_half, float dda_grid_size);

int mcl3dl_get_map_info(const mcl3dl_engine*, mcl3dl_map_info* out);

/* ---- Map window: large maps.
 * mcl3dl_set_map, mcl3dl_map_load and mcl3dl_map_append / mcl3dl_map_update_commit lay the likelihood search grid over
 * the whole map when its lattice fits: fewer than 2^31 cells, and no more than MCL3DL_MAP_MAX_CELLS (environment, read at
 * mcl3dl_create; default 2^31 - 1, a smaller value forces windows on small maps).  Otherwise the map is staged WINDOWED
 * instead of refused: its points and bounding boxes stay on every device and the search structures (CSR grid, near
 * fields, NN field, KD caster's near field) are built over the points inside a window, a box of raw map space around the
 * particles.  The DDA caster's grid stays whole-map as before (and is refused beyond its own int point_total limit).
 *   Rule: every call that reads the map (mcl3dl_measure, mcl3dl_measure_update, mcl3dl_beam_status, mcl3dl_beam_cast,
 *   mcl3dl_match_output, mcl3dl_particles_measure_update / _prepared) first reduces its inputs on the device to the box
 *   its searches need: the finite particle positions grown by the largest norm of a finite scan point or origin (times
 *   the particles' largest |q|^2), the searches' radii per axis in raw coordinates (likelihood rpad, the KD caster's
 *   second radius and its march, the match output's radius) and a relative pad for the float transform.  When that box
 *   is not inside the window, the window is rebuilt as the box grown by the scan reach on each side (less when that
 *   exceeds the cap).  One 32-byte copy back and one synchronise per device and call, on a windowed map only (a
 *   multi-device call enqueues every device's check with its inputs, then reads them; MCL3DL_TIMING's h2d_ms leaves
 *   them out); a whole-staged map
 *   runs exactly as before.  Each search returns the exact nearest neighbour within its radius, so the records are
 *   those of a whole staging.  Non-finite particles and points are left out of the box (they find nothing either way).
 *   Appends add to the device point list and rebuild the window (at the next call) only when an appended point lies
 *   inside it; an append that takes a whole-staged map over the lattice makes it windowed.  mcl3dl_map_get returns the
 *   whole map; mcl3dl_get_map_info reports the staged window's lattice (zero dimensions before the first window).
 *   Refused with MCL3DL_ERR_TOO_LARGE on a windowed map, as the whole map was before:
 *     - a call whose required box alone exceeds the cap (e.g. particles spread over the map): the window and the
 *       resident particle set stay as they were;
 *     - mcl3dl_measure_device and mcl3dl_measure_exchange_device (they run on the caller's stream or in a captured
 *       graph, where no synchronise may happen);
 *     - field mode (mcl3dl_field_mode, _field_nodes, _field_upload, and set_map in field mode): the volume is whole-map;
 *     - mcl3dl_global_localization: its seeds cover the whole map. */
typedef struct
{
  int32_t windowed;   /* 1: the staged map is windowed */
  int32_t staged;     /* 1: a window's structures are built */
  float box_min[3];   /* the window, raw map space */
  float box_max[3];
  int32_t dims[3];    /* its likelihood lattice, cells per axis */
  int32_t _pad;
  uint64_t rebuilds;  /* windows built since the map was staged (device 0) */
  double rebuild_ms;  /* stream time of the last one: the point selection plus the build, event to event; like
                         mcl3dl_map_info.build_ms it includes the build's own count readbacks, not the allocations
                         between the two */
} mcl3dl_window_info;
int mcl3dl_map_window_info(const mcl3dl_engine*, mcl3dl_window_info* out);

/* ---- Resident particle set (SURVEY.md §8 row f3; the per-particle arithmetic is verified on the host bit for bit
 * against the oracle, the kernels by tests/test_gpu_resident.py on an H100).
 * The particles of pf::ParticleFilter<State6DOF> stay in device memory between updates, so an update moves only the
 * scans and the odometry in and a summary out.  Engines with exactly one device.
 *
 * mcl3dl_state = the State6DOF fields that prediction, measurement and resampling touch
 * (include/mcl_3dl/state_6dof.h:55-63): pos_, rot_ (x y z w), noise_ll_/la_/al_/aa_, odom_err_integ_lin_/_ang_. */
typedef struct
{
  float pos[3];
  float rot[4];
  float noise_ll, noise_la, noise_al, noise_aa;
  float odom_err_integ_lin[3];
  float odom_err_integ_ang[3];
} mcl3dl_state; /* 68 bytes */

/* set() uploads a set built on the host (states + probability_), get() reads the set back (either pointer may be NULL).
 * pf_->init / initUsingNoiseGenerator, resizeParticle and the global localisation seed have device versions below. */
int mcl3dl_particles_set(mcl3dl_engine*, const mcl3dl_state* states, const float* prob, size_t n_particles);
int mcl3dl_particles_get(mcl3dl_engine*, mcl3dl_state* states, float* prob, size_t n_particles);
/* pf_->predict(motion_prediction_model) for MotionPredictionModelDifferentialDrive: setOdoms(odom_prev, odom_current,
 * time_diff) + predict() per particle (motion_prediction_models/motion_prediction_model_differential_drive.h:46-67;
 * src/mcl_3dl.cpp:227-232).  odom_* : position + rotation of the two odometry states. */
int mcl3dl_particles_predict(mcl3dl_engine*, const mcl3dl_pose* odom_prev, const mcl3dl_pose* odom_current, float time_diff,
                             float odom_err_integ_lin_tc, float odom_err_integ_ang_tc);
/* pf_->measure(measure_func) of src/mcl_3dl.cpp:398-426 on the resident set: both models, the odometry-error factor
 * NormalLikelihood(odom_err_integ_lin_sigma)(|odom_err_integ_lin_|) (sigma <= 0: factor 1), prior * likelihood,
 * normalisation, entropy, match-ratio min/max, arg max.  The posterior replaces the resident probabilities (or the
 * prior is kept when no particle survives, pf.h:274-278). */
int mcl3dl_particles_measure_update(mcl3dl_engine*, const mcl3dl_point* lik_pts, size_t n_lik, const mcl3dl_point* beam_pts,
                                    size_t n_beam, const float* origins_xyz, size_t n_origins, float odom_err_integ_lin_sigma,
                                    mcl3dl_update_summary* summary);
/* pf_->resample(State6DOF(sigma_pos, sigma_rpy)) (pf.h:182-225, src/mcl_3dl.cpp:809-815): sequential float prefix sum,
 * systematic pick from initial_p = initial_frac * pstep (the host draws initial_frac in [0, 1) with the node's engine),
 * noise on duplicates only, probability 1 / n.  Documented departures: the noise comes from a counter-based generator
 * (Philox-4x32-10 keyed by seed, output index and call count) instead of std::default_random_engine's stream, and
 * particles that tie in the accumulated probability are taken by lowest index instead of std::sort's order.  The call
 * count starts at 1 on a new engine and is not reset by mcl3dl_particles_set.  Given the noise draws, the picks, the
 * copies and the probabilities are exact; a duplicate differs from host arithmetic only through the device's logf /
 * sinf / cosf (a few ulp of the noise). */
int mcl3dl_particles_resample(mcl3dl_engine*, const float sigma_pos[3], const float sigma_rpy[3], float initial_frac,
                              uint64_t seed);

/* The node's other per-particle events on the resident set.  Single-device engines; synchronous; INVALID_ARG for a null
 * engine or pointer, no resident set or a multi-device engine.
 *
 * Random numbers: the documented departure of resample, Philox-4x32-10 keyed by seed (key words = its low and high 32
 * bits), one block per counter (particle index, call count, block, event).  The event word keeps the streams apart:
 * 0 resample (blocks 0 and 1), 1 the odometry-noise redraw (block 0), 2 the expansion noise (blocks 0 and 1), 3 the
 * initial seed (particles_init, blocks 0 and 1).  A block's
 * four output words w0..w3 give uniforms u(w) = float((w >> 8) + 1) * 2^-24 in (0, 1], and Box-Muller on a pair (u, v)
 * gives z = sqrtf(-2 logf(u)) * cosf(2 pi v) and z' = ... * sinf(2 pi v) (float, in that order).  Resample and the
 * expansion noise take the pairs (w0, w1), (w2, w3) of block 0 and (w0, w1) of block 1 for x, y, z, roll, pitch, yaw,
 * each times its sigma (0 where the sigma is 0).  Every entry point keeps its own call count: 1 on the first call of an
 * engine, never reset by particles_set.
 *
 * redraw_odom_noise: the node's update_noise_func through pf_->predict (src/mcl_3dl.cpp:817-825).  Block 0's two pairs give
 * z0..z3 and, in the node's draw order, noise_ll = float(double(z0) * lin_lin), noise_la = float(double(z1) * lin_ang),
 * noise_aa = float(double(z2) * ang_ang), noise_al = float(double(z3) * ang_lin).  Nothing else changes, the
 * probabilities included.  INVALID_ARG for a negative or non-finite sigma. */
int mcl3dl_particles_redraw_odom_noise(mcl3dl_engine*, double lin_lin, double lin_ang, double ang_lin, double ang_ang,
                                       uint64_t seed);
/* noise: pf_->noise(State6DOF(sigma_pos, sigma_rpy)) (pf.h:226-237), expansion resetting (src/mcl_3dl.cpp:853-864): every
 * particle becomes state + generateNoise, as resample treats a duplicate, with two differences the reference makes and
 * that are kept: the rotation is NOT normalised afterwards (rot = nrot * rot as it comes), and operator+ builds a fresh
 * State6DOF, so noise_ll/la/al/aa become 0 (the node calls this right after the redraw, whose values are discarded).  The
 * probabilities are unchanged.  INVALID_ARG for a negative or non-finite sigma. */
int mcl3dl_particles_noise(mcl3dl_engine*, const float sigma_pos[3], const float sigma_rpy[3], uint64_t seed);
/* imu_update: ImuMeasurementModelGravity::setAccMeasure(acc_measure) + pf_->measure(imu measure) (cbImu,
 * src/mcl_3dl.cpp:941-1018; imu_measurement_model_gravity.h:45-55; pf.h:252-279).  On the host, once: |acc_measure| as
 * Vec3::norm and NormalLikelihood<float>(float(acc_var)) (a = float(1.0 / sqrt(2 pi s s)), sq2 = float(float(s s) * 2.0)).
 * Per particle: acc_estim = rot.inv() * (0, 0, 1) with the RAW rot, diff = acosf(dot / (|acc_measure| |acc_estim|)),
 * likelihood = a * expf(-diff * diff / sq2), w = prior * likelihood; then the fold of mcl3dl_particles_measure_update
 * (double sums with a fixed tree, the posterior replaces the probabilities, kept = 0 keeps the prior).  The summary's
 * match_ratio_min and match_ratio_max are both 0: no likelihood model ran.  An acosf argument that rounds above 1 makes
 * that particle's likelihood NaN; as in the reference (sum > 0 is false), the whole update is then discarded: kept = 0,
 * weight_sum NaN, probabilities untouched.  Documented departure: INVALID_ARG when float(acc_var) is not finite and
 * positive (the reference would compute with it). */
int mcl3dl_particles_imu_update(mcl3dl_engine*, const float acc_measure[3], double acc_var, mcl3dl_update_summary* summary);

/* landmark_update: cbLandmark's pf_->measure (src/mcl_3dl.cpp:899-931; nd.h:61-83; pf.h:252-279).  The host builds the
 * reference's own NormalLikelihoodNd<float, 6> from the message's covariance, as cbLandmark does
 * (Eigen::Matrix<double, 6, 6>(covariance.data()).cast<float>(); Eigen maps that array column-major, so a non-symmetric
 * covariance enters transposed), and passes its a_ and sigma_inv_: Eigen's determinant and inverse stay on the host.
 * measured is the message's pose as received (RAW rotation; _pad ignored).  Per particle: diff = s - measured
 * (state_6dof.h:262-274: the position per axis in float, rot = measured.rot.inv() * rot with both rotations RAW,
 * Quat::inv = conj * float(1.0 / double(dot))), x = (diff.pos, diff.rot.getRPY()), likelihood = a * expf(q) with
 * q = -0.5 x^T S x evaluated in float in this fixed order (a documented departure: Eigen's order depends on its
 * vectorisation): h_k = -0.5 x_k, r_j = sum over k = 0..5 of h_k S(k, j), q = sum over j = 0..5 of r_j x_j, each sum
 * accumulated left to right from its first product.  Then the fold of mcl3dl_particles_imu_update: w = prior *
 * likelihood, double sums with a fixed tree, the posterior replaces the probabilities; match_ratio_min and _max are 0.
 * A NaN likelihood (e.g. a NaN rotation) or weights that all underflow to 0 (a landmark far from every particle)
 * discard the whole update, as the reference's sum > 0 test does: kept = 0, probabilities untouched.  The states never
 * change.  Documented departure: INVALID_ARG when nd_a, any sigma_inv entry or any of the measured pose's seven values
 * is not finite (the reference would compute with them). */
typedef struct
{
  mcl3dl_pose measured;  /* the message's pose: position + orientation as received (RAW) */
  float nd_a;            /* NormalLikelihoodNd<float, 6>::a_ */
  float sigma_inv[36];   /* NormalLikelihoodNd<float, 6>::sigma_inv_, row-major: [r * 6 + c] = sigma_inv_(r, c) */
} mcl3dl_landmark_params;
int mcl3dl_particles_landmark_update(mcl3dl_engine*, const mcl3dl_landmark_params* params, mcl3dl_update_summary* summary);
/* reset_odom_err_integ: the node's integ_reset_func through pf_->predict (the pose-jump branch of measure(),
 * src/mcl_3dl.cpp:653-658, and cbPosition, :190-195): odom_err_integ_lin and odom_err_integ_ang become +0.0f.  Nothing
 * else changes, the probabilities included. */
int mcl3dl_particles_reset_odom_err_integ(mcl3dl_engine*);
/* get_poses: what publishParticles (src/mcl_3dl.cpp:1101-1125) publishes, 32 bytes per particle instead of the 72 of
 * particles_get: out[i] = the position and rot.normalized() (quat.h:175-177: rot * float(1.0 / double(sqrtf(dot)))),
 * _pad = 0.  The resident set is not modified (the reference normalises a copy).  n must equal the resident count. */
int mcl3dl_particles_get_poses(mcl3dl_engine*, mcl3dl_pose* out, size_t n);

/* init: pf::ParticleFilter::initUsingNoiseGenerator(generator) (pf.h:169-181) on the device, for the configured start
 * (MCL3dlNode::configure's pf_->init(initial_pose, initial_pose_std): DiagonalNoiseGenerator, multivariate = 0) and for
 * cbPosition (MultivariateNoiseGenerator<float>(mean, msg->pose.covariance), multivariate = 1; src/mcl_3dl.cpp:155-198).
 * Creates or replaces the resident set at count n (no particles_set needed; after global localisation the node passes the
 * enlarged count, as the reference seeds particles_.size() particles).  Every particle gets probability float(1.0 /
 * double(n)) and the state of State6DOF::generateNoise (state_6dof.h:226-248):
 *   draws: the layout of resample's noise with event word 3: six standard normals z0..z5 (x y z roll pitch yaw) from
 *          the pairs (w0, w1), (w2, w3) of block 0 and (w0, w1) of block 1 of Philox (particle index, call count, block,
 *          3), z = sqrtf(-2 logf(u)) * cosf(2 pi v) and ... * sinf(2 pi v); the call count is init's own (1 on the first
 *          call of an engine, never reset);
 *   diagonal (DiagonalNoiseGenerator::operator(), diagonal_noise_generator.h:63-78): org_k = sigma_k == 0 ? mean_k :
 *          z_k * sigma_k + mean_k in float (libstdc++'s normal_distribution<float>), with sigma = setSigma(State6DOF):
 *          pos then rpy_.v_;
 *   multivariate (multivariate_noise_generator.h:51-91): org_i = mean_i + t_i, t_i = sum over k = 0..5 of T(i, k) z_k
 *          accumulated in float left to right from its first product, T = norm_transform_ = V sqrt(D) of the
 *          covariance read row-major (cov(i, j) = covariance[j + i * 6]; the eigensolver reads the lower triangle).
 *          The eigendecomposition stays on the host.  Documented departure: the fixed order of the product (Eigen's
 *          depends on its vectorisation);
 *   state: pos = org[0..2]; odom_err_integ_lin = org[0..2], the mean included (a reference quirk, kept);
 *          odom_err_integ_ang = org[3..5] - mean[3..5]; rot = Quat(Vec3(org[3..5])) (setRPY, quat.h:202-215), NOT
 *          normalised, as the reference leaves it; noise_ll/la/al/aa = 0.  cbPosition resets both integrals right
 *          after (particles_reset_odom_err_integ); the configured start does not.
 * Synchronous; single-device engines.  The other entry points' call counts are unchanged.  Errors, all before the set is
 * touched: INVALID_ARG for a null engine or params, a multi-device engine, n == 0 or n >= 2^31, multivariate not 0 or 1,
 * a non-finite mean, a diagonal sigma that is negative or not finite, or a multivariate transform entry that is not
 * finite.  The last is a documented departure: a covariance with a negative eigenvalue gives the reference NaN
 * particles (sqrt of a negative eigenvalue); here it is refused.  sigma is ignored when multivariate = 1, norm_transform
 * when multivariate = 0. */
typedef struct
{
  int32_t multivariate;     /* 0: DiagonalNoiseGenerator, 1: MultivariateNoiseGenerator */
  float mean[6];            /* NoiseGeneratorBase::getMean(): x y z roll pitch yaw */
  float sigma[6];           /* diagonal: DiagonalNoiseGenerator::sigma_ */
  float norm_transform[36]; /* multivariate: norm_transform_, row-major [r * 6 + c] */
} mcl3dl_init_params;
int mcl3dl_particles_init(mcl3dl_engine*, size_t n, const mcl3dl_init_params* params, uint64_t seed);

/* pf_->resizeParticle(num) (pf.h:399-436) on the resident set, as the node calls it after every update while the set is
 * larger than num_particles (src/mcl_3dl.cpp:875-888): sequential float prefix sum accum, pstep = accum_total / num in
 * float, the sequential float chain pscan += pstep (from 0, added before each pick), output i = the whole state of the
 * first particle with accum >= pscan_i; outputs whose pscan passes the total copy the last earlier output that found a
 * particle (particle 0 when none did); probability float(1.0 / num).  Shrink and growth.  Deterministic and exact;
 * the one departure is the one of resample: particles that tie in accum are taken by lowest index.  INVALID_ARG for
 * num == 0, num >= 2^31, no resident set or a multi-device engine.  Synchronous. */
int mcl3dl_particles_resize(mcl3dl_engine*, size_t num);

/* Global localisation (the node's global_localization service, src/mcl_3dl.cpp:1039-1099) on the device; the result
 * replaces the resident set.
 *   1. pcl::VoxelGrid of the cloud with leaf float(grid) on all three axes: the restatement of mcl3dl_scan_prepare
 *      (finite points only, PCL's INT32_MAX overflow rule leaves the cloud unfiltered, output in ascending voxel index,
 *      centroid float sums in input order; the label vote runs as there, the labels are unused).
 *   2. Free-space filter: a downsampled point p is dropped when some downsampled point lies within grid of
 *      q = (p.x, p.y, float(double(p.z) + (0.01 + grid))) — flann::L2_Simple d2 < float(grid * grid) in the space
 *      rescaled by dist_weight (KdTreeFLANN with the node's point representation; exact, the node's tree has no eps).
 *      The survivors (the seeds) keep their order.
 *   3. n_particles = n_seeds * div_yaw: particle i = State6DOF(seed[i / div_yaw], yaw[i % div_yaw]) with
 *      yaw[c] = (Quat(Vec3(0, 0, 2 pi c / div_yaw)) * imu_quat).normalized() (computed on the host in the reference's
 *      operation order), noise and odometry-error fields 0, and probability float(1.0 / float(n_seeds)) for every particle.
 *      That is the reference's own quirk, kept: the set sums to div_yaw, not 1.
 * pts == NULL: the staged map (set_map, appends included; n is ignored); nothing is uploaded.  Otherwise the host cloud
 * pts[0..n).
 * Only the resident set changes (count = n_particles, the resample call count is kept, as for particles_set); the
 * staged map and its structures, the prepared scans, the matched / unmatched buffers and the exchange buffers are
 * untouched.  n_seeds == 0 (e.g. an empty cloud): OK with zero counts and the resident set unchanged — a documented
 * departure, the reference would resize to 0.  Errors, all before the set is touched: INVALID_ARG for a null engine or
 * params, a multi-device engine, grid <= 0 or not finite, div_yaw < 1, a dist_weight component <= 0 or not finite,
 * or a host cloud of 2^31 points or more; NO_MAP for pts == NULL before set_map; TOO_LARGE
 * when n_seeds * div_yaw >= 2^31 or the free-space filter's grid would have 2^31 cells or more.  Synchronous. */
typedef struct
{
  double grid;          /* Parameters::global_localization_grid_ (node default 0.3) */
  int32_t div_yaw;      /* Parameters::global_localization_div_yaw_ = lround(2 pi / grid_ang) */
  float imu_quat[4];    /* the node's imu_quat_ (x y z w) */
  float dist_weight[3]; /* the node's point representation rescale (Parameters::dist_weight_) */
} mcl3dl_global_localization_params;
typedef struct
{
  uint64_t n_input, n_downsampled, n_seeds, n_particles;
  float probability; /* what every particle got (0 when n_seeds == 0) */
  double build_ms;   /* device time of the call (CUDA events on the engine's stream) */
} mcl3dl_global_localization_info;
int mcl3dl_global_localization(mcl3dl_engine*, const mcl3dl_point* pts, size_t n, const mcl3dl_global_localization_params*,
                               mcl3dl_global_localization_info* info);

/* The pose estimate the node takes from the filter after every measurement, on the resident set
 * (src/mcl_3dl.cpp:428-452,704-724): pf_->bias(bias_func) + pf_->expectationBiased() (pf.h:246-251,294-303;
 * ParticleWeightedMeanQuat, state_6dof.h:316-355), pf_->max() (pf.h:361-374) and pf_->covariance(1.0, .) (pf.h:304-360,
 * State6DOF::covElement state_6dof.h:162-184).  Only this summary leaves the device.
 *   state_prev == NULL: bias 1 for every particle (the node's branch for more particles than num_particles, :428-434);
 *   otherwise bias = NormalLikelihood(bias_var_dist)(|pos - prev.pos|) * NormalLikelihood(bias_var_ang)(angle) + 1e-6.
 * Sums are accumulated in double with a fixed tree (the reference: sequential float), so the values agree with the
 * reference to ~1e-5 relative.  Against the exact sums of the same float terms: with state_prev == NULL the weight
 * sum, the mean position and the position block of cov equal float(exact ratio) (away from rounding boundaries), the
 * mean rotation is within 1 ulp; the angle rows and the biased means carry the errors of the device's atan2f / asinf /
 * acosf / expf (tests/test_gpu_pf_exact.py derives the bars).  Documented departures: the covariance always uses every particle (the reference
 * subsamples randomly above num_particles "to reduce calculation cost", and its expectation(1.0) / covariance(1.0) stop
 * early if the float running total of the probabilities passes 1.0 before the last particle). */
typedef struct
{
  mcl3dl_pose mean_biased;  /* expectationBiased(): pos, rot as built by Quat(front, up) — normalise as the node does (:462) */
  mcl3dl_pose max_state;    /* max(): pos + raw rot of the first particle with the largest probability */
  uint32_t max_index;
  float weight_sum_biased;  /* sum of probability * bias */
  float cov[36];            /* row-major 6 x 6: x y z roll pitch yaw */
} mcl3dl_estimate;
int mcl3dl_particles_estimate(mcl3dl_engine*, const mcl3dl_pose* state_prev, float bias_var_dist, float bias_var_ang,
                              mcl3dl_estimate* out);

/* ---- Scan preprocessing on the device (SURVEY.md §8 row f4, scan half): the node's per-update treatment of the
 * accumulated raw cloud (src/mcl_3dl.cpp:363-383): pcl::VoxelGrid downsample (:363-367), then per model filter() = clip
 * by planar range and z window (src/lidar_measurement_model_likelihood.cpp:79-103, _beam.cpp:98-122) and
 * PointCloudUniformSampler::sample (point_cloud_uniform_sampler.h:56-74).  The prepared scans stay on the device for
 * mcl3dl_particles_measure_update_prepared; scan_get reads any stage back.  num_points are the values
 * setGlobalLocalizationStatus computed on the host (likelihood.cpp:63-77).  Departures: PCL's VoxelGrid is third-party
 * and unpinned (restated from its published algorithm; centroid float sums in input order, majority label, lowest on
 * ties); non-finite points are skipped by the VoxelGrid as for a cloud that is not dense, and more than INT32_MAX voxels
 * by PCL's count leave the cloud unfiltered, as PCL does (without downsampling, non-finite points reach filter()); the
 * sampler's draws come from Philox-4x32-10 (the reference seeds from std::random_device: not reproducible either). */
typedef struct
{
  float downsample[3]; /* VoxelGrid leaf size; any component <= 0: no downsampling */
  float lik_clip_near, lik_clip_far, lik_clip_z_min, lik_clip_z_max;
  float beam_clip_near, beam_clip_far, beam_clip_z_min, beam_clip_z_max;
  uint32_t lik_num_points, beam_num_points; /* sample sizes (0: that model gets an empty scan) */
  uint64_t seed;
} mcl3dl_scan_params;
typedef struct
{
  uint32_t n_raw, n_downsampled, n_lik_clipped, n_beam_clipped, n_lik, n_beam;
} mcl3dl_scan_info;
int mcl3dl_scan_prepare(mcl3dl_engine*, const mcl3dl_point* raw, size_t n_raw, const mcl3dl_scan_params*, mcl3dl_scan_info* info);
/* which: 0 downsampled cloud, 1 / 2 clipped cloud of the likelihood / beam model, 3 / 4 their sampled scans. */
int mcl3dl_scan_get(mcl3dl_engine*, int which, mcl3dl_point* out, size_t capacity, size_t* n_out);
/* mcl3dl_particles_measure_update on the scans left on the device by the last mcl3dl_scan_prepare. */
int mcl3dl_particles_measure_update_prepared(mcl3dl_engine*, const float* origins_xyz, size_t n_origins,
                                             float odom_err_integ_lin_sigma, mcl3dl_update_summary* summary);

/* ---- Cloud accumulation on the device (src/mcl_3dl.cpp:248-342): the cloud mcl3dl_scan_prepare receives, built where it
 * is used.  cbCloud -> CloudAccumulationLogic::push (src/cloud_accum.cpp:53-119) calls accumCloud / accumClear / measure();
 * with these entry points each incoming PointCloud2 crosses the bus once, as raw bytes, and measure() sends nothing but
 * the origins.
 *   accumulate (accumCloud, :274-302): tf2::doTransform of every point into the odom frame (odom_from_sensor), the
 *     conversion, label = the cloud's accumulation index k (k-th call since the last clear, from 0; :295-298), appended
 *     in row-major order.  Point (r, c) is read at data + r row_step + c point_step + offset[i] (FLOAT32, little-endian);
 *     the call reads (height - 1) row_step + width point_step bytes from data and returns after it no longer needs them.
 *     *n_clouds_out (may be NULL): the clouds accumulated, this one included.  Errors, all checked before data is read,
 *     leave the accumulation as it was: INVALID_ARG for a null engine / view / data / transform, a multi-device engine,
 *     width height == 0, an offset + 4 > point_step or row_step < width point_step; TOO_LARGE when the accumulated total
 *     would reach 2^30 points (mcl3dl_scan_prepare's limit).
 *   clear (accumClear, :266-272): empties the accumulation; the prepared scans stay.
 *   accumulated_get: the accumulated points in the odom frame, as they are (the prepare below does not change them).
 *   prepare_accumulated (measure(), :319-367): pcl::transformPointCloud of the accumulation into base_link
 *     (base_from_odom), then exactly mcl3dl_scan_prepare's pipeline on it (VoxelGrid, clip, uniform sample; scan_get,
 *     particles_measure_update_prepared, scan_sample_with_normal, match_output(pts = NULL) and beam_cast(beam_pts = NULL)
 *     read its result).  The beam labels are accumulation indices, so the caller's origins (one per accumulated header,
 *     :343-359) cover them.  The accumulation is not consumed.  INVALID_ARG, with nothing changed (the previous
 *     prepared scans stay valid), for a null engine / transform / params, a multi-device engine or an empty accumulation
 *     (the node logs and returns, :312-316).
 * The transforms (both; restating Eigen and PCL): R = Eigen::Quaternion<float>(float(w), float(x), float(y),
 * float(z)).toRotationMatrix() on the RAW quaternion (no normalisation; Eigen's formula: tx = 2x, .., twz = tz w, ..,
 * R00 = 1 - (tyy + tzz), R01 = txy - twz, ..), t = float(translation), out_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i with every
 * operation rounded on its own.  They are applied as two transforms, in the node's order, never composed.  The first
 * applies to every point (tf2_sensor_msgs iterates over all of them); the second, as pcl::transformPointCloud, to every
 * point when every accumulated cloud had is_dense, otherwise it leaves a point with any non-finite coordinate as it is
 * (visible without downsampling: the models' clip keeps NaN points and drops infinite ones).
 * Departures: PCL, tf2 and Eigen are third-party and absent from the reference tree, so the operation order above is
 * restated, "parity unpinned" as the VoxelGrid: PCL's SSE2 Transformer<float>::se3 may nest the sum the other way
 * (x c0 + (y c1 + (z c2 + t))), which would differ in the last ulp; this has not been checked against a PCL build.  The C++
 * adapter rejects what fromROSMsg would (no x / y / z field, an empty cloud) and, beyond it, x / y / z that are not
 * FLOAT32, a big-endian cloud, and a layout that does not hold its points (row_step < width point_step, data shorter
 * than (height - 1) row_step + width point_step, or a field that does not fit in point_step), which pcl::fromROSMsg
 * does not check and would read past the message's data.  Synchronous; single-device engines. */
typedef struct
{
  const void* data;                           /* PointCloud2::data */
  uint32_t width, height, point_step, row_step;
  uint32_t offset[3];                         /* byte offsets of the FLOAT32 fields x, y, z */
  int32_t is_dense;                           /* PointCloud2::is_dense */
} mcl3dl_cloud_view;
typedef struct
{
  double translation[3];
  double rotation[4]; /* x y z w, raw */
} mcl3dl_transform;
int mcl3dl_scan_accumulate(mcl3dl_engine*, const mcl3dl_cloud_view* cloud, const mcl3dl_transform* odom_from_sensor,
                           uint32_t* n_clouds_out);
int mcl3dl_scan_accumulate_clear(mcl3dl_engine*);
/* *n_out = the accumulated point count; out == NULL: count only; INVALID_ARG when capacity is below it. */
int mcl3dl_scan_accumulated_get(mcl3dl_engine*, mcl3dl_point* out, size_t capacity, size_t* n_out);
int mcl3dl_scan_prepare_accumulated(mcl3dl_engine*, const mcl3dl_transform* base_from_odom, const mcl3dl_scan_params*,
                                    mcl3dl_scan_info* info);

/* ---- Map intake on the device (src/mcl_3dl.cpp:127-153, 1150-1192, 1350-1378): the received map and its update patches
 * are converted and downsampled where they are staged, so the node runs no VoxelGrid on the map and keeps no host copy.
 *   load (cbMapcloud / cbLoadPCD -> loadMapCloud, :1150-1170): conversion, VoxelGrid at map_downsample, then staged
 *     exactly as mcl3dl_set_map(result, stamp, lik, beam) (it replaces the map; the same params rules and the same
 *     rebuild trigger).  A pending patch is dropped (pc_update_.reset(), :1154).
 *   update_set (cbMapcloudUpdate, :141-153): conversion and VoxelGrid at update_downsample into a pending patch on the
 *     device; it replaces a pending patch.  Allowed before any map; the staged map is untouched.
 *   update_commit (cbMapUpdateTimer, :1350-1378): mcl3dl_map_append(pending patch, stamp, info), moved device to device:
 *     the incremental and full paths and info are those of an append of the same points.  The patch is consumed.  NO_MAP
 *     before any map (the patch stays pending); with no pending patch OK and nothing changes (info: n_before = n_after =
 *     the staged count, incremental = 1).  A commit appends to the staged map: after load / commit / commit the map is
 *     the load's points, then the first patch's, then the second's.
 *   update_clear (cbPosition, :189): drops the pending patch.
 *   map_get: the staged map (pc_map2_, published as updated_map at :1371-1373) in staged order and one intensity per
 *     point.  *n_out = the staged count; out == NULL: count only; INVALID_ARG when capacity is below it;
 *     intensity_out may be NULL.  NO_MAP before any map.
 * Conversion (fromROSMsg into PointXYZIL): point (r, c) is read at data + r row_step + c point_step + offset, points in
 * row-major order; x / y / z (FLOAT32) are copied bit for bit; intensity from the FLOAT32 field at intensity_offset,
 * label from the UINT32 field at label_offset, each 0 when its offset is -1 (the PointXYZIL() defaults pcl::fromROSMsg
 * leaves when no field of that name and type exists; the caller passes an offset only for a field of the right type).
 * VoxelGrid: exactly mcl3dl_scan_prepare's (lattice, PCL's INT32_MAX overflow rule, centroid and label
 * vote); any leaf component <= 0 (or NaN) means no downsampling.  The intensity of a voxel is the float sum of its
 * points' intensities in input order over float(cnt), like x / y / z.
 * Departure: non-finite points never reach the staged map.  Downsampled, the VoxelGrid skips them; unfiltered (the
 * overflow rule, or no leaf) they are dropped with the order kept, as KdTreeFLANN::setInputCloud does with a cloud that
 * is not dense.  (mcl3dl_set_map takes its points as given: a NaN coordinate is ignored by the bounding box but
 * converts to cell 0 of the likelihood grid (clamped) and of the DDA grid, where it marks the corner cell occupied; an
 * infinite one makes the bounding box infinite, so the lattices' float-to-int conversions have no defined result.)
 * A load that leaves no point returns INVALID_ARG with the previous map kept; a patch that leaves none is a valid
 * empty patch, and its commit only sets the stamp (map_append with n == 0).
 * Intensity storage: one float per staged point.  Intake stores the VoxelGrid's; mcl3dl_set_map and mcl3dl_map_append
 * store 0 (host arrays carry none).  No kernel other than map_get's copy reads it.  It costs 4 more bytes of device
 * memory per staged point on every device, on the set_map / map_append paths as well (not counted in device_bytes).
 * Checks, all before data is read: INVALID_ARG for a null engine / map / data / leaf, width height == 0, row_step <
 * width point_step, an x / y / z offset + 4 > point_step, an intensity or label offset below -1 or with offset + 4 >
 * point_step, and (load) no params or set_map's lik params rules; TOO_LARGE for 2^30 raw points or more (the VoxelGrid's
 * key limit, as mcl3dl_scan_prepare) and (commit) a staged total of 2^31 or more.  An error leaves the staged map and
 * the pending patch as they were, except an error of the map build itself, which drops the map as mcl3dl_set_map's
 * does.  The resident particle set, the prepared scans, the accumulation and the exchange buffers are untouched; in
 * field mode the volume is restaged as by set_map / map_append.  Multi-device engines: the map and the pending patch
 * are built on every device, with byte-identical results.  Synchronous: data is not read after the call returns.
 * info (may be NULL): raw points, points staged (load) or pending (update_set), whether the VoxelGrid filtered, and the
 * device time of the intake (max over devices; the map build is mcl3dl_map_info.build_ms / append_info.build_ms). */
typedef struct
{
  mcl3dl_cloud_view view;   /* data, layout, FLOAT32 x / y / z offsets, is_dense */
  int32_t intensity_offset; /* FLOAT32 "intensity" field, -1: absent */
  int32_t label_offset;     /* UINT32 "label" field, -1: absent */
} mcl3dl_map_cloud;
typedef struct
{
  uint64_t n_input, n_staged;
  int32_t downsampled;
  double device_ms;
} mcl3dl_map_intake_info;
int mcl3dl_map_load(mcl3dl_engine*, const mcl3dl_map_cloud* map, const float leaf[3], uint64_t stamp, const mcl3dl_lik_params* lik,
                    const mcl3dl_beam_params* beam, mcl3dl_map_intake_info* info);
int mcl3dl_map_update_set(mcl3dl_engine*, const mcl3dl_map_cloud* patch, const float leaf[3], mcl3dl_map_intake_info* info);
int mcl3dl_map_update_commit(mcl3dl_engine*, uint64_t stamp, mcl3dl_map_append_info* info);
int mcl3dl_map_update_clear(mcl3dl_engine*);
int mcl3dl_map_get(mcl3dl_engine*, mcl3dl_point* out, float* intensity_out, size_t capacity, size_t* n_out);

/* The node's second sampler, PointCloudSamplerWithNormal (use_random_sampler_with_normal; point_cloud_random_samplers/
 * point_cloud_sampler_with_normal.h), on the clipped clouds the last mcl3dl_scan_prepare left on the device, once per
 * model.  It REPLACES that call's sampled scans (scan_get(3 | 4), particles_measure_update_prepared); the downsampled and
 * clipped clouds, the resident set, the staged map and the exchange buffers are untouched.
 *   Statistics (setParticleStatistics, :75-89): the caller passes SelfAdjointEigenSolver(|3 x 3 position block of
 *   covariance|)'s eigenvalues (ascending) and its eigenvector column 2, and expectation().rot_ raw.  On the host, in the
 *   reference's operation order: ratio = sqrt(l2 / l1); max_weight = 1 below perform_weighting_ratio, max_weight above
 *   max_weight_ratio, linear in between (double); fpc_local = mean_rot.inv() * Vec3(float(v)) (float Quat arithmetic).
 *   1. clipped <= num: the whole clipped cloud, in order, no draws; clipped == 0 or num == 0: empty.
 *   2. Normals (pcl::NormalEstimation with a fresh isotropic KdTree and radius r = normal_search_range), restated: the
 *      neighbours of a finite point q are every finite point p with flann::L2_Simple d2 < float(double r * r), q
 *      included, found in a grid of cell edge r (1 + 2^-10) (more margin for coordinates beyond ~8000 cells, so that
 *      the float cell index always keeps a neighbour within one cell); count, sum d and sum d d^T (d = p - q) in
 *      double, C = S / n - m m^T, the normal is the unit eigenvector of C's smallest eigenvalue from ten cyclic Jacobi
 *      sweeps in double, stored as float.  Fewer than 3 neighbours or a non-finite point: a NaN normal.  Its sign is
 *      unspecified; the weight takes |.|.
 *   3. Weight w = 1 + (max_weight - 1) ((pi/2 - acos(a)) / (pi/2)), a = min(1, |nx fx + ny fy + nz fz|) (float products
 *      and sums, widened to double; acos in double from +, -, *, /, sqrt), a NaN normal: 1.
 *   4. Fixed-point weights q = max(1, rint(w 2^F)), F = 32 - ceil(log2(max(1, max_weight))), and their exact uint64
 *      inclusive sum.
 *   5. Draw t of stream s (0 likelihood, 1 beam): Philox-4x32-10 keyed by the seed's two words at counter
 *      (t mod 2^32, s, 0x6e6f726d, t >> 32), r = high 64 bits of (w0 | w1 << 32) * total, index = the first i with
 *      cum_i > r (probability q_i / total).  Output j = the point of the j-th draw, in draw order, whose index was not
 *      drawn before; the draws stop at num outputs.  Draws run in rounds (the host reads one word per round); at most
 *      2^32 draws are made.  The expected number needed is at most n rho H_n (rho = max q / min q <= max(max_weight,
 *      1 / max_weight)), below 10^8 for the node's parameters and a million clipped points; a call that reaches the cap
 *      returns the points found so far (n_lik / n_beam < num) with draws = 2^32.
 * Documented departures: the normals are "parity unpinned" (PCL's NormalEstimation and eigen33 are third-party and
 * absent here; the restatement uses exact neighbour sets, a double covariance and a double eigen routine); Philox instead
 * of std::default_random_engine; output in first-draw order instead of std::unordered_set order; weights rounded to
 * 2^-F; a non-finite max_weight (l1 = l2 = 0, or a ratio exactly equal to equal thresholds: the reference's cumulative
 * weights are NaN there, its result undefined) becomes 1, uniform weights.  The normals and weights of both clipped
 * clouds are computed on every call (mcl3dl_scan_normals reads them), whatever num is.
 * Errors, all before any state changes (the previous samples stay valid): INVALID_ARG for a null engine or params, a
 * multi-device engine, no scan_prepare before, normal_search_range <= 0 or not finite, max_weight <= 0 or not finite,
 * or a non-finite ratio parameter, eigen value / vector entry or mean_rot entry; TOO_LARGE when a clipped cloud's
 * neighbour grid would need 2^31 cells or more (outliers in an unbounded clip window).  Synchronous; single-device. */
typedef struct
{
  double perform_weighting_ratio, max_weight_ratio, max_weight, normal_search_range; /* PointCloudSamplerWithNormalParameters */
  double eigen_values[3]; /* SelfAdjointEigenSolver(|pos cov|).eigenvalues(), ascending */
  double eigen_vector[3]; /* .eigenvectors().col(2) */
  float mean_rot[4];      /* expectation().rot_, raw, x y z w */
  uint32_t lik_num_points, beam_num_points;
  uint64_t seed;
} mcl3dl_normal_sampler_params;
typedef struct
{
  uint32_t n_lik, n_beam;   /* sample sizes: min(num, clipped count) */
  uint32_t n_normal[2];     /* clipped points with a finite normal (lik, beam) */
  uint32_t rounds[2];       /* draw rounds (0 when no draw was needed) */
  uint64_t draws[2];        /* draws made */
  double max_weight;        /* after step 2 and the non-finite rule */
  float fpc_local[3];
  int32_t weight_shift;     /* F of the fixed-point weights */
} mcl3dl_normal_sampler_info;
int mcl3dl_scan_sample_with_normal(mcl3dl_engine*, const mcl3dl_normal_sampler_params*, mcl3dl_normal_sampler_info* info);
/* Diagnostics of the last mcl3dl_scan_sample_with_normal, per clipped point of model `which` (0 likelihood, 1 beam), in
 * clipped order: the normal (3 floats, NaN where none), the neighbour count and the fixed-point weight q.  Each output
 * pointer may be NULL; *n_out = the clipped count.  INVALID_ARG with no such call since the last scan_prepare, a bad
 * `which`, or an output pointer with capacity below the count. */
int mcl3dl_scan_normals(mcl3dl_engine*, int which, float* normals_xyz, uint32_t* n_neighbours, uint64_t* weights_q, size_t capacity,
                        size_t* n_out);

/* ---- Matched / unmatched output (src/mcl_3dl.cpp:761-805): the scan transformed by the pose estimate e
 * (State6DOF::transform, normalised rotation) and split by kdtree_->radiusSearch(p, unmatch_output_dist, id, sqdist, 1)
 * on the map index ChunkedKdtree(chunk_length, max_search_radius):
 *   unmatched: no map point within unmatch_output_dist (the search radius);
 *   matched:   the nearest one has sqdist < match_output_dist^2 (squared in double, :777);
 *   neither:   every other point.
 * Both clouds keep input order and carry the transformed xyz; the label passes through.  Distances are those of the
 * likelihood search (dist_weight rescale, float L2), and which map points a query sees follows the chunk rule of
 * ChunkedKdtree exactly: its own chunk's sub-cloud, halo copies included (chunked_kdtree.h:124-263), which matters
 * because the radius is larger than max_search_radius.  Departures: a non-finite transformed point is unmatched (the
 * reference gets there through floor(NaN) -> INT_MIN on x86, a chunk that does not exist); FLANN's eps is not emulated
 * (the search is exact, as every search of this engine).
 * pts == NULL: the downsampled cloud of the last mcl3dl_scan_prepare (single-device engines; n is ignored).
 * matched / unmatched: host arrays with room for every input point, either may be NULL (count only).  Synchronous; on
 * multi-device engines host clouds run on device 0.  Errors: INVALID_ARG for a null engine, pose, params or count
 * pointer, a map staged without likelihood params, chunk_length <= 0, float(unmatch_output_dist) > chunk_length (the
 * reference throws, chunked_kdtree.h:224-225) or pts == NULL without a prepared scan; NO_MAP before set_map. */
typedef struct
{
  double match_output_dist;   /* Parameters::match_output_dist_   (node default 0.1) */
  double unmatch_output_dist; /* Parameters::unmatch_output_dist_ (node default 0.5): the search radius */
  float chunk_length;         /* ChunkedKdtree(map_chunk_, max_search_radius), src/mcl_3dl.cpp:1327 */
  float max_search_radius;
} mcl3dl_match_params;
int mcl3dl_match_output(mcl3dl_engine*, const mcl3dl_pose* pose, const mcl3dl_point* pts, size_t n,
                        const mcl3dl_match_params*, mcl3dl_point* matched, size_t* n_matched,
                        mcl3dl_point* unmatched, size_t* n_unmatched);

/* Record exchange over peer memory for the one-process-per-GPU layout (SURVEY §8e: particles sharded, ONE gather of the
 * 24-byte records, then the unchanged weight update of include/mcl_3dl/pf.h:252-279 on the full array).  There is no
 * collective call and no copy: the two measurement kernels store each particle's record straight into slot `rank` of
 * EVERY rank's gathered array over NVLink (peer memory mapped with CUDA IPC), and one 32-thread kernel then publishes
 * "rank r finished step s" to every peer and waits, on the device, for the other ranks' flags.  The launch sequence
 * of a step is identical every time (the step parity is read from device memory), so it can be captured in a CUDA
 * graph.  Engines with exactly one device; world <= 8; every rank holds n_local particles.
 *   create:  allocates this rank's buffer (two [world * n_local] record arrays used alternately, plus flags) and writes
 *            its CUDA IPC handle (MCL3DL_IPC_HANDLE_BYTES) for the caller to all-gather between the processes
 *            (once per engine: the peers keep the buffer mapped);
 *   open:    maps the other ranks' buffers from the gathered handles (rank order);
 *   measure_exchange_device: mcl3dl_measure_device for this rank's n_local particles + the exchange, enqueued on the
 *            caller's stream; when it retires, *d_all_out (device memory, valid until the call after next) holds every
 *            rank's records in rank order.  *d_all_out assumes eager calls; after CUDA-graph replays ask `current`;
 *   current: synchronises the stream and returns the array of the last completed step and whether a peer ever failed
 *            to show up within the signal kernel's bounded wait. */
#define MCL3DL_IPC_HANDLE_BYTES 64
int mcl3dl_exchange_create(mcl3dl_engine*, size_t n_local, int world, int rank, void* ipc_handle_out);
int mcl3dl_exchange_open(mcl3dl_engine*, const void* ipc_handles);
int mcl3dl_measure_exchange_device(mcl3dl_engine*, const mcl3dl_pose* d_poses, size_t n_local,
                                   const mcl3dl_point* d_lik_pts, size_t n_lik,
                                   const mcl3dl_point* d_beam_pts, size_t n_beam,
                                   const float* d_origins_xyz, size_t n_origins,
                                   void* cuda_stream, const mcl3dl_result** d_all_out);
int mcl3dl_exchange_current(mcl3dl_engine*, void* cuda_stream, const mcl3dl_result** d_all_out, int* failed_out);

/* The near-field screens staged by the last set_map ([0] likelihood search, [1] KD-tree raycaster's marching search):
 * dilation k (0 = no field staged) and bytes per device.  A screen is one bit per fine cell of the map's bounding box,
 * "a map point may lie within the search radius"; a clear bit skips the exact search, a set bit decides nothing, so
 * results are unchanged (no reference counterpart: ChunkedKdtree::radiusSearch, chunked_kdtree.h:218-251, always
 * descends the tree).  Environment: MCL3DL_NEAR_K / MCL3DL_NEAR_KD_K (0 disables), MCL3DL_NEAR_MAX_MB. */
int mcl3dl_near_field_info(const mcl3dl_engine*, int32_t k_out[2], uint64_t bytes_out[2]);

/* The NN field staged by the last set_map (exact per-voxel candidate lists, the default likelihood search structure;
 * no reference counterpart — ChunkedKdtree::radiusSearch, chunked_kdtree.h:218-251, descends a kd-tree per query):
 * out[0] = bytes per device (0: not staged, the CSR-window kernels serve the searches; after mcl3dl_map_append the
 * allocation, dead lists included), out[1] = candidates stored (live ones: those a fresh build stores),
 * out[2] = directory cells that overflowed (a voxel with more than 40 candidates: queries there fall back to the CSR
 * window search), out[3] = fine voxel edge in micrometres of the rescaled space, out[4] = wide cells (a voxel with 15..40
 * candidates: counts in a side table, one more dependent load).  A voxel-filtered map has neither kind.
 * Environment: MCL3DL_NNF=0 disables, MCL3DL_NNF_MAX_MB caps the size. */
int mcl3dl_nn_field_info(const mcl3dl_engine*, uint64_t out[5]);

/* Field mode (BASELINE.json north_star's literal likelihood kernel; OPT-IN and INEXACT): a dense Euclidean-distance
 * volume over the NN field's lattice, read by trilinear interpolation, replaces the exact nearest-neighbour distance of
 * LidarMeasurementModelLikelihood::measure (src/lidar_measurement_model_likelihood.cpp:124-135).  Interpolating a
 * distance field at 0.1 m voxels deviates by ~1e-1 relative from the reference's scores (SURVEY hard part 1), so the
 * engine never selects it on its own; bench.py / the tests report its deviation.  The beam model is unaffected.
 *   field_mode(1): stage the volume (once per map: node distances from the NN field on the device, a cudaMalloc3D
 *                  volume) and route the likelihood kernel through it; field_mode(0): back to the exact search.
 *                  Needs the NN field (MCL3DL_NNF != 0) and lik params; MCL3DL_ERR_TOO_LARGE above MCL3DL_FIELD_MAX_MB.
 *                  Environment: MCL3DL_LIK_MODE=field = field_mode(1) at create.
 *   field_nodes:   dims (nodes per axis), origin and edge of the lattice (rescaled space); nodes_out != NULL also
 *                  copies the node volume to the host (cudaMemcpy3D), x fastest, dims[0]*dims[1]*dims[2] floats.
 *   field_upload:  replace the node volume by host values of the same dims (cudaMemcpy3D H2D), e.g. an EDT computed
 *                  elsewhere; the per-cell corner layout the kernel reads is rebuilt on the device. */
int mcl3dl_field_mode(mcl3dl_engine*, int enable);
int mcl3dl_field_nodes(mcl3dl_engine*, float* nodes_out, int32_t dims_out[3], float origin_out[3], float* edge_out);
int mcl3dl_field_upload(mcl3dl_engine*, const float* nodes, const int32_t dims[3]);

/* Enable (and zero) / disable the work counters; read them (synchronises the devices). */
int mcl3dl_collect_stats(mcl3dl_engine*, int enable);
int mcl3dl_read_stats(mcl3dl_engine*, mcl3dl_work_stats* out);

/* Device times of the last mcl3dl_measure call (CUDA events on the engine's stream, max over
 * devices): host->device copies, the two kernels, device->host copy.  The events cost tens of
 * microseconds per update, so they are only recorded after mcl3dl_collect_timing(eng, 1)
 * (or with MCL3DL_TIMING=1 in the environment); otherwise the four values read 0. */
int mcl3dl_collect_timing(mcl3dl_engine*, int enable);
int mcl3dl_last_timing(const mcl3dl_engine*, double* h2d_ms, double* lik_kernel_ms, double* beam_kernel_ms,
                       double* d2h_ms);

/* Device work this engine enqueued since create (the bench's gpu_launches counter): one per successful kernel launch and
   one per device-wide CUB call (sort, scan, reduce), however many kernels CUB runs inside it. */
uint64_t mcl3dl_kernel_launches(const mcl3dl_engine*);

const char* mcl3dl_strerror(int code);
/* Text of the last CUDA failure seen by this engine ("" if none). */
const char* mcl3dl_last_error_detail(const mcl3dl_engine*);
int mcl3dl_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MCL3DL_B200_H */
