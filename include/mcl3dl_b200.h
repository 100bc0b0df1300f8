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

/* pf_->init()/resizeParticle() happen on the host; set() uploads the result (states + probability_), get() reads the
 * set back (either pointer may be NULL) — e.g. for pf_->expectationBiased()/covariance(), which stay host code. */
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
 * particles that tie in the accumulated probability are taken by lowest index instead of std::sort's order. */
int mcl3dl_particles_resample(mcl3dl_engine*, const float sigma_pos[3], const float sigma_rpy[3], float initial_frac,
                              uint64_t seed);

/* The pose estimate the node takes from the filter after every measurement, on the resident set
 * (src/mcl_3dl.cpp:428-452,704-724): pf_->bias(bias_func) + pf_->expectationBiased() (pf.h:246-251,294-303;
 * ParticleWeightedMeanQuat, state_6dof.h:316-355), pf_->max() (pf.h:361-374) and pf_->covariance(1.0, .) (pf.h:304-360,
 * State6DOF::covElement state_6dof.h:162-184).  Only this summary leaves the device.
 *   state_prev == NULL: bias 1 for every particle (the node's branch for more particles than num_particles, :428-434);
 *   otherwise bias = NormalLikelihood(bias_var_dist)(|pos - prev.pos|) * NormalLikelihood(bias_var_ang)(angle) + 1e-6.
 * Sums are accumulated in double with a fixed tree (the reference: sequential float), so the values agree with the
 * reference to ~1e-5 relative.  Documented departures: the covariance always uses every particle (the reference
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
 * and unpinned (restated from its published algorithm; centroid float sums in input order, majority label); the
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
 * out[0] = bytes per device (0: not staged, the CSR-window kernels serve the searches), out[1] = candidates stored,
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

/* Number of this library's kernels launched since create (the bench's gpu_launches counter). */
uint64_t mcl3dl_kernel_launches(const mcl3dl_engine*);

const char* mcl3dl_strerror(int code);
/* Text of the last CUDA failure seen by this engine ("" if none). */
const char* mcl3dl_last_error_detail(const mcl3dl_engine*);
int mcl3dl_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MCL3DL_B200_H */
