/*
 * limovelo_b200.h — C ABI of liblimovelo_b200.so
 *
 * H100-native (sm_90a) implementation of LIMO-Velo's per-sweep localization hot path:
 * Localizator::correct -> IKFoM update_iterated_dyn_share_modified -> per iteration
 * Mapper::match (exact 5-NN, plane fit, gates) -> Localizator::calculate_H -> HtH / Hth ->
 * 23-DoF state update.  Plain pointers and sizes only; no torch / Eigen / ROS types.
 *
 * Every entry point names the reference interface it replaces (paths relative to the
 * LIMO-Velo source tree; esekfom.hpp = include/IKFoM/IKFoM_toolkit/esekfom/esekfom.hpp).
 * INTEGRATION.md shows the reference-side glue (the h_share_model / Localizator / Mapper
 * call sites that would bind these).
 *
 * Threading: like the reference (single main thread, main.cpp:52-130) a handle is not
 * re-entrant.  Handles are independent of each other: one handle = one sequence = one
 * CUDA device + stream.
 *
 * There is NO CPU fallback: every compute entry point returns LV_ERR_CUDA when no CUDA
 * device is usable.
 */
#ifndef LIMOVELO_B200_H_
#define LIMOVELO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LV_STATE_LEN 26   /* flat state_ikfom, see lv_state_layout below                    */
#define LV_DOF 23         /* state_ikfom::DOF (use-ikfom.hpp:12-21)                         */
#define LV_MEAS_COLS 12   /* non-zero Jacobian columns (Localizator.cpp:31, esekfom.hpp:1647) */
#define LV_MAX_EVALS 8    /* capacity of the per-update log: MAX_NUM_ITERS + 1 <= 8          */

typedef struct lv_context* lv_handle;

typedef enum lv_status {
    LV_OK = 0,
    LV_EMPTY_MAP = 1,          /* Localizator.cpp:24 / Mapper.cpp:42 silent returns           */
    LV_TOO_FEW_MATCHES = 2,    /* Nm < 23: esekfom.hpp:1701-1709 branch (undefined in the ref) */
    LV_ERR_ARG = 3,
    LV_ERR_CUDA = 4,           /* no device / CUDA failure (see lv_last_error)                */
    LV_ERR_CAPACITY = 5,       /* more points than the handle was created for                 */
    LV_ERR_IO = 6,             /* YAML file unreadable                                        */
    LV_TOO_FEW_POINTS = 7      /* main.cpp:81: fewer points than MAX_POINTS2MATCH, no update (lv_correct_device_async) */
} lv_status;

/*
 * Flat state layout (26 doubles), field order of state_ikfom (use-ikfom.hpp:12-21),
 * quaternions in Eigen coeffs() order (x, y, z, w):
 *   [0:3) pos   [3:7) rot   [7:11) offset_R_L_I   [11:14) offset_T_L_I
 *   [14:17) vel [17:20) bg  [20:23) ba            [23:26) grav (S2, |grav| = 9.809)
 * Covariance P is 23 x 23 row-major in DOF order pos0 rot3 offR6 offT9 vel12 bg15 ba18 grav21.
 */

/* Configuration.  Upper-case / ROS-style names are the YAML keys read by fill_config
 * (src/main.cpp:135-176) with the same defaults; the last block is device tuning that has
 * no counterpart in the reference.                                                         */
typedef struct lv_params {
    /* Localizator */
    int32_t MAX_NUM_ITERS;            /* main.cpp:144, default 3                           */
    int32_t NUM_MATCH_POINTS;         /* main.cpp:146, must be 5                           */
    int32_t estimate_extrinsics;      /* main.cpp:139                                      */
    int32_t print_degeneracy_values;  /* main.cpp:156 (eigenvalues are returned in the log) */
    double MAX_DIST_PLANE;            /* main.cpp:148, default 2.0                         */
    float PLANES_THRESHOLD;           /* main.cpp:149, default 0.1                         */
    float pad0_;
    double LiDAR_noise;               /* main.cpp:152 -> R                                 */
    double degeneracy_threshold;      /* main.cpp:155 -> D                                 */
    double LIMITS[LV_DOF];            /* main.cpp:145, default 23 x 0.001                  */
    /* IMU process noise (Localizator.cpp:164-168) */
    double covariance_gyroscope, covariance_acceleration;
    double covariance_bias_gyroscope, covariance_bias_acceleration;
    /* extrinsics / gravity (Localizator.cpp:135-153) */
    float initial_gravity[3];
    float I_Translation_L[3];
    float I_Rotation_L[9];            /* row-major YAML list                               */
    float map_downsample_size;        /* ikd-Tree box_length, Mapper.cpp:65 = 0.2          */
    /* ---- device tuning (not in the reference) ---- */
    float voxel_size;                 /* edge of the hashed search voxels [m], default 0.4; rounded to a whole number
                                       * (1..3) of map_downsample_size cells: a voxel is k x k x k downsample cells */
    int32_t device;                   /* CUDA device ordinal                               */
    int32_t pad1_;                    /* reserved (keeps the layout of earlier releases), ignored */
    int64_t max_map_points;           /* capacity of the device map                        */
    int64_t max_points;               /* capacity of one sweep                             */
    void* stream;                     /* cudaStream_t to run on; NULL = own stream         */
} lv_params;

/* One record per h-evaluation of update_iterated_dyn_share_modified (esekfom.hpp:1634-1822) */
typedef struct lv_iter_log {
    int64_t n_matches;        /* Nm = rows of h_x (esekfom.hpp:1650)                       */
    int32_t converged;        /* dyn_share.converge after esekfom.hpp:1748-1762            */
    int32_t degenerate;       /* 1 if any eigenvalue of HTH[0:6,0:6] < D (esekfom.hpp:1740) */
    double HTH[144];          /* row-major 12 x 12 (esekfom.hpp:1723)                      */
    double HTh[12];           /* h_x^T h (esekfom.hpp:1727)                                */
    double dx[LV_DOF];        /* dx_ before the degeneracy mask (esekfom.hpp:1733)         */
    double x_after[LV_STATE_LEN];
} lv_iter_log;

typedef struct lv_profile {
    double measure_ms;        /* sum of device time of the measurement kernels (search + fit) */
    double solve_ms;          /* sum of device time of the IESKF step kernel               */
    double build_ms;          /* sum of device time of map (re)builds                      */
    int64_t measure_launches, solve_launches, build_launches;
    int64_t total_launches;   /* every kernel launched by this handle since the last reset */
    double idle_ms;           /* launches that found the update already finished (early exit) */
    int64_t idle_launches;
    /* measure_ms split by kernel (each launched once per h-evaluation) */
    double search_ms;         /* lv_search_kernel: exact 5-NN at level 0                   */
    double search_upper_ms;   /* lv_search_rings_kernel: the queries level 0 cannot certify */
    double fit_ms;            /* lv_fit_kernel: plane fit, Jacobian rows, normal equations  */
    double reuse_ms;          /* lv_reuse_kernel: neighbours carried over from the previous evaluation */
    double search_first_ms;   /* the part of search_ms spent in FIRST evaluations: those launches search every query of the
                               * sweep (later ones only the queries the reuse test handed back)                  */
    int64_t search_first_launches;
} lv_profile;

/* ------------------------------------------------------------------------------------------ */
/* configuration                                                                              */
void lv_default_params(lv_params* p);                         /* defaults of main.cpp:137-175 */
lv_status lv_params_from_yaml(const char* path, lv_params* p); /* config/<name>.yaml keys           */

/* lifetime: replaces the Localizator / Mapper singletons (Localizator.cpp:100-103,
 * Mapper.hpp:35-38): one handle owns one filter and one map.                                */
lv_status lv_create(const lv_params* p, lv_handle* out);
void lv_destroy(lv_handle h);
const char* lv_last_error(void);
const char* lv_version(void);
/* bytes one lv_correct() reads back from the device (state, covariance, logs): the D2H side of its e2e cost */
int64_t lv_result_bytes(void);

/* ---- Mapper boundary (include/Headers/Mapper.hpp:17-23) ---------------------------------- */
/* Mapper::add on an empty map == KD_TREE::Build, no downsampling (Mapper.cpp:26,68-71).      */
lv_status lv_map_build(lv_handle h, const float* xyz, int64_t m);
/* Mapper::add on an existing map == KD_TREE::Add_Points (Mapper.cpp:73-76,
 * ikd_Tree.cpp:478-573): 0.2 m voxel rule when downsample != 0.                              */
lv_status lv_map_add(lv_handle h, const float* xyz, int64_t n, int downsample);
/* Both are ASYNCHRONOUS on the handle's stream (no host round trip: every count lives on the device; the host
 * buffer may be reused when the call returns only if it is pinned — pageable memory is staged by the runtime).
 * Running out of table / arena space is flagged on the device and reported as LV_ERR_CAPACITY by the next call
 * that synchronises anyway (lv_map_size, lv_map_status, lv_correct, lv_last_logs).                              */
int64_t lv_map_size(lv_handle h);                             /* Mapper::size  (Mapper.cpp:32); synchronises */
int lv_map_exists(lv_handle h);                               /* Mapper::exists (Mapper.cpp:36) */
lv_status lv_map_status(lv_handle h);                         /* synchronises; LV_OK or LV_ERR_CAPACITY       */
/* KD_TREE::flatten: the map's points in insertion order; returns their number; synchronises  */
int64_t lv_map_points(lv_handle h, float* xyz_out, int64_t cap);
/* same as lv_map_build / lv_map_add but xyz is a DEVICE pointer (data already resident in HBM, e.g. the deskewed
 * sweep transformed by the update's own result): correct -> add never leaves the GPU.  The buffer must stay valid
 * until the stream has passed the call.                                                                        */
lv_status lv_map_build_device(lv_handle h, const float* d_xyz, int64_t m);
lv_status lv_map_add_device(lv_handle h, const float* d_xyz, int64_t n, int downsample);
/* main.cpp:99-105 on the device: `map.add(Xt2 * Xt2.I_Rt_L() * ds_compensated, t2, true)`.  The sweep is given in the
 * LiDAR frame (device memory) and is transformed by the filter's current state, i.e. the result of the lv_correct /
 * lv_correct_device that precedes the call, without that state ever visiting the host.  lv_map_add_last_sweep reuses
 * the sweep of that update (it is still resident), so one tick is lv_correct(...); lv_map_add_last_sweep(h, 1).
 * On an empty map both build it un-downsampled (Mapper.cpp:26).  That is how a sequence starts: the first tick's
 * lv_correct returns LV_EMPTY_MAP but keeps the sweep, and lv_map_add_last_sweep builds the map from it at the
 * current (propagated) state.  Asynchronous.                                                                      */
lv_status lv_map_add_sweep_device(lv_handle h, const float* d_xyz_lidar, int64_t n, int downsample);
lv_status lv_map_add_last_sweep(lv_handle h, int downsample);

/* ---- map capacity.  The ikd-Tree has none: it allocates nodes for as long as the sequence runs (Mapper.cpp:22-30,
 * ikd_Tree.cpp:478-573).  The device map is sized from lv_params.max_map_points at lv_create and can grow after it:
 * new, larger tables and arena, the old content re-hashed / copied into them on the handle's stream.  A growth keeps
 * the content, the point ids, the insertion order and every arena index, so results do not change: only the storage
 * behind the map gets bigger.  It never shrinks. */
/* grow now so that the map holds at least `points` points at the ratios of lv_create (4 voxel slots, 96 arena float4
 * per point).  Asynchronous.  No-op when `points` is not above the current capacity.  LV_ERR_CAPACITY (the map
 * untouched, lv_last_error names the ceiling) beyond 2^26 voxel slots or 0x7FFFFFF0 arena entries (ids are int32),
 * i.e. beyond 2^24 points; LV_ERR_CAPACITY with the CUDA error when the device is out of memory (map untouched). */
lv_status lv_map_reserve(lv_handle h, int64_t points);
/* automatic growth up to a capacity of `max_points` points (0: off, the default).  With it on, before every add
 * (lv_map_add*, lv_map_add_last_sweep) the host bounds what the map will hold after it from the newest counter snapshot
 * the device has finished (no synchronisation) plus the adds queued since: points + n, voxel slots + 27 n, block slots
 * + n, arena + 96 n; it doubles the capacity while a bound crosses its mark (points above capacity, slots or blocks
 * above half their table, arena above 3/4).  lv_map_build(_device) of m > capacity and adds of n > the add capacity grow
 * to fit instead of failing.  What this does NOT guarantee: the arena figure is a planning ratio, not a bound, and the
 * limit caps every growth, so an add can still overflow (one huge scattered add on a small limit); that is reported as
 * LV_ERR_CAPACITY by the next synchronising call exactly as without growth.  Growth past the limit is refused with
 * LV_ERR_CAPACITY where an add cannot even be staged (n above the add capacity at the limit).  Enabling synchronises
 * once (to read the counters). */
lv_status lv_map_set_growth(lv_handle h, int64_t max_points);
/* (a struct tag, not a typedef: the function below has the same name) */
struct lv_map_info {
    /* capacity */
    int64_t capacity_points;   /* points the tables and the arena are sized for                          */
    int64_t voxel_slots;       /* 32-byte slots of the voxel table                                        */
    int64_t block_slots;       /* 16-byte slots of the block table                                        */
    int64_t arena_entries;     /* float4 entries of the arena                                             */
    int64_t add_capacity;      /* most points one build / add takes                                       */
    int64_t bytes;             /* device bytes of the map: tables, arena, lists, add scratch               */
    /* usage (device counters) */
    int64_t points;
    int64_t slots_used;
    int64_t blocks_used;
    int64_t arena_top;         /* arena entries handed out (abandoned extents included)                   */
    /* growth */
    int64_t growths;           /* growths so far: lv_map_reserve and automatic                            */
    int64_t growth_limit;      /* lv_map_set_growth's max_points; 0 = off                                 */
    int64_t host_waits;        /* times the growth policy waited for a pending counter snapshot          */
    uint32_t error_flags;      /* device error flags (0: none; see LV_ERR_CAPACITY)                      */
    uint32_t pad_;
};
/* Mapper::size and more: capacity, usage and growth of the map; synchronises */
lv_status lv_map_info(lv_handle h, struct lv_map_info* out);

/* ---- operator boundary: the measurement model IKFoM calls (esekfom.hpp:128,1637) --------- */
/* compat mode: fills h_x (Nm x 12, COLUMN-major like Eigen::MatrixXd) and h (Nm) exactly as
 * IKFoM::h_share_model does (use-ikfom.cpp:16-37); rows in input-point order.                */
lv_status lv_measure(lv_handle h, const double* x /*LV_STATE_LEN*/, const float* xyz_lidar, int64_t n,
                     double* h_x, double* h_vec, int64_t* nm);
/* fast mode: what update_iterated_dyn_share_modified consumes when Nm >= 23
 * (esekfom.hpp:1722-1729): HTH = h_x^T h_x (row-major 12x12), HTh = h_x^T h.                 */
lv_status lv_measure_reduced(lv_handle h, const double* x, const float* xyz_lidar, int64_t n,
                             double* HTH, double* HTh, int64_t* nm);
/* Mapper::match without the compaction (Mapper.cpp:40-56): per input point the world point,
 * the 5 neighbours (indices into the current map order of lv_map_points, squared distances
 * ascending), the fitted plane (A,B,C,D), the point-to-plane distance and is_chosen().
 * Any output pointer may be NULL.  Neighbour data are defined for points whose 5th
 * neighbour is closer than MAX_DIST_PLANE (others report idx -1).                            */
lv_status lv_match_all(lv_handle h, const double* x, const float* xyz_lidar, int64_t n,
                       uint8_t* valid, int32_t* nn_idx, float* nn_sqd, float* plane, float* dist,
                       float* g_world);
/* The neighbours the LAST evaluation of the last lv_correct (or operator call) handed to the plane fit: nn_idx (n x 5,
 * indices as in lv_match_all, -1 where a query had fewer than five).  lv_match_all always searches afresh; inside an
 * update, evaluations after the first keep the stored five wherever the exact search provably returns them again
 * (the reference searches every time, Mapper.cpp:40-56) — this is the window on what the update really used.  */
lv_status lv_last_neighbours(lv_handle h, int64_t n, int32_t* nn_idx);

/* ---- module boundary: Localizator (include/Headers/Localizator.hpp:24-33) ---------------- */
lv_status lv_set_state(lv_handle h, const double* x, const double* P);   /* change_x / change_P */
lv_status lv_get_state(lv_handle h, double* x, double* P);               /* get_x / get_P       */
/* Localizator::init_IKFoM_state (Localizator.cpp:135-153); q_imu = (x,y,z,w)                 */
lv_status lv_init_state(lv_handle h, const float q_imu[4]);
/* Localizator::propagate -> esekf::predict (Localizator.cpp:159-173, esekfom.hpp:279-384)    */
lv_status lv_predict(lv_handle h, const double acc[3], const double gyro[3], double dt);
/* Localizator::propagate_to (Localizator.cpp:59-75) on the DEVICE: the k IMU samples between two sweeps (acc, gyro: k x 3,
 * dt: k) run through esekf::predict in one launch; the filter state stays in HBM, so update -> propagate -> update needs no
 * host round trip (lv_get_state fetches it when the caller wants to publish it).  Same arithmetic as lv_predict.        */
lv_status lv_propagate_device(lv_handle h, const double* acc, const double* gyro, const double* dt, int32_t k);
/* the same two host-side steps on caller-owned (x, P), no handle and no GPU involved           */
lv_status lv_init_state_host(const lv_params* p, const float q_imu[4], double* x, double* P);
lv_status lv_predict_host(const lv_params* p, const double acc[3], const double gyro[3], double dt,
                          double* x, double* P);
/* Localizator::correct(points, time) (Localizator.cpp:23-27): the whole iterated update.
 * xyz_lidar: HOST buffer of n deskewed points in the LiDAR frame.  logs (capacity
 * LV_MAX_EVALS) / n_evals / x_out / P_out may be NULL.
 * On an empty map it returns LV_EMPTY_MAP and leaves the state, the time and x_out / P_out untouched (Localizator.cpp:24),
 * but the sweep is still uploaded and becomes the one lv_map_add_last_sweep adds: the first tick builds the map.  */
lv_status lv_correct(lv_handle h, const float* xyz_lidar, int64_t n, double time,
                     lv_iter_log* logs, int32_t* n_evals, double* x_out, double* P_out);
/* same, but the points are already resident in HBM (DEVICE pointer) and nothing is copied
 * back except through lv_get_state / lv_last_logs.  On an empty map it returns LV_EMPTY_MAP
 * and records the sweep for lv_map_add_last_sweep, like lv_correct.                          */
lv_status lv_correct_device(lv_handle h, const float* d_xyz_lidar, int64_t n, double time);
lv_status lv_last_logs(lv_handle h, lv_iter_log* logs, int32_t* n_evals);
/* Localizator::last_time_updated; synchronises when an lv_correct_device_async is still to be resolved */
double lv_last_time_updated(lv_handle h);

/* ---- starting a sequence in a saved map (no counterpart in the reference: its README lists prelocalization in a saved map as
 * work in progress).  The update converges from errors well inside MAX_DIST_PLANE only; lv_prelocalize searches a window of
 * positions and headings about the gravity axis around the filter's state and moves the state to the best candidate.
 *
 * Semantics of lv_prelocalize:
 *   base state   the filter's current state on the device, the one lv_get_state would return after preceding
 *                lv_propagate_device / update work.  The call synchronises.
 *   axes         rotation axis g = grav / |grav| (the state's S2 field), right-hand rule.  Position axes
 *                u = normalize(e - (e.g) g) and v = g x u, with e the world x axis, or the y axis when |g_x| > 0.9.
 *   grid         I = floor(radius / step + 1e-9), K = floor(yaw_range / yaw_step + 1e-9) (in double);
 *                a_i = i step, b_j = j step for i, j in [-I, I]; theta_k = k yaw_step for k in [-K, K].
 *                Linear index ((k + K)(2I + 1) + (i + I))(2I + 1) + (j + I).  More than 2^24 candidates are refused.
 *   candidate    rot' = q(g, theta_k) (x) rot and pos' = pos + (a_i u + b_j v), both in fp64 (a_i u + b_j v: the products,
 *                then the sum); vel' = R(g, theta_k) vel; every other field unchanged.  theta_k = 0 keeps rot and vel as
 *                they are.
 *   score        the number of the S scored points whose world point lands in a voxel that holds map points (its
 *                block-mask bit is set).  The world point is fp32: F_k = make_frame(x with rot').lidar_to_world, once per
 *                heading; o_ij = (float)(a_i u + b_j v); t = fadd(F_k.t, o_ij); w = fadd(dot3f(F_k.R row, p), t) (rt_apply);
 *                the voxel of each axis as the map computes it (cell floor(w / map_downsample_size), voxel_size cells).
 *                A point with a coordinate not below 1e9 m in magnitude, or NaN, never scores (the map holds no such point).
 *                For k = i = j = 0 the world points are, by construction, bit for bit lv_match_all's g_world at the base.
 *   subset       S = min(n, max_points); point s is d_xyz_lidar[floor(s n / S)] (int64 arithmetic).
 *   winner       the highest score; ties go to the smaller |k|, then the smaller i^2 + j^2, then the smaller linear index.
 *                The selection does not depend on launch order (one packed 64-bit key per candidate, atomicMax).
 *   effect       the filter state becomes out->x, as lv_set_state(out->x, NULL) would set it; P, the map, the time and
 *                the recorded sweep (lv_map_add_last_sweep) are unchanged.
 *   empty map    LV_EMPTY_MAP and nothing changes, also after an asynchronous first build that the gate left empty.
 *   arguments    LV_ERR_ARG before any device work, also with a null handle, lv_last_error naming the problem: null params,
 *                result or points, n outside [1, 2^31 - 1], a parameter outside its range, more than 2^24 candidates.
 * scores_out (host, NULL or lv_preloc_count(p) entries) receives every candidate's score at its linear index: a second peak
 * far from the winner means the window is ambiguous (a corridor, a symmetric hall).  One kernel launch. */
typedef struct lv_preloc_params {
    float radius;       /* half-width (m) of the square of positions searched around the current position, >= 0          */
    float step;         /* grid step of positions (m), > 0; the voxel edge (voxel_size) is the natural choice              */
    float yaw_range;    /* half-width (rad) of the headings searched about the gravity axis, in [0, pi] (pi: 3.1415927f)   */
    float yaw_step;     /* rad, > 0                                                                                      */
    int32_t max_points; /* sweep points scored, 1 .. 4096 (evenly strided subset when the sweep has more)                 */
    int32_t pad_;
} lv_preloc_params;
typedef struct lv_preloc_result {
    double x[LV_STATE_LEN]; /* the winning candidate's state (written to the filter)                          */
    int64_t candidates;     /* (2K+1) (2I+1)^2                                                              */
    int64_t index;          /* linear index of the winner                                                  */
    int32_t k, i, j;        /* its heading and position indices                                            */
    int32_t score;          /* scored points that fall in an occupied voxel                                */
    int32_t points;         /* points scored (S)                                                           */
    int32_t pad_;
} lv_preloc_result;
/* the number of candidates (2K+1)(2I+1)^2 of p, or -1 for invalid params (or a count above 2^61); no GPU needed.  A count
 * above 2^24 is returned as it is: lv_prelocalize refuses it. */
int64_t lv_preloc_count(const lv_preloc_params* p);
/* d_xyz_lidar: DEVICE buffer of n sweep points in the LiDAR frame (e.g. the deskewed, voxel-grid downsampled first sweep) */
lv_status lv_prelocalize(lv_handle h, const float* d_xyz_lidar, int64_t n, const lv_preloc_params* p,
                         lv_preloc_result* out, int32_t* scores_out /* NULL or lv_preloc_count(p) entries */);

/* ---- the start pose anywhere in a saved map: an exact branch-and-bound form of the same search, for windows that cover a
 * whole map.
 *
 * Semantics of lv_prelocalize_global: base state, axes, grid, candidate, score, subset, winner, effect, empty map and
 * arguments as lv_prelocalize above, except:
 *   cap          up to 2^40 candidates and 2^20 headings (yaw_step >= about 6e-6 rad over every heading); more are refused
 *                (LV_ERR_ARG, "more than 2^40" / "more than 2^20").  There is no scores array: only a fraction of the
 *                candidates is ever scored.
 *   result       out holds exactly what lv_prelocalize would return for the same state, map, points and params: index,
 *                k, i, j, score, points, candidates, and x bit for bit; the filter state is set the same way.  P, the
 *                time, the map and the recorded sweep are untouched.
 *   how          a cell is one heading with an aligned block of 2^l x 2^l positions (clipped at the window's edge).
 *                Every step from (i, j) to a point's voxel is monotone per axis, so over a cell each voxel coordinate of
 *                a scored point lies between its values at the cell's four corners; the cell's upper bound counts the
 *                points whose voxel box may hold an occupied voxel.  A cell is pruned only when its bound is strictly
 *                below a score some candidate reaches, so every candidate that could win or tie is scored exactly with
 *                lv_prelocalize's arithmetic.  The cells are bounded at 32 x 32 positions (more for very large windows),
 *                taken in order of bound, and refined level by level; level-1 survivors are scored exactly.
 *   stats        NULL or filled.  Every count depends on the inputs only (not on launch order or timing).  Each candidate
 *                counts once in candidates_scored.  launches counts the search's launches; the map's occupancy summary
 *                (extent and bitmaps, two launches) is built once per map state and kept until an add, build or growth
 *                changes the map (those launches appear in the profile's total_launches, not in stats).
 *   environment  LV_PRELOC_NO_PRUNE=1 (read at each call) scores every candidate through the same exact kernel and
 *                selection, bounding nothing: the exhaustive reference for windows above lv_prelocalize's cap.
 * Covering every position inside the map's extent: lv_map_extent, then radius = the largest |(c - pos).u|, |(c - pos).v|
 * over the box's corners c (INTEGRATION.md B7).  Synchronises; several launches (stats->launches). */
typedef struct lv_preloc_stats {
    int64_t candidates;        /* (2K+1)(2I+1)^2 of the window                                              */
    int64_t cells_bounded;     /* cells (blocks of positions x one heading) whose upper bound was computed  */
    int64_t candidates_scored; /* candidates scored exactly (level 0)                                       */
    int64_t probes;            /* occupancy probes, all levels: S per bounded cell and per scored candidate */
    int32_t launches, pad_;    /* kernel launches of the search                                             */
} lv_preloc_stats;
lv_status lv_prelocalize_global(lv_handle h, const float* d_xyz_lidar, int64_t n, const lv_preloc_params* p,
                                lv_preloc_result* out, lv_preloc_stats* stats /* NULL or filled */);
/* axis-aligned box (world frame, metres) of the occupied voxels' extent: lo = the low face of the lowest occupied voxel,
 * hi = the high face of the highest (voxel_low of the next voxel), per axis.  A window built from it as above covers every
 * position inside the map's extent.  A sweep reaches beyond the vehicle, so a pose just outside the box can still see the
 * map: pad the radius by the sweep's range to include those.  Synchronises; LV_EMPTY_MAP on an empty map; LV_ERR_ARG for a
 * null handle, lo or hi. */
lv_status lv_map_extent(lv_handle h, double lo[3], double hi[3]);

/* ---- utilities --------------------------------------------------------------------------- */
void* lv_host_alloc(int64_t bytes);                           /* pinned host memory            */
void lv_host_free(void* p);
void* lv_device_alloc(lv_handle h, int64_t bytes);
void lv_device_free(lv_handle h, void* p);
lv_status lv_memcpy_h2d(lv_handle h, void* dst, const void* src, int64_t bytes);
lv_status lv_memcpy_d2h(lv_handle h, void* dst, const void* src, int64_t bytes);   /* both synchronise */
lv_status lv_synchronize(lv_handle h);
lv_status lv_profile_enable(lv_handle h, int on);             /* CUDA-event timing per kernel  */
lv_status lv_profile_get(lv_handle h, lv_profile* out, int reset);
lv_status lv_flush_l2(lv_handle h);                           /* writes a 256 MiB scratch      */

/* ---- Compensator boundary: deskew (include/Headers/Compensator.hpp, src/Modules/Compensator.cpp) ---- */
/* `State` of include/Headers/Objects.hpp:97-120 (single precision like the reference), row-major matrices */
typedef struct lv_state32 {
    float R[9];
    float pos[3], vel[3], bw[3], ba[3], g[3];
    float RLI[9], tLI[3];
    float a[3], w[3];          /* last controls (State.cpp:129-131) */
    double time;
} lv_state32;
/* State(const state_ikfom&, double) (State.cpp:40-62): x = flat state (layout above); a, w = the IMU sample that
 * follows `time` (Accumulator::get_next_imu); g = p->initial_gravity (State.cpp:21)                    */
void lv_state_from_ikfom(const lv_params* p, const double* x, double time, const float a[3], const float w[3],
                         lv_state32* out);
/* State::operator+=(const IMU&) (State.cpp:73-75 -> update :122-132 -> propagate_f :103-120), host */
void lv_state_add_imu(lv_state32* s, const float a[3], const float w[3], double time);
/* Compensator::upsample (Compensator.cpp:73-113): states (before t1 .. t2) + IMU samples (a, w: ni x 3, t: ni) ->
 * the integrated path; returns the number of states the path has (writes at most cap)                   */
int32_t lv_compensator_upsample(const lv_state32* states, int32_t ns, const float* imu_a, const float* imu_w,
                                const double* imu_t, int32_t ni, lv_state32* out, int32_t cap);
/* Compensator::get_t2 (Compensator.cpp:55-63) */
void lv_compensator_get_t2(const lv_state32* path, int32_t ns, double t2, lv_state32* out);
/* Compensator::compensate(states, Xt2, points) (Compensator.cpp:123-146): every point is carried from the pose at
 * its own timestamp to the LiDAR frame at t2.  xyz (n x 3) and t (n, ascending, inside [path[0].time,
 * path[ns-1].time]) are HOST buffers; xyz_out (n x 3, host) receives the deskewed points in input order, which is
 * what Localizator::correct takes.  LV_ERR_ARG if a timestamp lies outside the path (the reference asserts).   */
lv_status lv_compensate(lv_handle h, const lv_state32* path, int32_t ns, const lv_state32* Xt2, const float* xyz,
                        const double* t, int64_t n, float* xyz_out);
/* same on device-resident buffers (lv_device_alloc); d_xyz_out may alias d_xyz                              */
lv_status lv_compensate_device(lv_handle h, const lv_state32* path, int32_t ns, const lv_state32* Xt2,
                               const float* d_xyz, const double* d_t, int64_t n, float* d_xyz_out);

/* ---- downsamplers in front of the path (SURVEY 8f row 3) -------------------------------------------- */
/* PointCloudProcessor::downsample -> temporal_downsample (src/Utils/PointCloudProcessor.cpp:18-21,101-112): keeps
 * point i iff (downsample_rate <= 1 or (i + 1) % downsample_rate == 0) and min_dist < |p|, order preserved.
 * HOST buffers; xyz_out (n x 3) and idx_out (n, may be NULL: indices of the kept points, for the caller's other
 * per-point fields) receive *n_out entries.                                                             */
lv_status lv_temporal_downsample(lv_handle h, const float* xyz, int64_t n, int32_t downsample_rate, double min_dist,
                                 float* xyz_out, int32_t* idx_out, int64_t* n_out);
/* Compensator::downsample -> voxelgrid_downsample (src/Modules/Compensator.cpp:115-118,148-163): pcl::VoxelGrid with
 * leaf downsample_prec: one centroid per occupied leaf, leaves in ascending PCL cell index.  xyz_out needs room for
 * n points.  When the leaf is too small for the extent (cell index overflow) PCL warns and returns the input: so does
 * this (n_out = n, LV_OK, the warning in lv_last_error()).                                                          */
lv_status lv_voxelgrid_downsample(lv_handle h, const float* xyz, int64_t n, float downsample_prec, float* xyz_out,
                                  int64_t* n_out);
/* the same on device-resident buffers; LV_ERR_ARG (and a message in lv_last_error()) when the n-point ranges at
 * d_xyz and d_xyz_out overlap                                                                              */
lv_status lv_voxelgrid_downsample_device(lv_handle h, const float* d_xyz, int64_t n, float downsample_prec,
                                         float* d_xyz_out, int64_t* n_out);
/* lv_voxelgrid_downsample_full_device_async on HOST buffers of n points (the outputs need room for n; time_out, intensity_out and
 * range_out may be NULL); synchronises.  LV_ERR_ARG for a null handle or input, n outside [0, 2^31 - 1] or a leaf <= 0.  The
 * overflow pass-through returns LV_OK with *n_out = n and PCL's warning in lv_last_error(), as lv_voxelgrid_downsample. */
lv_status lv_voxelgrid_downsample_full(lv_handle h, const float* xyz, const double* time, const float* intensity, int64_t n,
                                       float downsample_prec, float* xyz_out, double* time_out, float* intensity_out, float* range_out,
                                       int64_t* n_out);

/* ---- wire format of the LiDAR message (SURVEY 8f row 4, last item) --------------------------------------
 * PointCloudProcessor::msg2points (src/Utils/PointCloudProcessor.cpp:24-99) on the raw `data` of a
 * sensor_msgs/PointCloud2: the point structs of include/Headers/Common.hpp:109-221 are read field by field at the
 * byte offsets the message declares (pcl::fromROSMsg maps fields by name), so no ROS / PCL type is needed here. */
typedef enum lv_lidar_type { LV_LIDAR_VELODYNE = 0, LV_LIDAR_HESAI = 1, LV_LIDAR_OUSTER = 2, LV_LIDAR_CUSTOM = 3 } lv_lidar_type;
typedef struct lv_cloud_layout {
    int32_t point_step;        /* bytes per point */
    int32_t off_x, off_y, off_z;           /* float32 */
    int32_t off_intensity;     /* velodyne / custom: float32 `intensity`; hesai: uint8 `intensity`; ouster: uint16 `reflectivity` */
    int32_t off_time;          /* velodyne: float32 `time`; hesai / custom: float64 `timestamp`; ouster: uint32 `t` (ns) */
    int32_t off_range;         /* ouster: uint32 `range`; others: unused (range = |p|, Point.cpp:166-169) */
} lv_cloud_layout;
/* the time semantics of the YAML (Common.hpp:56-107): stamp_beginning, offset_beginning, full_rotation_time.
 * header_stamp_us = pcl header stamp (microseconds).  Outputs (n entries each; intensity / range may be NULL):
 * xyz, absolute time per point (Point.cpp:37-111 + get_begin_time, PointCloudProcessor.cpp:42-88), intensity, range. */
lv_status lv_pointcloud2_to_points(lv_lidar_type type, const lv_cloud_layout* layout, const uint8_t* data, int64_t n,
                                   uint64_t header_stamp_us, int stamp_beginning, int offset_beginning,
                                   double full_rotation_time, float* xyz, double* time, float* intensity, float* range);
/* PointCloudProcessor::sort_points (PointCloudProcessor.cpp:114-123): order of the points by time (stable; the
 * reference's std::sort leaves equal stamps in unspecified order)                                          */
lv_status lv_time_sort_indices(const double* time, int64_t n, int32_t* idx_out);

/* lv_pointcloud2_to_points with the bounds pcl::fromROSMsg takes from the message: every field used lies inside point_step
 * and n points fit data_bytes (LV_ERR_ARG otherwise)                                                                    */
lv_status lv_pointcloud2_to_points_checked(lv_lidar_type type, const lv_cloud_layout* layout, const uint8_t* data, int64_t data_bytes,
                                           int64_t n, uint64_t header_stamp_us, int stamp_beginning, int offset_beginning,
                                           double full_rotation_time, float* xyz, double* time, float* intensity, float* range);

/* Accumulator::process (Accumulator.cpp:142-151) on the device: msg2points (PointCloudProcessor.cpp:24-99) ->
 * temporal_downsample (:101-112) -> sort_points (:114-123).  d_data: DEVICE copy of the message's point bytes
 * (data_bytes long, any alignment); layout / type / time flags as for lv_pointcloud2_to_points_checked.  Outputs are
 * DEVICE buffers with room for n points (d_intensity, d_range, d_idx may be NULL); *n_out = points kept.
 * Output ascending in time, ties in message order: d_xyz / d_time feed lv_compensate_device as they are.
 * d_idx = index of each output point in the message (for the caller's other fields, e.g. ring).  Synchronises (n_out).
 * Bit for bit lv_pointcloud2_to_points_checked, then the decimation rule of lv_temporal_downsample on the message index,
 * then lv_time_sort_indices on the kept times, then the gathers.  The begin time comes from the first and last point of
 * the whole message, as on the host.  LV_ERR_ARG, before any device work, for a null handle / layout / data / xyz / time /
 * n_out, n outside [0, 2^31 - 1], a layout _checked refuses, or an output range that overlaps [d_data, d_data +
 * data_bytes); LV_ERR_ARG after the device work when a kept point's time is NaN (the sort has no order for it).  A NaN
 * coordinate is no error: min_dist < |p| drops the point.  n == 0, or nothing kept: LV_OK with *n_out = 0. */
lv_status lv_process_cloud_device(lv_handle h, lv_lidar_type type, const lv_cloud_layout* layout,
                                  const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t header_stamp_us,
                                  int stamp_beginning, int offset_beginning, double full_rotation_time,
                                  int32_t downsample_rate, double min_dist,
                                  float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx,
                                  int64_t* n_out);

/* ---- Livox messages: livox_ros_driver/CustomMsg (livox_ros_driver2/CustomMsg has the same fields) -------------------------------
 * Not a PointCloud2: one uint64 time base (ns, the first point's time) per message, then packed 19-byte records
 *     uint32 offset_time (ns after timebase) | float32 x | float32 y | float32 z | uint8 reflectivity | uint8 tag | uint8 line
 * (little endian, a record at data + 19 i, any alignment; lv_bag_parse_livox finds them in a bag).  Per point:
 *   time       total = timebase + offset_time (uint64 ns), then (double)(int64)(total / 10^9) + (double)(total % 10^9) * 1e-9, the sum
 *              and the product unfused (Conversions::nanosec2Sec, Utils.cpp:25-30, with a 64-bit quotient).  Absolute, like the
 *              Hesai's: stamp_beginning, offset_beginning and full_rotation_time do not apply and the header stamp is not read.  A
 *              timebase above 2^64 - 2^32 is refused (the sum could wrap).
 *   tag        the point is dropped when (tag & tag_reject_mask) != 0: 0 keeps every point, 0x20 keeps the first and the single
 *              returns (tag bits 4-5 are the return number), 0x0F also drops what the sensor marks as noise (bits 0-3)
 *   outputs    xyz as stored, intensity = (float)reflectivity, range = the fp32 |p| (Point.cpp:166-169), idx = the index in the message
 *              (the caller reads tag and line through it). */
/* msg2points on the host: the tag-kept points, in message order, into xyz (n x 3), time, intensity, range and idx (n each; intensity,
 * range and idx may be NULL); *n_out = their count.  LV_ERR_ARG for null data / xyz / time / n_out, n outside [0, 2^31 - 1], n
 * records beyond data_bytes or the timebase limit. */
lv_status lv_livox_to_points(const uint8_t* data, int64_t data_bytes, int64_t n, uint64_t timebase_ns, uint8_t tag_reject_mask,
                             float* xyz, double* time, float* intensity, float* range, int32_t* idx, int64_t* n_out);
/* Accumulator::process on the device for a Livox message: the tag filter (msg2points) -> temporal_downsample on the RANK of the point
 * among the tag-kept points (not its message index; with mask 0 they are the same) -> sort_points (stable in time, equal times in
 * message order).  d_data: DEVICE copy of the records (data_bytes long, any alignment).  Outputs as lv_process_cloud_device: DEVICE
 * buffers with room for n points (d_intensity, d_range, d_idx may be NULL), ascending in time.  Bit for bit lv_livox_to_points, then
 * lv_temporal_downsample on its output, then lv_time_sort_indices on the kept times, then the gathers.  LV_ERR_ARG, before any device
 * work and also with a null handle, for null d_data / xyz / time / n_out, n outside [0, 2^31 - 1], n records beyond data_bytes, the
 * timebase limit, or an output range that overlaps [d_data, d_data + data_bytes).  Synchronises (n_out). */
lv_status lv_process_livox_device(lv_handle h, const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t timebase_ns,
                                  uint8_t tag_reject_mask, int32_t downsample_rate, double min_dist,
                                  float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out);

/* ---- Velodyne packets: velodyne_msgs/VelodyneScan of a VLP-16 or Puck Hi-Res (single return) --------------------------------------
 * The raw UDP packets of one rotation, as the Velodyne driver records them on /velodyne_packets; lv_bag_parse_velodyne_scan finds
 * them in a bag.  Packet k starts at packets + 1214 k (any alignment): uint32 stamp.sec | uint32 stamp.nsec | uint8[1206] data.
 * data: 12 blocks of 100 bytes, each a uint16 flag (0xEEFF), a uint16 azimuth A_b (0.01 deg) and 32 channels of (uint16 distance
 * in 2 mm, uint8 reflectivity); then the sensor's uint32 us timestamp (not read), the return mode (byte 1204: 0x37 strongest, 0x38
 * last, 0x39 dual) and the product id (not read).  All little endian.  The arithmetic follows the VLP-16 manual and the structure
 * of velodyne_pointcloud's RawData::unpack_vlp16; bit parity with that driver is not claimed.
 *   slots      message slot i: packet k = i / 384, r = i % 384, block b = r / 32, firing f = (r % 32) / 16, laser l = r % 16 (the
 *              driver's ring is a caller-side mapping of l); 384 n_packets slots, idx reports the slot
 *   points     a slot is a point when its packet's return mode is not 0x39, its block and every earlier block of the packet carry
 *              the flag 0xEEFF (the driver stops at the first bad block), and its distance is not 0
 *   azimuth    D_b = (A_{b+1} + 36000 - A_b) mod 36000 for b < 11 (from block b+1's raw bytes whatever its flag), D_11 = D_10;
 *              a = A_b + D_b (l 2.304 + f 55.296) / 110.592 in fp32, each product, sum and the quotient rounded, no contraction;
 *              q = round(a) (half away from zero) mod 36000
 *   tables     C[q] = (float)cos(q 0.01 pi / 180), S[q] = (float)sin(...) in double, rounded; per laser cv, sv, cr, sr = the
 *              floats of cos / sin of the vertical angle and the rotational correction, and the floats of dist, vo, ho
 *   xyz        fp32, each product and sum rounded, in this order:
 *                d = raw 0.002f + dist;  cosr = C[q] cr + S[q] sr;  sinr = S[q] cr - C[q] sr;  xy = d cv - vo sv
 *                X = xy sinr - ho cosr;  Y = xy cosr + ho sinr;  Z = d sv + vo cv;  (x, y, z) = (Y, -X, Z) (ROS: x forward, y left)
 *              so with zero calibration a return at range d, elevation e and azimuth A (clockwise from +x, seen from above) lies
 *              at d (cos e cos A, -cos e sin A, sin e)
 *   time       the packet stamp is the time of its first firing: total = sec 10^9 + nsec + (2b + f) 55296 + l 2304 ns (uint64),
 *              then seconds as for Livox.  nsec >= 10^9 cannot be converted.
 *   outputs    intensity = (float)reflectivity, range = the fp32 |p| (Point.cpp:166-169)
 * Out of scope: dual-return decoding, the HDL-32E / VLP-32C / HDL-64 block layouts, calibration files (a sensor's factory values go
 * in through lv_velodyne_calibration), the sensor's us timestamp and GPS time. */
typedef enum lv_velodyne_model { LV_VELODYNE_VLP16 = 0, LV_VELODYNE_PUCK_HIRES = 1 } lv_velodyne_model;
/* the fields of velodyne_pointcloud's calibration YAML, by laser id (= l) */
typedef struct lv_velodyne_calibration {
    double vert_correction[16];          /* vertical angle (rad)         */
    double rot_correction[16];           /* rotational correction (rad)  */
    double dist_correction[16];          /* distance correction (m)      */
    double vert_offset_correction[16];   /* vertical offset (m)          */
    double horiz_offset_correction[16];  /* horizontal offset (m)        */
} lv_velodyne_calibration;
/* the nominal calibration of a model: the vertical angles of its manual (VLP-16: -15, 1, -13, 3, ... 15 deg; Puck Hi-Res: -10,
 * 0.67, -8.67, 2, ... 10 deg), every other term 0.  LV_ERR_ARG for an unknown model or a null out. */
lv_status lv_velodyne_default_calibration(lv_velodyne_model model, lv_velodyne_calibration* out);
/* msg2points on the host: the points of the message, in slot order, into xyz (3 x 384 n_packets), time, intensity, range and idx
 * (384 n_packets each; intensity, range and idx may be NULL); *n_out = their count.  A dual-return packet contributes no points.
 * LV_ERR_ARG for null packets / cal / xyz / time / n_out, n_packets outside [0, (2^31 - 1) / 384], data_bytes < 1214 n_packets, a
 * non-finite calibration entry, or a packet stamp with nsec >= 10^9. */
lv_status lv_velodyne_to_points(const uint8_t* packets, int64_t data_bytes, int64_t n_packets, const lv_velodyne_calibration* cal,
                                float* xyz, double* time, float* intensity, float* range, int32_t* idx, int64_t* n_out);
/* Accumulator::process on the device for a VelodyneScan: msg2points -> temporal_downsample on the RANK of the point among the
 * msg2points points (not its slot) -> sort_points (stable in time, equal times in slot order).  d_packets: DEVICE copy of the
 * packets (data_bytes long, any alignment).  Outputs as lv_process_livox_device, DEVICE buffers with room for 384 n_packets points.
 * Bit for bit lv_velodyne_to_points, then lv_temporal_downsample on its output, then lv_time_sort_indices on the kept times, then
 * the gathers.  The first call on a handle uploads the 2 x 36000-float rotation tables (and waits for that copy); lv_destroy frees
 * them.  LV_ERR_ARG, before any device work and also with a null handle, for the host decoder's argument errors except the stamp,
 * or an output range that overlaps [d_packets, d_packets + data_bytes).  LV_ERR_ARG after the device work when a packet is a
 * dual-return one or its stamp has nsec >= 10^9 (the other packets' points are written, *n_out stays 0).  When 384 n_packets <
 * downsample_rate nothing can be kept and the packets are not read.  Synchronises (n_out). */
lv_status lv_process_velodyne_device(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                     const lv_velodyne_calibration* cal, int32_t downsample_rate, double min_dist,
                                     float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out);

/* ---- Ouster packets: ouster_ros/PacketMsg of an OS0 / OS1 / OS2 -----------------------------------------------------------------
 * The raw UDP packets the Ouster driver records on .../lidar_packets (one packet per message) and .../imu_packets, with the
 * sensor's metadata JSON; lv_bag_parse_ouster_packet finds a packet in a bag, lv_ouster_sensor_from_json reads the metadata and
 * its lidar UDP profile.  A packet holds 16 columns; packet k starts at packets + k B (B = the profile's packet bytes), at any
 * alignment.  All little endian.  H = pixels_per_column.
 *   LEGACY (firmware 1.x, and 2.x by default): B = 16 (20 + 12 H) (12 608 bytes for H = 64).  Column: uint64 timestamp (ns) |
 *              uint16 measurement_id m | uint16 frame_id | uint32 encoder count (not read) | H pixels of 12 bytes | uint32 status.
 *              Pixel: uint32 range word (r = its low 20 bits, mm) | uint16 reflectivity | signal and noise (not read).
 *   the profiles of firmware 2.2+ (RNG19_RFL8_SIG16_NIR16 is the default of firmware 3.x): B = 64 + 16 (12 + s H): a 32-byte
 *              packet header (not read) | 16 columns | a 32-byte packet footer (not read, so its CRC64 is not checked).  Column:
 *              uint64 timestamp (ns) | uint16 measurement_id m | uint16 status | H pixels of s bytes.  Pixel, by profile:
 *                profile                        s    r (mm)                      reflectivity   B for H = 64
 *                RNG19_RFL8_SIG16_NIR16         12   u32 @0 & 0x7FFFF            u8 @4          12 544
 *                RNG19_RFL8_SIG16_NIR16_DUAL    16   u32 @0 & 0x7FFFF (first)    u8 @3 (first)  16 640
 *                RNG15_RFL8_NIR8 (low data)     4    (u16 @0 & 0x7FFF) << 3      u8 @2          4 352
 *              The bits above each range mask (flags) are ignored.  Dual return gives the first return's points only: those of
 *              os_cloud_node's `points` topic; the second return is not read.  Low data gives ranges on an 8 mm grid.
 * These layouts follow the Ouster firmware manual's packet tables and the field table of ouster_client's packet_format; nobody
 * has checked the non-LEGACY ones against a recording from a real sensor.  The geometry is that of the Ouster driver's
 * make_xyz_lut in the LiDAR frame (os_lidar); bit parity with ouster_ros is not claimed.  Every profile decodes by the same rules:
 *   slots      message slot i = k 16 H + c H + p (packet k, column c, pixel p); idx reports the slot (the ring is i % H);
 *              16 H n_packets slots, and n_packets <= (2^31 - 1) / (16 H) (slot indices are int32)
 *   points     a slot is a point when bit 0 of its column's status is set (for LEGACY 0xFFFFFFFF is valid, 0 is not), m < W and
 *              r != 0
 *   tables     one column table for every W: C[q] = (float)cos(2 pi q / 2048), S[q] = (float)sin(...) for q in [0, 2048), in
 *              double, rounded; column m reads q = m (2048 / W).  Per beam p: ce, se, ca, sa = the floats of cos / sin of
 *              beam_altitude_angles[p] and beam_azimuth_angles[p] (degrees, times pi / 180 in double); nf = (float)(n 0.001)
 *   xyz        fp32, each product and sum rounded, no contraction, in this order:
 *                e = (float)r 0.001f - nf;  ch = C ca - S sa;  sh = S ca + C sa;  ee = e ce
 *                x = ee ch + nf C;  y = -(ee sh + nf S);  z = e se
 *              so with zero angles and n = 0 column m looks at the angle 2 pi m / W clockwise from +x, seen from above.  This is
 *              the frame the extrinsic of config/ouster.yaml describes; lidar_to_sensor_transform (os_sensor) is not applied
 *   time       the column's timestamp, in seconds as for Livox: absolute, so stamp_beginning, offset_beginning and
 *              full_rotation_time do not apply.  The conversion cannot fail
 *   outputs    intensity = (float)reflectivity, range = (float)r in mm: the range field os_cloud_node writes, which the Ouster
 *              PointCloud2 path passes through (lv_cloud_layout.off_range), so both Ouster paths give the buffer the same lanes
 * Out of scope: the second return of the dual profile, the FUSA profiles, the packet CRC, the packet header's init_id / serial
 * number checked against the metadata, columns_per_packet != 16, lidar_to_sensor_transform, signal and NIR, the driver's frame-id
 * dedup of late packets. */
typedef enum lv_ouster_profile {
    LV_OUSTER_LEGACY = 0,
    LV_OUSTER_RNG19_RFL8_SIG16_NIR16 = 1,
    LV_OUSTER_RNG19_RFL8_SIG16_NIR16_DUAL = 2,
    LV_OUSTER_RNG15_RFL8_NIR8 = 3
} lv_ouster_profile;
typedef struct lv_ouster_calibration {
    int32_t columns_per_frame;           /* W: 512, 1024 or 2048 (lidar_mode "1024x10" -> 1024)     */
    int32_t pixels_per_column;           /* H: 16, 32, 64 or 128                                     */
    double beam_altitude_angles[128];    /* degrees, the first H are read                           */
    double beam_azimuth_angles[128];     /* degrees, the first H are read                           */
    double lidar_origin_to_beam_origin_mm;   /* n; 0 for firmware that does not report it          */
} lv_ouster_calibration;
/* the sensor metadata JSON (len bytes of text, no terminator needed) -> *out and *profile.  A narrow reader, not a JSON library: the
 * keys are found at any depth (firmware 1.x puts them at the top level, 2.x nests them under beam_intrinsics, config_params and
 * lidar_data_format), the first occurrence counts.  Required: beam_altitude_angles and beam_azimuth_angles (arrays of equal
 * length H, finite numbers) and lidar_mode ("<W>x<rate>").  Optional: lidar_origin_to_beam_origin_mm (0 when absent) and
 * udp_profile_lidar ("LEGACY", "RNG19_RFL8_SIG16_NIR16", "RNG19_RFL8_SIG16_NIR16_DUAL" or "RNG15_RFL8_NIR8"; LEGACY when absent,
 * as on firmware 1.x).  Checked when present: pixels_per_column == H, columns_per_packet == 16.  LV_ERR_ARG for a null argument,
 * len < 0, a missing or malformed required key, W or H outside its set, any other profile (the FUSA ones, a misspelt name), or a
 * check that fails (*out and *profile are then zeroed).  Host code. */
lv_status lv_ouster_sensor_from_json(const char* text, int64_t len, lv_ouster_calibration* out, lv_ouster_profile* profile);
/* lv_ouster_sensor_from_json for LEGACY sensors: a profile other than LEGACY is LV_ERR_ARG, with *out zeroed. */
lv_status lv_ouster_calibration_from_json(const char* text, int64_t len, lv_ouster_calibration* out);
/* msg2points on the host: the points of the packets, in slot order, into xyz (3 x 16 H n_packets), time, intensity, range and idx
 * (16 H n_packets each; intensity, range and idx may be NULL); *n_out = their count.  LV_ERR_ARG for null packets / cal / xyz /
 * time / n_out, a profile outside lv_ouster_profile, W or H outside its set, a non-finite calibration entry (the first H angles,
 * n), n_packets outside [0, (2^31 - 1) / (16 H)] or data_bytes below n_packets packets of the profile. */
lv_status lv_ouster_packets_to_points(const uint8_t* packets, int64_t data_bytes, int64_t n_packets, const lv_ouster_calibration* cal,
                                      lv_ouster_profile profile, float* xyz, double* time, float* intensity, float* range, int32_t* idx,
                                      int64_t* n_out);
/* lv_ouster_packets_to_points with LV_OUSTER_LEGACY */
lv_status lv_ouster_to_points(const uint8_t* packets, int64_t data_bytes, int64_t n_packets, const lv_ouster_calibration* cal,
                              float* xyz, double* time, float* intensity, float* range, int32_t* idx, int64_t* n_out);
/* Accumulator::process on the device for Ouster packets of the given profile: msg2points -> temporal_downsample on the RANK of the
 * point among the msg2points points (not its slot) -> sort_points (stable in time, equal times in slot order, so within a column the
 * points stay in pixel order).  d_packets: DEVICE copy of the packets (data_bytes long, any alignment), e.g. the packets of one frame
 * batched into one upload.  Outputs as lv_process_livox_device, DEVICE buffers with room for 16 H n_packets points.  Bit for bit
 * lv_ouster_packets_to_points, then lv_temporal_downsample on its output, then lv_time_sort_indices on the kept times, then the
 * gathers.  The first call on a handle uploads the 2 x 2048-float column table (and waits for that copy); lv_destroy frees it.
 * LV_ERR_ARG, before any device work and also with a null handle, for the host decoder's argument errors or an output range that
 * overlaps [d_packets, d_packets + data_bytes).  When 16 H n_packets < downsample_rate nothing can be kept and the packets are not
 * read.  Synchronises (n_out). */
lv_status lv_process_ouster_packets_device(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                           const lv_ouster_calibration* cal, lv_ouster_profile profile, int32_t downsample_rate,
                                           double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                           int32_t* d_idx, int64_t* n_out);
/* lv_process_ouster_packets_device with LV_OUSTER_LEGACY */
lv_status lv_process_ouster_device(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                   const lv_ouster_calibration* cal, int32_t downsample_rate, double min_dist,
                                   float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out);

/* ---- the tick without a host wait (main.cpp:76-105)------------------------------------------------------------------------
 * Stream-ordered forms of the tick's device calls.  Each takes its input count from DEVICE memory (d_n, an int64_t) and writes
 * its output count to device memory (d_n_out), so that one stage hands its count to the next without the host: none of them
 * synchronises.  n_max is a host-known upper bound of the count (the message's n, or max_points) in [1, min(max_points,
 * 2^31 - 1)]: it sizes the grids and the sorts, which run over n_max slots with padding keys that sort last.  A device count
 * outside [0, n_max] is clamped to it and flagged.  Errors found on the device are not returned: they are recorded and
 * reported (and cleared) by lv_async_status, which names the stage.  Argument errors are LV_ERR_ARG before any device work.
 * Each call's results equal those of its synchronous form bit for bit (counts, values, order). */
/* Accumulator::process (Accumulator.cpp:142-151) as lv_process_cloud_device; *d_n_out = points kept.  A kept point whose time
 * is NaN is a deferred error.  The output buffers have room for n points. */
lv_status lv_process_cloud_device_async(lv_handle h, lv_lidar_type type, const lv_cloud_layout* layout,
                                        const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t header_stamp_us,
                                        int stamp_beginning, int offset_beginning, double full_rotation_time,
                                        int32_t downsample_rate, double min_dist,
                                        float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx,
                                        int64_t* d_n_out);
/* lv_process_livox_device with *d_n_out = points kept; feeds lv_lidar_push_full_device_async (d_intensity, d_range) or
 * lv_lidar_push_device_async directly.  The output buffers have room for n points. */
lv_status lv_process_livox_device_async(lv_handle h, const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t timebase_ns,
                                        uint8_t tag_reject_mask, int32_t downsample_rate, double min_dist,
                                        float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx,
                                        int64_t* d_n_out);
/* lv_process_velodyne_device with *d_n_out = points kept; feeds lv_lidar_push_full_device_async or lv_lidar_merge_device_async
 * directly.  The output buffers have room for 384 n_packets points.  A dual-return packet or a stamp with nsec >= 10^9 is a deferred
 * error (the other packets' points are kept). */
lv_status lv_process_velodyne_device_async(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                           const lv_velodyne_calibration* cal, int32_t downsample_rate, double min_dist,
                                           float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx,
                                           int64_t* d_n_out);
/* lv_process_ouster_packets_device with *d_n_out = points kept; feeds lv_lidar_push_full_device_async or
 * lv_lidar_merge_device_async directly.  The output buffers have room for 16 H n_packets points.  No deferred error of its own. */
lv_status lv_process_ouster_packets_device_async(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                                 const lv_ouster_calibration* cal, lv_ouster_profile profile, int32_t downsample_rate,
                                                 double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                                 int32_t* d_idx, int64_t* d_n_out);
/* lv_process_ouster_packets_device_async with LV_OUSTER_LEGACY */
lv_status lv_process_ouster_device_async(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                         const lv_ouster_calibration* cal, int32_t downsample_rate, double min_dist,
                                         float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx,
                                         int64_t* d_n_out);
/* Compensator::compensate (Compensator.cpp:123-146) as lv_compensate_device over *d_n points.  The path and Xt2 stay host-built
 * (Compensator::upsample / get_t2); they are staged through pinned memory, so the host buffers may be reused on return.  A
 * timestamp outside the path (or out of order) is a deferred error.  d_xyz_out may equal d_xyz; other overlaps of the
 * n_max-point ranges of d_xyz, d_t and d_xyz_out are refused. */
lv_status lv_compensate_device_async(lv_handle h, const lv_state32* path, int32_t ns, const lv_state32* Xt2, const float* d_xyz,
                                     const double* d_t, const int64_t* d_n, int64_t n_max, float* d_xyz_out);
/* Compensator::downsample -> voxelgrid_downsample (Compensator.cpp:115-118,148-163) as lv_voxelgrid_downsample_device over *d_n
 * points; *d_n_out = leaves.  PCL's cell-index overflow pass-through (d_xyz_out = the input, *d_n_out = *d_n) is decided on the
 * device.  The n_max-point ranges of d_xyz and d_xyz_out must not overlap. */
lv_status lv_voxelgrid_downsample_device_async(lv_handle h, const float* d_xyz, const int64_t* d_n, int64_t n_max,
                                               float downsample_prec, float* d_xyz_out, int64_t* d_n_out);
/* Compensator::voxelgrid_downsample (Compensator.cpp:148-163) of full points, as the reference runs it on full_info::Points
 * (Processor::fill -> pcl::VoxelGrid<full_info::Point> -> Point(const full_info::Point&), Point.cpp:21-25,164-168): per leaf the xyz
 * centroid of lv_voxelgrid_downsample_device_async (bit for bit the same), intensity = the fp32 sum of the leaf's intensities in the
 * same order divided by the count (CentroidPoint's AccumulatorIntensity), range = the fp32 norm of the centroid, time = 0 (no
 * accumulator carries timestamp).  On a cell-index overflow PCL hands the input on: xyz, time and intensity are passed through,
 * and range is the fp32 norm of each passed point, because Compensator.cpp:161 builds every output point with Point(p), whose
 * set_attributes sets range = |p| (Point.cpp:166-169).  So range is always the norm of the output xyz, and no input range is
 * taken.  The three inputs are required (time is read by the pass-through only); d_time_out, d_intensity_out and d_range_out may
 * each be NULL.  No output range may overlap an input range or another output range (n_max points each, 8 bytes for a count). */
lv_status lv_voxelgrid_downsample_full_device_async(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity,
                                                    const int64_t* d_n, int64_t n_max, float downsample_prec, float* d_xyz_out,
                                                    double* d_time_out, float* d_intensity_out, float* d_range_out, int64_t* d_n_out);
/* main.cpp:81-88: `if (ds_compensated.size() < MAX_POINTS2MATCH) break; localizator.correct(ds_compensated, t2)` on *d_n points of
 * d_xyz (device, LiDAR frame).  Below max(min_points, 1) points the update does not run: state, P and last_time_updated are left
 * as they are and the status lv_last_logs fetches is LV_TOO_FEW_POINTS.  On a map the host knows to be empty it returns
 * LV_EMPTY_MAP at once, like lv_correct_device; after an asynchronous first build (which the gate may have left empty) the device
 * checks the map's point count and records LV_EMPTY_MAP the same way (Localizator.cpp:24).  last_time_updated becomes `time` when
 * the update runs, resolved by the next call that fetches the results (lv_last_logs, lv_get_state, ...).  The sweep and its
 * device count are recorded for lv_map_add_last_sweep, which then adds *d_n points, or none when the gate stopped the tick
 * (main.cpp:81 breaks before map.add), the first tick's build included; its growth bound (lv_map_set_growth) uses n_max. */
lv_status lv_correct_device_async(lv_handle h, const float* d_xyz, const int64_t* d_n, int64_t n_max, int64_t min_points,
                                  double time);
/* ---- the tick's output and mapping step (main.cpp:88-117) without a host wait.  Stream-ordered like the calls above: counts in
 * device memory, n_max in [1, min(max_points, 2^31 - 1)], argument errors LV_ERR_ARG before any device work (a null handle too),
 * deferred errors through lv_async_status.  Whether to publish, map online or map offline (mapping_online, high_quality_publish,
 * Mapper::hasToMap with full_rotation_time) stays with the caller, as does the time management. */
/* `Xt2 * Xt2.I_Rt_L() * points` (main.cpp:91-93, 111; State.cpp:79-89) in fp32 with the filter state on the device: the state the
 * preceding update left, or the propagated state when there was none (an empty map, Localizator.cpp:24).  The same arithmetic and
 * the same kernel as lv_map_add_last_sweep's transform and Mapper::match's.  *d_n points (clamped to [0, n_max]) of d_xyz_lidar
 * (n_max x 3) go to d_xyz_world; *d_n_out = their count, or 0 when the preceding lv_correct_device_async's gate stopped the tick
 * (main.cpp:81 breaks before publishing), the rule lv_map_add_last_sweep follows.  d_xyz_world may equal d_xyz_lidar and d_n_out
 * may equal d_n; other overlaps of the outputs with the inputs are refused.  Two launches. */
lv_status lv_sweep_to_world_device_async(lv_handle h, const float* d_xyz_lidar, const int64_t* d_n, int64_t n_max, float* d_xyz_world,
                                         int64_t* d_n_out);
/* Mapper::add (Mapper.cpp:22-30) of *d_n points (clamped to [0, n_max]) of d_xyz (device, world frame): nothing when the count is
 * 0; a map without points is built without downsampling, else Add_Points with the 0.2 m rule when downsample != 0.  No gate of its
 * own.  Content, point ids, order and lv_map_info counters equal those of lv_map_add_device with the count on the host; the growth
 * bound (lv_map_set_growth) uses n_max. */
lv_status lv_map_add_device_async(lv_handle h, const float* d_xyz, const int64_t* d_n, int64_t n_max, int downsample);
/* Publishers::pointcloud's header stamp (Publishers.hpp:51-60 -> Processor::fill, PointCloudProcessor.cpp:125-133): starting from 0,
 * the maximum over the *d_n (clamped to [0, n_max]) times of d_time of Conversions::sec2Microsec(t) = std::round(t * 1e6) as uint64
 * (Utils.cpp:14-16: the product in double, rounded half away from zero), written to *d_stamp_us; 0 for a count of 0.  Specified
 * for finite, non-negative times below 2^64 us only (the reference's conversion is undefined elsewhere).  The downsampled clouds'
 * times are all 0 (lv_voxelgrid_downsample_full), so their stamp is 0, as in the reference; where the voxel grid passed its input
 * through (cell-index overflow) the times are the input's and the stamp is their maximum.  One launch of one block. */
lv_status lv_cloud_stamp_device_async(lv_handle h, const double* d_time, const int64_t* d_n, int64_t n_max, uint64_t* d_stamp_us);
/* the deferred errors of the _async calls since the last lv_async_status, and the map's capacity flags (as lv_map_status):
 * LV_ERR_ARG (lv_last_error names the stage), LV_ERR_CAPACITY or LV_OK.  Clears them; the handle stays usable.  Synchronises. */
lv_status lv_async_status(lv_handle h);

/* ---- the LiDAR buffer in HBM (Accumulator::BUFFER_L, include/Headers/Accumulator.hpp:3) ------------------------------------------
 * main.cpp:61-79 localizes on a time window [t1, t2] that is usually much shorter than a message: Compensator::compensate(t1, t2)
 * takes its points from the Accumulator's LiDAR buffer (Compensator.cpp:23 -> Accumulator::get_points -> get, Accumulator.hpp:61-74),
 * which receive_lidar fills one processed message at a time (Accumulator.cpp:39-48) and clear_lidar empties from its old end
 * (main.cpp:122, Buffer.cpp:66-70).  These calls keep that buffer on the device: a message goes lv_process_cloud_device_async ->
 * scratch -> lv_lidar_push_device_async, a tick's window comes out of lv_lidar_get_points_device_async into the buffers that
 * lv_compensate_device_async reads, and nothing about the buffer's fill state is known on the host.  Time management (t2, the
 * delta schedule, the field-of-view check) stays with the caller.
 * The results are the reference's bit for bit, quirks included: the buffer is in arrival order (a late or overlapping message
 * leaves it unsorted, and get still runs its binary search with the reference's probe sequence), and of m points whose time
 * equals t2 exactly only min(m, 2) are returned (the walk starts one before the last of them; t1 is inclusive, so the next
 * window picks up the rest).  Point times that are NaN follow the reference's comparisons.  The buffer holds xyz (float) and
 * time (double) per point: 20 bytes.  All calls are stream-ordered on the handle's stream.  Argument errors are LV_ERR_ARG
 * before any device work, also with a null handle: null pointers, n_max outside [1, 2^31 - 1], a NaN time argument, a push, get
 * or clear before lv_lidar_reserve, and ranges that overlap each other or the buffer.  lv_destroy releases the buffer. */
/* sizes the buffer for `capacity` points (1 .. 2^30; the deque has no bound, so size it for empty_lidar_time of data plus the
 * messages a tick may leave behind); the live points stay, in order.  LV_ERR_CAPACITY when more points are live than fit.
 * Synchronises. */
lv_status lv_lidar_reserve(lv_handle h, int64_t capacity);
/* BUFFER_L holds whole Points (Accumulator.hpp:3,61-74): lv_lidar_reserve with two more float lanes per point, intensity and range
 * (28 bytes per point), which lv_lidar_push_full_device_async fills and lv_lidar_get_points_full_device_async returns.  Live points
 * keep their lanes across any later reserve (lv_lidar_reserve keeps the lanes of a ring that has them); points that arrived before
 * the ring had lanes get intensity 0 and range 0, as does every point of a plain lv_lidar_push_device_async onto a ring with lanes.
 * Synchronises. */
lv_status lv_lidar_reserve_full(lv_handle h, int64_t capacity);
/* Accumulator::receive_lidar's `for (Point p : points) this->add(p);` (Accumulator.cpp:47): appends the *d_n points (clamped to
 * [0, n_max]) of d_xyz (n x 3) / d_time in that order, the last one becoming content[0].  Points that do not fit are a deferred
 * error (lv_async_status) and leave the buffer unchanged: nothing is dropped silently. */
lv_status lv_lidar_push_device_async(lv_handle h, const float* d_xyz, const double* d_time, const int64_t* d_n, int64_t n_max);
/* the same with the points' intensity and range (n_max each), e.g. lv_process_cloud_device_async's d_intensity / d_range
 * (Point.cpp:164-173: the message's intensity, Ouster reflectivity or Hesai uint8; the Ouster's range field, |p| otherwise).  LV_ERR_ARG
 * on a ring without lanes (lv_lidar_reserve_full first). */
lv_status lv_lidar_push_full_device_async(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity, const float* d_range,
                                          const int64_t* d_n, int64_t n_max);
/* Accumulator::get_points(t1, t2) (Accumulator.cpp:93-95, Accumulator.hpp:61-74): the points of the window, oldest inserted first,
 * into d_xyz (n_max x 3) / d_time (n_max); *d_n_out = their count.  A window of more than n_max points writes count 0 and is a
 * deferred error: the tick that follows is gated off (LV_TOO_FEW_POINTS) and lv_async_status names the stage. */
lv_status lv_lidar_get_points_device_async(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, int64_t n_max,
                                           int64_t* d_n_out);
/* the same window (the same binary search, ties at t2, order and count) with its intensity and range into d_intensity / d_range
 * (n_max each).  Deskew keeps the attributes and the order (RotTransl.cpp:43-48), so these lanes stay aligned with
 * lv_compensate_device_async's output and lv_sweep_to_world_device_async's.  LV_ERR_ARG on a ring without lanes. */
lv_status lv_lidar_get_points_full_device_async(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, float* d_intensity,
                                                float* d_range, int64_t n_max, int64_t* d_n_out);
/* the same kernels, then the count read back into *n_out (host); a window above n_max returns LV_ERR_CAPACITY with *n_out = 0
 * and lv_last_error() naming its size.  Synchronises. */
lv_status lv_lidar_get_points_device(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, int64_t n_max, int64_t* n_out);
/* Accumulator::clear_lidar(t) (Accumulator.cpp:68-70, Buffer.cpp:66-70): drops the oldest points while t >= their time, stopping
 * at the first one, in insertion order, that is newer than t */
lv_status lv_lidar_clear_async(lv_handle h, double t);
struct lv_lidar_info {
    int64_t points;            /* live points: content.size()                                   */
    int64_t capacity;          /* lv_lidar_reserve's capacity (0: not reserved)                  */
    double oldest_time;        /* content.back().time  (NaN when empty)                          */
    double newest_time;        /* content.front().time (NaN when empty)                          */
};
/* the buffer's fill state; synchronises */
lv_status lv_lidar_info(lv_handle h, struct lv_lidar_info* out);

/* ---- several LiDARs into one buffer: the time-ordered merge ----------------------------------------------------------------------
 * The push keeps arrival order, so messages of two sensors whose time spans overlap leave the buffer unsorted, and get's binary
 * search then answers from whichever points it probes.  The merge puts each message where its times belong instead, after moving
 * its points into the primary LiDAR's frame (the frame I_Rotation_L / I_Translation_L describe).  Let L be the live points, oldest
 * first, and B the message (time-sorted, as the message front end leaves it).  The split s is one past the newest live point whose
 * time is <= B[0].time, and T_tail the live points after it.  When T_tail and B are each non-decreasing in time with no NaN, the
 * points from s on become std::merge(T_tail, B) by time, buffered points first on equal times, and the points before s do not move.
 * A message that starts no earlier than the newest live point is exactly the push: the same slots, bits and counters.  Otherwise
 * (a NaN time, a batch that is not sorted, or T_tail left unsorted by an earlier push) the message is appended as the push does,
 * and lv_async_status reports that the buffer is no longer time-ordered.  An empty message changes nothing.
 * Each point is written as rt_apply(T, p) (RotTransl * Point in fp32, unfused); T = NULL writes the points bit for bit unchanged.
 * Intensity and range move with their points; range stays the sensor-frame value the front end computed (|p| in the sensor's
 * frame, or the Ouster's range field).  Deferred errors, each leaving the buffer unchanged: T_tail larger than the merge reserve,
 * and points that do not fit the capacity.  Three launches per call whatever the overlap; no host wait.
 * Argument errors are LV_ERR_ARG before any device work, also with a null handle: null pointers, n_max outside [1, 2^31 - 1], a
 * non-finite entry of T, input ranges that overlap each other or the buffer, a merge before lv_lidar_reserve and
 * lv_lidar_reserve_merge, and a _full merge on a buffer without lanes. */
/* room for `overlap_points` (1 .. 2^30) buffered points that one merge may move (T_tail); the scratch has lanes when the buffer has
 * them, and gains them when lv_lidar_reserve_full adds them.  LV_ERR_CAPACITY when the allocation fails (merges are refused until a
 * reserve succeeds).  Synchronises. */
lv_status lv_lidar_reserve_merge(lv_handle h, int64_t overlap_points);
/* merge the *d_n points (clamped to [0, n_max]) of d_xyz (n x 3) / d_time; T: 12 host floats, R row-major then t, mapping the
 * sensor's frame into the primary LiDAR's frame (L0_T_Lk), or NULL.  On a buffer with lanes the points get intensity 0 and range 0,
 * as with the push. */
lv_status lv_lidar_merge_device_async(lv_handle h, const float* d_xyz, const double* d_time, const int64_t* d_n, int64_t n_max,
                                      const float* T);
/* the same with the points' intensity and range (n_max each); a buffer reserved with lv_lidar_reserve_full */
lv_status lv_lidar_merge_full_device_async(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity, const float* d_range,
                                           const int64_t* d_n, int64_t n_max, const float* T);

/* ---- rosbag reader (format 2.0; replaces roscpp / `rosbag play` in front of Accumulator::receive_lidar / receive_imu,
 * src/main.cpp:27-39, src/Modules/Accumulator.cpp:39-60).  Sequential read of uncompressed bags (bz2 / lz4 chunks are
 * refused with LV_ERR_IO: `rosbag decompress` first).  Host code.                                                       */
typedef struct lv_bag lv_bag;
typedef struct lv_bag_message {
    int32_t conn;              /* connection id                                                   */
    const char* topic;         /* e.g. "/velodyne_points"; valid while the bag is open            */
    const char* type;          /* e.g. "sensor_msgs/PointCloud2"                                  */
    uint32_t sec, nsec;        /* receive time of the record                                      */
    const uint8_t* data;       /* the serialised message (points into the bag's buffer)           */
    int64_t size;
} lv_bag_message;
lv_status lv_bag_open(const char* path, lv_bag** out);
void lv_bag_close(lv_bag* bag);
void lv_bag_rewind(lv_bag* bag);
int32_t lv_bag_connection_count(const lv_bag* bag);
/* next message in file order: 1 = *msg filled, 0 = end of the bag, -1 = malformed */
int lv_bag_next(lv_bag* bag, lv_bag_message* msg);
/* sensor_msgs/PointCloud2 -> a view of the point bytes + the offsets of the fields `type`'s point struct uses
 * (include/Headers/Common.hpp:109-221), ready for lv_pointcloud2_to_points_checked                                      */
typedef struct lv_pointcloud2_view {
    uint32_t stamp_sec, stamp_nsec;      /* header.stamp                                          */
    uint32_t height, width, point_step, row_step;
    int32_t is_bigendian, is_dense;
    int64_t n_points;                    /* height x width                                        */
    const uint8_t* data;
    int64_t data_bytes;
    lv_cloud_layout layout;
} lv_pointcloud2_view;
lv_status lv_bag_parse_pointcloud2(const uint8_t* msg, int64_t size, lv_lidar_type type, lv_pointcloud2_view* out);
/* sensor_msgs/Imu (what Accumulator::receive_imu reads: IMU.cpp:18-40) */
typedef struct lv_imu_sample {
    uint32_t stamp_sec, stamp_nsec;
    double orientation[4];               /* x y z w                                                */
    double angular_velocity[3];
    double linear_acceleration[3];
} lv_imu_sample;
lv_status lv_bag_parse_imu(const uint8_t* msg, int64_t size, lv_imu_sample* out);
/* livox_ros_driver(2)/CustomMsg -> a view of the 19-byte records, ready for lv_livox_to_points / lv_process_livox_device
 * (data, data_bytes, n_points, timebase).  LV_ERR_ARG for a null argument, a truncated message, bytes after the records, or a
 * point_num that differs from the record count (the driver always writes them equal). */
typedef struct lv_livox_view {
    uint32_t stamp_sec, stamp_nsec;      /* header.stamp                                          */
    uint64_t timebase;                   /* ns: the time of the first point                       */
    uint32_t point_num;
    uint8_t lidar_id;
    int64_t n_points;                    /* records in `points`                                   */
    const uint8_t* data;                 /* the first record (any alignment)                      */
    int64_t data_bytes;                  /* 19 x n_points                                         */
} lv_livox_view;
lv_status lv_bag_parse_livox(const uint8_t* msg, int64_t size, lv_livox_view* out);
/* velodyne_msgs/VelodyneScan -> a view of its packets, ready for lv_velodyne_to_points / lv_process_velodyne_device (packets,
 * data_bytes, n_packets).  LV_ERR_ARG for a null argument, a truncated message or bytes after the packets. */
typedef struct lv_velodyne_view {
    uint32_t stamp_sec, stamp_nsec;      /* header.stamp                                          */
    int64_t n_packets;
    const uint8_t* packets;              /* the first packet's stamp (any alignment)              */
    int64_t data_bytes;                  /* 1214 x n_packets                                      */
} lv_velodyne_view;
lv_status lv_bag_parse_velodyne_scan(const uint8_t* msg, int64_t size, lv_velodyne_view* out);
/* ouster_ros/PacketMsg (uint8[] buf: a uint32 length, then the bytes) -> a view of its one packet: a LiDAR packet for
 * lv_ouster_packets_to_points / lv_process_ouster_packets_device, or an IMU packet for lv_ouster_imu_packet.  LV_ERR_ARG for a
 * null argument, a
 * truncated message or bytes after the packet. */
typedef struct lv_ouster_packet_view {
    const uint8_t* data;                 /* the packet's first byte (any alignment)               */
    int64_t bytes;
} lv_ouster_packet_view;
lv_status lv_bag_parse_ouster_packet(const uint8_t* msg, int64_t size, lv_ouster_packet_view* out);
/* an Ouster IMU packet (48 bytes, little endian: uint64 sys ts | uint64 accel ts | uint64 gyro ts (ns) | float32 accel xyz (g) |
 * float32 gyro xyz (deg/s)) -> the sample Accumulator::receive_imu reads: stamp = the gyro ts split into sec / nsec,
 * linear_acceleration = (double)a 9.80665, angular_velocity = ((double)w pi) / 180, orientation = {0, 0, 0, 0} (IMU::has_orientation
 * reads that as no orientation).  The stamp is in the sensor's clock, the clock of the LiDAR packets' column times.  LV_ERR_ARG for
 * a null argument, bytes != 48 or a gyro ts whose seconds exceed 2^32 - 1. */
lv_status lv_ouster_imu_packet(const uint8_t* pkt, int64_t bytes, lv_imu_sample* out);

/* ---- PCD map files (the map format of PCL, pcl::io::savePCDFileBinary, and of most LiDAR SLAM tools).  Host code.
 * Saving the device map: lv_map_points -> lv_pcd_write.  Loading it: lv_pcd_read -> lv_map_build (KD_TREE::Build: file order
 * becomes insertion order and point ids).  INTEGRATION.md B7. */
/* PCD v0.7, DATA binary, FIELDS x y z, SIZE 4 4 4, TYPE F F F, COUNT 1 1 1, WIDTH n, HEIGHT 1, VIEWPOINT 0 0 0 1 0 0 0,
 * POINTS n; the floats as they are (bit for bit).  LV_ERR_IO for a failed open, a short write or a failed close;
 * LV_ERR_ARG for a null path, null xyz with n > 0, or n < 0. */
lv_status lv_pcd_write(const char* path, const float* xyz, int64_t n);
/* DATA ascii or binary (VERSION 0.7 or .7, '#' comment lines; no COUNT line means counts of 1).  x, y and z must each be
 * TYPE F, SIZE 4, COUNT 1; every other field (SIZE 1, 2, 4 or 8, any COUNT, '_' padding) is skipped by its bytes.  Points
 * with a non-finite coordinate are dropped, file order is kept; *n = points kept.  xyz == NULL: only *n is set.
 * LV_ERR_CAPACITY when cap < *n (nothing is written).  LV_ERR_IO, lv_last_error naming it, for an unreadable file,
 * DATA binary_compressed (convert it with pcl_convert_pcd_ascii_binary), a missing or ill-typed coordinate field,
 * POINTS != WIDTH x HEIGHT, a data section shorter than POINTS records, or another malformed header. */
lv_status lv_pcd_read(const char* path, float* xyz, int64_t cap, int64_t* n);

#ifdef __cplusplus
}
#endif
#endif /* LIMOVELO_B200_H_ */
