/*
 * lv_internal.h — launcher declarations shared by the translation units of liblimovelo_b200.so.
 */
#ifndef LV_INTERNAL_H_
#define LV_INTERNAL_H_

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/limovelo_b200.h"
#include "lv_buffers.h"
#include "lv_ieskf.h"
#include "lv_preloc_bound.h"
#include "lv_voxel_search.h"
#include "lv_wire.h"

namespace lv {

/* SMs of one H100 SXM: fixed grids that stride over device-side work are sized in multiples of it */
enum { kNumSMs = 132 };

/* The stream-ordered (_async) entry points report errors through one device word of the handle, read and cleared by
 * lv_async_status.  Bits: */
enum : uint32_t { kAsyncCloudNaN = 1u, kAsyncDeskewPath = 2u, kAsyncCount = 4u, kAsyncLidarFull = 8u, kAsyncLidarWindow = 16u,
                  kAsyncLidarUnsorted = 32u, kAsyncLidarOverlap = 64u, kAsyncVelodyne = 128u };
/* device words of the async tick: the deferred errors and what lv_correct_device_async decided */
struct AsyncWords {
    uint32_t err;              /* kAsync* bits since the last lv_async_status              */
    int32_t time_set;          /* 1: an async update ran since the last fetch; time_updated is its time */
    double time_updated;
    uint32_t world_n;          /* the count lv_sweep_to_world_device_async's transform reads */
    uint32_t pad;
};
#ifdef __CUDACC__
/* a count in device memory (NULL: the host-known n_max) clamped to [0, n_max]; one thread flags a count outside it */
__device__ __forceinline__ int64_t device_count(const int64_t* d_n, int64_t n_max, uint32_t* err) {
    if (!d_n) return n_max;
    const int64_t v = *d_n;
    if (v >= 0 && v <= n_max) return v;
    if (err && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(err, kAsyncCount);
    return v < 0 ? 0 : n_max;
}
#endif

/* what lv_correct_device_async hands the begin kernel (all zero / NULL for the synchronous forms) */
struct UpdateGate {
    const int64_t* n = nullptr;              /* device count of the sweep (NULL: the host-known n) */
    int64_t min_points = 0;                  /* main.cpp:81 MAX_POINTS2MATCH: fewer points -> LV_TOO_FEW_POINTS, no update */
    const uint32_t* map_counters = nullptr;  /* non-NULL: LV_EMPTY_MAP when the map holds no point (host cannot know it) */
    AsyncWords* words = nullptr;             /* non-NULL: the time of an update that runs goes to words->time_updated */
    double time = 0.0;
};
/* the fit kernel's grid: 4 blocks of kMeasureThreads resident per SM is ample; one partial row per block */
enum { kMeasureThreads = 128, kPartialStride = 96, kStepThreads = 512, kPartialGroup = 32, kMeasureGridCap = kNumSMs * 4 };
inline int partial_groups(int grid) { return (grid + kPartialGroup - 1) / kPartialGroup; }
/* The search kernel appends its uncertified queries to one of 32 lists picked by block index: thousands of atomics on
 * ONE counter give it a long tail on the first evaluation of an update (tools/timeline.py). */
enum { kHardBuckets = 32, kCounters = 4 + kHardBuckets };
/* a bucket receives the queries of every 32nd block: at most n / 32 + (queries per block <= 128) of them */
inline uint32_t hard_segment(int64_t n) { return (uint32_t)((n + kHardBuckets - 1) / kHardBuckets + 160); }

/* the sweep of an update replayed from a CUDA graph: written by the begin kernel (whose arguments are the
 * only thing patched per launch), read by the measurement kernels instead of MeasureArgs::xyz / n / n_tiles */
struct MeasureJob {
    const float* xyz;
    int32_t n;
    int32_t n_tiles;
};

/* per-launch constants of the measurement kernels (reuse, search, search-upper, fit) */
struct MeasureArgs {
    const float* xyz;          /* n x 3 packed, LiDAR frame                               */
    int32_t n;                 /* with `job`: the capacity the grids were sized for       */
    int32_t n_tiles;           /* ceil(n / kMeasureThreads)                               */
    const MeasureJob* job;     /* non-NULL: xyz / n / n_tiles come from device memory      */
    VoxelMapView map;
    const UpdateCtrl* ctrl;    /* frame + done flag                                       */
    UpdateCtrl* prep;          /* non-NULL: block 0 of the fit kernel runs ieskf_prepare() */
    float max_d2;              /* smallest float >= MAX_DIST_PLANE^2 (search radius^2)    */
    double gate_d2;            /* MAX_DIST_PLANE^2 in double (Plane.cpp:42)               */
    float planes_threshold;
    int32_t estimate_extrinsics;
    double* partials;          /* [grid][kPartialStride]: 78 + 12 sums, count             */
    double* group_rows;        /* [partial_groups(grid)][kPartialStride]: the partials summed in groups of kPartialGroup rows */
    uint32_t* group_tickets;   /* [partial_groups(grid)]: blocks of the group that have finished (fit kernel)                  */
    /* optional per-point outputs (NULL on the hot path) */
    uint8_t* valid;
    int32_t* nn_idx;
    float* nn_sqd;
    float* plane;
    float* dist;
    float* g_world;
    double* rows;              /* n x 13 (row[12], h)                                     */
    int4* nn_a;                /* n: search result handed from K1 to K2 (neighbours 0..3)      */
    int2* nn_b;                /* n: (neighbour 4, bits of the 5th squared distance)         */
    uint32_t* hard_list;       /* queries level 0 could not certify (K1 -> K1b): kHardBuckets segments of hard_seg entries */
    uint32_t hard_seg;         /* capacity of one segment                                      */
    uint32_t* hard_count;      /* [2] length of redo_list, [4 .. 4 + kHardBuckets) lengths of the segments; kCounters words */
    /* reuse of neighbours across the evaluations of one update (NULL: off) */
    float4* ref;               /* n: world position the stored neighbours were searched from + outsider bound */
    uint32_t* redo_list;       /* n: queries whose neighbours could not be reused (Kv -> K1)  */
};

/* device map storage (layout: lv_voxel_map.h) + scratch of one add */
struct MapBuffers {
    MapGrid grid;
    uint4* table;              /* voxel slots (2 x uint4 each)                               */
    uint32_t slots;
    uint4* btable;             /* block slots                                                 */
    uint32_t bslots;
    float4* arena;             /* own extents + halo buckets                                  */
    uint32_t arena_cap;
    uint32_t* counters;        /* kMapCounters device words                                   */
    uint32_t* h_counters;      /* pinned mirror (map_fetch_counters)                          */
    uint32_t* touched;
    uint32_t* dirty;
    uint32_t list_cap;
    float* stage_xyz;          /* device copy of host points handed to lv_map_build / lv_map_add: add_cap x 3 */
    uint32_t *skeys, *skeys_alt, *svals, *svals_alt;   /* sort of the new points (add_cap each) */
    void* sort_tmp;
    size_t sort_tmp_bytes;
    int sort_bits;
    int64_t cap;               /* max_map_points, then what the last growth sized for (tables and arena) */
    int64_t add_cap;           /* most points one build / add can take                        */
    int64_t max_points;        /* lv_params.max_points: add_cap never drops below it          */
    bool empty;                /* nothing was ever added (Mapper::exists, Mapper.cpp:32-34)   */
    cudaStream_t stream;       /* the stream the buffers were allocated on (stream-ordered)   */
};

/* what map_alloc / map_grow allocate for a capacity of `cap` points */
enum : uint32_t { kMaxSlots = 1u << 26, kMaxArena = 0x7FFFFFF0u };   /* hard ceilings: slot << kCellBits and point ids are 32-bit */
struct MapSizes {
    uint32_t slots, bslots, arena_cap;
    int64_t add_cap;
    size_t sort_tmp_bytes;
};
MapSizes map_sizes(int64_t cap, int64_t max_points, bool scratch = true);   /* scratch: size the radix sort's temporary too */
/* NULL when `cap` points fit under the hard ceilings, else the name of the ceiling it crosses */
const char* map_ceiling(int64_t cap);
int64_t map_bytes(const MapBuffers& b);

cudaError_t map_alloc(MapBuffers& b, int64_t max_map_points, int64_t max_points, float voxel_size, float ds, cudaStream_t st);
void map_free(MapBuffers& b);
/* grow to a capacity of `cap` points (no-op when cap <= b.cap); keeps content, ids, insertion order and arena indices */
cudaError_t map_grow(MapBuffers& b, int64_t cap, cudaStream_t st, int* launches);
/* empty the map (table, block table, counters); asynchronous */
cudaError_t map_clear(MapBuffers& b, cudaStream_t st, int* launches);
/* the count of an add that lives in device memory (lv_correct_device_async -> lv_map_add_last_sweep): the add takes
 * *n points (clamped to the host bound), none when *n < max(min_points, 1) (main.cpp:81 breaks before map.add); with
 * build_if_empty an add that finds the map without points builds it (no downsampling, Mapper.cpp:26) */
struct MapAddCount {
    const int64_t* n = nullptr;
    int64_t min_points = 0;
    int build_if_empty = 0;
    uint32_t* err = nullptr;
};
/* KD_TREE::Build (downsample = 0 on an empty map) / Add_Points: n points in DEVICE memory (or *cnt.n of them, n = the
 * host-known bound the sort runs over); asynchronous, no host round trip.  With to_world the points are a sweep (LiDAR frame)
 * transformed by the state in to_world->x first: main.cpp:99-105 without leaving the GPU */
cudaError_t map_add(MapBuffers& b, const float* d_xyz, int64_t n, int downsample, cudaStream_t st, int* launches,
                    const MapAddCount& cnt = MapAddCount(), const UpdateCtrl* to_world = nullptr);
/* main.cpp:91-93 (lv_sweep_to_world_device_async): *d_n points (clamped to [0, n_max]) of d_xyz (LiDAR frame) transformed by the
 * state in d_ctrl->x into d_out (may equal d_xyz); *d_n_out and *count (a device word the transform reads) = that count, or 0 when
 * gate_n is given and its count (clamped to [0, gate_max]) is below max(gate_min, 1) (main.cpp:81 breaks before publishing) */
cudaError_t launch_sweep_to_world(const UpdateCtrl* d_ctrl, const float* d_xyz, const int64_t* d_n, int64_t n_max, const int64_t* gate_n,
                                  int64_t gate_max, int64_t gate_min, float* d_out, int64_t* d_n_out, uint32_t* count, uint32_t* err,
                                  cudaStream_t st, int* launches);
cudaError_t map_fetch_counters(MapBuffers& b, cudaStream_t st);
cudaError_t map_points_sorted(MapBuffers& b, float* host_out, int64_t cap, int64_t* n_out, cudaStream_t st);
VoxelMapView map_view(const MapBuffers& b);

int measure_grid(int n);
/* `probe` (optional) is called on the launching thread before the search (stage 0), after it (1), after the
 * upper-level search (2) and after the fit (3): the profiler records its events there */
struct MeasureProbe { void (*at)(void* ctx, int stage); void* ctx; };
/* reuse = index of the evaluation within its update; != 0 (needs a.ref): lv_reuse_kernel first, then the search only
 * over the queries it could not vouch for; the probe then sees stage 4 before the reuse kernel.  The index also picks
 * the shape of the level-0 search kernel (search_group() in lv_measure.cu). */
cudaError_t launch_measure(const MeasureArgs& a, int grid, cudaStream_t st, const MeasureProbe* probe = nullptr,
                           int reuse = 0, int pdl = 0);
cudaError_t launch_ieskf_begin(UpdateCtrl* c, MeasureJob* job, const float* xyz, int n, uint32_t* counters, const UpdateGate& gate,
                               cudaStream_t st);
const void* ieskf_begin_kernel_ptr();
/* the constant tables of the fit and step kernels on the current device: copied on st and waited for by the first call per
 * device (thread-safe); the launchers above and below need it done, so lv_create calls it on the handle's stream, never inside
 * a capture.  Without a stream (a harness that runs the launchers on the legacy stream) the copy runs on the legacy stream */
cudaError_t measure_init(cudaStream_t st = 0);
cudaError_t launch_ieskf_step(UpdateCtrl* c, const IeskfParams& prm, const double* partials, int n_partials,
                              cudaStream_t st, int pdl = 0);
/* stand-alone reduction of the partials (operator-boundary calls): out[0:144) HTH, [144:156) HTh, [156] Nm */
cudaError_t launch_reduce_partials(const double* partials, int n_partials, double* out, cudaStream_t st);
struct PredictNoise;
cudaError_t launch_predict(UpdateCtrl* c, const PredictNoise& noise, const double* d_imu, int k, cudaStream_t st);
cudaError_t launch_set_frame(UpdateCtrl* c, cudaStream_t st);   /* frame from c->x, done = 0 */
cudaError_t launch_l2_flush(void* buf, size_t bytes, cudaStream_t st);

/* lv_downsample.cu: PointCloudProcessor::temporal_downsample and Compensator::voxelgrid_downsample */
struct GridBox;
struct DownsampleScratch {
    int64_t cap = 0;               /* points every per-point array holds (0 until all of them are allocated) */
    DeviceBuf<uint32_t> keys, keys_sorted, vals, vals_sorted;
    DeviceBuf<uint64_t> keys64, keys64_sorted;   /* time keys of lv_cloud.cu */
    DeviceBuf<uint8_t> flags;
    DeviceBuf<int32_t> sel;
    DeviceBuf<uint8_t> tmp;        /* cub's temporary storage: tmp.size() bytes */
    DeviceBuf<GridBox> box;
    DeviceBuf<int> count;          /* [0] output count, [1] NaN-time flag (velodyne: packet flag), [2] tag-kept count of a livox
                                    * message / point count of a velodyne or ouster one (lv_cloud.cu) */
    PinnedBuf<int> h_count;        /* [0] output count, [1] overflow flag (voxel grid) / NaN-time or packet flag (cloud) */
};
cudaError_t ds_reserve(DownsampleScratch& s, int64_t n);
/* the attribute lanes of a full voxel grid (lv_voxelgrid_downsample_full): the inputs (intensity summed per leaf; time read by
 * the overflow pass-through only; range is never read: every output's range is |output xyz|) and the outputs, any of which may
 * be NULL */
struct VoxelLanes {
    const double* time = nullptr;
    const float* intensity = nullptr;
    double* time_out = nullptr;
    float* intensity_out = nullptr;
    float* range_out = nullptr;
};
/* the voxel grid over d_n ? *d_n : n_max points (the sort runs over n_max, padding keys last), the PCL cell-index overflow
 * pass-through decided on the device; afterwards s.count[0] = output count (also written to *d_n_out when non-NULL),
 * s.h_count[0] / [1] = output count / overflow flag after a stream sync.  lanes non-NULL: the full points' attributes too */
cudaError_t launch_voxelgrid(DownsampleScratch& s, const float* d_xyz, const int64_t* d_n, int64_t n_max, float leaf, float* d_out,
                             int64_t* d_n_out, uint32_t* err, cudaStream_t st, int* launches, const VoxelLanes* lanes = nullptr);
cudaError_t launch_temporal(DownsampleScratch& s, const float* d_xyz, int64_t n, int rate, double min_dist, float* d_out,
                            int32_t* d_idx_out, cudaStream_t st, int* launches);

/* lv_cloud.cu: Accumulator::process (msg2points -> temporal_downsample -> sort_points) on the message bytes in HBM */
struct CloudArgs {
    const uint8_t* data;       /* the message's point bytes (device, any alignment) */
    int64_t n;
    lv_cloud_layout layout;
    lv_lidar_type type;
    uint64_t stamp_us;
    int32_t stamp_beginning, offset_beginning;
    double full_rotation_time;
    int32_t rate;
    double min_dist;
};
struct CloudOut { float* xyz; double* time; float* intensity; float* range; int32_t* idx; };   /* intensity / range / idx may be NULL */
/* most points the decimator can keep: the slots the sort runs over */
int64_t cloud_bound(int64_t n, int rate);
/* enqueues everything (needs ds_reserve(s, n) and cloud_bound > 0); afterwards s.h_count[0] = points kept, s.h_count[1] = 1 if a
 * kept point's time is NaN (after a stream sync).  d_n_out (may be NULL) receives the count on the device; err (may be NULL)
 * gets kAsyncCloudNaN for a NaN time */
cudaError_t launch_process_cloud(DownsampleScratch& s, const CloudArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err, cudaStream_t st,
                                 int* launches);
/* the same for a livox CustomMsg: the tag filter, then the decimator on the rank among the tag-kept points (lv_wire.h) */
struct LivoxArgs {
    const uint8_t* data;       /* the message's 19-byte records (device, any alignment) */
    int64_t n;
    uint64_t timebase_ns;
    uint32_t tag_reject_mask;
    int32_t rate;
    double min_dist;
};
cudaError_t launch_process_livox(DownsampleScratch& s, const LivoxArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err, cudaStream_t st,
                                 int* launches);
/* the same for a velodyne_msgs/VelodyneScan: msg2points (return mode, block flags, distance), then the decimator on the rank among
 * its points (lv_wire.h).  s.h_count[1] = 1 (after a stream sync) and err gets kAsyncVelodyne when a packet is a dual-return one or
 * its stamp does not convert */
struct VelodyneArgs {
    const uint8_t* data;       /* the packets (device, any alignment) */
    int64_t n_packets;
    int64_t n;                 /* 384 n_packets slots */
    const float* table;        /* C then S, kVelodyneTable floats each (velodyne_tables, device) */
    VelodyneCalib cal;
    int32_t rate;
    double min_dist;
};
cudaError_t launch_process_velodyne(DownsampleScratch& s, const VelodyneArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err,
                                    cudaStream_t st, int* launches);
/* the same for Ouster packets of any UDP profile: msg2points (column status, measurement id, range), then the decimator on the rank
 * among its points (lv_wire.h).  No deferred error of its own: a column's time always converts */
struct OusterArgs {
    const uint8_t* data;       /* the packets (device, any alignment) */
    int64_t n;                 /* 16 H n_packets slots */
    const float* table;        /* C then S, kOusterTable floats each (ouster_table, device) */
    OusterCalib cal;           /* the beam terms, by value: the kernels read them from the parameter bank */
    OusterFormat fmt;          /* where the profile keeps a column's fields (ouster_format), by value */
    int32_t rate;
    double min_dist;
};
cudaError_t launch_process_ouster(DownsampleScratch& s, const OusterArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err,
                                  cudaStream_t st, int* launches);
/* Processor::fill's header stamp (PointCloudProcessor.cpp:125-133): *d_stamp_us = max over the *d_n (clamped to [0, n_max]) times of
 * round(t * 1e6) as uint64 (Conversions::sec2Microsec, Utils.cpp:14-16), 0 for no point.  One launch */
cudaError_t launch_cloud_stamp(const double* d_time, const int64_t* d_n, int64_t n_max, uint64_t* d_stamp_us, uint32_t* err, cudaStream_t st,
                               int* launches);

/* lv_deskew.cu: Compensator::compensate over d_n ? *d_n : n_max points.  d_bad (one int) is set when a timestamp is out of
 * range / out of order; err (may be NULL) gets kAsyncDeskewPath then too */
int deskew_max_states();
cudaError_t launch_deskew(const lv_state32* d_path, int ns, const lv_state32& Xt2, double t_lo, double t_hi, const float* d_xyz,
                          const double* d_t, const int64_t* d_n, int64_t n_max, float* d_out, int* d_bad, uint32_t* err, cudaStream_t st);

/* lv_lidar_buffer.cu: Accumulator::BUFFER_L as a ring in HBM (index arithmetic: lv_lidar_buffer.h) */
struct LidarWords {
    int64_t head, tail;        /* live positions [head, tail); position p in slot p % cap          */
    int64_t window;            /* points the last get's window holds (also when above its n_max)    */
    int64_t count;             /* points the last get wrote (0 when the window was above n_max)     */
    uint32_t ticket;           /* blocks of a push or of a merge kernel that have finished          */
    uint32_t merge_bad;        /* a block of the merge's split kernel found T_tail or B out of order */
    int64_t merge_split;       /* the last merge's split s, its point count and its mode (kLidarMerge*) */
    int64_t merge_n;
    uint32_t merge_mode;
    uint32_t pad;
};
struct LidarRing {
    DeviceBuf<float> xyz;      /* cap x 3 */
    DeviceBuf<double> time;    /* cap     */
    DeviceBuf<float> intensity;   /* cap, or empty: a ring without attribute lanes (lv_lidar_reserve_full adds them) */
    DeviceBuf<float> range;       /* cap, with intensity */
    int64_t cap = 0;           /* 0: not reserved yet */
    DeviceBuf<LidarWords> words;
    PinnedBuf<LidarWords> h_words;
    /* the merge's overlap scratch (lv_lidar_reserve_merge): T_tail is staged here before the merge overwrites it */
    DeviceBuf<float> merge_xyz;        /* merge_cap x 3 */
    DeviceBuf<double> merge_time;      /* merge_cap     */
    DeviceBuf<float> merge_intensity;  /* merge_cap, when the ring has lanes */
    DeviceBuf<float> merge_range;
    int64_t merge_cap = 0;     /* 0: no merge before lv_lidar_reserve_merge */
};
/* push *d_n (clamped to [0, n_max]) points; kAsyncLidarFull and nothing appended when they do not fit.  On a ring with lanes the
 * points' intensity and range go with them (NULL: 0) */
cudaError_t launch_lidar_push(const LidarRing& r, const float* xyz, const double* time, const int64_t* d_n, int64_t n_max, uint32_t* err,
                              cudaStream_t st, int* launches, const float* intensity = nullptr, const float* range = nullptr);
/* Accumulator::get(BUFFER_L, t1, t2) into xyz / time; the count goes to words->count and to *d_n_out (may be NULL); a window
 * above n_max writes count 0 and raises kAsyncLidarWindow (err may be NULL).  intensity / range non-NULL (a ring with lanes
 * only): the window's lanes too */
cudaError_t launch_lidar_get(const LidarRing& r, double t1, double t2, float* xyz, double* time, int64_t n_max, int64_t* d_n_out, uint32_t* err,
                             cudaStream_t st, int* launches, float* intensity = nullptr, float* range = nullptr);
/* merge *d_n (clamped to [0, n_max]) time-ordered points into the ring by time (lv_lidar_buffer.h), each through T when
 * `transform`: three launches whatever the overlap, the counts and the decision on the device.  Unsorted input is appended with
 * kAsyncLidarUnsorted; an overlap above merge_cap (kAsyncLidarOverlap) or points that do not fit (kAsyncLidarFull) change nothing.
 * intensity / range as in launch_lidar_push */
cudaError_t launch_lidar_merge(const LidarRing& r, const float* xyz, const double* time, const int64_t* d_n, int64_t n_max, bool transform,
                               const Rt32& T, uint32_t* err, cudaStream_t st, int* launches, const float* intensity = nullptr,
                               const float* range = nullptr);
cudaError_t launch_lidar_clear(const LidarRing& r, double t, cudaStream_t st, int* launches);
/* copy the `live` live points of `from` into the arrays of a ring of capacity cap (the counters stay as they are); intensity /
 * range non-NULL: into those lanes too (0 where `from` has none) */
cudaError_t launch_lidar_move(const LidarRing& from, int64_t live, float* xyz, double* time, int64_t cap, cudaStream_t st, int* launches,
                              float* intensity = nullptr, float* range = nullptr);

/* lv_preloc.cu: the scoring kernel of lv_prelocalize (arithmetic: lv_preloc.h) */
enum { kPrelocThreads = 256, kPrelocPosPerCta = 64 };
struct PrelocArgs {
    const float* xyz;          /* the sweep, n x 3, LiDAR frame (device)                                  */
    int64_t n;
    int32_t S;                 /* scored points: xyz[floor(s n / S)], s < S <= kPrelocMaxPoints             */
    int64_t I, K;              /* half-widths of the position and heading grids                           */
    int64_t headings;          /* 2K + 1                                                                  */
    int64_t positions;         /* (2I + 1)^2                                                              */
    const float* frames;       /* headings x 12: lidar_to_world R (row-major) and t of each heading       */
    const float4* offsets;     /* positions: the fp32 offset (x, y, z, 0) of each position                */
    VoxelMapView map;
    int32_t* scores;           /* headings x positions, or NULL                                           */
    unsigned long long* best;  /* the largest selection key (preloc_key); 0 before the launch             */
};
cudaError_t launch_preloc(const PrelocArgs& a, cudaStream_t st, int* launches);

/* lv_preloc_global.cu: the occupancy summary, the cell bounds and the exact cell scores of lv_prelocalize_global
 * (arithmetic and schedule: lv_preloc_bound.h) */
enum { kPrelocGlobalThreads = 256 };
struct PrelocGlobalArgs {
    const float* xyz;          /* the sweep, n x 3, LiDAR frame (device)                                  */
    int64_t n;
    int32_t S;                 /* scored points: xyz[floor(s n / S)]                                       */
    float step;                /* position grid step (m)                                                   */
    int64_t I, K;              /* half-widths of the position and heading grids                           */
    PrelocAxes ax;             /* u, v: the position offsets are computed in the kernel (preloc_offset)  */
    const float* frames;       /* (2K + 1) x 12: lidar_to_world R (row-major) and t of each heading       */
    PrelocOcc occ;
    const PrelocCell* cells;   /* the cells of one launch                                                 */
    int64_t count;
    int32_t* bounds;           /* bound launch: the bound of each cell                                    */
    PrelocBest* best;          /* exact launch: the best candidate of each cell                           */
};
/* ext: 6 words, lo (x, y, z) then hi; set to 0xFFFFFFFF / 0 before the launch */
cudaError_t launch_occ_extent(const VoxelMapView& m, uint32_t bslots, uint32_t* ext, cudaStream_t st, int* launches);
/* o.bits zeroed before the launch; o.lo / o.hi, the levels and offsets from occ_layout */
cudaError_t launch_occ_bits(const PrelocOcc& o, uint32_t bslots, uint32_t* bits, cudaStream_t st, int* launches);
cudaError_t launch_preloc_bounds(const PrelocGlobalArgs& a, cudaStream_t st, int* launches);
cudaError_t launch_preloc_exact(const PrelocGlobalArgs& a, cudaStream_t st, int* launches);

}  // namespace lv
#endif
