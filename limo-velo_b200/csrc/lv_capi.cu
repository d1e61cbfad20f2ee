/*
 * lv_capi.cu — context object and the C ABI of liblimovelo_b200.so (include/limovelo_b200.h).
 *
 * One lv_context replaces the Localizator + Mapper singletons of the reference
 * (src/Modules/Localizator.cpp:100-103, include/Headers/Mapper.hpp:35-38): it owns the IKFoM
 * state mirror, the device map and the device buffers of one sequence, on one CUDA stream.
 * No CPU fallback exists: without a usable CUDA device every compute call returns LV_ERR_CUDA.
 */
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <utility>
#include <vector>

#include "../../include/limovelo_b200.h"
#include "lv_host.h"
#include "lv_internal.h"
#include "lv_lidar_buffer.h"
#include "lv_preloc.h"
#include "lv_preloc_bound.h"
#include "lv_predict.h"
#include "lv_wire.h"

using namespace lv;

static_assert(sizeof(lv_iter_log) == sizeof(IterLog), "lv_iter_log must mirror lv::IterLog");
static_assert(LV_MAX_EVALS == kMaxEvals, "log capacity");
static_assert(LV_STATE_LEN == kStateLen && LV_DOF == kDof, "state layout");

static thread_local std::string g_last_error;
static void set_error(const std::string& s) { g_last_error = s; }
void lvh_set_error(const char* msg) { set_error(msg); }

#define LV_CUDA(call)                                                                            \
    do {                                                                                         \
        cudaError_t e__ = (call);                                                                \
        if (e__ != cudaSuccess) {                                                                \
            char buf__[512];                                                                     \
            snprintf(buf__, sizeof(buf__), "%s:%d: %s -> %s", __FILE__, __LINE__, #call,         \
                     cudaGetErrorString(e__));                                                   \
            set_error(buf__);                                                                    \
            return LV_ERR_CUDA;                                                                  \
        }                                                                                        \
    } while (0)

/* what an event pair times; search, search-upper and fit are in the order of launch_measure's probe stages 0, 1, 2 */
enum ProfKind { kProfSolve, kProfMap, kProfSearch, kProfSearchUpper, kProfFit, kProfReuse };
struct EventPair { cudaEvent_t a, b; ProfKind kind; int upd; int slot; };
enum { kNevalsRing = 4096 };

struct lv_context {
    lv_params prm;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    MapBuffers map;
    /* reserved once, by create_buffers (as are d_job and d_async): the update graphs bake these pointers into their nodes */
    DeviceBuf<float> d_sweep;          /* max_points x 3 */
    DeviceBuf<UpdateCtrl> d_ctrl;
    PinnedBuf<UpdateCtrl> h_ctrl;      /* mirror for the D2H of results */
    DeviceBuf<double> d_partials;
    DeviceBuf<double> d_group_rows;    /* partials pre-reduced in groups of kPartialGroup rows (fit kernel) */
    DeviceBuf<uint32_t> d_group_tickets;
    DeviceBuf<int4> d_nn_a;            /* max_points: K1 -> K2 hand-over */
    DeviceBuf<int2> d_nn_b;
    DeviceBuf<uint32_t> d_hard_list;   /* kHardBuckets segments of hard_segment(max_points) entries, then kCounters counters */
    DeviceBuf<float4> d_ref;           /* max_points: reuse reference (lv_reuse_kernel) */
    DeviceBuf<uint32_t> d_redo;        /* max_points */
    DeviceBuf<double> d_imu;           /* kImuBatch x 7: lv_propagate_device (lazily allocated) */
    PinnedBuf<double> h_imu;
    /* recorded after the last H2D copy out of h_imu / h_ctrl: the calls return before those copies run (they queue behind
     * the update), so the next refill of the pinned buffer waits for this event, not for the whole stream */
    Event imu_copied;
    Event ctrl_copied;
    /* the sweep of the last update (correct_enqueue), for lv_map_add_last_sweep and lv_sweep_to_world_device_async */
    struct TickSweep {
        const float* xyz = nullptr;    /* device pointer */
        int64_t n = 0;                 /* its points, or with d_n the host bound of its device count */
        const int64_t* d_n = nullptr;  /* lv_correct_device_async: the device count ... */
        int64_t min_points = 0;        /* ... and its MAX_POINTS2MATCH gate */
    } tick;
    /* the async tick: deferred errors and the time of the last update that ran (lv_correct_device_async) */
    DeviceBuf<AsyncWords> d_async;
    PinnedBuf<AsyncWords> h_async;
    bool time_pending = false;         /* last_time_updated waits for the device's decision (next fetch) */
    bool map_unknown = false;          /* an async add may have left the map without points: the device checks it */
    Event path_copied;                 /* the last H2D copy out of h_path (lv_compensate_device_async returns before it runs) */
    LidarRing lidar;                   /* Accumulator::BUFFER_L (lv_lidar_reserve) */
    bool use_reuse = true;
    bool use_pdl = true;               /* programmatic dependent launch between the kernels of an update */
    /* Compensator (deskew) staging: lazily allocated */
    DeviceBuf<lv_state32> d_path;      /* deskew_max_states() */
    PinnedBuf<lv_state32> h_path;
    DeviceBuf<double> d_times;         /* max_points */
    DeviceBuf<float> d_deskew_in;      /* max_points x 3 */
    DeviceBuf<int> d_bad;
    PinnedBuf<int> h_bad;
    DownsampleScratch ds;              /* downsamplers: grows with the largest cloud seen */
    DeviceBuf<float> d_velodyne_tables;   /* cos then sin of the 36000 azimuths (velodyne_tables): the first Velodyne call */
    bool velodyne_tables_ok = false;      /* uploaded: a failed upload is retried on the next call */
    DeviceBuf<float> d_ouster_table;      /* cos then sin of the 2048 column angles (ouster_table): the first Ouster call */
    bool ouster_table_ok = false;         /* uploaded: a failed upload is retried on the next call */
    DeviceBuf<float> d_ds_in;          /* staging for the host-buffer variants (ds_stage) */
    DeviceBuf<float> d_ds_out;
    DeviceBuf<uint8_t> d_ds_lanes;     /* attribute staging of lv_voxelgrid_downsample_full: 28 B per point */
    DeviceBuf<double> d_reduced;       /* 157 doubles */
    PinnedBuf<double> h_reduced;
    DeviceBuf<uint8_t> d_flush;
    /* per-point debug outputs (lazily allocated, max_points) */
    DeviceBuf<uint8_t> d_valid; DeviceBuf<int32_t> d_nn_idx; DeviceBuf<float> d_nn_sqd;
    DeviceBuf<float> d_plane; DeviceBuf<float> d_dist; DeviceBuf<float> d_gworld; DeviceBuf<double> d_rows;
    /* lv_prelocalize: winner key, heading frames, position offsets, scores (lazily allocated, grows) */
    DeviceBuf<uint8_t> d_preloc;
    /* lv_prelocalize_global / lv_map_extent: extent, heading frames, cell lists and results, occupancy bitmaps (grows) */
    DeviceBuf<uint8_t> d_pglob;
    /* the occupancy summary (extent, bitmap pyramid) of the map as of map_gen occ_gen; rebuilt when the map changed since */
    uint64_t map_gen = 0;              /* bumped by every add, build and growth (map_enqueue, map_grow_to) */
    uint64_t occ_gen = ~0ull;
    PrelocOcc occ;
    DeviceBuf<uint32_t> d_occ;         /* extent (8 words), then the bitmaps */
    /* host mirror of the filter (get_x / get_P) */
    double x[LV_STATE_LEN];
    double P[LV_DOF * LV_DOF];
    bool state_dirty = true;           /* host mirror newer than d_ctrl->x/P */
    bool pending_fetch = false;        /* device holds results not yet mirrored (lv_correct_device) */
    double last_time_updated = -1;
    lv_iter_log logs[LV_MAX_EVALS];
    int32_t n_evals = 0;
    int32_t last_status = LV_OK;
    /* profiling */
    bool profile = false;
    std::vector<EventPair> pending;
    std::vector<EventPair> pool;
    lv_profile prof;
    PinnedBuf<int32_t> h_nevals;       /* ring: n_evals of profiled updates */
    uint32_t update_seq = 0;
    IeskfParams iprm;
    /* one update = begin + (MAX_NUM_ITERS + 1) x (search, search-upper, fit, step): replayed as a CUDA graph
     * (one per sweep-capacity bucket) so that the host pays one launch instead of ~21 */
    struct UpdateGraph {
        int64_t cap;
        cudaGraph_t graph;
        cudaGraphExec_t exec;
        cudaGraphNode_t begin_node;
    };
    std::vector<UpdateGraph> graphs;
    DeviceBuf<MeasureJob> d_job;
    bool use_graph = true;
    /* map growth (lv_map_set_growth): after every add the 64 B of map counters are copied into a pinned ring and an event is
     * recorded; before the next add the host bounds the map from the newest snapshot the device has finished */
    enum { kSnapRing = 4 };
    int64_t grow_limit = 0;            /* 0: off */
    int64_t growths = 0;
    int64_t grow_waits = 0;
    int64_t waited_at_cap = 0;         /* capacity at which the policy last waited for a snapshot */
    PinnedBuf<uint32_t> h_snap;        /* kSnapRing x kMapCounters */
    Event snap_ev[kSnapRing];
    int64_t snap_seq[kSnapRing] = {-1, -1, -1, -1};   /* add sequence number a slot holds (-1: none) */
    int64_t snap_cum[kSnapRing] = {};  /* points enqueued up to and including that add */
    int64_t add_seq = 0;               /* adds enqueued since the last clear */
    int64_t add_cum = 0;               /* points of those adds */
    uint32_t known[kMapCounters] = {}; /* newest finished snapshot (or the cleared map) */
    int64_t known_seq = 0, known_cum = 0;
    /* the owners above free their buffers and events after this */
    ~lv_context() {
        if (stream) cudaStreamSynchronize(stream);
        for (auto& e : pending) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
        for (auto& e : pool) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
        for (auto& u : graphs) { cudaGraphExecDestroy(u.exec); cudaGraphDestroy(u.graph); }
        map_free(map);
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
};

static lv_status drain_events(lv_context* h) {
    if (h->pending.empty()) return LV_OK;
    LV_CUDA(cudaStreamSynchronize(h->stream));
    for (auto& e : h->pending) {
        float ms = 0;
        LV_CUDA(cudaEventElapsedTime(&ms, e.a, e.b));
        /* launches enqueued after the update had already finished return immediately: keep them apart */
        const bool idle = e.upd >= 0 && e.slot >= h->h_nevals[e.upd % kNevalsRing];
        if (idle) { h->prof.idle_ms += ms; h->prof.idle_launches++; }
        else if (e.kind == kProfSearch) {
            h->prof.search_ms += ms; h->prof.measure_ms += ms; h->prof.measure_launches++;
            if (e.slot <= 0) { h->prof.search_first_ms += ms; h->prof.search_first_launches++; }
        }
        else if (e.kind == kProfSearchUpper) { h->prof.search_upper_ms += ms; h->prof.measure_ms += ms; }
        else if (e.kind == kProfFit) { h->prof.fit_ms += ms; h->prof.measure_ms += ms; }
        else if (e.kind == kProfReuse) { h->prof.reuse_ms += ms; h->prof.measure_ms += ms; }
        else if (e.kind == kProfSolve) { h->prof.solve_ms += ms; h->prof.solve_launches++; }
        else { h->prof.build_ms += ms; h->prof.build_launches++; }
        h->pool.push_back(e);
    }
    h->pending.clear();
    return LV_OK;
}
static bool prof_begin(lv_context* h, ProfKind kind, EventPair* ep) {
    if (!h->profile) return false;
    if (h->pending.size() > 2048) drain_events(h);
    if (h->pool.empty()) {
        EventPair e;
        if (cudaEventCreate(&e.a) != cudaSuccess || cudaEventCreate(&e.b) != cudaSuccess) return false;
        h->pool.push_back(e);
    }
    *ep = h->pool.back();
    h->pool.pop_back();
    ep->kind = kind;
    ep->upd = -1;
    ep->slot = 0;
    cudaEventRecord(ep->a, h->stream);
    return true;
}
static void prof_end(lv_context* h, EventPair* ep) {
    cudaEventRecord(ep->b, h->stream);
    h->pending.push_back(*ep);
}

static void fill_iprm(lv_context* h) {
    h->iprm.R = h->prm.LiDAR_noise;
    h->iprm.D = h->prm.degeneracy_threshold;
    for (int i = 0; i < kN; ++i) h->iprm.limits[i] = h->prm.LIMITS[i];
    h->iprm.max_iter = h->prm.MAX_NUM_ITERS;
    h->iprm.estimate_extrinsics = h->prm.estimate_extrinsics;
}

static MeasureArgs make_measure_args(lv_context* h, const float* d_xyz, int64_t n) {
    MeasureArgs a;
    memset(&a, 0, sizeof(a));
    a.xyz = d_xyz;
    a.n = (int32_t)n;
    a.n_tiles = (int32_t)((n + kMeasureThreads - 1) / kMeasureThreads);
    a.map = map_view(h->map);
    a.ctrl = h->d_ctrl;
    const double md = h->prm.MAX_DIST_PLANE;
    a.gate_d2 = md * md;
    float f = (float)a.gate_d2;
    if ((double)f < a.gate_d2) f = nextafterf(f, INFINITY);
    a.max_d2 = f;
    a.planes_threshold = h->prm.PLANES_THRESHOLD;
    a.estimate_extrinsics = h->prm.estimate_extrinsics;
    a.partials = h->d_partials;
    a.group_rows = h->d_group_rows;
    a.group_tickets = h->d_group_tickets;
    a.nn_a = h->d_nn_a;
    a.nn_b = h->d_nn_b;
    a.hard_list = h->d_hard_list;
    a.hard_seg = hard_segment(h->prm.max_points);
    a.hard_count = h->d_hard_list + (size_t)kHardBuckets * a.hard_seg;
    return a;
}

/* argument checks of the _async forms; `what` names the call in the message */
static bool n_max_ok(const char* what, int64_t n_max) {
    if (n_max >= 1 && n_max <= 0x7fffffff) return true;
    set_error(std::string(what) + ": n_max outside [1, 2^31 - 1]");
    return false;
}
static bool handle_ok(const char* what, const lv_context* h, int64_t n_max) {
    if (!h) { set_error(std::string(what) + ": null handle"); return false; }
    if (n_max > h->prm.max_points) { set_error(std::string(what) + ": n_max above max_points"); return false; }
    return true;
}
/* the byte ranges share a byte (ranges that only touch do not) */
static bool ranges_overlap(const void* a, int64_t a_bytes, const void* b, int64_t b_bytes) {
    return (uintptr_t)a < (uintptr_t)b + (uintptr_t)b_bytes && (uintptr_t)b < (uintptr_t)a + (uintptr_t)a_bytes;
}
struct ByteRange {
    const void* p;
    int64_t bytes;
};
/* two of the n ranges share a byte, NULL pointers skipped; the first `shared` ranges may share bytes with each other */
static bool any_ranges_overlap(const ByteRange* r, int n, int shared = 0) {
    for (int b = shared > 1 ? shared : 1; b < n; ++b)
        for (int a = 0; a < b; ++a)
            if (r[a].p && r[b].p && ranges_overlap(r[a].p, r[a].bytes, r[b].p, r[b].bytes)) return true;
    return false;
}

extern "C" {

const char* lv_last_error(void) { return g_last_error.c_str(); }
const char* lv_version(void) { return "limovelo_b200 0.1 (sm_90a)"; }
int64_t lv_result_bytes(void) { return (int64_t)sizeof(UpdateCtrl); }

/* the stream and the buffers of a new context; lv_create destroys the context when this fails */
static lv_status create_buffers(lv_context* h) {
    const lv_params* p = &h->prm;
    if (p->stream) { h->stream = (cudaStream_t)p->stream; h->own_stream = false; }
    else { LV_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true; }
    LV_CUDA(map_alloc(h->map, p->max_map_points, p->max_points, p->voxel_size, p->map_downsample_size, h->stream));
    { int l = 0; LV_CUDA(map_clear(h->map, h->stream, &l)); }
    LV_CUDA(h->d_sweep.reserve(3 * (size_t)p->max_points));
    LV_CUDA(h->d_nn_a.reserve(p->max_points));
    LV_CUDA(h->d_nn_b.reserve(p->max_points));
    LV_CUDA(h->d_hard_list.reserve((size_t)kHardBuckets * hard_segment(p->max_points) + kCounters));
    LV_CUDA(h->d_ref.reserve(p->max_points));
    LV_CUDA(h->d_redo.reserve(p->max_points + 64));   /* + one block of slack: read speculatively */
    /* hand-over buffers start defined: lv_search_kernel<.., LIST> reads redo_list[] before it knows the list's length, and a
     * first update's reuse kernel must not see stale neighbours (also keeps compute-sanitizer initcheck quiet).  Every clear of
     * a context runs on its own stream: the stream orders it before the context's first kernel, and no clear touches the legacy
     * stream, which would wait for (or, while one is being captured, break) other threads' work on blocking streams */
    LV_CUDA(cudaMemsetAsync(h->d_redo, 0, sizeof(uint32_t) * (p->max_points + 64), h->stream));
    LV_CUDA(cudaMemsetAsync(h->d_nn_a, 0xFF, sizeof(int4) * p->max_points, h->stream));
    LV_CUDA(cudaMemsetAsync(h->d_nn_b, 0xFF, sizeof(int2) * p->max_points, h->stream));
    LV_CUDA(cudaMemsetAsync(h->d_ref, 0, sizeof(float4) * p->max_points, h->stream));
    LV_CUDA(cudaMemsetAsync(h->d_hard_list, 0, sizeof(uint32_t) * ((size_t)kHardBuckets * hard_segment(p->max_points) + kCounters), h->stream));
    h->use_reuse = getenv("LV_NO_REUSE") == nullptr;
    h->use_pdl = getenv("LV_NO_PDL") == nullptr;
    LV_CUDA(h->d_job.reserve(1));
    LV_CUDA(measure_init(h->stream));
    h->use_graph = getenv("LV_NO_GRAPH") == nullptr;
    LV_CUDA(h->d_ctrl.reserve(1));
    LV_CUDA(cudaMemsetAsync(h->d_ctrl, 0, sizeof(UpdateCtrl), h->stream));
    LV_CUDA(h->h_ctrl.reserve(1));
    LV_CUDA(h->imu_copied.create());
    LV_CUDA(h->ctrl_copied.create());
    LV_CUDA(h->path_copied.create());
    LV_CUDA(h->d_async.reserve(1));
    LV_CUDA(cudaMemsetAsync(h->d_async, 0, sizeof(AsyncWords), h->stream));
    LV_CUDA(h->h_async.reserve(1));
    LV_CUDA(h->d_partials.reserve((size_t)kPartialStride * (kMeasureGridCap + 8)));
    LV_CUDA(cudaMemsetAsync(h->d_partials, 0, sizeof(double) * kPartialStride * (kMeasureGridCap + 8), h->stream));
    LV_CUDA(h->d_group_rows.reserve((size_t)kPartialStride * 32));
    LV_CUDA(cudaMemsetAsync(h->d_group_rows, 0, sizeof(double) * kPartialStride * 32, h->stream));
    LV_CUDA(h->d_group_tickets.reserve(32));
    LV_CUDA(cudaMemsetAsync(h->d_group_tickets, 0, sizeof(uint32_t) * 32, h->stream));
    LV_CUDA(h->d_reduced.reserve(160));
    LV_CUDA(h->h_reduced.reserve(160));
    LV_CUDA(h->h_nevals.reserve(kNevalsRing));
    return LV_OK;
}

lv_status lv_create(const lv_params* p, lv_handle* out) {
    if (!p || !out) return LV_ERR_ARG;
    *out = nullptr;
    /* all argument checks come before the first allocation */
    if (p->NUM_MATCH_POINTS != 5) { set_error("NUM_MATCH_POINTS must be 5 (5x3 plane fit)"); return LV_ERR_ARG; }
    if (p->MAX_NUM_ITERS < 0 || p->MAX_NUM_ITERS + 1 > LV_MAX_EVALS) {   /* 0: a single h-evaluation (esekfom.hpp:1634 runs i = -1 .. max-1) */
        set_error("MAX_NUM_ITERS out of range");
        return LV_ERR_ARG;
    }
    if (!(p->voxel_size > 0.f) || !(p->map_downsample_size > 0.f) || p->max_map_points <= 0 || p->max_points <= 0) {
        set_error("bad capacity / voxel_size / map_downsample_size");
        return LV_ERR_ARG;
    }
    if (p->max_map_points > (1ll << 24) || p->max_points > (1ll << 24)) { set_error("capacity beyond 2^24 points"); return LV_ERR_ARG; }
    if (!(p->MAX_DIST_PLANE > 0.0) || p->MAX_DIST_PLANE > 48.0 * (double)p->map_downsample_size) {
        set_error("MAX_DIST_PLANE must be positive and at most 48 map_downsample_size (ring search bound)");
        return LV_ERR_ARG;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        set_error("no CUDA device available (there is no CPU fallback)");
        return LV_ERR_CUDA;
    }
    LV_CUDA(cudaSetDevice(p->device));
    lv_context* h = new lv_context();
    h->prm = *p;
    memset(&h->prof, 0, sizeof(h->prof));
    memset(h->logs, 0, sizeof(h->logs));
    memset(&h->map, 0, sizeof(h->map));
    fill_iprm(h);
    const lv_status s = create_buffers(h);
    if (s != LV_OK) { lv_destroy(h); return s; }                 /* nothing of a half-built context survives */
    /* default filter state: identity pose, P = I (esekf constructor); callers normally follow
     * with lv_init_state or lv_set_state */
    for (int i = 0; i < LV_STATE_LEN; ++i) h->x[i] = 0;
    h->x[kRot + 3] = 1; h->x[kOffR + 3] = 1; h->x[kGrav] = LV_S2_LEN;
    for (int i = 0; i < LV_DOF * LV_DOF; ++i) h->P[i] = (i % (LV_DOF + 1) == 0) ? 1.0 : 0.0;
    *out = h;
    return LV_OK;
}

void lv_destroy(lv_handle h) {
    if (!h) return;
    cudaSetDevice(h->prm.device);
    delete h;
}

/* ---- Mapper ---------------------------------------------------------------------------------- */
/* device-side error flags of the map (table / arena exhausted) -> status.  Call after a stream synchronisation that
 * followed map_fetch_counters(). */
static lv_status map_status_from_mirror(lv_context* h) {
    const uint32_t err = h->map.h_counters[kCtrError];
    if (!err) return LV_OK;
    char buf[256];
    snprintf(buf, sizeof(buf), "device map out of capacity (flags 0x%x: 1 voxel table, 2 arena, 4 extent too large, 8 list, 16 block table): raise max_map_points",
             err);
    set_error(buf);
    return LV_ERR_CAPACITY;
}
static void count_map_launches(lv_context* h, int launches) { h->prof.total_launches += launches; }

/* ---- map growth (lv_map_reserve, lv_map_set_growth) ------------------------------------------ */
enum : int64_t { kMaxCapPoints = (int64_t)kMaxSlots / 4 };   /* the largest capacity under both ceilings */

static void drop_update_graphs(lv_context* h) {
    /* the update graphs bake the map view (table, masks, arena) into their kernel arguments; a graph
     * still in flight is freed when it completes */
    for (auto& u : h->graphs) { cudaGraphExecDestroy(u.exec); cudaGraphDestroy(u.graph); }
    h->graphs.clear();
}
static lv_status map_grow_to(lv_context* h, int64_t cap) {
    if (cap <= h->map.cap) return LV_OK;
    char buf[512];
    if (const char* c = map_ceiling(cap)) {
        snprintf(buf, sizeof(buf), "map capacity of %lld points is past the %s", (long long)cap, c);
        set_error(buf);
        return LV_ERR_CAPACITY;
    }
    EventPair ep;
    const bool pr = prof_begin(h, kProfMap, &ep);
    const int64_t old_cap = h->map.cap;
    int launches = 0;
    h->map_gen++;                                                  /* new tables: the occupancy summary is rebuilt */
    const cudaError_t e = map_grow(h->map, cap, h->stream, &launches);
    if (pr) prof_end(h, &ep);
    if (e != cudaSuccess) {
        snprintf(buf, sizeof(buf), "map growth from %lld to %lld points: %s", (long long)old_cap, (long long)cap, cudaGetErrorString(e));
        set_error(buf);
        return h->map.cap == old_cap ? LV_ERR_CAPACITY : LV_ERR_CUDA;   /* allocation failed: the old map is intact */
    }
    drop_update_graphs(h);
    h->growths++;
    count_map_launches(h, launches);
    return LV_OK;
}
/* the smallest capacity, doubling from the current one, at which every bound lies under its mark (DESIGN.md §3) */
static int64_t grow_target(const lv_context* h, const uint32_t* c, int64_t pend) {
    const int64_t pts = (int64_t)(int32_t)c[kCtrPoints] + pend;
    const int64_t slots = (int64_t)c[kCtrSlotsUsed] + 27 * pend;    /* own voxel + 26 dilated neighbours per new point */
    const int64_t blocks = (int64_t)c[kCtrBlocksUsed] + pend;       /* a new block needs a newly occupied voxel */
    const int64_t arena = (int64_t)c[kCtrArenaTop] + 96 * pend;     /* map_alloc's planning ratio */
    int64_t cap = h->map.cap;
    for (;;) {
        const MapSizes z = map_sizes(cap, h->map.max_points, false);
        if (pts <= cap && 2 * slots <= (int64_t)z.slots && 2 * blocks <= (int64_t)z.bslots && 4 * arena <= 3 * (int64_t)z.arena_cap) return cap;
        if (cap >= kMaxCapPoints) return cap;
        cap = cap * 2 < kMaxCapPoints ? cap * 2 : kMaxCapPoints;
    }
}
/* newest finished counter snapshot -> h->known; returns the ring slot of the newest one still pending (-1: none).  Never blocks. */
static int snap_absorb(lv_context* h) {
    int pending = -1;
    for (int i = 0; i < lv_context::kSnapRing; ++i) {
        if (h->snap_seq[i] <= h->known_seq) continue;
        const cudaError_t q = cudaEventQuery(h->snap_ev[i]);
        if (q == cudaErrorNotReady) {
            if (pending < 0 || h->snap_seq[i] > h->snap_seq[pending]) pending = i;
            continue;
        }
        if (q != cudaSuccess) continue;
        memcpy(h->known, h->h_snap + (size_t)i * kMapCounters, sizeof(h->known));
        h->known_seq = h->snap_seq[i];
        h->known_cum = h->snap_cum[i];
    }
    if (pending >= 0 && h->snap_seq[pending] <= h->known_seq) pending = -1;
    if (cudaPeekAtLastError() == cudaErrorNotReady) cudaGetLastError();
    return pending;
}
/* before an add of n points (clears: a build, which empties the map first): grow when the bounds call for it */
static lv_status grow_before_add(lv_context* h, int64_t n, bool clears) {
    if (!h->grow_limit) return LV_OK;
    int64_t want;
    if (clears) {
        uint32_t zero[kMapCounters] = {};
        want = grow_target(h, zero, n);
    } else {
        const int pending = snap_absorb(h);
        want = grow_target(h, h->known, h->add_cum - h->known_cum + n);
        /* maybe only stale: wait for the newest snapshot, once per capacity (a map that sits near a mark would otherwise
         * wait on every tick; the next decision at this capacity grows on the stale bound instead) */
        if (want > h->map.cap && pending >= 0 && h->waited_at_cap != h->map.cap) {
            LV_CUDA(cudaEventSynchronize(h->snap_ev[pending]));
            h->waited_at_cap = h->map.cap;
            h->grow_waits++;
            snap_absorb(h);
            want = grow_target(h, h->known, h->add_cum - h->known_cum + n);
        }
    }
    const int64_t lim = h->grow_limit < kMaxCapPoints ? h->grow_limit : kMaxCapPoints;
    if (want > lim) want = lim;                                    /* at the limit: the add is enqueued as without growth */
    return map_grow_to(h, want);
}
/* after an add: its counters into the pinned ring, behind it on the stream */
static lv_status snap_after_add(lv_context* h, int64_t n) {
    h->add_seq++;
    h->add_cum += n;
    if (!h->grow_limit) return LV_OK;
    const int i = (int)(h->add_seq % lv_context::kSnapRing);
    LV_CUDA(cudaMemcpyAsync(h->h_snap + (size_t)i * kMapCounters, h->map.counters, sizeof(uint32_t) * kMapCounters,
                            cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaEventRecord(h->snap_ev[i], h->stream));
    h->snap_seq[i] = h->add_seq;
    h->snap_cum[i] = h->add_cum;
    return LV_OK;
}
static void snap_reset_cleared(lv_context* h) {                    /* map_clear: the counters are known again */
    memset(h->known, 0, sizeof(h->known));
    h->known[kCtrArenaTop] = 16u;
    h->known_seq = h->known_cum = h->add_seq = h->add_cum = 0;
    for (int i = 0; i < lv_context::kSnapRing; ++i) h->snap_seq[i] = -1;
}
static lv_status capacity_error(lv_context* h, const char* what) {
    char buf[256];
    if (h->grow_limit)
        snprintf(buf, sizeof(buf), "%s: map growth limit reached (%lld points, lv_map_set_growth)", what, (long long)h->grow_limit);
    else
        snprintf(buf, sizeof(buf), "%s", what);
    set_error(buf);
    return LV_ERR_CAPACITY;
}

lv_status lv_map_reserve(lv_handle h, int64_t points) {
    if (!h || points < 0) return LV_ERR_ARG;
    if (points <= h->map.cap) return LV_OK;
    LV_CUDA(cudaSetDevice(h->prm.device));
    return map_grow_to(h, points);
}
lv_status lv_map_set_growth(lv_handle h, int64_t max_points) {
    if (!h || max_points < 0) return LV_ERR_ARG;
    if (max_points == 0) { h->grow_limit = 0; return LV_OK; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(h->h_snap.reserve((size_t)kMapCounters * lv_context::kSnapRing));
    for (Event& e : h->snap_ev) LV_CUDA(e.create());
    if (!h->grow_limit) {                                          /* the counters as of now: the base of the bounds */
        LV_CUDA(map_fetch_counters(h->map, h->stream));
        LV_CUDA(cudaStreamSynchronize(h->stream));
        memcpy(h->known, h->map.h_counters, sizeof(h->known));
        h->known_seq = h->add_seq;
        h->known_cum = h->add_cum;
        for (int i = 0; i < lv_context::kSnapRing; ++i) h->snap_seq[i] = -1;
    }
    h->grow_limit = max_points;
    return LV_OK;
}
lv_status lv_map_info(lv_handle h, struct lv_map_info* out) {
    if (!h || !out) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(map_fetch_counters(h->map, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    const MapBuffers& b = h->map;
    memset(out, 0, sizeof(*out));
    out->capacity_points = b.cap;
    out->voxel_slots = b.slots;
    out->block_slots = b.bslots;
    out->arena_entries = b.arena_cap;
    out->add_capacity = b.add_cap;
    out->bytes = map_bytes(b);
    out->points = (int64_t)(int32_t)b.h_counters[kCtrPoints];
    out->slots_used = b.h_counters[kCtrSlotsUsed];
    out->blocks_used = b.h_counters[kCtrBlocksUsed];
    out->arena_top = b.h_counters[kCtrArenaTop];
    out->growths = h->growths;
    out->growth_limit = h->grow_limit;
    out->host_waits = h->grow_waits;
    out->error_flags = b.h_counters[kCtrError];
    return LV_OK;
}

static lv_status upload_state(lv_context* h, const double* x, const double* P);
/* the host mirror into d_ctrl when it is the newer copy (lv_set_state, lv_init_state, lv_predict) */
static lv_status sync_device_state(lv_context* h) {
    if (!h->state_dirty) return LV_OK;
    const lv_status s = upload_state(h, h->x, h->P);
    if (s == LV_OK) h->state_dirty = false;
    return s;
}

/* Mapper::add on the device, every form, from its argument checks on: n points of xyz, or with cnt.n the host bound of their
 * device count.  Points on the host (on_host) are staged once the add is known to fit.  `build` empties the map first and
 * adds without downsampling (KD_TREE::Build, Mapper.cpp:68-71), and its points must fit the map's capacity; any other add
 * must fit one add's scratch.  An add that finds the map without points builds it (Mapper.cpp:26): emptied first too, except
 * a sweep (to_world: its points transformed by the state on the device), which adds without downsampling to the map as it
 * stands. */
static lv_status map_enqueue(lv_context* h, const float* xyz, bool on_host, int64_t n, bool build, int downsample,
                             const MapAddCount& cnt = MapAddCount(), bool to_world = false) {
    if (!h || (!xyz && n > 0)) return LV_ERR_ARG;
    if (n <= 0) return LV_OK;                                    /* Mapper.cpp:23 */
    LV_CUDA(cudaSetDevice(h->prm.device));
    const bool empty = h->map.empty;
    const bool clears = build || (empty && !to_world);
    lv_status s = to_world ? sync_device_state(h) : LV_OK;
    if (s != LV_OK) return s;
    s = grow_before_add(h, n, clears);
    if (s != LV_OK) return s;
    if (build ? n > h->map.cap : n > h->map.add_cap)
        return capacity_error(h, build ? "map capacity exceeded" : "more points than one lv_map_add can take (max_map_points)");
    if (on_host) {
        LV_CUDA(cudaMemcpyAsync(h->map.stage_xyz, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
        xyz = h->map.stage_xyz;
    }
    if (cnt.n && empty) h->map_unknown = true;                   /* a device count of 0 leaves the map without a point */
    h->map_gen++;                                                  /* the occupancy summary of lv_prelocalize_global is stale */
    EventPair ep;
    const bool pr = prof_begin(h, kProfMap, &ep);
    int launches = 0;
    if (clears) LV_CUDA(map_clear(h->map, h->stream, &launches));
    LV_CUDA(map_add(h->map, xyz, n, (!build && !empty && downsample) ? 1 : 0, h->stream, &launches, cnt, to_world ? h->d_ctrl.get() : nullptr));
    if (pr) prof_end(h, &ep);
    count_map_launches(h, launches);
    if (clears) snap_reset_cleared(h);
    return snap_after_add(h, n);
}

lv_status lv_map_build(lv_handle h, const float* xyz, int64_t m) { return map_enqueue(h, xyz, true, m, true, 0); }
lv_status lv_map_build_device(lv_handle h, const float* d_xyz, int64_t m) { return map_enqueue(h, d_xyz, false, m, true, 0); }
int64_t lv_map_size(lv_handle h) {
    if (!h || h->map.empty) return 0;
    if (cudaSetDevice(h->prm.device) != cudaSuccess) return -1;
    if (map_fetch_counters(h->map, h->stream) != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess) return -1;
    map_status_from_mirror(h);
    return (int64_t)(int32_t)h->map.h_counters[kCtrPoints];
}
int lv_map_exists(lv_handle h) { return (h && !h->map.empty) ? 1 : 0; }
lv_status lv_map_status(lv_handle h) {
    if (!h) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(map_fetch_counters(h->map, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return map_status_from_mirror(h);
}
int64_t lv_map_points(lv_handle h, float* out, int64_t cap) {
    if (!h || h->map.empty) return 0;
    if (cudaSetDevice(h->prm.device) != cudaSuccess) return -1;
    int64_t n = 0;
    if (map_points_sorted(h->map, out, cap, &n, h->stream) != cudaSuccess) return -1;
    return n;
}

lv_status lv_map_add(lv_handle h, const float* xyz, int64_t n, int downsample) {
    return map_enqueue(h, xyz, true, n, h && h->map.empty, downsample);   /* Mapper.cpp:26: lv_map_build on a map without points */
}
lv_status lv_map_add_device(lv_handle h, const float* d_xyz, int64_t n, int downsample) {
    return map_enqueue(h, d_xyz, false, n, false, downsample);
}
lv_status lv_map_add_device_async(lv_handle h, const float* d_xyz, const int64_t* d_n, int64_t n_max, int downsample) {
    if (!d_xyz || !d_n) { set_error("map add async: null points or count"); return LV_ERR_ARG; }
    if (!n_max_ok("map add async", n_max) || !handle_ok("map add async", h, n_max)) return LV_ERR_ARG;
    /* Mapper.cpp:22-30: *d_n points, none when it is 0; a map without points (also one an earlier device count left empty) is
     * built without downsampling.  The add capacity is at least max_points, so n_max always fits. */
    MapAddCount cnt;
    cnt.n = d_n;
    cnt.build_if_empty = 1;
    cnt.err = &h->d_async->err;
    return map_enqueue(h, d_xyz, false, n_max, false, downsample, cnt);
}

/* ---- the tick on the device: main.cpp:99-105 ------------------------------------------------- */
/* how the tick's map add and world cloud count the sweep of the last update: after lv_correct_device_async its gate decides for
 * the whole tick (*d_n points, none when it stopped the tick; a map that an earlier gated build left without points is built,
 * Mapper.cpp:26); after the synchronous forms the host knows the count */
static MapAddCount tick_count(const lv_context* h) {
    MapAddCount c;
    if (!h->tick.d_n) return c;
    c.n = h->tick.d_n;
    c.min_points = h->tick.min_points;
    c.build_if_empty = 1;
    c.err = &h->d_async->err;
    return c;
}
lv_status lv_map_add_sweep_device(lv_handle h, const float* d_xyz_lidar, int64_t n, int downsample) {
    return map_enqueue(h, d_xyz_lidar, false, n, false, downsample, MapAddCount(), true);
}
lv_status lv_map_add_last_sweep(lv_handle h, int downsample) {
    if (!h) return LV_ERR_ARG;
    if (!h->tick.xyz || h->tick.n <= 0) { set_error("no sweep has been corrected yet"); return LV_ERR_ARG; }
    return map_enqueue(h, h->tick.xyz, false, h->tick.n, false, downsample, tick_count(h), true);
}
lv_status lv_sweep_to_world_device_async(lv_handle h, const float* d_xyz_lidar, const int64_t* d_n, int64_t n_max, float* d_xyz_world,
                                         int64_t* d_n_out) {
    if (!d_xyz_lidar || !d_n || !d_xyz_world || !d_n_out) { set_error("sweep to world: null input, count, output or output count"); return LV_ERR_ARG; }
    if (!n_max_ok("sweep to world", n_max)) return LV_ERR_ARG;
    /* one thread reads a point and then writes the same point: in place is fine, a shifted overlap is not.  The counts are read
     * and written by one thread before any point: the output count may equal the input count, but not lie among the points. */
    const int64_t b = 12 * n_max;
    if ((d_xyz_world != d_xyz_lidar && ranges_overlap(d_xyz_world, b, d_xyz_lidar, b)) || ranges_overlap(d_n_out, 8, d_xyz_lidar, b) ||
        ranges_overlap(d_n_out, 8, d_xyz_world, b) || ranges_overlap(d_n, 8, d_xyz_world, b) ||
        (d_n_out != d_n && ranges_overlap(d_n_out, 8, d_n, 8))) {
        set_error("sweep to world: an output range overlaps another range");
        return LV_ERR_ARG;
    }
    if (!handle_ok("sweep to world", h, n_max)) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    const lv_status s = sync_device_state(h);                     /* the transform uses the device copy of the state */
    if (s != LV_OK) return s;
    const MapAddCount gate = tick_count(h);
    int launches = 0;
    LV_CUDA(launch_sweep_to_world(h->d_ctrl, d_xyz_lidar, d_n, n_max, gate.n, h->tick.n, gate.min_points, d_xyz_world, d_n_out,
                                  &h->d_async->world_n, &h->d_async->err, h->stream, &launches));
    h->prof.total_launches += launches;
    return LV_OK;
}

/* ---- state ----------------------------------------------------------------------------------- */
static lv_status fetch_results(lv_context* h);
static lv_status sync_mirror(lv_context* h) {   /* bring the host mirror up to date after lv_correct_device */
    if (!h->pending_fetch) return LV_OK;
    if (cudaSetDevice(h->prm.device) != cudaSuccess) return LV_ERR_CUDA;
    fetch_results(h);
    return LV_OK;
}

lv_status lv_set_state(lv_handle h, const double* x, const double* P) {
    if (!h) return LV_ERR_ARG;
    if (!(x && P)) sync_mirror(h);
    if (x) memcpy(h->x, x, sizeof(h->x));
    if (P) memcpy(h->P, P, sizeof(h->P));
    h->state_dirty = true;
    return LV_OK;
}
lv_status lv_get_state(lv_handle h, double* x, double* P) {
    if (!h) return LV_ERR_ARG;
    sync_mirror(h);
    if (x) memcpy(x, h->x, sizeof(h->x));
    if (P) memcpy(P, h->P, sizeof(h->P));
    return LV_OK;
}
lv_status lv_init_state(lv_handle h, const float q_imu[4]) {
    if (!h || !q_imu) return LV_ERR_ARG;
    lvh_init_state(h->prm, q_imu, h->x, h->P);
    h->state_dirty = true;
    return LV_OK;
}
lv_status lv_predict(lv_handle h, const double acc[3], const double gyro[3], double dt) {
    if (!h || !acc || !gyro) return LV_ERR_ARG;
    sync_mirror(h);
    lvh_predict(h->prm, acc, gyro, dt, h->x, h->P);
    h->state_dirty = true;
    return LV_OK;
}
/* Localizator::propagate_to on the device (Localizator.cpp:59-75): k IMU samples, one launch, no host round trip */
lv_status lv_propagate_device(lv_handle h, const double* acc, const double* gyro, const double* dt, int32_t k) {
    enum { kImuBatch = 512 };
    if (!h || !acc || !gyro || !dt || k < 0) return LV_ERR_ARG;
    if (k == 0) return LV_OK;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(h->d_imu.reserve(7 * kImuBatch));
    LV_CUDA(h->h_imu.reserve(7 * kImuBatch));
    const lv_status s = sync_device_state(h);                     /* the host mirror may be newer (lv_set_state / lv_predict) */
    if (s != LV_OK) return s;
    const PredictNoise noise = {h->prm.covariance_gyroscope, h->prm.covariance_acceleration, h->prm.covariance_bias_gyroscope,
                                h->prm.covariance_bias_acceleration};
    for (int32_t s0 = 0; s0 < k; s0 += kImuBatch) {
        const int32_t kb = k - s0 < kImuBatch ? k - s0 : kImuBatch;
        /* the pinned staging buffer is reused: the previous copy out of it (an earlier batch, or an earlier call still
         * queued behind an update) must have run before it is refilled */
        LV_CUDA(cudaEventSynchronize(h->imu_copied));
        for (int32_t i = 0; i < kb; ++i) {
            for (int a = 0; a < 3; ++a) { h->h_imu[7 * i + a] = acc[3 * (s0 + i) + a]; h->h_imu[7 * i + 3 + a] = gyro[3 * (s0 + i) + a]; }
            h->h_imu[7 * i + 6] = dt[s0 + i];
        }
        LV_CUDA(cudaMemcpyAsync(h->d_imu, h->h_imu, sizeof(double) * 7 * kb, cudaMemcpyHostToDevice, h->stream));
        LV_CUDA(cudaEventRecord(h->imu_copied, h->stream));
        LV_CUDA(launch_predict(h->d_ctrl, noise, h->d_imu, kb, h->stream));
        h->prof.total_launches += 1;
    }
    h->pending_fetch = true;                                      /* the device now holds the newest (x, P) */
    return LV_OK;
}
double lv_last_time_updated(lv_handle h) {
    if (!h) return -1;
    if (h->time_pending) sync_mirror(h);                          /* an async update's time is known once its results are */
    return h->last_time_updated;
}

static lv_status upload_state(lv_context* h, const double* x, const double* P) {
    /* x, P are staged through the pinned mirror so the copy is truly asynchronous; an earlier upload may still be queued
     * behind an update (lv_correct_device, lv_propagate_device return without synchronising) */
    LV_CUDA(cudaEventSynchronize(h->ctrl_copied));
    memcpy(h->h_ctrl->x, x, sizeof(double) * kStateLen);
    if (P) memcpy(h->h_ctrl->P, P, sizeof(double) * kN * kN);
    /* x and P are adjacent in UpdateCtrl: one copy (each small copy costs several microseconds of latency) */
    static_assert(offsetof(UpdateCtrl, P) == offsetof(UpdateCtrl, x) + sizeof(double) * kStateLen, "x, P adjacent");
    LV_CUDA(cudaMemcpyAsync(h->d_ctrl->x, h->h_ctrl->x, sizeof(double) * (kStateLen + (P ? kN * kN : 0)),
                            cudaMemcpyHostToDevice, h->stream));
    LV_CUDA(cudaEventRecord(h->ctrl_copied, h->stream));
    return LV_OK;
}

/* launch_measure() with one CUDA-event pair per kernel when profiling is on (never inside a capture) */
static cudaError_t launch_measure_timed(lv_context* h, const MeasureArgs& a, int grid, int allow_events, int reuse,
                                        int upd, int slot, int pdl = 0) {
    if (!h->profile || !allow_events) return launch_measure(a, grid, h->stream, nullptr, reuse, pdl);
    struct Ctx { lv_context* h; EventPair ep; bool on; int upd, slot; } ctx = {h, EventPair(), false, upd, slot};
    MeasureProbe probe;
    probe.ctx = &ctx;
    probe.at = [](void* p, int stage) {
        Ctx* c = static_cast<Ctx*>(p);
        if (c->on) prof_end(c->h, &c->ep);
        c->on = false;
        if (stage != 3) {         /* 4: reuse kernel follows, 0: search, 1: search-upper, 2: fit, 3: end */
            c->on = prof_begin(c->h, stage == 4 ? kProfReuse : (ProfKind)(kProfSearch + stage), &c->ep);
            c->ep.upd = c->upd; c->ep.slot = c->slot;
        }
    };
    return launch_measure(a, grid, h->stream, &probe, reuse, 0);   /* events between the kernels: no pdl */
}

/* ---- the update ------------------------------------------------------------------------------ */
static MeasureArgs update_measure_args(lv_context* h, const float* d_xyz, int64_t n, bool as_job) {
    MeasureArgs a = make_measure_args(h, d_xyz, n);
    a.prep = h->d_ctrl;                                           /* ieskf_prepare rides in the fit kernel */
    if (as_job) a.job = h->d_job;
    if (h->use_reuse) { a.ref = h->d_ref; a.redo_list = h->d_redo; }
    return a;
}

/* enqueue begin + all evaluations on h->stream; with `as_job` the sweep comes from device memory (graph capture, or a count
 * in device memory), `capture`: inside a stream capture */
static lv_status enqueue_update_kernels(lv_context* h, const float* d_xyz, int64_t n, bool as_job, bool capture, const UpdateGate& gate);

static lv_status build_update_graph(lv_context* h, int64_t cap, lv_context::UpdateGraph* out) {
    cudaGraph_t graph = nullptr;
    LV_CUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    lv_status s = enqueue_update_kernels(h, nullptr, cap, true, true, UpdateGate());
    cudaError_t e = cudaStreamEndCapture(h->stream, &graph);
    if (s != LV_OK || e != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return LV_ERR_CUDA; }
        return s;
    }
    out->cap = cap;
    out->graph = graph;                 /* kept: the node handles below belong to it */
    LV_CUDA(cudaGraphInstantiate(&out->exec, graph, 0));
    /* the one node patched per launch is the begin kernel (sweep pointer and size); the measurement kernels' arguments
     * embed the map view, which never changes over the life of a handle (tables and arena are allocated once) */
    size_t n_nodes = 0;
    LV_CUDA(cudaGraphGetNodes(graph, nullptr, &n_nodes));
    std::vector<cudaGraphNode_t> nodes(n_nodes);
    LV_CUDA(cudaGraphGetNodes(graph, nodes.data(), &n_nodes));
    out->begin_node = nullptr;
    for (cudaGraphNode_t nd : nodes) {
        cudaGraphNodeType t;
        LV_CUDA(cudaGraphNodeGetType(nd, &t));
        if (t != cudaGraphNodeTypeKernel) continue;
        cudaKernelNodeParams kp;
        LV_CUDA(cudaGraphKernelNodeGetParams(nd, &kp));
        if (kp.func == ieskf_begin_kernel_ptr()) out->begin_node = nd;
    }
    if (!out->begin_node) { set_error("update graph: begin node not found"); return LV_ERR_CUDA; }
    return LV_OK;
}

/* n: the sweep's points, or with gate.n the host bound of its device count (the graph bucket is chosen by it) */
static lv_status enqueue_update(lv_context* h, const float* d_xyz, int64_t n, UpdateGate gate) {
    const lv_status s = sync_device_state(h);
    if (s != LV_OK) return s;
    if (h->profile || !h->use_graph) return enqueue_update_kernels(h, d_xyz, n, gate.n != nullptr, false, gate);
    int64_t cap = 4096;
    while (cap < n) cap <<= 1;
    if (cap > h->prm.max_points) cap = h->prm.max_points;
    lv_context::UpdateGraph* g = nullptr;
    for (auto& u : h->graphs) if (u.cap == cap) g = &u;
    if (!g) {
        lv_context::UpdateGraph u;
        lv_status s = build_update_graph(h, cap, &u);
        if (s != LV_OK) return s;
        h->graphs.push_back(u);
        g = &h->graphs.back();
    }
    UpdateCtrl* c = h->d_ctrl;
    MeasureJob* job = h->d_job;
    int n32 = (int)n;
    uint32_t* counters = h->d_hard_list + (size_t)kHardBuckets * hard_segment(h->prm.max_points);
    void* args[6] = {&c, &job, &d_xyz, &n32, &counters, &gate};
    cudaKernelNodeParams kp = {};
    kp.func = const_cast<void*>(ieskf_begin_kernel_ptr());
    kp.gridDim = dim3(1, 1, 1);
    kp.blockDim = dim3(256, 1, 1);
    kp.kernelParams = args;
    LV_CUDA(cudaGraphExecKernelNodeSetParams(g->exec, g->begin_node, &kp));
    LV_CUDA(cudaGraphLaunch(g->exec, h->stream));
    h->prof.total_launches += 1 + 4 * (h->prm.MAX_NUM_ITERS + 1) + (h->use_reuse ? h->prm.MAX_NUM_ITERS : 0);
    return LV_OK;
}

static lv_status enqueue_update_kernels(lv_context* h, const float* d_xyz, int64_t n, bool as_job, bool capture, const UpdateGate& gate) {
    const int pdl = (h->use_pdl && !h->profile) ? 1 : 0;
    uint32_t* counters = h->d_hard_list + (size_t)kHardBuckets * hard_segment(h->prm.max_points);
    LV_CUDA(launch_ieskf_begin(h->d_ctrl, as_job ? h->d_job.get() : nullptr, d_xyz, (int)n, counters, gate, h->stream));
    if (!capture) h->prof.total_launches += 1;
    MeasureArgs a = update_measure_args(h, d_xyz, n, as_job);
    const int grid = measure_grid((int)n);
    for (int e = 0; e <= h->prm.MAX_NUM_ITERS; ++e) {            /* i = -1 .. max_iter-1, esekfom.hpp:1634 */
        EventPair ep;
        bool pr;
        LV_CUDA(launch_measure_timed(h, a, grid, capture ? 0 : 1, e /* evaluation index: > 0 = reuse + work list */, (int)(h->update_seq % kNevalsRing), e, pdl));
        pr = prof_begin(h, kProfSolve, &ep);
        ep.upd = (int)(h->update_seq % kNevalsRing); ep.slot = e;
        LV_CUDA(launch_ieskf_step(h->d_ctrl, h->iprm, h->d_group_rows, partial_groups(grid), h->stream, pdl));
        if (pr) prof_end(h, &ep);
        if (!capture) h->prof.total_launches += 4 + ((e > 0 && h->use_reuse) ? 1 : 0);
    }
    if (h->profile) {
        LV_CUDA(cudaMemcpyAsync(&h->h_nevals[h->update_seq % kNevalsRing], &h->d_ctrl->n_evals, sizeof(int32_t),
                                cudaMemcpyDeviceToHost, h->stream));
        h->update_seq++;
    }
    return LV_OK;
}

/* settles map_unknown (an async first build the gate may have left without points) from the map counters, which are fetched
 * first unless they are already on the host (on_host) */
static lv_status settle_map_unknown(lv_context* h, bool on_host) {
    if (!h->map_unknown) return LV_OK;
    if (!on_host) {
        LV_CUDA(map_fetch_counters(h->map, h->stream));
        LV_CUDA(cudaStreamSynchronize(h->stream));
    }
    if ((int32_t)h->map.h_counters[kCtrPoints] == 0) h->map.empty = true;
    h->map_unknown = false;
    return LV_OK;
}

static lv_status fetch_results(lv_context* h) {
    LV_CUDA(cudaMemcpyAsync(h->h_ctrl, h->d_ctrl, sizeof(UpdateCtrl), cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(map_fetch_counters(h->map, h->stream));       /* 64 bytes: the map's error flags ride along */
    if (h->time_pending) {                                /* what the async updates decided about last_time_updated */
        LV_CUDA(cudaMemcpyAsync(h->h_async, h->d_async, sizeof(AsyncWords), cudaMemcpyDeviceToHost, h->stream));
        LV_CUDA(cudaMemsetAsync(&h->d_async->time_set, 0, sizeof(int32_t), h->stream));
    }
    LV_CUDA(cudaStreamSynchronize(h->stream));
    if (h->time_pending) {
        if (h->h_async->time_set) h->last_time_updated = h->h_async->time_updated;
        h->time_pending = false;
    }
    settle_map_unknown(h, true);                          /* LV_OK: the counters came with the results */
    const UpdateCtrl* c = h->h_ctrl;
    memcpy(h->x, c->x, sizeof(h->x));
    /* a gated update (LV_TOO_FEW_POINTS, or LV_EMPTY_MAP found on the device) leaves P as it was on the device, which may be
     * newer than the mirror (lv_propagate_device) */
    if (c->status == LV_OK || c->status == LV_TOO_FEW_POINTS || c->status == LV_EMPTY_MAP) memcpy(h->P, c->P, sizeof(h->P));
    h->n_evals = c->n_evals;
    memcpy(h->logs, c->logs, sizeof(h->logs));
    h->last_status = c->status;
    h->state_dirty = false;
    h->pending_fetch = false;
    if (c->status == LV_OK && map_status_from_mirror(h) != LV_OK) return LV_ERR_CAPACITY;
    return (lv_status)c->status;
}

/* Localizator::correct (Localizator.cpp:22-27) enqueued, every form: the sweep's n points, or with d_n its device count (n is
 * then the bound) and the MAX_POINTS2MATCH gate min_points (main.cpp:81).  The sweep is recorded even on an empty map: the
 * first tick's lv_map_add_last_sweep builds the map from it.  Who decides last_time_updated: with `fetched` (lv_correct, which
 * fetches the results at once) the caller, from the status; otherwise the host now, unless only the device knows whether the
 * update runs (a device count, or a map an async build may have left without points): then the device, read at the next fetch. */
static lv_status correct_enqueue(lv_context* h, const float* d_xyz, int64_t n, const int64_t* d_n, int64_t min_points, double time,
                                 bool fetched) {
    h->tick = {d_xyz, n, d_n, min_points};
    if (h->map.empty) return LV_EMPTY_MAP;                        /* Localizator.cpp:24: the state is left as it is */
    LV_CUDA(cudaSetDevice(h->prm.device));
    UpdateGate gate;
    gate.n = d_n;
    gate.min_points = min_points;
    if (h->map_unknown) gate.map_counters = h->map.counters;      /* an async build may have added nothing */
    const bool device_time = d_n || (h->map_unknown && !fetched);
    if (device_time) {
        gate.words = h->d_async;
        gate.time = time;
    } else if (!fetched && h->time_pending) {                     /* this time supersedes what an earlier async update recorded */
        LV_CUDA(cudaMemsetAsync(&h->d_async->time_set, 0, sizeof(int32_t), h->stream));
    }
    const lv_status s = enqueue_update(h, d_xyz, n, gate);
    if (fetched) return s;
    h->time_pending = device_time;
    if (!device_time) h->last_time_updated = time;
    h->pending_fetch = true;
    return s;
}

lv_status lv_correct(lv_handle h, const float* xyz, int64_t n, double time, lv_iter_log* logs, int32_t* n_evals,
                     double* x_out, double* P_out) {
    if (!h || !xyz || n <= 0) return LV_ERR_ARG;
    if (n_evals) *n_evals = 0;
    if (n > h->prm.max_points) { set_error("sweep capacity exceeded"); return LV_ERR_CAPACITY; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaMemcpyAsync(h->d_sweep, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
    lv_status s = correct_enqueue(h, h->d_sweep, n, nullptr, 0, time, true);
    if (s != LV_OK) return s;
    s = fetch_results(h);
    if (s != LV_EMPTY_MAP) h->last_time_updated = time;          /* Localizator.cpp:26 (LV_EMPTY_MAP: an async build added nothing) */
    if (logs) memcpy(logs, h->logs, sizeof(lv_iter_log) * (size_t)h->n_evals);
    if (n_evals) *n_evals = h->n_evals;
    if (x_out) memcpy(x_out, h->x, sizeof(h->x));
    if (P_out) memcpy(P_out, h->P, sizeof(h->P));
    return s;
}

lv_status lv_correct_device(lv_handle h, const float* d_xyz, int64_t n, double time) {
    if (!h || !d_xyz || n <= 0) return LV_ERR_ARG;
    return correct_enqueue(h, d_xyz, n, nullptr, 0, time, false);
}

lv_status lv_correct_device_async(lv_handle h, const float* d_xyz, const int64_t* d_n, int64_t n_max, int64_t min_points, double time) {
    if (!d_xyz || !d_n) { set_error("correct async: null sweep or count"); return LV_ERR_ARG; }
    if (!n_max_ok("correct async", n_max)) return LV_ERR_ARG;
    if (min_points < 0) { set_error("correct async: negative min_points"); return LV_ERR_ARG; }
    if (!handle_ok("correct async", h, n_max)) return LV_ERR_ARG;
    return correct_enqueue(h, d_xyz, n_max, d_n, min_points, time, false);
}

lv_status lv_last_logs(lv_handle h, lv_iter_log* logs, int32_t* n_evals) {
    if (!h) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    lv_status s = fetch_results(h);
    if (logs) memcpy(logs, h->logs, sizeof(lv_iter_log) * (size_t)h->n_evals);
    if (n_evals) *n_evals = h->n_evals;
    return s;
}

/* ---- operator boundary ----------------------------------------------------------------------- */
static lv_status run_measure_once(lv_context* h, const double* x, const float* xyz, int64_t n, bool want_rows,
                                  bool want_debug) {
    if (n > h->prm.max_points) { set_error("sweep capacity exceeded"); return LV_ERR_CAPACITY; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaMemcpyAsync(h->d_sweep, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
    lv_status s = upload_state(h, x, nullptr);
    if (s != LV_OK) return s;
    h->state_dirty = true;   /* d_ctrl->x no longer mirrors the filter */
    LV_CUDA(launch_set_frame(h->d_ctrl, h->stream));
    MeasureArgs a = make_measure_args(h, h->d_sweep, n);
    const size_t mp = (size_t)h->prm.max_points;
    if (want_rows) { LV_CUDA(h->d_rows.reserve(13 * mp)); LV_CUDA(h->d_valid.reserve(mp)); a.rows = h->d_rows; a.valid = h->d_valid; }
    if (want_debug) {
        LV_CUDA(h->d_valid.reserve(mp)); LV_CUDA(h->d_nn_idx.reserve(5 * mp)); LV_CUDA(h->d_nn_sqd.reserve(5 * mp));
        LV_CUDA(h->d_plane.reserve(4 * mp)); LV_CUDA(h->d_dist.reserve(mp)); LV_CUDA(h->d_gworld.reserve(3 * mp));
        a.valid = h->d_valid; a.nn_idx = h->d_nn_idx; a.nn_sqd = h->d_nn_sqd; a.plane = h->d_plane; a.dist = h->d_dist;
        a.g_world = h->d_gworld;
    }
    const int grid = measure_grid((int)n);
    LV_CUDA(launch_measure_timed(h, a, grid, 1, 0, -1, 0));
    LV_CUDA(launch_reduce_partials(h->d_group_rows, partial_groups(grid), h->d_reduced, h->stream));
    LV_CUDA(cudaMemcpyAsync(h->h_reduced, h->d_reduced, sizeof(double) * 157, cudaMemcpyDeviceToHost, h->stream));
    h->prof.total_launches += 5;
    return LV_OK;
}

lv_status lv_measure_reduced(lv_handle h, const double* x, const float* xyz, int64_t n, double* HTH, double* HTh,
                             int64_t* nm) {
    if (!h || !x || !xyz || n <= 0) return LV_ERR_ARG;
    if (nm) *nm = 0;
    if (h->map.empty) return LV_EMPTY_MAP;
    lv_status s = run_measure_once(h, x, xyz, n, false, false);
    if (s != LV_OK) return s;
    LV_CUDA(cudaStreamSynchronize(h->stream));
    if (HTH) memcpy(HTH, h->h_reduced, sizeof(double) * 144);
    if (HTh) memcpy(HTh, h->h_reduced + 144, sizeof(double) * 12);
    if (nm) *nm = (int64_t)h->h_reduced[156];
    return LV_OK;
}

lv_status lv_measure(lv_handle h, const double* x, const float* xyz, int64_t n, double* h_x, double* h_vec, int64_t* nm) {
    if (!h || !x || !xyz || n <= 0 || !nm) return LV_ERR_ARG;
    *nm = 0;
    if (h->map.empty) return LV_EMPTY_MAP;
    lv_status s = run_measure_once(h, x, xyz, n, true, false);
    if (s != LV_OK) return s;
    std::vector<double> rows(13 * (size_t)n);
    std::vector<uint8_t> valid((size_t)n);
    LV_CUDA(cudaMemcpyAsync(rows.data(), h->d_rows, sizeof(double) * 13 * n, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaMemcpyAsync(valid.data(), h->d_valid, (size_t)n, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    /* compaction in input order = the single-thread order of Mapper::match (Mapper.cpp:46-53);
     * layout: column-major Nm x 12 like Eigen::MatrixXd (Localizator.cpp:31) */
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; ++i) cnt += valid[i] ? 1 : 0;
    int64_t k = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (!valid[i]) continue;
        if (h_x)
            for (int c = 0; c < 12; ++c) h_x[(size_t)c * cnt + k] = rows[13 * (size_t)i + c];
        if (h_vec) h_vec[k] = rows[13 * (size_t)i + 12];
        ++k;
    }
    *nm = cnt;
    return LV_OK;
}

lv_status lv_match_all(lv_handle h, const double* x, const float* xyz, int64_t n, uint8_t* valid, int32_t* nn_idx,
                       float* nn_sqd, float* plane, float* dist, float* g_world) {
    if (!h || !x || !xyz || n <= 0) return LV_ERR_ARG;
    if (h->map.empty) return LV_EMPTY_MAP;
    lv_status s = run_measure_once(h, x, xyz, n, false, true);
    if (s != LV_OK) return s;
    if (valid) LV_CUDA(cudaMemcpyAsync(valid, h->d_valid, (size_t)n, cudaMemcpyDeviceToHost, h->stream));
    if (nn_idx) LV_CUDA(cudaMemcpyAsync(nn_idx, h->d_nn_idx, sizeof(int32_t) * 5 * n, cudaMemcpyDeviceToHost, h->stream));
    if (nn_sqd) LV_CUDA(cudaMemcpyAsync(nn_sqd, h->d_nn_sqd, sizeof(float) * 5 * n, cudaMemcpyDeviceToHost, h->stream));
    if (plane) LV_CUDA(cudaMemcpyAsync(plane, h->d_plane, sizeof(float) * 4 * n, cudaMemcpyDeviceToHost, h->stream));
    if (dist) LV_CUDA(cudaMemcpyAsync(dist, h->d_dist, sizeof(float) * n, cudaMemcpyDeviceToHost, h->stream));
    if (g_world) LV_CUDA(cudaMemcpyAsync(g_world, h->d_gworld, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return LV_OK;
}


/* the neighbours the LAST evaluation of the last update (or operator call) handed to the plane fit, as map point ids:
 * after an update with neighbour reuse these are the stored five where lv_reuse_kernel vouched for them and the fresh
 * search's elsewhere — what lv_match_all (always a fresh search) cannot show */
__global__ void lv_neighbour_ids_kernel(const int4* nn_a, const int2* nn_b, const float4* arena, int n, int32_t* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int4 a = nn_a[i];
    const int2 b = nn_b[i];
    const int id[5] = {a.x, a.y, a.z, a.w, b.x};
    for (int k = 0; k < 5; ++k) out[5 * i + k] = (b.x >= 0 && id[k] >= 0) ? __float_as_int(arena[id[k]].w) : -1;
}
lv_status lv_last_neighbours(lv_handle h, int64_t n, int32_t* nn_idx) {
    if (!h || !nn_idx || n <= 0 || n > h->prm.max_points) return LV_ERR_ARG;
    if (h->map.empty) return LV_EMPTY_MAP;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(h->d_nn_idx.reserve(5 * (size_t)h->prm.max_points));
    lv_neighbour_ids_kernel<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(h->d_nn_a, h->d_nn_b, h->map.arena, (int)n, h->d_nn_idx);
    LV_CUDA(cudaGetLastError());
    LV_CUDA(cudaMemcpyAsync(nn_idx, h->d_nn_idx, sizeof(int32_t) * 5 * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return LV_OK;
}

/* ---- start pose in a saved map (lv_prelocalize, and the host path both searches share) -------- */
/* NULL when p is valid (I, K and the candidate count filled in), else what is wrong with it */
static const char* preloc_params_error(const lv_preloc_params* p, int64_t* I, int64_t* K, int64_t* count) {
    if (!(p->radius >= 0.f && p->radius <= 3.402823466e38f)) return "radius outside [0, inf)";
    if (!(p->step > 0.f && p->step <= 3.402823466e38f)) return "step not a positive finite number";
    if (!(p->yaw_range >= 0.f && p->yaw_range <= 3.14159274f)) return "yaw_range outside [0, pi]";
    if (!(p->yaw_step > 0.f && p->yaw_step <= 3.402823466e38f)) return "yaw_step not a positive finite number";
    if (p->max_points < 1 || p->max_points > kPrelocMaxPoints) return "max_points outside [1, 4096]";
    const double hi = preloc_half(p->radius, p->step), hk = preloc_half(p->yaw_range, p->yaw_step);
    if ((2.0 * hk + 1.0) * (2.0 * hi + 1.0) * (2.0 * hi + 1.0) > 2305843009213693952.0) return "more than 2^61 candidates";
    *I = (int64_t)hi;
    *K = (int64_t)hk;
    *count = (2 * *K + 1) * (2 * *I + 1) * (2 * *I + 1);
    return nullptr;
}
int64_t lv_preloc_count(const lv_preloc_params* p) {
    int64_t I, K, c;
    if (!p || preloc_params_error(p, &I, &K, &c)) return -1;
    return c;
}
/* the argument checks of both searches, `what` prefixing the messages: LV_OK with I, K and the candidate count filled in when
 * there are at most max_candidates (a power of two) */
static lv_status preloc_args(const std::string& what, const float* d_xyz, int64_t n, const lv_preloc_params* p, const lv_preloc_result* out,
                             int64_t max_candidates, int64_t* I, int64_t* K, int64_t* count) {
    if (!p || !out || !d_xyz) { set_error(what + ": null params, result or points"); return LV_ERR_ARG; }
    if (n < 1 || n > 0x7fffffff) { set_error(what + ": n outside [1, 2^31 - 1]"); return LV_ERR_ARG; }
    if (const char* e = preloc_params_error(p, I, K, count)) { set_error(what + ": " + e); return LV_ERR_ARG; }
    if (*count > max_candidates) {
        set_error(what + ": " + std::to_string((long long)*count) + " candidates, more than 2^" + std::to_string(__builtin_ctzll(max_candidates)));
        return LV_ERR_ARG;
    }
    return LV_OK;
}
/* the handle's checks of both searches, after the argument checks: LV_OK with the base state (what lv_get_state returns) in h->x
 * and a map that holds points */
static lv_status preloc_ready(lv_context* h, const std::string& what) {
    if (!h) { set_error(what + ": null handle"); return LV_ERR_ARG; }
    if (h->map.empty) { set_error(what + ": the map is empty"); return LV_EMPTY_MAP; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    sync_mirror(h);
    if (lv_status s = settle_map_unknown(h, false)) return s;
    if (h->map.empty) { set_error(what + ": the map is empty"); return LV_EMPTY_MAP; }
    return LV_OK;
}
/* one frame per heading k = -K..K about the base state: R (9 floats), then t (3) */
static std::vector<float> preloc_frames(const double* x, const PrelocAxes& ax, int64_t K, float yaw_step) {
    std::vector<float> frames((size_t)(2 * K + 1) * 12);
    for (int64_t k = -K; k <= K; ++k) {
        const Rt32 F = preloc_heading_frame(x, ax, (double)k * (double)yaw_step);
        memcpy(&frames[(size_t)(k + K) * 12], F.R, sizeof(float) * 9);
        memcpy(&frames[(size_t)(k + K) * 12 + 9], F.t, sizeof(float) * 3);
    }
    return frames;
}
/* the winning candidate (index idx in heading-major order, its score over S points) into out and into the state, as
 * lv_set_state(out->x, NULL) */
static void preloc_finish(lv_context* h, const lv_preloc_params* p, int64_t I, int64_t K, int64_t count, int64_t idx, int32_t score,
                          int32_t S, lv_preloc_result* out) {
    const int64_t W = 2 * I + 1, P = W * W, hk = idx / P, q = idx % P;
    memset(out, 0, sizeof(*out));
    out->candidates = count;
    out->index = idx;
    out->k = (int32_t)(hk - K);
    out->i = (int32_t)(q / W - I);
    out->j = (int32_t)(q % W - I);
    out->score = score;
    out->points = S;
    preloc_candidate(h->x, preloc_axes(h->x), (double)out->k * (double)p->yaw_step, (double)out->i * (double)p->step,
                     (double)out->j * (double)p->step, out->x);
    memcpy(h->x, out->x, sizeof(h->x));
    h->state_dirty = true;
}
lv_status lv_prelocalize(lv_handle h, const float* d_xyz_lidar, int64_t n, const lv_preloc_params* p, lv_preloc_result* out,
                         int32_t* scores_out) {
    int64_t I = 0, K = 0, count = 0;
    if (lv_status s = preloc_args("prelocalize", d_xyz_lidar, n, p, out, LV_PRELOC_MAX_CANDIDATES, &I, &K, &count)) return s;
    if (lv_status s = preloc_ready(h, "prelocalize")) return s;

    const int64_t H = 2 * K + 1, W = 2 * I + 1, P = W * W;
    const int32_t S = (int32_t)(n < p->max_points ? n : p->max_points);
    const PrelocAxes ax = preloc_axes(h->x);
    const std::vector<float> frames = preloc_frames(h->x, ax, K, p->yaw_step);
    std::vector<float4> offsets((size_t)P);
    for (int64_t i = -I; i <= I; ++i)
        for (int64_t j = -I; j <= I; ++j) {
            float o[3];
            preloc_offset(ax, (double)i * (double)p->step, (double)j * (double)p->step, o);
            offsets[(size_t)((i + I) * W + (j + I))] = make_float4(o[0], o[1], o[2], 0.f);
        }
    /* scratch: key (256 B slot), frames, offsets, scores */
    const size_t off_frames = 256, off_offsets = (off_frames + sizeof(float) * frames.size() + 255) & ~(size_t)255;
    const size_t off_scores = (off_offsets + sizeof(float4) * offsets.size() + 255) & ~(size_t)255;
    const size_t bytes = off_scores + (scores_out ? sizeof(int32_t) * (size_t)count : 0);
    LV_CUDA(h->d_preloc.reserve(bytes));
    uint8_t* base = h->d_preloc;
    PrelocArgs a;
    a.xyz = d_xyz_lidar;
    a.n = n;
    a.S = S;
    a.I = I;
    a.K = K;
    a.headings = H;
    a.positions = P;
    a.frames = reinterpret_cast<const float*>(base + off_frames);
    a.offsets = reinterpret_cast<const float4*>(base + off_offsets);
    a.map = map_view(h->map);
    a.scores = scores_out ? reinterpret_cast<int32_t*>(base + off_scores) : nullptr;
    a.best = reinterpret_cast<unsigned long long*>(base);
    LV_CUDA(cudaMemcpyAsync(base + off_frames, frames.data(), sizeof(float) * frames.size(), cudaMemcpyHostToDevice, h->stream));
    LV_CUDA(cudaMemcpyAsync(base + off_offsets, offsets.data(), sizeof(float4) * offsets.size(), cudaMemcpyHostToDevice, h->stream));
    LV_CUDA(cudaMemsetAsync(base, 0, sizeof(unsigned long long), h->stream));
    int launches = 0;
    LV_CUDA(launch_preloc(a, h->stream, &launches));
    h->prof.total_launches += launches;
    unsigned long long key = 0;
    LV_CUDA(cudaMemcpyAsync(&key, base, sizeof(key), cudaMemcpyDeviceToHost, h->stream));
    if (scores_out) LV_CUDA(cudaMemcpyAsync(scores_out, a.scores, sizeof(int32_t) * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    preloc_finish(h, p, I, K, count, preloc_key_index(key), preloc_key_score(key), S, out);
    return LV_OK;
}

/* ---- start pose anywhere in a saved map (lv_prelocalize_global, lv_map_extent) ---------------- */
static size_t pglob_align(size_t b) { return (b + 255) & ~(size_t)255; }
/* the occupancy summary of the map (h->occ: extent, bitmap pyramid in h->d_occ), rebuilt only when the map changed since it
 * was built (map_gen); LV_EMPTY_MAP when no block holds an occupied voxel */
static lv_status pglob_occupancy(lv_context* h, const char* what, int* launches) {
    if (h->occ_gen != h->map_gen) {
        LV_CUDA(h->d_occ.reserve(64));
        uint32_t ext[6];
        LV_CUDA(cudaMemsetAsync(h->d_occ, 0xFF, 3 * sizeof(uint32_t), h->stream));
        LV_CUDA(cudaMemsetAsync(h->d_occ + 3, 0, 3 * sizeof(uint32_t), h->stream));
        LV_CUDA(launch_occ_extent(map_view(h->map), h->map.bslots, h->d_occ, h->stream, launches));
        LV_CUDA(cudaMemcpyAsync(ext, h->d_occ, 6 * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
        LV_CUDA(cudaStreamSynchronize(h->stream));
        PrelocOcc& o = h->occ;
        memset(&o, 0, sizeof(o));
        for (int a = 0; a < 3; ++a) { o.lo[a] = ext[a]; o.hi[a] = ext[3 + a]; }
        if (ext[0] <= ext[3]) {
            const size_t words = (size_t)occ_layout(o);
            LV_CUDA(h->d_occ.reserve(64 + words));                 /* a growth loses the extent: copied out above */
            uint32_t* bits = h->d_occ + 64;
            o.map = map_view(h->map);
            o.bits = bits;
            LV_CUDA(cudaMemsetAsync(bits, 0, sizeof(uint32_t) * words, h->stream));
            LV_CUDA(launch_occ_bits(o, h->map.bslots, bits, h->stream, launches));
        }
        h->occ_gen = h->map_gen;
    }
    if (h->occ.lo[0] > h->occ.hi[0]) { set_error(std::string(what) + ": the map is empty"); return LV_EMPTY_MAP; }
    h->occ.map = map_view(h->map);
    return LV_OK;
}

lv_status lv_map_extent(lv_handle h, double lo[3], double hi[3]) {
    if (!h) { set_error("map_extent: null handle"); return LV_ERR_ARG; }
    if (!lo || !hi) { set_error("map_extent: null lo or hi"); return LV_ERR_ARG; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    if (lv_status s = settle_map_unknown(h, false)) return s;
    if (h->map.empty) { set_error("map_extent: the map is empty"); return LV_EMPTY_MAP; }
    int launches = 0;
    const lv_status s = pglob_occupancy(h, "map_extent", &launches);
    h->prof.total_launches += launches;
    if (s != LV_OK) return s;
    for (int a = 0; a < 3; ++a) {
        lo[a] = (double)voxel_low(h->map.grid, h->occ.lo[a]);
        hi[a] = (double)voxel_low(h->map.grid, h->occ.hi[a] + 1);
    }
    return LV_OK;
}

namespace {
/* PrelocSearch's evaluator on the device: one launch per call, the results read back (the schedule decides on the host) */
struct DevicePrelocEval {
    cudaStream_t st;
    PrelocGlobalArgs a;
    PrelocCell* d_cells;
    int32_t* d_bounds;
    PrelocBest* d_best;
    cudaError_t err;
    int launches;
    void bounds(const PrelocCell* c, int64_t n, int32_t* out) {
        if (err == cudaSuccess) err = cudaMemcpyAsync(d_cells, c, sizeof(PrelocCell) * (size_t)n, cudaMemcpyHostToDevice, st);
        a.cells = d_cells;
        a.count = n;
        if (err == cudaSuccess) err = launch_preloc_bounds(a, st, &launches);
        if (err == cudaSuccess) err = cudaMemcpyAsync(out, d_bounds, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, st);
        if (err == cudaSuccess) err = cudaStreamSynchronize(st);
        if (err != cudaSuccess) std::fill(out, out + n, -2);        /* below any score: the search winds down */
    }
    void exact(const PrelocCell* c, int64_t n, PrelocBest* out) {
        if (err == cudaSuccess) err = cudaMemcpyAsync(d_cells, c, sizeof(PrelocCell) * (size_t)n, cudaMemcpyHostToDevice, st);
        a.cells = d_cells;
        a.count = n;
        if (err == cudaSuccess) err = launch_preloc_exact(a, st, &launches);
        if (err == cudaSuccess) err = cudaMemcpyAsync(out, d_best, sizeof(PrelocBest) * (size_t)n, cudaMemcpyDeviceToHost, st);
        if (err == cudaSuccess) err = cudaStreamSynchronize(st);
        if (err != cudaSuccess)
            for (int64_t t = 0; t < n; ++t) { out[t].score = -1; out[t].pad_ = 0; out[t].tie = 0; out[t].idx = 0; }
    }
};
}  // namespace

lv_status lv_prelocalize_global(lv_handle h, const float* d_xyz_lidar, int64_t n, const lv_preloc_params* p, lv_preloc_result* out,
                                lv_preloc_stats* stats) {
    int64_t I = 0, K = 0, count = 0;
    if (lv_status s = preloc_args("prelocalize_global", d_xyz_lidar, n, p, out, LV_PRELOC_GLOBAL_MAX_CANDIDATES, &I, &K, &count)) return s;
    if (2 * K + 1 > kPrelocMaxTopCells) {
        set_error("prelocalize_global: " + std::to_string((long long)(2 * K + 1)) + " headings, more than 2^20");
        return LV_ERR_ARG;
    }
    if (lv_status s = preloc_ready(h, "prelocalize_global")) return s;

    int launches = 0;
    {
        const lv_status s = pglob_occupancy(h, "prelocalize_global", &launches);
        h->prof.total_launches += launches;
        if (s != LV_OK) return s;
    }
    const PrelocOcc occ = h->occ;
    const int32_t S = (int32_t)(n < p->max_points ? n : p->max_points);
    const PrelocAxes ax = preloc_axes(h->x);
    const std::vector<float> frames = preloc_frames(h->x, ax, K, p->yaw_step);
    /* scratch: frames, cells, bounds, best */
    const size_t off_frames = 0, off_cells = pglob_align(off_frames + sizeof(float) * frames.size());
    const size_t off_bounds = pglob_align(off_cells + sizeof(PrelocCell) * kPrelocChunk);
    const size_t off_best = pglob_align(off_bounds + sizeof(int32_t) * kPrelocChunk);
    LV_CUDA(h->d_pglob.reserve(off_best + sizeof(PrelocBest) * kPrelocChunk));
    uint8_t* base = h->d_pglob;
    LV_CUDA(cudaMemcpyAsync(base + off_frames, frames.data(), sizeof(float) * frames.size(), cudaMemcpyHostToDevice, h->stream));

    DevicePrelocEval ev;
    ev.st = h->stream;
    memset(&ev.a, 0, sizeof(ev.a));
    ev.a.xyz = d_xyz_lidar;
    ev.a.n = n;
    ev.a.S = S;
    ev.a.step = p->step;
    ev.a.I = I;
    ev.a.K = K;
    ev.a.ax = ax;
    ev.a.frames = reinterpret_cast<const float*>(base + off_frames);
    ev.a.occ = occ;
    ev.a.bounds = reinterpret_cast<int32_t*>(base + off_bounds);
    ev.a.best = reinterpret_cast<PrelocBest*>(base + off_best);
    ev.d_cells = reinterpret_cast<PrelocCell*>(base + off_cells);
    ev.d_bounds = ev.a.bounds;
    ev.d_best = ev.a.best;
    ev.err = cudaSuccess;
    ev.launches = 0;
    const char* np = getenv("LV_PRELOC_NO_PRUNE");
    PrelocSearch<DevicePrelocEval> search(ev, I, K, S, !(np && np[0] == '1'));
    try {
        search.run();
    } catch (const std::bad_alloc&) {                             /* the cell lists are host vectors */
        h->prof.total_launches += ev.launches;
        set_error("prelocalize_global: out of host memory for the cell lists");
        return LV_ERR_CAPACITY;
    }
    h->prof.total_launches += ev.launches;
    LV_CUDA(ev.err);

    if (stats) {
        memset(stats, 0, sizeof(*stats));
        stats->candidates = search.st.candidates;
        stats->cells_bounded = search.st.cells_bounded;
        stats->candidates_scored = search.st.candidates_scored;
        stats->probes = search.st.probes;
        stats->launches = search.st.launches;
    }
    preloc_finish(h, p, I, K, count, search.best.idx, search.best.score, S, out);
    return LV_OK;
}

/* ---- utilities ------------------------------------------------------------------------------- */
void* lv_host_alloc(int64_t bytes) {
    void* p = nullptr;
    if (bytes <= 0 || cudaMallocHost(&p, (size_t)bytes) != cudaSuccess) return nullptr;
    return p;
}
void lv_host_free(void* p) { if (p) cudaFreeHost(p); }
void* lv_device_alloc(lv_handle h, int64_t bytes) {
    if (!h || bytes <= 0) return nullptr;
    void* p = nullptr;
    cudaSetDevice(h->prm.device);
    if (cudaMalloc(&p, (size_t)bytes) != cudaSuccess) return nullptr;
    return p;
}
void lv_device_free(lv_handle h, void* p) { if (h && p) { cudaSetDevice(h->prm.device); cudaFree(p); } }
lv_status lv_memcpy_h2d(lv_handle h, void* dst, const void* src, int64_t bytes) {
    if (!h || !dst || !src || bytes < 0) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyHostToDevice, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return LV_OK;
}
lv_status lv_memcpy_d2h(lv_handle h, void* dst, const void* src, int64_t bytes) {
    if (!h || !dst || !src || bytes < 0) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return LV_OK;
}
/* ---- Compensator::compensate ------------------------------------------------------------------ */
/* d_n: NULL (n points, the flag is read back into h_bad) or the device count of the async form (n is its bound) */
static lv_status deskew_common(lv_context* h, const lv_state32* path, int32_t ns, const lv_state32* Xt2,
                               const float* d_xyz, const double* d_t, const int64_t* d_n, int64_t n, float* d_out) {
    LV_CUDA(h->d_path.reserve(deskew_max_states()));
    LV_CUDA(h->h_path.reserve(deskew_max_states()));
    LV_CUDA(h->d_bad.reserve(1));
    LV_CUDA(h->h_bad.reserve(1));
    /* the pinned staging buffer is reused: the copy out of it queued by an earlier async call must have run */
    LV_CUDA(cudaEventSynchronize(h->path_copied));
    memcpy(h->h_path, path, sizeof(lv_state32) * (size_t)ns);
    LV_CUDA(cudaMemcpyAsync(h->d_path, h->h_path, sizeof(lv_state32) * (size_t)ns, cudaMemcpyHostToDevice, h->stream));
    LV_CUDA(cudaEventRecord(h->path_copied, h->stream));
    LV_CUDA(launch_deskew(h->d_path, ns, *Xt2, path[0].time, path[ns - 1].time, d_xyz, d_t, d_n, n, d_out, h->d_bad,
                          d_n ? &h->d_async->err : nullptr, h->stream));
    if (!d_n) LV_CUDA(cudaMemcpyAsync(h->h_bad, h->d_bad, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    h->prof.total_launches += 2;
    return LV_OK;
}
/* the path's checks, with the sweep's capacity between them (the async form has checked n against max_points already) */
static lv_status deskew_path_ok(const lv_context* h, const lv_state32* path, int32_t ns, int64_t n) {
    if (ns > deskew_max_states()) { set_error("deskew path too long"); return LV_ERR_CAPACITY; }
    if (n > h->prm.max_points) { set_error("sweep capacity exceeded"); return LV_ERR_CAPACITY; }
    for (int32_t s = 1; s < ns; ++s)
        if (!(path[s - 1].time <= path[s].time)) { set_error("deskew path not sorted by time"); return LV_ERR_ARG; }
    return LV_OK;
}
static lv_status deskew_args_ok(const lv_context* h, const lv_state32* path, int32_t ns, const lv_state32* Xt2, const void* a,
                                const void* b, int64_t n, const void* c) {
    if (!h || !path || !Xt2 || !a || !b || !c || n <= 0 || ns < 2) return LV_ERR_ARG;
    return deskew_path_ok(h, path, ns, n);
}
lv_status lv_compensate_device(lv_handle h, const lv_state32* path, int32_t ns, const lv_state32* Xt2,
                               const float* d_xyz, const double* d_t, int64_t n, float* d_xyz_out) {
    lv_status s = deskew_args_ok(h, path, ns, Xt2, d_xyz, d_t, n, d_xyz_out);
    if (s != LV_OK) return s;
    LV_CUDA(cudaSetDevice(h->prm.device));
    s = deskew_common(h, path, ns, Xt2, d_xyz, d_t, nullptr, n, d_xyz_out);
    if (s != LV_OK) return s;
    LV_CUDA(cudaStreamSynchronize(h->stream));
    if (*h->h_bad) { set_error("deskew: a timestamp lies outside the path or the points are not time-sorted"); return LV_ERR_ARG; }
    return LV_OK;
}
lv_status lv_compensate_device_async(lv_handle h, const lv_state32* path, int32_t ns, const lv_state32* Xt2, const float* d_xyz,
                                     const double* d_t, const int64_t* d_n, int64_t n_max, float* d_xyz_out) {
    if (!path || !Xt2 || !d_xyz || !d_t || !d_n || !d_xyz_out) { set_error("compensate async: null path, Xt2, xyz, t, count or output"); return LV_ERR_ARG; }
    if (!n_max_ok("compensate async", n_max)) return LV_ERR_ARG;
    if (ns < 2) { set_error("compensate async: a path needs two states"); return LV_ERR_ARG; }
    /* one thread reads a point and then writes the same point: in place is fine, a shifted overlap is not */
    if ((d_xyz_out != d_xyz && ranges_overlap(d_xyz_out, 12 * n_max, d_xyz, 12 * n_max)) || ranges_overlap(d_xyz_out, 12 * n_max, d_t, 8 * n_max)) {
        set_error("compensate async: the output range overlaps an input range");
        return LV_ERR_ARG;
    }
    if (!handle_ok("compensate async", h, n_max)) return LV_ERR_ARG;
    const lv_status s = deskew_path_ok(h, path, ns, n_max);
    if (s != LV_OK) return s;
    LV_CUDA(cudaSetDevice(h->prm.device));
    return deskew_common(h, path, ns, Xt2, d_xyz, d_t, d_n, n_max, d_xyz_out);
}
lv_status lv_compensate(lv_handle h, const lv_state32* path, int32_t ns, const lv_state32* Xt2, const float* xyz,
                        const double* t, int64_t n, float* xyz_out) {
    lv_status s = deskew_args_ok(h, path, ns, Xt2, xyz, t, n, xyz_out);
    if (s != LV_OK) return s;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(h->d_times.reserve(h->prm.max_points));
    LV_CUDA(h->d_deskew_in.reserve(3 * (size_t)h->prm.max_points));
    LV_CUDA(cudaMemcpyAsync(h->d_deskew_in, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
    LV_CUDA(cudaMemcpyAsync(h->d_times, t, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
    s = deskew_common(h, path, ns, Xt2, h->d_deskew_in, h->d_times, nullptr, n, h->d_deskew_in);
    if (s != LV_OK) return s;
    LV_CUDA(cudaMemcpyAsync(xyz_out, h->d_deskew_in, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    if (*h->h_bad) { set_error("deskew: a timestamp lies outside the path or the points are not time-sorted"); return LV_ERR_ARG; }
    return LV_OK;
}

/* ---- downsamplers ------------------------------------------------------------------------------- */
/* in / out xyz of the host forms, grown with slack; both are freed first, and d_ds_out, reserved last, is empty unless both fit */
static lv_status ds_stage(lv_context* h, int64_t n) {
    if (3 * (size_t)n <= h->d_ds_out.size()) return LV_OK;
    const size_t cap = (size_t)(n + n / 4 + 1024);
    h->d_ds_in.reset();
    h->d_ds_out.reset();
    LV_CUDA(h->d_ds_in.reserve(3 * cap));
    LV_CUDA(h->d_ds_out.reserve(3 * cap));
    return LV_OK;
}
/* the synchronous voxel grid of n > 0 device points (lanes: the full form's attributes): the async form's kernels over the
 * host-known count, then the count read back */
static lv_status voxelgrid_sync(lv_context* h, const float* d_xyz, int64_t n, float leaf, float* d_xyz_out, const VoxelLanes* lanes,
                                int64_t* n_out) {
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(ds_reserve(h->ds, n));
    int launches = 0;
    LV_CUDA(launch_voxelgrid(h->ds, d_xyz, nullptr, n, leaf, d_xyz_out, nullptr, nullptr, h->stream, &launches, lanes));
    h->prof.total_launches += launches;
    LV_CUDA(cudaStreamSynchronize(h->stream));
    /* the pass-through (input copied, count n) is done on the device; the host keeps PCL's warning */
    if (h->ds.h_count[1]) set_error("voxel grid: leaf size too small for the extent of the cloud (cell index overflows): input passed through");
    *n_out = h->ds.h_count[0];
    return LV_OK;
}
/* both host forms for n > 0 points: xyz (and, when time is given, time and intensity) staged, the synchronous voxel grid, then
 * whichever outputs are non-NULL copied back */
static lv_status voxelgrid_host(lv_context* h, const float* xyz, const double* time, const float* intensity, int64_t n, float leaf,
                                float* xyz_out, double* time_out, float* intensity_out, float* range_out, int64_t* n_out) {
    LV_CUDA(cudaSetDevice(h->prm.device));
    lv_status s = ds_stage(h, n);
    if (s != LV_OK) return s;
    /* device staging of the attributes, grown with slack as ds_stage: in / out time, then in / out intensity and out range */
    VoxelLanes lanes;
    double* t_in = nullptr;
    float* f = nullptr;
    if (time) {
        if (28 * (size_t)n > h->d_ds_lanes.size()) LV_CUDA(h->d_ds_lanes.reserve(28 * (size_t)(n + n / 4 + 1024)));
        const int64_t c = (int64_t)(h->d_ds_lanes.size() / 28);
        t_in = reinterpret_cast<double*>(h->d_ds_lanes.get());
        f = reinterpret_cast<float*>(t_in + 2 * c);
        lanes.time = t_in; lanes.time_out = t_in + c;
        lanes.intensity = f; lanes.intensity_out = f + c; lanes.range_out = f + 2 * c;
    }
    LV_CUDA(cudaMemcpyAsync(h->d_ds_in, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
    if (time) {
        LV_CUDA(cudaMemcpyAsync(t_in, time, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
        LV_CUDA(cudaMemcpyAsync(f, intensity, sizeof(float) * n, cudaMemcpyHostToDevice, h->stream));
    }
    s = voxelgrid_sync(h, h->d_ds_in, n, leaf, h->d_ds_out, time ? &lanes : nullptr, n_out);
    if (s != LV_OK) return s;
    const size_t m = (size_t)*n_out;
    LV_CUDA(cudaMemcpyAsync(xyz_out, h->d_ds_out, sizeof(float) * 3 * m, cudaMemcpyDeviceToHost, h->stream));
    if (time_out) LV_CUDA(cudaMemcpyAsync(time_out, lanes.time_out, sizeof(double) * m, cudaMemcpyDeviceToHost, h->stream));
    if (intensity_out) LV_CUDA(cudaMemcpyAsync(intensity_out, lanes.intensity_out, sizeof(float) * m, cudaMemcpyDeviceToHost, h->stream));
    if (range_out) LV_CUDA(cudaMemcpyAsync(range_out, lanes.range_out, sizeof(float) * m, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return LV_OK;
}
lv_status lv_voxelgrid_downsample_device(lv_handle h, const float* d_xyz, int64_t n, float leaf, float* d_xyz_out, int64_t* n_out) {
    /* the centroid kernel reads every input point of a leaf while other threads write their leaves' centroids: an output
     * range that overlaps the input would be read after it is overwritten */
    if (d_xyz && d_xyz_out && n > 0 && n <= 0x7fffffff && ranges_overlap(d_xyz_out, 12 * n, d_xyz, 12 * n)) {
        set_error("voxel grid: the output range overlaps the input range");
        return LV_ERR_ARG;
    }
    if (!h || !d_xyz || !d_xyz_out || !n_out || n < 0 || !(leaf > 0.f) || n > 0x7fffffff) return LV_ERR_ARG;
    *n_out = 0;
    if (n == 0) return LV_OK;
    return voxelgrid_sync(h, d_xyz, n, leaf, d_xyz_out, nullptr, n_out);
}
/* the handle's checks and the launch of both async voxel grids, after their own checks; `what` names the call in the messages */
static lv_status voxelgrid_async(lv_context* h, const char* what, const float* d_xyz, const int64_t* d_n, int64_t n_max, float leaf,
                                 float* d_xyz_out, int64_t* d_n_out, const VoxelLanes* lanes) {
    if (!handle_ok(what, h, n_max)) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(ds_reserve(h->ds, n_max));
    int launches = 0;
    LV_CUDA(launch_voxelgrid(h->ds, d_xyz, d_n, n_max, leaf, d_xyz_out, d_n_out, &h->d_async->err, h->stream, &launches, lanes));
    h->prof.total_launches += launches;
    return LV_OK;
}
lv_status lv_voxelgrid_downsample_device_async(lv_handle h, const float* d_xyz, const int64_t* d_n, int64_t n_max, float leaf,
                                               float* d_xyz_out, int64_t* d_n_out) {
    if (!d_xyz || !d_n || !d_xyz_out || !d_n_out) { set_error("voxel grid async: null input, count, output or output count"); return LV_ERR_ARG; }
    if (!n_max_ok("voxel grid async", n_max)) return LV_ERR_ARG;
    if (!(leaf > 0.f)) { set_error("voxel grid async: leaf size must be positive"); return LV_ERR_ARG; }
    /* the centroid kernel reads every input point of a leaf while other threads write their leaves' centroids */
    if (ranges_overlap(d_xyz, 12 * n_max, d_xyz_out, 12 * n_max)) { set_error("voxel grid async: the output range overlaps the input range"); return LV_ERR_ARG; }
    return voxelgrid_async(h, "voxel grid async", d_xyz, d_n, n_max, leaf, d_xyz_out, d_n_out, nullptr);
}
lv_status lv_voxelgrid_downsample_full_device_async(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity,
                                                    const int64_t* d_n, int64_t n_max, float leaf, float* d_xyz_out, double* d_time_out,
                                                    float* d_intensity_out, float* d_range_out, int64_t* d_n_out) {
    if (!d_xyz || !d_time || !d_intensity || !d_n || !d_xyz_out || !d_n_out) {
        set_error("voxel grid full: null xyz, time, intensity, count, output or output count");
        return LV_ERR_ARG;
    }
    if (!n_max_ok("voxel grid full", n_max)) return LV_ERR_ARG;
    if (!(leaf > 0.f)) { set_error("voxel grid full: leaf size must be positive"); return LV_ERR_ARG; }
    /* the centroid kernel reads a leaf's inputs while other threads write: an output may overlap no input and no other output */
    const ByteRange r[9] = {{d_xyz, 12 * n_max}, {d_time, 8 * n_max}, {d_intensity, 4 * n_max}, {d_n, 8}, {d_xyz_out, 12 * n_max},
                            {d_time_out, 8 * n_max}, {d_intensity_out, 4 * n_max}, {d_range_out, 4 * n_max}, {d_n_out, 8}};
    if (any_ranges_overlap(r, 9, 4)) { set_error("voxel grid full: an output range overlaps an input or another output"); return LV_ERR_ARG; }
    VoxelLanes lanes;
    lanes.time = d_time; lanes.intensity = d_intensity;
    lanes.time_out = d_time_out; lanes.intensity_out = d_intensity_out; lanes.range_out = d_range_out;
    return voxelgrid_async(h, "voxel grid full", d_xyz, d_n, n_max, leaf, d_xyz_out, d_n_out, &lanes);
}
lv_status lv_voxelgrid_downsample(lv_handle h, const float* xyz, int64_t n, float leaf, float* xyz_out, int64_t* n_out) {
    if (!h || !xyz || !xyz_out || !n_out || n < 0 || !(leaf > 0.f) || n > 0x7fffffff) return LV_ERR_ARG;
    *n_out = 0;
    if (n == 0) return LV_OK;
    return voxelgrid_host(h, xyz, nullptr, nullptr, n, leaf, xyz_out, nullptr, nullptr, nullptr, n_out);
}
lv_status lv_voxelgrid_downsample_full(lv_handle h, const float* xyz, const double* time, const float* intensity, int64_t n, float leaf,
                                       float* xyz_out, double* time_out, float* intensity_out, float* range_out, int64_t* n_out) {
    if (n_out) *n_out = 0;
    if (!xyz || !time || !intensity || !xyz_out || !n_out) {
        set_error("voxel grid full: null xyz, time, intensity, output or n_out");
        return LV_ERR_ARG;
    }
    if (n < 0 || n > 0x7fffffff) { set_error("voxel grid full: n outside [0, 2^31 - 1]"); return LV_ERR_ARG; }
    if (!(leaf > 0.f)) { set_error("voxel grid full: leaf size must be positive"); return LV_ERR_ARG; }
    if (!h) { set_error("voxel grid full: null handle"); return LV_ERR_ARG; }
    if (n == 0) return LV_OK;
    return voxelgrid_host(h, xyz, time, intensity, n, leaf, xyz_out, time_out, intensity_out, range_out, n_out);
}
lv_status lv_temporal_downsample(lv_handle h, const float* xyz, int64_t n, int32_t rate, double min_dist, float* xyz_out,
                                 int32_t* idx_out, int64_t* n_out) {
    if (!h || !xyz || !xyz_out || !n_out || n < 0 || n > 0x7fffffff) return LV_ERR_ARG;
    *n_out = 0;
    if (n == 0) return LV_OK;
    LV_CUDA(cudaSetDevice(h->prm.device));
    lv_status s = ds_stage(h, n);
    if (s != LV_OK) return s;
    LV_CUDA(ds_reserve(h->ds, n));
    LV_CUDA(cudaMemcpyAsync(h->d_ds_in, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
    int launches = 0;
    LV_CUDA(launch_temporal(h->ds, h->d_ds_in, n, rate, min_dist, h->d_ds_out, nullptr, h->stream, &launches));
    h->prof.total_launches += launches;
    LV_CUDA(cudaStreamSynchronize(h->stream));
    const int64_t m = h->ds.h_count[0];
    LV_CUDA(cudaMemcpyAsync(xyz_out, h->d_ds_out, sizeof(float) * 3 * (size_t)m, cudaMemcpyDeviceToHost, h->stream));
    if (idx_out) LV_CUDA(cudaMemcpyAsync(idx_out, h->ds.sel, sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    *n_out = m;
    return LV_OK;
}

/* ---- Accumulator::process ------------------------------------------------------------------------ */
/* the argument checks and the launches of every message format: d_n_out NULL = the synchronous form (*n_out read back).
 * null_args: a required pointer is NULL (null_what names them); layout_error() runs once the pointers and n are known good;
 * launch(launches, err) enqueues the pipeline; `deferred` says what the pipeline's flag word (ds.count[1]) means */
static const char* const kCloudNaN = "a kept point's timestamp is NaN (the time sort has no order for it)";
extern "C++" {
template <class LayoutError, class Launch>
static lv_status front_end_impl(lv_handle h, const std::string& what, bool null_args, const char* null_what, const uint8_t* d_data,
                                int64_t data_bytes, int64_t n, int32_t downsample_rate, const CloudOut& o, int64_t* n_out, int64_t* d_n_out,
                                LayoutError layout_error, Launch launch, const char* deferred = kCloudNaN) {
    /* every check before the first device call */
    if (n_out) *n_out = 0;
    if (null_args || !n_out) { set_error(what + ": null " + null_what); return LV_ERR_ARG; }
    if (n < 0 || n > 0x7fffffff) { set_error(what + ": n outside [0, 2^31 - 1] (point indices are int32)"); return LV_ERR_ARG; }
    if (const char* why = layout_error()) { set_error(what + ": " + why); return LV_ERR_ARG; }
    /* the gather decodes the message while it writes the outputs: an output that overlaps the bytes would be read after it is
     * overwritten (the outputs may overlap each other) */
    const ByteRange r[6] = {{o.xyz, 12 * n}, {o.time, 8 * n}, {o.intensity, 4 * n}, {o.range, 4 * n}, {o.idx, 4 * n}, {d_data, data_bytes}};
    if (n > 0 && any_ranges_overlap(r, 6, 5)) { set_error(what + ": an output range overlaps the message bytes"); return LV_ERR_ARG; }
    if (!h) { set_error(what + ": null handle"); return LV_ERR_ARG; }
    if (cloud_bound(n, downsample_rate) == 0) {                  /* nothing can be kept */
        if (d_n_out) {
            LV_CUDA(cudaSetDevice(h->prm.device));
            LV_CUDA(cudaMemsetAsync(d_n_out, 0, sizeof(int64_t), h->stream));
        }
        return LV_OK;
    }
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(ds_reserve(h->ds, n));
    int launches = 0;
    LV_CUDA(launch(&launches, d_n_out ? &h->d_async->err : nullptr));
    h->prof.total_launches += launches;
    if (d_n_out) return LV_OK;
    LV_CUDA(cudaStreamSynchronize(h->stream));
    if (h->ds.h_count[1]) {                                       /* never raised for Livox: its times are never NaN */
        set_error(what + ": " + deferred);
        return LV_ERR_ARG;
    }
    *n_out = h->ds.h_count[0];
    return LV_OK;
}
}  // extern "C++"
static lv_status process_cloud_impl(lv_handle h, lv_lidar_type type, const lv_cloud_layout* layout, const uint8_t* d_data, int64_t data_bytes,
                                    int64_t n, uint64_t header_stamp_us, int stamp_beginning, int offset_beginning, double full_rotation_time,
                                    int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                    int32_t* d_idx, int64_t* n_out, int64_t* d_n_out) {
    const CloudOut o{d_xyz, d_time, d_intensity, d_range, d_idx};
    return front_end_impl(
        h, "process cloud", !layout || !d_data || !d_xyz || !d_time, "layout, data, xyz, time or n_out", d_data, data_bytes, n, downsample_rate,
        o, n_out, d_n_out, [&] { return cloud_layout_error(type, *layout, n, data_bytes); },
        [&](int* launches, uint32_t* err) {
            const CloudArgs a = {d_data, n, *layout, type, header_stamp_us, stamp_beginning, offset_beginning, full_rotation_time, downsample_rate,
                                 min_dist};
            return launch_process_cloud(h->ds, a, o, d_n_out, err, h->stream, launches);
        });
}
lv_status lv_process_cloud_device(lv_handle h, lv_lidar_type type, const lv_cloud_layout* layout, const uint8_t* d_data, int64_t data_bytes,
                                  int64_t n, uint64_t header_stamp_us, int stamp_beginning, int offset_beginning, double full_rotation_time,
                                  int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                  int32_t* d_idx, int64_t* n_out) {
    return process_cloud_impl(h, type, layout, d_data, data_bytes, n, header_stamp_us, stamp_beginning, offset_beginning, full_rotation_time,
                              downsample_rate, min_dist, d_xyz, d_time, d_intensity, d_range, d_idx, n_out, nullptr);
}
lv_status lv_process_cloud_device_async(lv_handle h, lv_lidar_type type, const lv_cloud_layout* layout, const uint8_t* d_data, int64_t data_bytes,
                                        int64_t n, uint64_t header_stamp_us, int stamp_beginning, int offset_beginning, double full_rotation_time,
                                        int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time, float* d_intensity,
                                        float* d_range, int32_t* d_idx, int64_t* d_n_out) {
    int64_t unused = 0;                                           /* the count stays on the device */
    if (!d_n_out) { set_error("process cloud: null layout, data, xyz, time or n_out"); return LV_ERR_ARG; }
    return process_cloud_impl(h, type, layout, d_data, data_bytes, n, header_stamp_us, stamp_beginning, offset_beginning, full_rotation_time,
                              downsample_rate, min_dist, d_xyz, d_time, d_intensity, d_range, d_idx, &unused, d_n_out);
}

/* a Livox CustomMsg's records (lv_wire.h): the tag filter, then the decimator on the rank among the tag-kept points */
static lv_status process_livox_impl(lv_handle h, const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t timebase_ns, uint8_t tag_reject_mask,
                                    int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                    int32_t* d_idx, int64_t* n_out, int64_t* d_n_out) {
    const CloudOut o{d_xyz, d_time, d_intensity, d_range, d_idx};
    return front_end_impl(
        h, "process livox", !d_data || !d_xyz || !d_time, "data, xyz, time or n_out", d_data, data_bytes, n, downsample_rate, o, n_out, d_n_out,
        [&] { return livox_layout_error(n, data_bytes, timebase_ns); },
        [&](int* launches, uint32_t* err) {
            const LivoxArgs a = {d_data, n, timebase_ns, tag_reject_mask, downsample_rate, min_dist};
            return launch_process_livox(h->ds, a, o, d_n_out, err, h->stream, launches);
        });
}
lv_status lv_process_livox_device(lv_handle h, const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t timebase_ns, uint8_t tag_reject_mask,
                                  int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                  int32_t* d_idx, int64_t* n_out) {
    return process_livox_impl(h, d_data, data_bytes, n, timebase_ns, tag_reject_mask, downsample_rate, min_dist, d_xyz, d_time, d_intensity,
                              d_range, d_idx, n_out, nullptr);
}
lv_status lv_process_livox_device_async(lv_handle h, const uint8_t* d_data, int64_t data_bytes, int64_t n, uint64_t timebase_ns,
                                        uint8_t tag_reject_mask, int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time,
                                        float* d_intensity, float* d_range, int32_t* d_idx, int64_t* d_n_out) {
    int64_t unused = 0;                                           /* the count stays on the device */
    if (!d_n_out) { set_error("process livox: null data, xyz, time or n_out"); return LV_ERR_ARG; }
    return process_livox_impl(h, d_data, data_bytes, n, timebase_ns, tag_reject_mask, downsample_rate, min_dist, d_xyz, d_time, d_intensity,
                              d_range, d_idx, &unused, d_n_out);
}

/* a VelodyneScan's packets (lv_wire.h): msg2points, then the decimator on the rank among its points.  The first call uploads the
 * rotation tables, which the context keeps */
static const char* const kVelodyneDeferred = "a packet is a dual-return one (not decoded) or its stamp has nsec >= 10^9";
static cudaError_t velodyne_tables_ready(lv_handle h) {
    if (h->velodyne_tables_ok) return cudaSuccess;
    std::vector<float> t(2 * kVelodyneTable);
    velodyne_tables(t.data(), t.data() + kVelodyneTable);
    cudaError_t e = h->d_velodyne_tables.reserve(t.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->d_velodyne_tables, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);   /* t is pageable and goes out of scope */
    h->velodyne_tables_ok = e == cudaSuccess;
    return e;
}
static lv_status process_velodyne_impl(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                       const lv_velodyne_calibration* cal, int32_t downsample_rate, double min_dist, float* d_xyz,
                                       double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out, int64_t* d_n_out) {
    const CloudOut o{d_xyz, d_time, d_intensity, d_range, d_idx};
    /* n_packets out of range leaves n at 0 here, and velodyne_layout_error names it */
    const int64_t n = n_packets >= 0 && n_packets <= kVelodyneMaxPackets ? n_packets * kVelodyneSlots : 0;
    return front_end_impl(
        h, "process velodyne", !d_packets || !cal || !d_xyz || !d_time, "packets, cal, xyz, time or n_out", d_packets, data_bytes, n,
        downsample_rate, o, n_out, d_n_out,
        [&]() -> const char* {
            if (const char* why = velodyne_layout_error(n_packets, data_bytes)) return why;
            return velodyne_calib_finite(*cal) ? nullptr : "a calibration entry is not finite";
        },
        [&](int* launches, uint32_t* err) {
            const cudaError_t e = velodyne_tables_ready(h);
            if (e != cudaSuccess) return e;
            const VelodyneArgs a = {d_packets, n_packets, n, h->d_velodyne_tables, velodyne_calib(*cal), downsample_rate, min_dist};
            return launch_process_velodyne(h->ds, a, o, d_n_out, err, h->stream, launches);
        },
        kVelodyneDeferred);
}
lv_status lv_process_velodyne_device(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                     const lv_velodyne_calibration* cal, int32_t downsample_rate, double min_dist, float* d_xyz,
                                     double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out) {
    return process_velodyne_impl(h, d_packets, data_bytes, n_packets, cal, downsample_rate, min_dist, d_xyz, d_time, d_intensity, d_range,
                                 d_idx, n_out, nullptr);
}
lv_status lv_process_velodyne_device_async(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                           const lv_velodyne_calibration* cal, int32_t downsample_rate, double min_dist, float* d_xyz,
                                           double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* d_n_out) {
    int64_t unused = 0;                                           /* the count stays on the device */
    if (!d_n_out) { set_error("process velodyne: null packets, cal, xyz, time or n_out"); return LV_ERR_ARG; }
    return process_velodyne_impl(h, d_packets, data_bytes, n_packets, cal, downsample_rate, min_dist, d_xyz, d_time, d_intensity, d_range,
                                 d_idx, &unused, d_n_out);
}

/* Ouster packets of any UDP profile (lv_wire.h): msg2points through the profile's layout, then the decimator on the rank among its
 * points.  The first call uploads the column table, which the context keeps */
static cudaError_t ouster_table_ready(lv_handle h) {
    if (h->ouster_table_ok) return cudaSuccess;
    std::vector<float> t(2 * kOusterTable);
    ouster_table(t.data(), t.data() + kOusterTable);
    cudaError_t e = h->d_ouster_table.reserve(t.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->d_ouster_table, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);   /* t is pageable and goes out of scope */
    h->ouster_table_ok = e == cudaSuccess;
    return e;
}
static lv_status process_ouster_impl(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                     const lv_ouster_calibration* cal, lv_ouster_profile profile, int32_t downsample_rate, double min_dist,
                                     float* d_xyz, double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out,
                                     int64_t* d_n_out) {
    const CloudOut o{d_xyz, d_time, d_intensity, d_range, d_idx};
    /* a calibration, profile or n_packets out of range leaves n at 0 here, and the layout check names it */
    const bool cal_ok = cal && !ouster_calib_error(*cal);
    const int H = cal_ok ? cal->pixels_per_column : 0;
    OusterFormat fmt{};
    const bool fmt_ok = cal_ok && ouster_format(profile, H, &fmt);
    const int64_t n = fmt_ok && n_packets >= 0 && n_packets <= ouster_max_packets(H) ? n_packets * kOusterColumns * H : 0;
    return front_end_impl(
        h, "process ouster", !d_packets || !cal || !d_xyz || !d_time, "packets, cal, xyz, time or n_out", d_packets, data_bytes, n,
        downsample_rate, o, n_out, d_n_out,
        [&]() -> const char* {
            if (const char* why = ouster_calib_error(*cal)) return why;
            if (!fmt_ok) return "profile is not an lv_ouster_profile";
            return ouster_layout_error(fmt, n_packets, data_bytes, H);
        },
        [&](int* launches, uint32_t* err) {
            const cudaError_t e = ouster_table_ready(h);
            if (e != cudaSuccess) return e;
            const OusterArgs a = {d_packets, n, h->d_ouster_table, ouster_calib(*cal), fmt, downsample_rate, min_dist};
            return launch_process_ouster(h->ds, a, o, d_n_out, err, h->stream, launches);
        });
}
lv_status lv_process_ouster_packets_device(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                           const lv_ouster_calibration* cal, lv_ouster_profile profile, int32_t downsample_rate,
                                           double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                           int32_t* d_idx, int64_t* n_out) {
    return process_ouster_impl(h, d_packets, data_bytes, n_packets, cal, profile, downsample_rate, min_dist, d_xyz, d_time, d_intensity,
                               d_range, d_idx, n_out, nullptr);
}
lv_status lv_process_ouster_packets_device_async(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                                 const lv_ouster_calibration* cal, lv_ouster_profile profile, int32_t downsample_rate,
                                                 double min_dist, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                                 int32_t* d_idx, int64_t* d_n_out) {
    int64_t unused = 0;                                           /* the count stays on the device */
    if (!d_n_out) { set_error("process ouster: null packets, cal, xyz, time or n_out"); return LV_ERR_ARG; }
    return process_ouster_impl(h, d_packets, data_bytes, n_packets, cal, profile, downsample_rate, min_dist, d_xyz, d_time, d_intensity,
                               d_range, d_idx, &unused, d_n_out);
}
lv_status lv_process_ouster_device(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                   const lv_ouster_calibration* cal, int32_t downsample_rate, double min_dist, float* d_xyz, double* d_time,
                                   float* d_intensity, float* d_range, int32_t* d_idx, int64_t* n_out) {
    return lv_process_ouster_packets_device(h, d_packets, data_bytes, n_packets, cal, LV_OUSTER_LEGACY, downsample_rate, min_dist, d_xyz,
                                            d_time, d_intensity, d_range, d_idx, n_out);
}
lv_status lv_process_ouster_device_async(lv_handle h, const uint8_t* d_packets, int64_t data_bytes, int64_t n_packets,
                                         const lv_ouster_calibration* cal, int32_t downsample_rate, double min_dist, float* d_xyz,
                                         double* d_time, float* d_intensity, float* d_range, int32_t* d_idx, int64_t* d_n_out) {
    return lv_process_ouster_packets_device_async(h, d_packets, data_bytes, n_packets, cal, LV_OUSTER_LEGACY, downsample_rate, min_dist,
                                                  d_xyz, d_time, d_intensity, d_range, d_idx, d_n_out);
}

/* the deferred errors of the _async calls (AsyncWords::err) and the map's flags; clears the former */
lv_status lv_async_status(lv_handle h) {
    if (!h) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaMemcpyAsync(&h->h_async->err, &h->d_async->err, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaMemsetAsync(&h->d_async->err, 0, sizeof(uint32_t), h->stream));
    LV_CUDA(map_fetch_counters(h->map, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    const uint32_t err = h->h_async->err;
    if (err) {
        std::string msg;
        if (err & kAsyncCloudNaN) msg += "process cloud: a kept point's timestamp is NaN (the time sort has no order for it); ";
        if (err & kAsyncDeskewPath) msg += "compensate: a timestamp lies outside the path or the points are not time-sorted; ";
        if (err & kAsyncCount) msg += "a device point count lies outside [0, n_max] (clamped); ";
        if (err & kAsyncLidarFull) msg += "lidar push or merge: the points do not fit the buffer's capacity (nothing appended; lv_lidar_reserve); ";
        if (err & kAsyncLidarWindow) msg += "lidar get points: the window holds more than n_max points (count 0); ";
        if (err & kAsyncLidarUnsorted)
            msg += "lidar merge: the message or the buffered points after its first time are not time-ordered (appended as a push does); ";
        if (err & kAsyncLidarOverlap)
            msg += "lidar merge: the message reaches back over more buffered points than the merge reserve (nothing merged; lv_lidar_reserve_merge); ";
        if (err & kAsyncVelodyne) msg += std::string("process velodyne: ") + kVelodyneDeferred + "; ";
        msg.resize(msg.size() - 2);
        set_error(msg);
        return LV_ERR_ARG;
    }
    return map_status_from_mirror(h);
}

/* ---- Accumulator::BUFFER_L (lv_lidar_buffer.cu) ---------------------------------------------------------------------------------- */
static bool overlaps_lidar(const lv_context* h, const void* p, int64_t bytes) {
    const LidarRing& r = h->lidar;
    return ranges_overlap(p, bytes, r.xyz, 12 * r.cap) || ranges_overlap(p, bytes, r.time, 8 * r.cap) ||
           ranges_overlap(p, bytes, r.words, (int64_t)sizeof(LidarWords)) ||
           (r.intensity && (ranges_overlap(p, bytes, r.intensity, 4 * r.cap) || ranges_overlap(p, bytes, r.range, 4 * r.cap))) ||
           ranges_overlap(p, bytes, r.merge_xyz, 4 * (int64_t)r.merge_xyz.size()) ||
           ranges_overlap(p, bytes, r.merge_time, 8 * (int64_t)r.merge_time.size()) ||
           ranges_overlap(p, bytes, r.merge_intensity, 4 * (int64_t)r.merge_intensity.size()) ||
           ranges_overlap(p, bytes, r.merge_range, 4 * (int64_t)r.merge_range.size());
}
/* lv_lidar_reserve (lanes: keep the ring's) and lv_lidar_reserve_full (lanes: always); `what` names the call in the messages */
static lv_status lidar_resize(lv_handle h, int64_t capacity, bool full, const char* what) {
    if (capacity < 1 || capacity > kLidarMaxCapacity) { set_error(std::string(what) + ": capacity outside [1, 2^30]"); return LV_ERR_ARG; }
    if (!h) { set_error(std::string(what) + ": null handle"); return LV_ERR_ARG; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    LidarRing& r = h->lidar;
    if (!r.h_words) {                                             /* the first call, or a retry of one that failed */
        LV_CUDA(r.words.reserve(1));
        LV_CUDA(r.h_words.reserve(1));
        LV_CUDA(cudaMemsetAsync(r.words, 0, sizeof(LidarWords), h->stream));
    }
    LV_CUDA(cudaMemcpyAsync(r.h_words, r.words, sizeof(LidarWords), cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    const bool lanes = full || r.intensity;
    if (capacity == r.cap && lanes == (r.intensity != nullptr)) return LV_OK;
    const int64_t live = r.h_words->tail - r.h_words->head;
    if (live > capacity) {
        char buf[160];
        snprintf(buf, sizeof(buf), "%s: %lld points are live, more than a capacity of %lld", what, (long long)live, (long long)capacity);
        set_error(buf);
        return LV_ERR_CAPACITY;
    }
    /* the new arrays are allocated while the old ones still hold the live points */
    DeviceBuf<float> xyz, intensity, range;
    DeviceBuf<double> time;
    cudaError_t e = lanes && r.merge_cap ? r.merge_intensity.reserve(r.merge_cap) : cudaSuccess;   /* the merge scratch gains lanes too */
    if (e == cudaSuccess && lanes && r.merge_cap) e = r.merge_range.reserve(r.merge_cap);
    if (e == cudaSuccess) e = xyz.reserve(3 * (size_t)capacity);
    if (e == cudaSuccess) e = time.reserve(capacity);
    if (e == cudaSuccess && lanes) e = intensity.reserve(capacity);
    if (e == cudaSuccess && lanes) e = range.reserve(capacity);
    int launches = 0;
    if (e == cudaSuccess) e = launch_lidar_move(r, live, xyz, time, capacity, h->stream, &launches, intensity, range);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) {                                       /* the buffer stays as it was */
        cudaGetLastError();
        set_error(std::string(what) + ": " + cudaGetErrorString(e));
        return LV_ERR_CAPACITY;
    }
    h->prof.total_launches += launches;
    r.xyz = std::move(xyz); r.time = std::move(time);
    r.intensity = std::move(intensity); r.range = std::move(range);
    r.cap = capacity;
    return LV_OK;
}
lv_status lv_lidar_reserve(lv_handle h, int64_t capacity) { return lidar_resize(h, capacity, false, "lidar reserve"); }
lv_status lv_lidar_reserve_full(lv_handle h, int64_t capacity) { return lidar_resize(h, capacity, true, "lidar reserve full"); }
/* lv_lidar_reserve_merge: the overlap scratch of the merge (with lanes when the ring has them); the stream is drained first, since
 * an enqueued merge may still read the old scratch */
lv_status lv_lidar_reserve_merge(lv_handle h, int64_t overlap_points) {
    if (overlap_points < 1 || overlap_points > kLidarMaxCapacity) { set_error("lidar reserve merge: overlap outside [1, 2^30]"); return LV_ERR_ARG; }
    if (!h) { set_error("lidar reserve merge: null handle"); return LV_ERR_ARG; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    LidarRing& r = h->lidar;
    r.merge_cap = 0;                                              /* until every array fits: a failure leaves merges refused */
    cudaError_t e = r.merge_xyz.reserve(3 * (size_t)overlap_points);
    if (e == cudaSuccess) e = r.merge_time.reserve(overlap_points);
    if (e == cudaSuccess && r.intensity) e = r.merge_intensity.reserve(overlap_points);
    if (e == cudaSuccess && r.intensity) e = r.merge_range.reserve(overlap_points);
    if (e != cudaSuccess) {
        set_error(std::string("lidar reserve merge: ") + cudaGetErrorString(e));
        return LV_ERR_CAPACITY;
    }
    r.merge_cap = overlap_points;
    return LV_OK;
}
/* the checks after the null-pointer check and the launch of both pushes and both merges: intensity / range NULL = the plain form;
 * merge: the time-ordered merge through the 12 floats of T (NULL: no transform) */
static lv_status lidar_push_impl(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity, const float* d_range,
                                 const int64_t* d_n, int64_t n_max, const char* what, bool merge = false, const float* T = nullptr) {
    const std::string w(what);
    if (!n_max_ok(what, n_max)) return LV_ERR_ARG;
    Rt32 rt{};
    if (merge) {
        for (int k = 0; T && k < 12; ++k)
            if (!std::isfinite(T[k])) { set_error(w + ": a transform entry is not finite"); return LV_ERR_ARG; }
        if (T) {
            memcpy(rt.R, T, sizeof(rt.R));
            memcpy(rt.t, T + 9, sizeof(rt.t));
        }
        /* the split kernel reads the times and the count while the write kernel reads the points: they must be distinct arrays */
        const ByteRange in[5] = {{d_xyz, 12 * n_max}, {d_time, 8 * n_max}, {d_n, 8}, {d_intensity, 4 * n_max}, {d_range, 4 * n_max}};
        if (any_ranges_overlap(in, 5)) { set_error(w + ": the input ranges overlap"); return LV_ERR_ARG; }
    }
    if (!h) { set_error(w + ": null handle"); return LV_ERR_ARG; }
    if (!h->lidar.cap) { set_error(w + ": the buffer has no capacity (lv_lidar_reserve first)"); return LV_ERR_ARG; }
    if (d_intensity && !h->lidar.intensity) { set_error(w + ": the buffer has no attribute lanes (lv_lidar_reserve_full first)"); return LV_ERR_ARG; }
    if (merge && !h->lidar.merge_cap) { set_error(w + ": the buffer has no merge reserve (lv_lidar_reserve_merge first)"); return LV_ERR_ARG; }
    /* the kernel reads the count and the points while it writes the buffer */
    if (overlaps_lidar(h, d_xyz, 12 * n_max) || overlaps_lidar(h, d_time, 8 * n_max) || overlaps_lidar(h, d_n, 8) ||
        (d_intensity && (overlaps_lidar(h, d_intensity, 4 * n_max) || overlaps_lidar(h, d_range, 4 * n_max)))) {
        set_error(w + ": an input range overlaps the buffer");
        return LV_ERR_ARG;
    }
    LV_CUDA(cudaSetDevice(h->prm.device));
    int launches = 0;
    if (merge)
        LV_CUDA(launch_lidar_merge(h->lidar, d_xyz, d_time, d_n, n_max, T != nullptr, rt, &h->d_async->err, h->stream, &launches, d_intensity,
                                   d_range));
    else
        LV_CUDA(launch_lidar_push(h->lidar, d_xyz, d_time, d_n, n_max, &h->d_async->err, h->stream, &launches, d_intensity, d_range));
    h->prof.total_launches += launches;
    return LV_OK;
}
lv_status lv_lidar_merge_device_async(lv_handle h, const float* d_xyz, const double* d_time, const int64_t* d_n, int64_t n_max, const float* T) {
    if (!d_xyz || !d_time || !d_n) { set_error("lidar merge: null xyz, time or count"); return LV_ERR_ARG; }
    return lidar_push_impl(h, d_xyz, d_time, nullptr, nullptr, d_n, n_max, "lidar merge", true, T);
}
lv_status lv_lidar_merge_full_device_async(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity, const float* d_range,
                                           const int64_t* d_n, int64_t n_max, const float* T) {
    if (!d_xyz || !d_time || !d_intensity || !d_range || !d_n) {
        set_error("lidar merge full: null xyz, time, intensity, range or count");
        return LV_ERR_ARG;
    }
    return lidar_push_impl(h, d_xyz, d_time, d_intensity, d_range, d_n, n_max, "lidar merge full", true, T);
}
lv_status lv_lidar_push_device_async(lv_handle h, const float* d_xyz, const double* d_time, const int64_t* d_n, int64_t n_max) {
    if (!d_xyz || !d_time || !d_n) { set_error("lidar push: null xyz, time or count"); return LV_ERR_ARG; }
    return lidar_push_impl(h, d_xyz, d_time, nullptr, nullptr, d_n, n_max, "lidar push");
}
lv_status lv_lidar_push_full_device_async(lv_handle h, const float* d_xyz, const double* d_time, const float* d_intensity, const float* d_range,
                                          const int64_t* d_n, int64_t n_max) {
    if (!d_xyz || !d_time || !d_intensity || !d_range || !d_n) { set_error("lidar push full: null xyz, time, intensity, range or count"); return LV_ERR_ARG; }
    return lidar_push_impl(h, d_xyz, d_time, d_intensity, d_range, d_n, n_max, "lidar push full");
}
/* the checks and the launch of every form of get: d_n_out NULL = the synchronous form; intensity / range NULL = a plain get */
static lv_status lidar_get_impl(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, float* d_intensity, float* d_range, int64_t n_max,
                                const void* count, int64_t* d_n_out, const char* what) {
    const std::string w(what);
    if (!d_xyz || !d_time || !count) { set_error(w + ": null xyz, time or count"); return LV_ERR_ARG; }
    if (!n_max_ok(what, n_max)) return LV_ERR_ARG;
    if (isnan(t1) || isnan(t2)) { set_error(w + ": t1 or t2 is NaN"); return LV_ERR_ARG; }
    const ByteRange outs[5] = {{d_xyz, 12 * n_max}, {d_time, 8 * n_max}, {d_n_out, 8}, {d_intensity, 4 * n_max}, {d_range, 4 * n_max}};
    if (any_ranges_overlap(outs, 5)) { set_error(w + ": the output ranges overlap"); return LV_ERR_ARG; }
    if (!h) { set_error(w + ": null handle"); return LV_ERR_ARG; }
    if (!h->lidar.cap) { set_error(w + ": the buffer has no capacity (lv_lidar_reserve first)"); return LV_ERR_ARG; }
    if (d_intensity && !h->lidar.intensity) { set_error(w + ": the buffer has no attribute lanes (lv_lidar_reserve_full first)"); return LV_ERR_ARG; }
    for (const ByteRange& o : outs)
        if (o.p && overlaps_lidar(h, o.p, o.bytes)) {
            set_error(w + ": an output range overlaps the buffer");
            return LV_ERR_ARG;
        }
    LV_CUDA(cudaSetDevice(h->prm.device));
    int launches = 0;
    LV_CUDA(launch_lidar_get(h->lidar, t1, t2, d_xyz, d_time, n_max, d_n_out, d_n_out ? &h->d_async->err : nullptr, h->stream, &launches,
                             d_intensity, d_range));
    h->prof.total_launches += launches;
    return LV_OK;
}
lv_status lv_lidar_get_points_device_async(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, int64_t n_max, int64_t* d_n_out) {
    return lidar_get_impl(h, t1, t2, d_xyz, d_time, nullptr, nullptr, n_max, d_n_out, d_n_out, "lidar get points");
}
lv_status lv_lidar_get_points_full_device_async(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, float* d_intensity,
                                                float* d_range, int64_t n_max, int64_t* d_n_out) {
    if (!d_intensity || !d_range) { set_error("lidar get points full: null intensity or range"); return LV_ERR_ARG; }
    return lidar_get_impl(h, t1, t2, d_xyz, d_time, d_intensity, d_range, n_max, d_n_out, d_n_out, "lidar get points full");
}
lv_status lv_lidar_get_points_device(lv_handle h, double t1, double t2, float* d_xyz, double* d_time, int64_t n_max, int64_t* n_out) {
    if (n_out) *n_out = 0;
    lv_status s = lidar_get_impl(h, t1, t2, d_xyz, d_time, nullptr, nullptr, n_max, n_out, nullptr, "lidar get points");
    if (s != LV_OK) return s;
    LidarRing& r = h->lidar;
    LV_CUDA(cudaMemcpyAsync(r.h_words, r.words, sizeof(LidarWords), cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    if (r.h_words->window > n_max) {
        char buf[160];
        snprintf(buf, sizeof(buf), "lidar get points: the window holds %lld points, more than n_max = %lld", (long long)r.h_words->window,
                 (long long)n_max);
        set_error(buf);
        return LV_ERR_CAPACITY;
    }
    *n_out = r.h_words->count;
    return LV_OK;
}
lv_status lv_lidar_clear_async(lv_handle h, double t) {
    if (isnan(t)) { set_error("lidar clear: t is NaN"); return LV_ERR_ARG; }
    if (!h) { set_error("lidar clear: null handle"); return LV_ERR_ARG; }
    if (!h->lidar.cap) { set_error("lidar clear: the buffer has no capacity (lv_lidar_reserve first)"); return LV_ERR_ARG; }
    LV_CUDA(cudaSetDevice(h->prm.device));
    int launches = 0;
    LV_CUDA(launch_lidar_clear(h->lidar, t, h->stream, &launches));
    h->prof.total_launches += launches;
    return LV_OK;
}
lv_status lv_cloud_stamp_device_async(lv_handle h, const double* d_time, const int64_t* d_n, int64_t n_max, uint64_t* d_stamp_us) {
    if (!d_time || !d_n || !d_stamp_us) { set_error("cloud stamp: null time, count or stamp"); return LV_ERR_ARG; }
    if (!n_max_ok("cloud stamp", n_max)) return LV_ERR_ARG;
    /* one block reads the times and the count, then writes the stamp */
    if (ranges_overlap(d_stamp_us, 8, d_time, 8 * n_max) || ranges_overlap(d_stamp_us, 8, d_n, 8)) {
        set_error("cloud stamp: the stamp overlaps the times or the count");
        return LV_ERR_ARG;
    }
    if (!handle_ok("cloud stamp", h, n_max)) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    int launches = 0;
    LV_CUDA(launch_cloud_stamp(d_time, d_n, n_max, d_stamp_us, &h->d_async->err, h->stream, &launches));
    h->prof.total_launches += launches;
    return LV_OK;
}
lv_status lv_lidar_info(lv_handle h, struct lv_lidar_info* out) {
    if (!h || !out) { set_error("lidar info: null handle or output"); return LV_ERR_ARG; }
    const LidarRing& r = h->lidar;
    out->points = 0;
    out->capacity = r.cap;
    out->oldest_time = out->newest_time = NAN;
    if (!r.cap) return LV_OK;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaMemcpyAsync(r.h_words, r.words, sizeof(LidarWords), cudaMemcpyDeviceToHost, h->stream));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    const int64_t head = r.h_words->head, tail = r.h_words->tail;
    out->points = tail - head;
    if (tail > head) {
        LV_CUDA(cudaMemcpyAsync(&out->oldest_time, r.time + lidar_slot(head, r.cap), sizeof(double), cudaMemcpyDeviceToHost, h->stream));
        LV_CUDA(cudaMemcpyAsync(&out->newest_time, r.time + lidar_slot(tail - 1, r.cap), sizeof(double), cudaMemcpyDeviceToHost, h->stream));
        LV_CUDA(cudaStreamSynchronize(h->stream));
    }
    return LV_OK;
}

lv_status lv_synchronize(lv_handle h) {
    if (!h) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    LV_CUDA(cudaStreamSynchronize(h->stream));
    return LV_OK;
}
lv_status lv_profile_enable(lv_handle h, int on) {
    if (!h) return LV_ERR_ARG;
    h->profile = on != 0;
    return LV_OK;
}
lv_status lv_profile_get(lv_handle h, lv_profile* out, int reset) {
    if (!h || !out) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    lv_status s = drain_events(h);
    if (s != LV_OK) return s;
    *out = h->prof;
    if (reset) memset(&h->prof, 0, sizeof(h->prof));
    return LV_OK;
}
lv_status lv_flush_l2(lv_handle h) {
    if (!h) return LV_ERR_ARG;
    LV_CUDA(cudaSetDevice(h->prm.device));
    const size_t bytes = 256ull << 20;
    LV_CUDA(h->d_flush.reserve(bytes));
    LV_CUDA(launch_l2_flush(h->d_flush, bytes, h->stream));
    h->prof.total_launches += 1;
    return LV_OK;
}

}  // extern "C"
