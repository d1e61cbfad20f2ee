/*
 * tests/cpu_shim/shim.cpp — TEST-ONLY host build of the product's host+device headers.
 *
 * The device math of liblimovelo_b200.so lives in limo-velo_b200/csrc/ headers that compile for
 * both nvcc and g++ (lv_voxel_search.h, lv_point_math.h, lv_ieskf.h, ...).  This file instantiates
 * them on the CPU (ExecSerial = one "thread", no barriers) so that `pytest -m "not gpu"` can check
 * the very code the kernels run against the oracle, in a container without a GPU.
 *
 * It is NOT part of the product, is not linked into liblimovelo_b200.so and is not reachable from
 * the C ABI; the product has no CPU path.  The map is built, updated and grown by the product's own per-item functions
 * (lv_voxel_map.h), called from plain host loops in the order lv_map.cu launches its kernels.
 *
 * liblv_cpushim.so is this file, lidar_ring.cpp (the LiDAR buffer) and preloc.cpp (the start-pose searches); tests/shim_binding.py
 * loads it.
 */
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../limo-velo_b200/csrc/lv_ieskf.h"
#include "../../limo-velo_b200/csrc/lv_voxel_search.h"
#include "../gpu_shim/manifold_ops.h"

using namespace lv;

struct ShimMap {
    std::vector<uint4> table, btable;
    std::vector<float4> arena;
    std::vector<uint32_t> counters, touched, dirty;
    VoxelMapRW rw;
    VoxelMapView view;
    uint32_t n_inserted = 0;
};

struct ShimParams {
    int32_t max_iter;
    int32_t estimate_extrinsics;
    double max_dist_plane;
    float planes_threshold;
    float voxel_size;
    double R, D;
    double limits[23];
};

extern "C" {

/* the product's map update (lv_voxel_map.h: map_point_key, map_merge_run, map_dilate_item, map_halo_voxel_serial) run
 * serially, in the order lv_map.cu launches the kernels: keys -> stable sort -> merge -> dilate -> halo */
static void shim_add_impl(ShimMap* sm, const float* xyz, int64_t n, int downsample) {
    VoxelMapRW& m = sm->rw;
    m.counters[kCtrTouched] = 0;
    m.counters[kCtrDirty] = 0;
    std::vector<uint32_t> keys(n), vals(n);
    for (int64_t i = 0; i < n; ++i) { keys[i] = map_point_key(m, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]); vals[i] = (uint32_t)i; }
    std::stable_sort(vals.begin(), vals.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
    std::vector<uint32_t> ks(n);
    for (int64_t j = 0; j < n; ++j) ks[j] = keys[vals[j]];
    for (int64_t j = 0; j < n; ++j) {
        if (ks[j] == 0xFFFFFFFFu) continue;
        if (j > 0 && (ks[j - 1] >> kCellBits) == (ks[j] >> kCellBits)) continue;
        map_merge_run(m, ks.data(), vals.data(), (uint32_t)j, (uint32_t)n, xyz, sm->n_inserted, downsample);
    }
    const uint32_t nt = m.counters[kCtrTouched];
    for (uint32_t t = 0; t < nt * 27u; ++t) map_dilate_item(m, m.touched[t / 27u], (int)(t % 27u));
    const uint32_t nd = m.counters[kCtrDirty];
    for (uint32_t d = 0; d < nd; ++d) map_halo_voxel_serial(m, m.dirty[d]);
    sm->n_inserted += (uint32_t)n;
}

/* empty tables and a zeroed arena for `cap` map points: 8 table slots and 64 arena entries per point; returns the slots */
static uint32_t alloc_tables(int64_t cap, std::vector<uint4>& table, std::vector<uint4>& btable, std::vector<float4>& arena) {
    uint32_t slots = 1u << 14;
    while (slots < 8 * (uint64_t)(cap + 65536)) slots <<= 1;
    uint4 empty; empty.x = empty.y = 0xFFFFFFFFu; empty.z = empty.w = 0;
    uint4 zero; zero.x = zero.y = zero.z = zero.w = 0;
    table.assign(2 * (size_t)slots, zero);
    for (uint32_t s = 0; s < slots; ++s) table[2 * (size_t)s] = empty;
    btable.assign(slots / 4, empty);
    arena.assign((size_t)64 * (size_t)(cap + 65536) + (1u << 20), float4{});
    return slots;
}

/* cap: map points the tables are sized for (at least m) */
ShimMap* shim_map_create_cap(const float* xyz, int64_t m, int64_t cap, float cell) {
    ShimMap* sm = new ShimMap();
    const float ds = 0.2f;
    int k = (int)floor((double)cell / (double)ds + 0.5);
    k = k < 1 ? 1 : (k > kMaxCellsPerVoxel ? kMaxCellsPerVoxel : k);
    if (cap < m) cap = m;
    const uint32_t slots = alloc_tables(cap, sm->table, sm->btable, sm->arena);
    sm->counters.assign(kMapCounters, 0u);
    sm->counters[kCtrArenaTop] = 16u;
    sm->touched.resize(slots);
    sm->dirty.resize(slots);
    VoxelMapRW& r = sm->rw;
    r.table = sm->table.data(); r.mask = slots - 1; r.btable = sm->btable.data(); r.bmask = slots / 4 - 1;
    r.arena = sm->arena.data(); r.arena_cap = (uint32_t)sm->arena.size(); r.counters = sm->counters.data();
    r.touched = sm->touched.data(); r.dirty = sm->dirty.data(); r.list_cap = slots;
    r.grid.ds = ds; r.grid.k = k; r.grid.cell0 = (float)k * ds;
    sm->view = map_view_of(r);
    if (m > 0) shim_add_impl(sm, xyz, m, 0);
    return sm;
}
ShimMap* shim_map_create(const float* xyz, int64_t m, float cell, double max_dist) {
    (void)max_dist;
    return shim_map_create_cap(xyz, m, m, cell);
}
/* Mapper::add on an existing map (KD_TREE::Add_Points) */
void shim_map_add(ShimMap* sm, const float* xyz, int64_t n, int downsample) { shim_add_impl(sm, xyz, n, downsample); }
int64_t shim_map_size(const ShimMap* sm) { return (int64_t)(int32_t)sm->counters[kCtrPoints]; }
uint32_t shim_map_error(const ShimMap* sm) { return sm->counters[kCtrError]; }
/* all points, ascending id (insertion order) */
int64_t shim_map_points(const ShimMap* sm, float* out, int64_t cap) {
    std::vector<float4> all;
    for (uint32_t s = 0; s <= sm->rw.mask; ++s) {
        const uint4 t = sm->table[2 * (size_t)s];
        if ((t.x & t.y) == 0xFFFFFFFFu) continue;
        for (uint32_t k = 0; k < t.w; ++k) all.push_back(sm->arena[t.z + k]);
    }
    std::sort(all.begin(), all.end(), [](const float4& a, const float4& b) { uint32_t ia, ib; memcpy(&ia, &a.w, 4); memcpy(&ib, &b.w, 4); return ia < ib; });
    const int64_t n = (int64_t)all.size() < cap ? (int64_t)all.size() : cap;
    for (int64_t i = 0; i < n; ++i) { out[3 * i] = all[i].x; out[3 * i + 1] = all[i].y; out[3 * i + 2] = all[i].z; }
    return (int64_t)all.size();
}
/* structural invariants of the layout (tests): every halo bucket equals the concatenation of the 27 own extents */
int shim_map_check(const ShimMap* sm) {
    const VoxelMapRW& m = sm->rw;
    for (uint32_t s = 0; s <= m.mask; ++s) {
        const uint32_t* s32 = reinterpret_cast<const uint32_t*>(m.table + 2 * (size_t)s);
        if ((s32[0] & s32[1]) == 0xFFFFFFFFu) continue;
        if (s32[7] != 0u) return 1;                                         /* dirty flag left set */
        if (s32[3] > caps_own(s32[6]) || s32[5] > caps_halo(s32[6])) return 2;
        const uint64_t key = (uint64_t)s32[0] | ((uint64_t)s32[1] << 32);
        const int bx = (int)((uint32_t)key & 0x1FFFFFu), by = (int)((uint32_t)(key >> 21) & 0x1FFFFFu), bz = (int)((uint32_t)(key >> 42) & 0x1FFFFFu);
        uint32_t w = s32[4], total = 0;
        bool any_occupied_nb = false;
        for (int l = 0; l < 27; ++l) {
            const int nb = halo_lane_to_nb(l);
            const int cx = bx + nb % 3 - 1, cy = by + (nb / 3) % 3 - 1, cz = bz + nb / 9 - 1;
            if (cx < 0 || cy < 0 || cz < 0) continue;
            const int ns = voxel_find_rw(m, voxel_key((uint32_t)cx, (uint32_t)cy, (uint32_t)cz));
            if (ns < 0) { if (s32[3] > 0) return 3; continue; }             /* an occupied voxel has all 26 neighbour slots */
            const uint32_t* n32 = reinterpret_cast<const uint32_t*>(m.table + 2 * (size_t)ns);
            any_occupied_nb = any_occupied_nb || n32[3] > 0;
            for (uint32_t t = 0; t < n32[3]; ++t, ++w)
                if (memcmp(&m.arena[w], &m.arena[n32[2] + t], sizeof(float4)) != 0) return 4;
            total += n32[3];
        }
        if (total != s32[5]) return 5;
        if (s32[3] > 0) {                                                   /* block occupancy bit */
            if (!((block_find(sm->view, voxel_key((uint32_t)bx >> 2, (uint32_t)by >> 2, (uint32_t)bz >> 2)) >> block_bit((uint32_t)bx, (uint32_t)by, (uint32_t)bz)) & 1ull)) return 6;
        }
    }
    return 0;
}
/* sizes of the layout: dims = {voxel slots, block slots, arena_top, list capacity}; counters = the kMapCounters words */
void shim_map_dims(const ShimMap* sm, uint32_t* dims, uint32_t* counters) {
    dims[0] = sm->rw.mask + 1u;
    dims[1] = sm->rw.bmask + 1u;
    dims[2] = sm->counters[kCtrArenaTop];
    dims[3] = sm->rw.list_cap;
    memcpy(counters, sm->counters.data(), sizeof(uint32_t) * kMapCounters);
}
/* the whole layout as it stands (tests/map_ref.py checks it): both tables, arena[0, arena_top), the touched and dirty lists
 * of the last add (as many entries as their counters say, at most the list capacity) */
void shim_map_dump(const ShimMap* sm, uint32_t* table, uint32_t* btable, float* arena, uint32_t* touched, uint32_t* dirty) {
    memcpy(table, sm->table.data(), sizeof(uint4) * sm->table.size());
    memcpy(btable, sm->btable.data(), sizeof(uint4) * sm->btable.size());
    memcpy(arena, sm->arena.data(), sizeof(float4) * (size_t)sm->counters[kCtrArenaTop]);
    memcpy(touched, sm->touched.data(), sizeof(uint32_t) * std::min(sm->counters[kCtrTouched], sm->rw.list_cap));
    memcpy(dirty, sm->dirty.data(), sizeof(uint32_t) * std::min(sm->counters[kCtrDirty], sm->rw.list_cap));
}
/* lv_map.cu's map_grow: fresh tables for `cap` points, every old slot re-inserted by the product's voxel_rehash_item /
 * block_rehash_item (the functions the rehash kernel runs), the used prefix of the arena copied with its indices unchanged */
void shim_map_grow(ShimMap* sm, int64_t cap) {
    std::vector<uint4> table, btable;
    std::vector<float4> arena;
    const uint32_t slots = alloc_tables(cap, table, btable, arena);
    if (arena.size() < sm->arena.size()) arena.resize(sm->arena.size());
    const uint32_t top = std::min<uint32_t>(sm->counters[kCtrArenaTop], (uint32_t)sm->arena.size());
    std::copy(sm->arena.begin(), sm->arena.begin() + top, arena.begin());
    VoxelMapRW r = sm->rw;
    r.table = table.data(); r.mask = slots - 1; r.btable = btable.data(); r.bmask = slots / 4 - 1;
    r.arena = arena.data(); r.arena_cap = (uint32_t)arena.size();
    sm->counters[kCtrSlotsUsed] = 0;
    sm->counters[kCtrBlocksUsed] = 0;
    for (uint32_t s = 0; s <= sm->rw.mask; ++s) voxel_rehash_item(r, sm->table.data(), s);
    for (uint32_t s = 0; s <= sm->rw.bmask; ++s) block_rehash_item(r, sm->btable.data(), s);
    sm->table.swap(table);              /* the buffers move with the swap: r's pointers stay valid */
    sm->btable.swap(btable);
    sm->arena.swap(arena);
    sm->touched.assign(slots, 0u);
    sm->dirty.assign(slots, 0u);
    r.touched = sm->touched.data(); r.dirty = sm->dirty.data(); r.list_cap = slots;
    sm->rw = r;
    sm->view = map_view_of(r);
}
/* one device counter of the map (lv_voxel_map.h kCtr*) */
uint32_t shim_map_counter(const ShimMap* sm, int k) { return sm->counters[k]; }
void shim_map_destroy(ShimMap* m) { delete m; }

static void search_setup(const ShimParams* p, float cell, float* max_d2, double* gate, int* max_ring) {
    (void)cell;
    *gate = p->max_dist_plane * p->max_dist_plane;
    float f = (float)*gate;
    if ((double)f < *gate) f = nextafterf(f, INFINITY);
    *max_d2 = f;
    *max_ring = (int)ceil(p->max_dist_plane / (double)cell);
    if (*max_ring < 1) *max_ring = 1;
}

/* per-point outputs like lv_match_all; rows (n x 13) optional */
void shim_match_all(const ShimMap* sm, const double* x, const ShimParams* p, const float* xyz, int64_t n,
                    uint8_t* valid, int32_t* nn_idx, float* nn_sqd, float* plane, float* dist, float* g_world,
                    double* rows) {
    Frame fr;
    make_frame(x, &fr);
    float max_d2; double gate; int max_ring;
    search_setup(p, sm->view.grid.cell0, &max_d2, &gate, &max_ring);
    for (int64_t i = 0; i < n; ++i) {
        float g[3];
        rt_apply(fr.lidar_to_world, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], g);
        Top5 t;
        const float4* src = sm->view.arena;                    /* the two tiers of the search kernels */
        uint32_t bs, bc;
        const bool has_bucket = level0_probe(sm->view, g[0], g[1], g[2], &bs, &bc) >= 0;
        if (!level0_scan<GroupSerial>(sm->view, g[0], g[1], g[2], max_d2, bs, bc, has_bucket, t)) {
            const float bound0 = t.i4 >= 0 ? t.d4 : max_d2;
            knn5_rings<GroupSerial>(sm->view, g[0], g[1], g[2], max_d2, bound0, t);
        }
        float abcd[4] = {0, 0, 0, 0}, d = 0;
        double row[12] = {0}, h = 0;
        bool chosen = false;
        int ids[5] = {t.i0, t.i1, t.i2, t.i3, t.i4};
        float ds[5] = {t.d0, t.d1, t.d2, t.d3, t.d4};
        float q[5][3];
        if (t.i4 >= 0) {                                     /* map point ids, as the fit kernel orders them */
            for (int k = 0; k < 5; ++k) {
                q[k][0] = src[ids[k]].x; q[k][1] = src[ids[k]].y; q[k][2] = src[ids[k]].z;
                memcpy(&ids[k], &src[ids[k]].w, 4);
            }
            canonical_neighbour_order(q, ds, ids);
        }
        if (t.i4 >= 0 && (double)t.d4 < gate) {
            chosen = plane_fit(q, p->planes_threshold, abcd);
            if (chosen) {
                d = plane_dist(abcd, g);
                jacobian_row(fr, g, abcd, d, p->estimate_extrinsics != 0, row, &h);
            } else {
                abcd[0] = abcd[1] = abcd[2] = abcd[3] = 0;
            }
        }
        if (valid) valid[i] = chosen;
        if (g_world) memcpy(g_world + 3 * i, g, sizeof(g));
        for (int k = 0; k < 5; ++k) {
            if (nn_idx) nn_idx[5 * i + k] = t.i4 >= 0 ? ids[k] : -1;
            if (nn_sqd) nn_sqd[5 * i + k] = t.i4 >= 0 ? ds[k] : INFINITY;
        }
        if (plane) memcpy(plane + 4 * i, abcd, sizeof(abcd));
        if (dist) dist[i] = d;
        if (rows) {
            for (int k = 0; k < 12; ++k) rows[13 * i + k] = chosen ? row[k] : 0.0;
            rows[13 * i + 12] = chosen ? h : 0.0;
        }
    }
}

static void reduce_rows(const double* rows, const uint8_t* valid, int64_t n, double* HTH, double* HTh, int64_t* nm) {
    for (int i = 0; i < 144; ++i) HTH[i] = 0;
    for (int i = 0; i < 12; ++i) HTh[i] = 0;
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (!valid[i]) continue;
        const double* r = rows + 13 * i;
        for (int a = 0; a < 12; ++a) {
            for (int b = 0; b < 12; ++b) HTH[a * 12 + b] += r[a] * r[b];
            HTh[a] += r[a] * r[12];
        }
        ++cnt;
    }
    *nm = cnt;
}

/* whole update with the product's ieskf_begin / ieskf_step run serially; returns status */
int shim_update(const ShimMap* sm, double* x, double* P, const ShimParams* p, const float* xyz, int64_t n,
                IterLog* logs, int32_t* n_evals) {
    UpdateCtrl* c = new UpdateCtrl();
    IeskfWork* w = new IeskfWork();
    memset(c, 0, sizeof(*c));
    memcpy(c->x, x, sizeof(double) * kStateLen);
    memcpy(c->P, P, sizeof(double) * kN * kN);
    IeskfParams prm;
    prm.R = p->R; prm.D = p->D; prm.max_iter = p->max_iter; prm.estimate_extrinsics = p->estimate_extrinsics;
    for (int i = 0; i < kN; ++i) prm.limits[i] = p->limits[i];
    ExecSerial ex;
    PrepWork* pw = new PrepWork();
    ieskf_begin(ex, c);
    std::vector<double> rows(13 * n);
    std::vector<uint8_t> valid(n);
    for (int e = 0; e <= p->max_iter && !c->done; ++e) {
        shim_match_all(sm, c->x, p, xyz, n, valid.data(), nullptr, nullptr, nullptr, nullptr, nullptr, rows.data());
        reduce_rows(rows.data(), valid.data(), n, w->HTH, w->HTh, &w->n_matches);
        ieskf_prepare(ex, c, pw);
        ieskf_load(ex, c, w);
        ieskf_step(ex, prm, c, w);
    }
    memcpy(x, c->x, sizeof(double) * kStateLen);
    if (c->status == 0) memcpy(P, c->P, sizeof(double) * kN * kN);
    *n_evals = c->n_evals;
    memcpy(logs, c->logs, sizeof(IterLog) * kMaxEvals);
    const int st = c->status;
    delete c;
    delete w;
    delete pw;
    return st;
}

/* the 23x23 step alone, measurement supplied */
int shim_step(const double* x_prop, const double* P_prop, const double* x_cur, const ShimParams* p, const double* HTH,
              const double* HTh, int64_t nm, int iter, int t_in, double* dx_out, double* x_new, double* P_out,
              int32_t* done) {
    UpdateCtrl* c = new UpdateCtrl();
    IeskfWork* w = new IeskfWork();
    memset(c, 0, sizeof(*c));
    memcpy(c->x_prop, x_prop, sizeof(double) * kStateLen);
    memcpy(c->P_prop, P_prop, sizeof(double) * kN * kN);
    memcpy(c->x, x_cur, sizeof(double) * kStateLen);
    c->iter = iter; c->t = t_in;
    IeskfParams prm;
    prm.R = p->R; prm.D = p->D; prm.max_iter = p->max_iter; prm.estimate_extrinsics = p->estimate_extrinsics;
    for (int i = 0; i < kN; ++i) prm.limits[i] = p->limits[i];
    memcpy(w->HTH, HTH, sizeof(double) * 144);
    memcpy(w->HTh, HTh, sizeof(double) * 12);
    w->n_matches = nm;
    ExecSerial ex;
    PrepWork* pw = new PrepWork();
    ieskf_prepare(ex, c, pw);
    delete pw;
    ieskf_load(ex, c, w);
    ieskf_step(ex, prm, c, w);
    memcpy(dx_out, c->logs[0].dx, sizeof(double) * kN);
    memcpy(x_new, c->x, sizeof(double) * kStateLen);
    if (c->done && c->status == 0) memcpy(P_out, c->P, sizeof(double) * kN * kN);
    *done = c->done;
    const int st = c->status;
    delete c;
    delete w;
    return st;
}

/* tests/gpu_shim's gs_manifold on the host: manifold_op (manifold_ops.h) over n rows */
void shim_manifold(const int* op, const double* in, double* out, int n) {
    for (int i = 0; i < n; ++i) manifold_op(op[i], in + (size_t)kManIn * i, out + (size_t)kManOut * i);
}
void shim_boxplus(double* x, const double* d) { state_boxplus(x, d); }
void shim_boxminus(const double* x, const double* y, double* d) { state_boxminus(x, y, d); }
void shim_plane_fit(const float* pts5, float thr, float* abcd, int* ok) {
    float q[5][3];
    memcpy(q, pts5, sizeof(q));
    *ok = plane_fit(q, thr, abcd) ? 1 : 0;
}
/* tests/gpu_shim's gs_fit_sets on the host: per set, distances from g, the tie order, fit, distance and row */
void shim_fit_sets(const float* q_in, const float* g_in, const int* id_in, const double* x, float thr, int est, int n, int* id_out,
                   float* abcd_out, int* ok_out, float* dist_out, double* row_out) {
    Frame fr;
    make_frame(x, &fr);
    for (int i = 0; i < n; ++i) {
        float q[5][3], d[5], abcd[4];
        int id[5];
        const float g[3] = {g_in[3 * i], g_in[3 * i + 1], g_in[3 * i + 2]};
        for (int k = 0; k < 5; ++k) {
            for (int a = 0; a < 3; ++a) q[k][a] = q_in[15 * i + 3 * k + a];
            d[k] = sq_dist(g[0], g[1], g[2], q[k][0], q[k][1], q[k][2]);
            id[k] = id_in[5 * i + k];
        }
        canonical_neighbour_order(q, d, id);
        ok_out[i] = plane_fit(q, thr, abcd) ? 1 : 0;
        const float dist = plane_dist(abcd, g);
        double row[12], h;
        jacobian_row(fr, g, abcd, dist, est != 0, row, &h);
        memcpy(id_out + 5 * i, id, sizeof(id));
        memcpy(abcd_out + 4 * i, abcd, sizeof(abcd));
        dist_out[i] = dist;
        memcpy(row_out + 13 * (size_t)i, row, sizeof(row));
        row_out[13 * (size_t)i + 12] = h;
    }
}
int shim_sizeof_iterlog() { return (int)sizeof(IterLog); }
unsigned long long shim_block_cube_mask(int cbx, int cby, int cbz, int r) { return block_cube_mask(cbx, cby, cbz, r); }

}  // extern "C"

/* neighbour reuse (query_reusable): search every query from state x0 keeping the reuse reference, then judge
 * from state x1.  reused[i] = 1 when the stored five were vouched for; for those, same[i] = 1 iff a fresh search
 * from x1 returns the same map points (by original index) with bit-identical distances in the same order. */
extern "C" void shim_reuse_check(const ShimMap* sm, const double* x0, const double* x1, double max_dist, const float* xyz,
                                 int64_t n, uint8_t* reused, uint8_t* same) {
    Frame f0, f1;
    make_frame(x0, &f0);
    make_frame(x1, &f1);
    const double gate = max_dist * max_dist;
    float max_d2 = (float)gate;
    if ((double)max_d2 < gate) max_d2 = nextafterf(max_d2, INFINITY);
    auto search = [&](const float* g, Top5& t, float* lb) -> const float4* {
        uint32_t bs, bc;
        float region = 0.f;
        const bool hb = level0_probe(sm->view, g[0], g[1], g[2], &bs, &bc) >= 0;
        if (level0_scan<GroupSerial>(sm->view, g[0], g[1], g[2], max_d2, bs, bc, hb, t, &region)) {
            *lb = outsider_bound(t.d5, region);
            return sm->view.arena;
        }
        const float bound0 = t.i4 >= 0 ? t.d4 : max_d2;
        knn5_rings<GroupSerial>(sm->view, g[0], g[1], g[2], max_d2, bound0, t, &region);
        *lb = outsider_bound(t.d5, region);
        return sm->view.arena;
    };
    for (int64_t i = 0; i < n; ++i) {
        float g0[3], g1[3];
        rt_apply(f0.lidar_to_world, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], g0);
        rt_apply(f1.lidar_to_world, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], g1);
        Top5 t0, t1, tr;
        float lb0 = 0.f, lb1 = 0.f;
        const float4* src0 = search(g0, t0, &lb0);
        const float ref[4] = {g0[0], g0[1], g0[2], lb0};
        const int id[5] = {t0.i0, t0.i1, t0.i2, t0.i3, t0.i4};
        float q[5][3];
        for (int k = 0; k < 5; ++k)
            if (id[k] >= 0) { q[k][0] = src0[id[k]].x; q[k][1] = src0[id[k]].y; q[k][2] = src0[id[k]].z; }
        reused[i] = query_reusable(ref, g1, q, id, max_d2, tr) ? 1 : 0;
        same[i] = 0;
        if (!reused[i]) continue;
        const float4* src1 = search(g1, t1, &lb1);
        const int a[5] = {tr.i0, tr.i1, tr.i2, tr.i3, tr.i4}, b[5] = {t1.i0, t1.i1, t1.i2, t1.i3, t1.i4};
        const float da[5] = {tr.d0, tr.d1, tr.d2, tr.d3, tr.d4}, db[5] = {t1.d0, t1.d1, t1.d2, t1.d3, t1.d4};
        bool ok = true;
        for (int k = 0; k < 5; ++k) {
            if (b[k] < 0) { ok = false; break; }
            int oa, ob;
            memcpy(&oa, &src0[a[k]].w, 4);
            memcpy(&ob, &src1[b[k]].w, 4);
            ok = ok && oa == ob && da[k] == db[k];
        }
        same[i] = ok ? 1 : 0;
    }
}

/* diagnostics: which queries level 0 settles */
extern "C" void shim_query_stats(const ShimMap* sm, const double* x, const float* xyz, int64_t n, double max_dist,
                                 int32_t* level_out, int32_t* scanned_out) {
    Frame fr;
    make_frame(x, &fr);
    const double gate = max_dist * max_dist;
    float max_d2 = (float)gate;
    if ((double)max_d2 < gate) max_d2 = nextafterf(max_d2, INFINITY);
    for (int64_t i = 0; i < n; ++i) {
        float g[3];
        rt_apply(fr.lidar_to_world, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], g);
        Top5 t;
        uint32_t bs, bc;
        const int slot = level0_probe(sm->view, g[0], g[1], g[2], &bs, &bc);
        const bool ok = level0_scan<GroupSerial>(sm->view, g[0], g[1], g[2], max_d2, bs, bc, slot >= 0, t);
        level_out[i] = ok ? 0 : (slot < 0 ? 2 : 1);    /* 0 settled, 1 bucket but not certified, 2 no slot */
        scanned_out[i] = slot >= 0 ? (int)bc : 0;
    }
}
