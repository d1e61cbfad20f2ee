/*
 * limovelo_synth_main.cpp — the tick of the reference driver (src/main.cpp:52-130) on the synthetic
 * reader: propagate_to -> compensate -> downsample -> correct -> map.add, with LIMO-Velo's module
 * names (Modules.hpp) on top of liblimovelo_b200.so.
 *
 *   limovelo_synth <config.yaml> [sweeps=10] [map_points=200000] [rings=64] [azimuths=1024] [downsample_leaf=0] [mapping_online=1]
 *
 * mapping_online=0 runs main.cpp:106-117 instead of the online map add: once per full_rotation_time the last full rotation goes to
 * the world frame, through the voxel grid (when a leaf is given) and into the map, on the device.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <chrono>

#include "../../include/lv_synth.h"
#include "Modules.hpp"

int main(int argc, char** argv) {
    if (argc < 2) {
        fprintf(stderr, "usage: %s config.yaml [sweeps] [map_points] [rings] [azimuths] [downsample_leaf] [mapping_online]\n", argv[0]);
        return 2;
    }
    const int sweeps = argc > 2 ? atoi(argv[2]) : 10;
    const int64_t map_points = argc > 3 ? atoll(argv[3]) : 200000;
    const int rings = argc > 4 ? atoi(argv[4]) : 64, azimuths = argc > 5 ? atoi(argv[5]) : 1024;
    const float leaf = argc > 6 ? (float)atof(argv[6]) : 0.f;
    const bool mapping_online = argc > 7 ? atoi(argv[7]) != 0 : true;
    try {
        lv_params prm;
        lv_default_params(&prm);
        lv::check(lv_params_from_yaml(argv[1], &prm), "config");
        prm.max_map_points = map_points + (int64_t)(sweeps + 2) * rings * azimuths;
        prm.max_points = (int64_t)rings * azimuths;
        lv::Context ctx(prm);
        lv::Mapper map(ctx);
        lv::Localizator loc(ctx);
        lv::Compensator comp(ctx);
        lv::Accumulator accum;

        lv_synth_world* world = lv_synth_world_create(20260924, map_points);
        std::vector<float> buf(3 * (size_t)map_points);
        lv_synth_world_map(world, buf.data(), map_points);
        lv::Points cloud((size_t)map_points);
        for (int64_t i = 0; i < map_points; ++i) cloud[i] = lv::Point{buf[3 * i], buf[3 * i + 1], buf[3 * i + 2], 0.0};
        map.add(cloud, 0.0, false);                                   /* first map.add builds (main.cpp:101) */

        const float q0[4] = {0, 0, 0, 1};
        loc.initialize(q0, 0.0);
        double truth[LV_STATE_LEN];
        lv_synth_pose(world, 10.0, &prm, truth);
        lv::check(lv_set_state(ctx.h, truth, nullptr), "seed pose");
        double P0[LV_DOF * LV_DOF];
        lv::check(lv_get_state(ctx.h, nullptr, P0), "P0");

        std::vector<float> sw(3 * (size_t)rings * azimuths);
        /* mapping offline: the full rotation (device), its world-frame copy and its voxel grid, each with a device count */
        const int64_t n_sweep = (int64_t)rings * azimuths;
        float* d_full = (float*)lv_device_alloc(ctx.h, 12 * n_sweep);
        float* d_world = (float*)lv_device_alloc(ctx.h, 12 * n_sweep);
        float* d_ds = (float*)lv_device_alloc(ctx.h, 12 * n_sweep);
        int64_t* d_counts = (int64_t*)lv_device_alloc(ctx.h, 3 * sizeof(int64_t));
        if (!d_full || !d_world || !d_ds || !d_counts) throw std::runtime_error("device buffers for mapping offline");
        for (int k = 0; k < sweeps; ++k) {
            const double t2 = 0.1 * (k + 1);
            lv_synth_pose(world, 10.0 + 1.5 * (k + 1), &prm, truth);   /* 15 m/s at 10 Hz */
            lv_synth_sweep(world, truth, rings, azimuths, -24.8, 2.0, 4.0, 0.02, 100 + k, sw.data());
            lv::Points pts((size_t)rings * azimuths);
            for (size_t i = 0; i < pts.size(); ++i) pts[i] = lv::Point{sw[3 * i], sw[3 * i + 1], sw[3 * i + 2], t2};
            accum.receive_lidar(pts);
            /* constant-velocity IMU between sweeps: the accelerometer reads -grav at rest (f = R a + grav,
             * use-ikfom.cpp:49-61, with grav = -initial_gravity, Localizator.cpp:138) */
            {
                lv::State cur = loc.latest_state();
                for (int s = 1; s <= 4; ++s)
                    accum.receive_imu(lv::IMU{{-cur.x[23], -cur.x[24], -cur.x[25]}, {0, 0, 0}, t2 - 0.1 + 0.025 * s});
            }
            loc.propagate_to_device(accum.get_imus(t2 - 0.1, t2), t2);   /* main.cpp:76: all IMU samples in one device launch */
            /* the synthetic vehicle is kinematic (no simulated IMU dynamics): take pose and velocity of the
             * prediction from the ground truth plus a 3 cm offset, and re-open the covariance to P0 so that
             * the offset is a consistent prior error */
            lv::State pred = loc.latest_state();
            double prev[LV_STATE_LEN];
            lv_synth_pose(world, 10.0 + 1.5 * k, &prm, prev);
            for (int i = 0; i < 7; ++i) pred.x[i] = truth[i] + (i < 3 ? 0.03 : 0.0);
            for (int i = 0; i < 3; ++i) pred.x[14 + i] = (truth[i] - prev[i]) / 0.1;
            lv::check(lv_set_state(ctx.h, pred.x, P0), "prediction");
            /* main.cpp:79-80: the synthetic sweep arrives deskewed (rays cast from the pose at t2); the voxel-grid downsample
             * (Compensator::downsample, leaf downsample_prec) runs on the GPU when a leaf is given on the command line */
            lv::Points ds = leaf > 0.f ? comp.downsample(comp.compensate(accum.points), leaf) : comp.downsample(comp.compensate(accum.points));
            const auto t0 = std::chrono::steady_clock::now();
            const int evals = loc.correct(ds, t2);                    /* main.cpp:84 */
            /* main.cpp:101-105: the sweep joins the map in the world frame of the corrected state, under the 0.2 m rule —
             * on the device, with the state the update left there (no copy of the sweep, no copy of the state) */
            if (mapping_online) map.add_corrected_sweep(t2, true);
            else if (map.hasToMap(t2)) {                              /* main.cpp:106-117 */
                /* the synthetic sweep is one full rotation, deskewed at t2: [t2 - full_rotation_time, t2] */
                const int64_t n_full = (int64_t)accum.points.size();
                lv::check(lv_memcpy_h2d(ctx.h, d_full, sw.data(), 12 * n_full), "full rotation");
                lv::check(lv_memcpy_h2d(ctx.h, d_counts, &n_full, sizeof(int64_t)), "full rotation");
                loc.to_world_device(d_full, d_counts, n_sweep, d_world, d_counts + 1);
                if (leaf > 0.f) {
                    lv::check(lv_voxelgrid_downsample_device_async(ctx.h, d_world, d_counts + 1, n_sweep, leaf, d_ds, d_counts + 2),
                              "Compensator::downsample");
                    map.add_device(d_ds, d_counts + 2, n_sweep, t2, true);
                } else {
                    map.add_device(d_world, d_counts + 1, n_sweep, t2, true);
                }
            }
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            lv::State X = loc.latest_state();
            const double err = sqrt(pow(X.x[0] - truth[0], 2) + pow(X.x[1] - truth[1], 2) + pow(X.x[2] - truth[2], 2));
            printf("sweep %2d  t=%.1f  points=%zu  evals=%d  Nm=%lld  correct()+map.add()=%.3f ms  |pos error|=%.4f m  map=%d\n", k, t2, ds.size(), evals,
                   evals ? (long long)loc.logs[evals - 1].n_matches : 0LL, ms, err, map.size());
        }
        for (void* p : {(void*)d_full, (void*)d_world, (void*)d_ds, (void*)d_counts}) lv_device_free(ctx.h, p);
        lv_synth_world_destroy(world);
    } catch (const std::exception& e) {
        fprintf(stderr, "limovelo_synth: %s\n", e.what());
        return 1;
    }
    return 0;
}
