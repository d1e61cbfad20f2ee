/*
 * Modules.hpp — LIMO-Velo's module boundaries on top of the C ABI (header-only C++).
 *
 * The reference driver (src/main.cpp:52-130) talks to four singletons: Accumulator, Compensator,
 * Localizator, Mapper.  These classes keep their names and the method names / argument meaning of the
 * calls that sit on the per-sweep path, so the tick of main.cpp reads the same; the bodies forward to
 * liblimovelo_b200.so.  One `Context` (= one lv_handle) replaces the singletons' hidden coupling
 * (use-ikfom.cpp:18-19 reaches Localizator::getInstance() / Mapper::getInstance()).
 *
 *   reference                                      here
 *   Points = std::deque<Point> (Common.hpp:231)    lv::Points = std::vector<lv::Point> (xyz, time, intensity, range)
 *   State (Objects.hpp:97-137, fp32)               lv::State  = flat state_ikfom layout (26 doubles) + time
 *   Mapper::add(Points&, t, downsample)            Mapper::add(...)          -> lv_map_build / lv_map_add
 *   Mapper::exists() / size()                      same                      -> lv_map_exists / lv_map_size
 *   Localizator::correct(const Points&, t)         same                      -> lv_correct
 *   Localizator::propagate_to(t)                   propagate(IMU) per sample -> lv_predict
 *   Localizator::latest_state()                    same                      -> lv_get_state
 *   Compensator::compensate / downsample           identity hooks (input is already deskewed; SURVEY 8f-2/3)
 *   Accumulator::receive_* / get_*                 plain buffers fed by the synthetic / rosbag reader
 */
#ifndef LIMOVELO_B200_MODULES_HPP_
#define LIMOVELO_B200_MODULES_HPP_

#include <deque>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/limovelo_b200.h"

namespace lv {

/* Point (Objects.hpp): xyz, time and the attributes the publishers send (Point::toPCL, Point.cpp:113-122) */
struct Point { float x, y, z; double time; float intensity, range; };
typedef std::vector<Point> Points;
struct IMU { double a[3]; double w[3]; double time; };
typedef std::deque<IMU> IMUs;

struct State {
    double x[LV_STATE_LEN];
    double time;
    const double* pos() const { return x; }
    const double* rot() const { return x + 3; }       /* quaternion x, y, z, w */
};

inline void check(lv_status s, const char* what) {
    if (s != LV_OK) throw std::runtime_error(std::string(what) + ": " + lv_last_error());
}

/* one sequence on one GPU: owns the handle the modules share */
class Context {
   public:
    explicit Context(const lv_params& p) : params(p) { check(lv_create(&params, &h), "lv_create"); }
    explicit Context(const std::string& yaml) {
        lv_default_params(&params);
        check(lv_params_from_yaml(yaml.c_str(), &params), "lv_params_from_yaml");
        check(lv_create(&params, &h), "lv_create");
    }
    ~Context() { lv_destroy(h); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    lv_handle h = nullptr;
    lv_params params;
};

class Mapper {
   public:
    explicit Mapper(Context& c) : ctx(c) {}
    double last_map_time = -1;
    bool exists() { return lv_map_exists(ctx.h) != 0; }                       /* Mapper.cpp:36-38 */
    int size() { return (int)lv_map_size(ctx.h); }                            /* Mapper.cpp:32-34 */
    /* Mapper.cpp:22-30: build on the first call, Add_Points (0.2 m voxel rule if downsample) afterwards */
    void add(const Points& points, double time, bool downsample = false) {
        if (points.empty()) return;
        std::vector<float> xyz(3 * points.size());
        for (size_t i = 0; i < points.size(); ++i) { xyz[3 * i] = points[i].x; xyz[3 * i + 1] = points[i].y; xyz[3 * i + 2] = points[i].z; }
        lv_status s = exists() ? lv_map_add(ctx.h, xyz.data(), (int64_t)points.size(), downsample ? 1 : 0)
                               : lv_map_build(ctx.h, xyz.data(), (int64_t)points.size());
        check(s, "Mapper::add");
        last_map_time = time;
    }
    /* main.cpp:99-105 without leaving the GPU: the sweep Localizator::correct has just used (still resident on the device)
     * is transformed by the corrected state and merged (lv_map_add_last_sweep); nothing is copied to or from the host */
    void add_corrected_sweep(double time, bool downsample = true) {
        check(lv_map_add_last_sweep(ctx.h, downsample ? 1 : 0), "Mapper::add_corrected_sweep");
        last_map_time = time;
    }
    /* Mapper::add of a device cloud whose count is on the device (lv_map_add_device_async), e.g. main.cpp:111-114's
     * global_full_ds_compensated.  The reference skips an empty cloud without touching last_map_time; the host does not know the
     * count here, so last_map_time becomes `time` either way (a full rotation of LiDAR data is not empty in practice). */
    void add_device(const float* d_xyz, const int64_t* d_n, int64_t n_max, double time, bool downsample = true) {
        check(lv_map_add_device_async(ctx.h, d_xyz, d_n, n_max, downsample ? 1 : 0), "Mapper::add_device");
        last_map_time = time;
    }
    /* Mapper.cpp:58-61: with mapping_online false, whether the tick at t maps the last full rotation */
    double full_rotation_time = 0.1;                                            /* Config.full_rotation_time (YAML) */
    bool hasToMap(double t) { return has_to_map(last_map_time, t, full_rotation_time); }
    static bool has_to_map(double& last_map_time, double t, double full_rotation_time) {
        if (last_map_time < 0) last_map_time = t;
        return t - last_map_time >= full_rotation_time;
    }
    /* the ikd-Tree has no capacity (ikd_Tree.cpp:478-573): grow the device map now to hold `points`, or let it grow by itself
     * before the adds that may not fit, up to `max_points` (0: off) — lv_map_reserve / lv_map_set_growth */
    void reserve(int64_t points) { check(lv_map_reserve(ctx.h, points), "Mapper::reserve"); }
    void set_growth(int64_t max_points) { check(lv_map_set_growth(ctx.h, max_points), "Mapper::set_growth"); }

   private:
    Context& ctx;
};

class Localizator {
   public:
    explicit Localizator(Context& c) : ctx(c) {}
    double last_time_integrated = -1;
    double last_time_updated = -1;
    bool initialized = false;
    /* Localizator.cpp:119-127,135-153 */
    void initialize(const float q_imu[4], double t) {
        check(lv_init_state(ctx.h, q_imu), "Localizator::initialize");
        last_time_integrated = t;
        initialized = true;
    }
    /* Localizator.cpp:159-173: one IMU sample */
    void propagate(const IMU& imu) {
        if (last_time_integrated < 0) last_time_integrated = imu.time;
        check(lv_predict(ctx.h, imu.a, imu.w, imu.time - last_time_integrated), "Localizator::propagate");
        last_time_integrated = imu.time;
    }
    /* Localizator.cpp:59-75 over an explicit IMU list (the Accumulator lookup is the caller's) */
    void propagate_to(const IMUs& imus, double t) {
        for (const IMU& imu : imus) propagate(imu);
        if (!imus.empty()) { IMU last = imus.back(); last.time = t; propagate(last); }
    }
    /* the same with every IMU sample in ONE device launch (lv_propagate_device): the filter state stays in HBM between the
     * previous update and the next one */
    void propagate_to_device(const IMUs& imus, double t) {
        if (imus.empty()) return;
        std::vector<double> a, w, dt;
        double last = last_time_integrated < 0 ? imus.front().time : last_time_integrated;
        for (const IMU& imu : imus) {
            for (int k = 0; k < 3; ++k) { a.push_back(imu.a[k]); w.push_back(imu.w[k]); }
            dt.push_back(imu.time - last);
            last = imu.time;
        }
        for (int k = 0; k < 3; ++k) { a.push_back(imus.back().a[k]); w.push_back(imus.back().w[k]); }   /* Localizator.cpp:70-74: the last sample up to t */
        dt.push_back(t - last);
        check(lv_propagate_device(ctx.h, a.data(), w.data(), dt.data(), (int32_t)dt.size()), "Localizator::propagate_to_device");
        last_time_integrated = t;
    }
    /* Localizator.cpp:23-27.  Returns the number of h-evaluations (0 when the map is empty). */
    int correct(const Points& points, double time) {
        if (points.empty()) return 0;
        std::vector<float> xyz(3 * points.size());
        for (size_t i = 0; i < points.size(); ++i) { xyz[3 * i] = points[i].x; xyz[3 * i + 1] = points[i].y; xyz[3 * i + 2] = points[i].z; }
        int32_t n_evals = 0;
        const lv_status s = lv_correct(ctx.h, xyz.data(), (int64_t)points.size(), time, logs, &n_evals, nullptr, nullptr);
        if (s == LV_EMPTY_MAP) return 0;                                       /* Localizator.cpp:24 */
        if (s != LV_TOO_FEW_MATCHES) check(s, "Localizator::correct");
        last_time_updated = time;
        return n_evals;
    }
    /* `Xt2 * Xt2.I_Rt_L() * points` (main.cpp:91-93, 111) on the device with the state the last correct left there
     * (lv_sweep_to_world_device_async): global_ds_compensated and global_compensated for the publishers, or the full rotation of
     * the offline map add.  *d_n_out = 0 when the MAX_POINTS2MATCH gate of correct_device_async stopped the tick. */
    void to_world_device(const float* d_xyz_lidar, const int64_t* d_n, int64_t n_max, float* d_xyz_world, int64_t* d_n_out) {
        check(lv_sweep_to_world_device_async(ctx.h, d_xyz_lidar, d_n, n_max, d_xyz_world, d_n_out), "Localizator::to_world_device");
    }
    State latest_state() {                                                     /* Localizator.cpp:77-98 */
        State s;
        check(lv_get_state(ctx.h, s.x, nullptr), "Localizator::latest_state");
        s.time = last_time_updated >= 0 ? last_time_updated : last_time_integrated;
        return s;
    }
    lv_iter_log logs[LV_MAX_EVALS];

   private:
    Context& ctx;
};

/* Deskew (lv_compensate) and voxel-grid downsample (lv_voxelgrid_downsample) on the GPU. */
class Compensator {
   public:
    explicit Compensator(Context& c) : ctx(c) {}
    /* Compensator::compensate(states, Xt2, points) (Compensator.cpp:123-146): `path` as Compensator::upsample
     * leaves it (lv_compensator_upsample), `Xt2` from lv_compensator_get_t2; points sorted by time */
    Points compensate(const std::vector<lv_state32>& path, const lv_state32& Xt2, const Points& sweep) {
        if (sweep.empty()) return Points();                                    /* Compensator.cpp:24 */
        std::vector<float> xyz(3 * sweep.size()), out(3 * sweep.size());
        std::vector<double> t(sweep.size());
        for (size_t i = 0; i < sweep.size(); ++i) {
            xyz[3 * i] = sweep[i].x; xyz[3 * i + 1] = sweep[i].y; xyz[3 * i + 2] = sweep[i].z;
            t[i] = sweep[i].time;
        }
        if (lv_compensate(ctx.h, path.data(), (int32_t)path.size(), &Xt2, xyz.data(), t.data(), (int64_t)sweep.size(),
                          out.data()) != LV_OK)
            throw std::runtime_error(lv_last_error());
        Points res = sweep;                                                    /* attributes ride along (RotTransl.cpp:43-48) */
        for (size_t i = 0; i < res.size(); ++i) { res[i].x = out[3 * i]; res[i].y = out[3 * i + 1]; res[i].z = out[3 * i + 2]; }
        return res;
    }
    Points compensate(const Points& sweep) { return sweep; }                   /* a sweep that arrives deskewed (synthetic reader) */
    /* Compensator::downsample -> voxelgrid_downsample (Compensator.cpp:115-118,148-163) of full points: per leaf the centroid, time 0,
     * the mean intensity and range = |centroid| (Point(const full_info::Point&), Point.cpp:21-25) — lv_voxelgrid_downsample_full.
     * When PCL passes the input through (cell-index overflow) the points keep xyz, time and intensity, and range becomes |p| */
    Points downsample(const Points& sweep, float downsample_prec) {
        if (sweep.empty()) return Points();
        const size_t n = sweep.size();
        std::vector<float> xyz(3 * n), out(3 * n), in_i(n), out_i(n), out_r(n);
        std::vector<double> t(n), out_t(n);
        for (size_t i = 0; i < n; ++i) {
            xyz[3 * i] = sweep[i].x; xyz[3 * i + 1] = sweep[i].y; xyz[3 * i + 2] = sweep[i].z;
            t[i] = sweep[i].time; in_i[i] = sweep[i].intensity;
        }
        int64_t m = 0;
        check(lv_voxelgrid_downsample_full(ctx.h, xyz.data(), t.data(), in_i.data(), (int64_t)n, downsample_prec, out.data(), out_t.data(),
                                           out_i.data(), out_r.data(), &m),
              "Compensator::downsample");                                      /* the overflow pass-through is LV_OK, done on the device */
        Points res((size_t)m);
        for (int64_t i = 0; i < m; ++i) res[(size_t)i] = Point{out[3 * i], out[3 * i + 1], out[3 * i + 2], out_t[i], out_i[i], out_r[i]};
        return res;
    }
    Points downsample(const Points& sweep) { return sweep; }                   /* a sweep that arrives downsampled */

   private:
    Context& ctx;
};

/* Plain time-ordered buffers (Accumulator.hpp:61-74), fed by a reader instead of ROS callbacks; with a Context the LiDAR buffer
 * (BUFFER_L) lives in HBM instead (lv_lidar_*), so the tick reads like main.cpp:61-122:
 *
 *     accum.receive_lidar_device(msg);                                  // Accumulator.cpp:39-48: process -> push, on the device
 *     ... t2, delta, t1 = max(t2 - delta, loc.last_time_updated); if (t2 - t1 < delta - 1e-6) break;   (host, main.cpp:61-71)
 *     accum.get_points_device(t1, t2, d_xyz, d_time, n_max, d_n);        // Compensator.cpp:23
 *     lv_compensate_device_async(...); lv_voxelgrid_downsample_device_async(...); lv_correct_device_async(...); ...
 *     accum.clear_lidar(t2 - empty_lidar_time);                         // main.cpp:122
 */
class Accumulator {
   public:
    Accumulator() = default;
    /* full: BUFFER_L keeps each point's intensity and range too (lv_lidar_reserve_full), for the *_full forms below */
    explicit Accumulator(Context& c, int64_t lidar_capacity, bool full = false) : ctx(&c) {
        check(full ? lv_lidar_reserve_full(c.h, lidar_capacity) : lv_lidar_reserve(c.h, lidar_capacity), "Accumulator");
    }
    void receive_lidar(const Points& sweep) { points = sweep; }                /* Accumulator.cpp:39-48 */
    /* Accumulator::receive_lidar on the message's bytes in device memory: Accumulator::process (lv_process_cloud_device_async into
     * the caller's scratch d_xyz / d_time / d_n, room for msg_n points) -> every point pushed onto BUFFER_L; no host wait */
    struct DeviceMessage {
        lv_lidar_type type; const lv_cloud_layout* layout; const uint8_t* d_data; int64_t data_bytes, n; uint64_t stamp_us;
        int stamp_beginning, offset_beginning; double full_rotation_time; int32_t downsample_rate; double min_dist;
    };
    void receive_lidar_device(const DeviceMessage& m, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_cloud_device_async(ctx->h, m.type, m.layout, m.d_data, m.data_bytes, m.n, m.stamp_us, m.stamp_beginning,
                                            m.offset_beginning, m.full_rotation_time, m.downsample_rate, m.min_dist, d_xyz, d_time,
                                            nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_lidar_device");
        if (m.n > 0) check(lv_lidar_push_device_async(ctx->h, d_xyz, d_time, d_n, m.n), "Accumulator::receive_lidar_device");
    }
    /* the same with whole Points: the message's intensity and range (Point.cpp:164-173) go into the caller's d_intensity / d_range
     * and onto a BUFFER_L made with `full` */
    void receive_lidar_device_full(const DeviceMessage& m, float* d_xyz, double* d_time, float* d_intensity, float* d_range, int64_t* d_n) {
        check(lv_process_cloud_device_async(ctx->h, m.type, m.layout, m.d_data, m.data_bytes, m.n, m.stamp_us, m.stamp_beginning,
                                            m.offset_beginning, m.full_rotation_time, m.downsample_rate, m.min_dist, d_xyz, d_time,
                                            d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_lidar_device_full");
        if (m.n > 0)
            check(lv_lidar_push_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, m.n), "Accumulator::receive_lidar_device_full");
    }
    /* receive_lidar_device for a Livox CustomMsg (lv_process_livox_device_async: tag filter, decimation on the rank among the tag-kept
     * points, time sort); the records in device memory, e.g. lv_bag_parse_livox's view uploaded */
    struct DeviceLivoxMessage {
        const uint8_t* d_data; int64_t data_bytes, n; uint64_t timebase_ns; uint8_t tag_reject_mask; int32_t downsample_rate; double min_dist;
    };
    void receive_livox_device(const DeviceLivoxMessage& m, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_livox_device_async(ctx->h, m.d_data, m.data_bytes, m.n, m.timebase_ns, m.tag_reject_mask, m.downsample_rate, m.min_dist,
                                            d_xyz, d_time, nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_livox_device");
        if (m.n > 0) check(lv_lidar_push_device_async(ctx->h, d_xyz, d_time, d_n, m.n), "Accumulator::receive_livox_device");
    }
    /* the same with whole Points: intensity = reflectivity, range = |p| */
    void receive_livox_device_full(const DeviceLivoxMessage& m, float* d_xyz, double* d_time, float* d_intensity, float* d_range, int64_t* d_n) {
        check(lv_process_livox_device_async(ctx->h, m.d_data, m.data_bytes, m.n, m.timebase_ns, m.tag_reject_mask, m.downsample_rate, m.min_dist,
                                            d_xyz, d_time, d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_livox_device_full");
        if (m.n > 0)
            check(lv_lidar_push_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, m.n), "Accumulator::receive_livox_device_full");
    }
    /* receive_lidar_device for a VelodyneScan (lv_process_velodyne_device_async: the packets decoded, decimation on the rank among the
     * points, time sort); the packets in device memory, e.g. lv_bag_parse_velodyne_scan's view uploaded.  The output buffers hold
     * 384 n_packets points. */
    struct DeviceVelodyneMessage {
        const uint8_t* d_packets; int64_t data_bytes, n_packets; const lv_velodyne_calibration* cal; int32_t downsample_rate; double min_dist;
    };
    void receive_velodyne_device(const DeviceVelodyneMessage& m, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_velodyne_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.downsample_rate, m.min_dist, d_xyz,
                                               d_time, nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_velodyne_device");
        if (m.n_packets > 0) check(lv_lidar_push_device_async(ctx->h, d_xyz, d_time, d_n, 384 * m.n_packets), "Accumulator::receive_velodyne_device");
    }
    /* the same with whole Points: intensity = reflectivity, range = |p| */
    void receive_velodyne_device_full(const DeviceVelodyneMessage& m, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                      int64_t* d_n) {
        check(lv_process_velodyne_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.downsample_rate, m.min_dist, d_xyz,
                                               d_time, d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_velodyne_device_full");
        if (m.n_packets > 0)
            check(lv_lidar_push_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, 384 * m.n_packets),
                  "Accumulator::receive_velodyne_device_full");
    }
    /* receive_lidar_device for Ouster packets (lv_process_ouster_packets_device_async: the packets of the sensor's lidar UDP profile
     * decoded through the beam intrinsics, decimation on the rank among the points, time sort); the packets in device memory, e.g. the
     * PacketMsgs of one frame batched into one upload.  The output buffers hold 16 H n_packets points (H = cal->pixels_per_column).
     * profile: the metadata's udp_profile_lidar (lv_ouster_sensor_from_json), LEGACY when left out. */
    struct DeviceOusterMessage {
        const uint8_t* d_packets; int64_t data_bytes, n_packets; const lv_ouster_calibration* cal; int32_t downsample_rate; double min_dist;
        lv_ouster_profile profile = LV_OUSTER_LEGACY;
        int64_t slots() const { return 16 * (int64_t)cal->pixels_per_column * n_packets; }
    };
    void receive_ouster_device(const DeviceOusterMessage& m, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_ouster_packets_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.profile, m.downsample_rate,
                                                     m.min_dist, d_xyz, d_time, nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_ouster_device");
        if (m.n_packets > 0) check(lv_lidar_push_device_async(ctx->h, d_xyz, d_time, d_n, m.slots()), "Accumulator::receive_ouster_device");
    }
    /* the same with whole Points: intensity = reflectivity, range = the range in mm */
    void receive_ouster_device_full(const DeviceOusterMessage& m, float* d_xyz, double* d_time, float* d_intensity, float* d_range,
                                    int64_t* d_n) {
        check(lv_process_ouster_packets_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.profile, m.downsample_rate,
                                                     m.min_dist, d_xyz, d_time, d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_ouster_device_full");
        if (m.n_packets > 0)
            check(lv_lidar_push_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, m.slots()),
                  "Accumulator::receive_ouster_device_full");
    }
    /* Several LiDARs: the same calls with the sensor's extrinsic L0_T_Lk (12 floats, R row-major then t: its frame into the primary
     * LiDAR's, nullptr for the primary itself) merge the message by time instead of pushing it (lv_lidar_merge_device_async), so
     * the buffer stays time-ordered when the sensors' messages overlap.  Needs lv_lidar_reserve_merge on the context's handle. */
    void receive_lidar_device(const DeviceMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_cloud_device_async(ctx->h, m.type, m.layout, m.d_data, m.data_bytes, m.n, m.stamp_us, m.stamp_beginning,
                                            m.offset_beginning, m.full_rotation_time, m.downsample_rate, m.min_dist, d_xyz, d_time,
                                            nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_lidar_device");
        if (m.n > 0) check(lv_lidar_merge_device_async(ctx->h, d_xyz, d_time, d_n, m.n, L0_T_Lk), "Accumulator::receive_lidar_device");
    }
    void receive_lidar_device_full(const DeviceMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, float* d_intensity,
                                   float* d_range, int64_t* d_n) {
        check(lv_process_cloud_device_async(ctx->h, m.type, m.layout, m.d_data, m.data_bytes, m.n, m.stamp_us, m.stamp_beginning,
                                            m.offset_beginning, m.full_rotation_time, m.downsample_rate, m.min_dist, d_xyz, d_time,
                                            d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_lidar_device_full");
        if (m.n > 0)
            check(lv_lidar_merge_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, m.n, L0_T_Lk),
                  "Accumulator::receive_lidar_device_full");
    }
    void receive_livox_device(const DeviceLivoxMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_livox_device_async(ctx->h, m.d_data, m.data_bytes, m.n, m.timebase_ns, m.tag_reject_mask, m.downsample_rate, m.min_dist,
                                            d_xyz, d_time, nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_livox_device");
        if (m.n > 0) check(lv_lidar_merge_device_async(ctx->h, d_xyz, d_time, d_n, m.n, L0_T_Lk), "Accumulator::receive_livox_device");
    }
    void receive_livox_device_full(const DeviceLivoxMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, float* d_intensity,
                                   float* d_range, int64_t* d_n) {
        check(lv_process_livox_device_async(ctx->h, m.d_data, m.data_bytes, m.n, m.timebase_ns, m.tag_reject_mask, m.downsample_rate, m.min_dist,
                                            d_xyz, d_time, d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_livox_device_full");
        if (m.n > 0)
            check(lv_lidar_merge_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, m.n, L0_T_Lk),
                  "Accumulator::receive_livox_device_full");
    }
    void receive_velodyne_device(const DeviceVelodyneMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_velodyne_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.downsample_rate, m.min_dist, d_xyz,
                                               d_time, nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_velodyne_device");
        if (m.n_packets > 0)
            check(lv_lidar_merge_device_async(ctx->h, d_xyz, d_time, d_n, 384 * m.n_packets, L0_T_Lk), "Accumulator::receive_velodyne_device");
    }
    void receive_velodyne_device_full(const DeviceVelodyneMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, float* d_intensity,
                                      float* d_range, int64_t* d_n) {
        check(lv_process_velodyne_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.downsample_rate, m.min_dist, d_xyz,
                                               d_time, d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_velodyne_device_full");
        if (m.n_packets > 0)
            check(lv_lidar_merge_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, 384 * m.n_packets, L0_T_Lk),
                  "Accumulator::receive_velodyne_device_full");
    }
    void receive_ouster_device(const DeviceOusterMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, int64_t* d_n) {
        check(lv_process_ouster_packets_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.profile, m.downsample_rate,
                                                     m.min_dist, d_xyz, d_time, nullptr, nullptr, nullptr, d_n),
              "Accumulator::receive_ouster_device");
        if (m.n_packets > 0)
            check(lv_lidar_merge_device_async(ctx->h, d_xyz, d_time, d_n, m.slots(), L0_T_Lk), "Accumulator::receive_ouster_device");
    }
    void receive_ouster_device_full(const DeviceOusterMessage& m, const float* L0_T_Lk, float* d_xyz, double* d_time, float* d_intensity,
                                    float* d_range, int64_t* d_n) {
        check(lv_process_ouster_packets_device_async(ctx->h, m.d_packets, m.data_bytes, m.n_packets, m.cal, m.profile, m.downsample_rate,
                                                     m.min_dist, d_xyz, d_time, d_intensity, d_range, nullptr, d_n),
              "Accumulator::receive_ouster_device_full");
        if (m.n_packets > 0)
            check(lv_lidar_merge_full_device_async(ctx->h, d_xyz, d_time, d_intensity, d_range, d_n, m.slots(), L0_T_Lk),
                  "Accumulator::receive_ouster_device_full");
    }
    /* Accumulator::get_points(t1, t2) (Accumulator.hpp:61-74) into device buffers of n_max points; the count goes to *d_n_out */
    void get_points_device(double t1, double t2, float* d_xyz, double* d_time, int64_t n_max, int64_t* d_n_out) {
        check(lv_lidar_get_points_device_async(ctx->h, t1, t2, d_xyz, d_time, n_max, d_n_out), "Accumulator::get_points_device");
    }
    /* the same window with its intensity and range */
    void get_points_device_full(double t1, double t2, float* d_xyz, double* d_time, float* d_intensity, float* d_range, int64_t n_max,
                                int64_t* d_n_out) {
        check(lv_lidar_get_points_full_device_async(ctx->h, t1, t2, d_xyz, d_time, d_intensity, d_range, n_max, d_n_out),
              "Accumulator::get_points_device_full");
    }
    void clear_lidar(double t) { check(lv_lidar_clear_async(ctx->h, t), "Accumulator::clear_lidar"); }   /* Accumulator.cpp:68-70 */
    void receive_imu(const IMU& imu) { imus.push_back(imu); }
    IMUs get_imus(double t1, double t2) {
        IMUs out;
        for (const IMU& i : imus) if (i.time > t1 && i.time <= t2) out.push_back(i);
        return out;
    }
    Points points;
    IMUs imus;

   private:
    Context* ctx = nullptr;
};

}  // namespace lv
#endif
