/*
 * lv_wire_host.cpp — the LiDAR message's wire format, on the host as in the reference:
 *   PointCloudProcessor::msg2points / to_points / get_begin_time   src/Utils/PointCloudProcessor.cpp:24-99
 *   Point(const <driver>::Point&, double time_offset)               src/Objects/Point.cpp:37-111,153-175
 *   Conversions::microsec2Sec / nanosec2Sec                         src/Utils/Utils.cpp:18-30
 *   PointCloudProcessor::sort_points                                src/Utils/PointCloudProcessor.cpp:114-123
 * One pass over the message bytes per sweep (a few MB); the per-point arithmetic is csrc/lv_wire.h, which
 * lv_process_cloud_device (csrc/lv_cloud.cu) runs on the device.  lv_livox_to_points is the same for a Livox CustomMsg
 * (lv_process_livox_device on the device), lv_velodyne_to_points for a VelodyneScan's packets (lv_process_velodyne_device),
 * lv_ouster_packets_to_points for Ouster packets of any UDP profile (lv_process_ouster_packets_device).
 */
#include <math.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/limovelo_b200.h"
#include "../csrc/lv_wire.h"

extern "C" {

lv_status lv_pointcloud2_to_points(lv_lidar_type type, const lv_cloud_layout* layout, const uint8_t* data, int64_t n,
                                   uint64_t header_stamp_us, int stamp_beginning, int offset_beginning,
                                   double full_rotation_time, float* xyz, double* time, float* intensity, float* range) {
    if (!layout || !data || !xyz || !time || n < 0 || layout->point_step <= 0) return LV_ERR_ARG;
    if (type != LV_LIDAR_VELODYNE && type != LV_LIDAR_HESAI && type != LV_LIDAR_OUSTER && type != LV_LIDAR_CUSTOM) return LV_ERR_ARG;
    if (n == 0) return LV_OK;
    const lv_cloud_layout& L = *layout;
    const double begin = lv::wire_begin_time(type, L, data, n, header_stamp_us, stamp_beginning);
    for (int64_t i = 0; i < n; ++i) {
        const uint8_t* p = data + (size_t)i * L.point_step;
        const float x = lv::wire_f32(p + L.off_x), y = lv::wire_f32(p + L.off_y), z = lv::wire_f32(p + L.off_z);
        xyz[3 * i] = x; xyz[3 * i + 1] = y; xyz[3 * i + 2] = z;
        time[i] = lv::wire_time(type, L, p, offset_beginning, full_rotation_time, begin);
        if (intensity) intensity[i] = lv::wire_intensity(type, L, p);
        if (range) range[i] = lv::wire_range(type, L, p, x, y, z);
    }
    return LV_OK;
}

lv_status lv_livox_to_points(const uint8_t* data, int64_t data_bytes, int64_t n, uint64_t timebase_ns, uint8_t tag_reject_mask,
                             float* xyz, double* time, float* intensity, float* range, int32_t* idx, int64_t* n_out) {
    if (n_out) *n_out = 0;
    if (!data || !xyz || !time || !n_out || n > 0x7fffffff || lv::livox_layout_error(n, data_bytes, timebase_ns)) return LV_ERR_ARG;
    int64_t m = 0;
    for (int64_t i = 0; i < n; ++i) {
        const uint8_t* p = lv::livox_point(data, i);
        if (!lv::livox_tag_keep(p, tag_reject_mask)) continue;
        const float x = lv::wire_f32(p + 4), y = lv::wire_f32(p + 8), z = lv::wire_f32(p + 12);
        xyz[3 * m] = x; xyz[3 * m + 1] = y; xyz[3 * m + 2] = z;
        time[m] = lv::livox_time(timebase_ns, p);
        if (intensity) intensity[m] = lv::livox_reflectivity(p);
        if (range) range[m] = lv::wire_norm(x, y, z);
        if (idx) idx[m] = (int32_t)i;
        ++m;
    }
    *n_out = m;
    return LV_OK;
}

lv_status lv_velodyne_default_calibration(lv_velodyne_model model, lv_velodyne_calibration* out) {
    static const double vlp16[16] = {-15, 1, -13, 3, -11, 5, -9, 7, -7, 9, -5, 11, -3, 13, -1, 15};
    static const double hires[16] = {-10, 0.67, -8.67, 2, -7.33, 3.33, -6, 4.67, -4.67, 6, -3.33, 7.33, -2, 8.67, -0.67, 10};
    if (!out || (model != LV_VELODYNE_VLP16 && model != LV_VELODYNE_PUCK_HIRES)) return LV_ERR_ARG;
    *out = lv_velodyne_calibration{};
    for (int l = 0; l < 16; ++l) out->vert_correction[l] = (model == LV_VELODYNE_VLP16 ? vlp16 : hires)[l] * M_PI / 180.0;
    return LV_OK;
}

lv_status lv_velodyne_to_points(const uint8_t* packets, int64_t data_bytes, int64_t n_packets, const lv_velodyne_calibration* cal,
                                float* xyz, double* time, float* intensity, float* range, int32_t* idx, int64_t* n_out) {
    if (n_out) *n_out = 0;
    if (!packets || !cal || !xyz || !time || !n_out || lv::velodyne_layout_error(n_packets, data_bytes) || !lv::velodyne_calib_finite(*cal))
        return LV_ERR_ARG;
    for (int64_t k = 0; k < n_packets; ++k)
        if (!lv::velodyne_stamp_ok(lv::velodyne_packet(packets, k))) return LV_ERR_ARG;
    static const std::vector<float> tables = [] {
        std::vector<float> t(2 * lv::kVelodyneTable);
        lv::velodyne_tables(t.data(), t.data() + lv::kVelodyneTable);
        return t;
    }();
    const float *C = tables.data(), *S = C + lv::kVelodyneTable;
    const lv::VelodyneCalib k = lv::velodyne_calib(*cal);
    int64_t m = 0;
    for (int64_t i = 0; i < n_packets * lv::kVelodyneSlots; ++i) {
        const uint8_t* pkt = lv::velodyne_packet(packets, i / lv::kVelodyneSlots);
        const int r = (int)(i % lv::kVelodyneSlots);
        if (!lv::velodyne_slot_valid(pkt, r)) continue;
        float x, y, z;
        lv::velodyne_xyz(pkt, r, C, S, k, x, y, z);
        xyz[3 * m] = x; xyz[3 * m + 1] = y; xyz[3 * m + 2] = z;
        time[m] = lv::velodyne_time(pkt, r);
        if (intensity) intensity[m] = lv::velodyne_reflectivity(pkt, r);
        if (range) range[m] = lv::wire_norm(x, y, z);
        if (idx) idx[m] = (int32_t)i;
        ++m;
    }
    *n_out = m;
    return LV_OK;
}

lv_status lv_ouster_packets_to_points(const uint8_t* packets, int64_t data_bytes, int64_t n_packets, const lv_ouster_calibration* cal,
                                      lv_ouster_profile profile, float* xyz, double* time, float* intensity, float* range, int32_t* idx,
                                      int64_t* n_out) {
    if (n_out) *n_out = 0;
    lv::OusterFormat f;
    if (!packets || !cal || !xyz || !time || !n_out || lv::ouster_calib_error(*cal) ||
        !lv::ouster_format(profile, cal->pixels_per_column, &f) || lv::ouster_layout_error(f, n_packets, data_bytes, cal->pixels_per_column))
        return LV_ERR_ARG;
    static const std::vector<float> table = [] {
        std::vector<float> t(2 * lv::kOusterTable);
        lv::ouster_table(t.data(), t.data() + lv::kOusterTable);
        return t;
    }();
    const float *C = table.data(), *S = C + lv::kOusterTable;
    const lv::OusterCalib k = lv::ouster_calib(*cal);
    int64_t m = 0;
    for (int64_t i = 0; i < n_packets * lv::kOusterColumns * k.H; ++i) {
        const uint8_t* col = lv::ouster_column(f, packets, i, k.H);
        const int p = (int)(i % k.H);
        if (!lv::ouster_slot_valid(f, col, p, k.W)) continue;
        float x, y, z;
        lv::ouster_xyz(f, col, p, C, S, k, x, y, z);
        xyz[3 * m] = x; xyz[3 * m + 1] = y; xyz[3 * m + 2] = z;
        time[m] = lv::ouster_time(col);
        if (intensity) intensity[m] = lv::ouster_reflectivity(f, col, p);
        if (range) range[m] = lv::ouster_range(f, col, p);
        if (idx) idx[m] = (int32_t)i;
        ++m;
    }
    *n_out = m;
    return LV_OK;
}
lv_status lv_ouster_to_points(const uint8_t* packets, int64_t data_bytes, int64_t n_packets, const lv_ouster_calibration* cal, float* xyz,
                              double* time, float* intensity, float* range, int32_t* idx, int64_t* n_out) {
    return lv_ouster_packets_to_points(packets, data_bytes, n_packets, cal, LV_OUSTER_LEGACY, xyz, time, intensity, range, idx, n_out);
}

lv_status lv_time_sort_indices(const double* time, int64_t n, int32_t* idx_out) {
    if (!time || !idx_out || n < 0 || n > 0x7fffffff) return LV_ERR_ARG;
    std::iota(idx_out, idx_out + n, 0);
    std::stable_sort(idx_out, idx_out + n, [time](int32_t a, int32_t b) { return time[a] < time[b]; });
    return LV_OK;
}

}  // extern "C"
