/*
 * lv_wire.h — the per-point arithmetic of the LiDAR message, compiled by the host (lv_pointcloud2_to_points, lv_livox_to_points,
 * lv_velodyne_to_points, lv_ouster_to_points) and the device (lv_process_cloud_device, lv_process_livox_device,
 * lv_process_velodyne_device, lv_process_ouster_device, the temporal decimator) alike, so that both give the same bits:
 *   PointCloudProcessor::msg2points / get_begin_time   src/Utils/PointCloudProcessor.cpp:24-99
 *   Point(const <driver>::Point&, double time_offset)   src/Objects/Point.cpp:37-111,153-175
 *   Conversions::microsec2Sec / nanosec2Sec             src/Utils/Utils.cpp:18-30
 *   PointCloudProcessor::temporal_downsample            src/Utils/PointCloudProcessor.cpp:101-112
 * Fields sit at whatever byte offsets the message declares and the message itself may start at any address, so every
 * value is assembled from single bytes (little endian): no 2-, 4- or 8-byte load is ever misaligned.  The doubles go
 * through lv::dadd / lv::dmul so that nvcc cannot contract them into FMAs the host build does not form.
 */
#ifndef LV_WIRE_H_
#define LV_WIRE_H_

#include <stdint.h>
#include <string.h>

#include "../../include/limovelo_b200.h"
#include "lv_hd.h"

namespace lv {

LV_HD uint32_t wire_u8(const uint8_t* p) { return p[0]; }
LV_HD uint32_t wire_u16(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8; }
LV_HD uint32_t wire_u32(const uint8_t* p) {
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}
LV_HD float wire_f32(const uint8_t* p) {
    const uint32_t u = wire_u32(p);
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
LV_HD double wire_f64(const uint8_t* p) {
    const uint64_t u = (uint64_t)wire_u32(p) | (uint64_t)wire_u32(p + 4) << 32;
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double d;
    memcpy(&d, &u, 8);
    return d;
#endif
}

/* Utils.cpp:18-23: int arithmetic on the quotient and the remainder, as written (the int cast keeps the low 32 bits) */
LV_HD double microsec2sec(uint64_t t) {
    const int order = 1000000;
    const int secs = (int)(t / (uint64_t)order);
    const int musecs = (int)(t % (uint64_t)order);
    return dadd((double)secs, dmul((double)musecs, 1e-6));
}
LV_HD double nanosec2sec(uint32_t t) {   /* Utils.cpp:25-30 */
    const int order = 1000000000;
    const int secs = (int)(t / (uint32_t)order);
    const int nsecs = (int)(t % (uint32_t)order);
    return dadd((double)secs, dmul((double)nsecs, 1e-9));
}

/* the point's own time field in seconds, before any offset */
LV_HD double wire_raw_time(lv_lidar_type type, const lv_cloud_layout& L, const uint8_t* p) {
    switch (type) {
        case LV_LIDAR_VELODYNE: return (double)wire_f32(p + L.off_time);
        case LV_LIDAR_OUSTER: return nanosec2sec(wire_u32(p + L.off_time));
        default: return wire_f64(p + L.off_time);                          /* hesai, custom: absolute */
    }
}
LV_HD bool wire_relative(lv_lidar_type type) { return type == LV_LIDAR_VELODYNE || type == LV_LIDAR_OUSTER; }

/* get_begin_time (PointCloudProcessor.cpp:42-88), from the first and the last point of the whole message: relative stamps
 * hang off the header stamp, absolute ones get 0 */
LV_HD double wire_begin_time(lv_lidar_type type, const lv_cloud_layout& L, const uint8_t* data, int64_t n, uint64_t header_stamp_us,
                             int stamp_beginning) {
    if (!wire_relative(type) || n <= 0) return 0.0;
    const double front = wire_raw_time(type, L, data), back = wire_raw_time(type, L, data + (uint64_t)(n - 1) * (uint64_t)L.point_step);
    const double s = dadd(microsec2sec(header_stamp_us), front);
    return stamp_beginning ? s : dsub(s, back);
}
/* absolute time of one point: Point.cpp:58-60,77-79 (full_rotation_time + t unless offset_beginning), then + begin */
LV_HD double wire_time(lv_lidar_type type, const lv_cloud_layout& L, const uint8_t* p, int offset_beginning, double full_rotation_time,
                       double begin) {
    double t = wire_raw_time(type, L, p);
    if (wire_relative(type) && !offset_beginning) t = dadd(full_rotation_time, t);
    return dadd(t, begin);
}

LV_HD float wire_norm(float x, float y, float z) { return fsqrt(fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z))); }
LV_HD float wire_intensity(lv_lidar_type type, const lv_cloud_layout& L, const uint8_t* p) {
    return type == LV_LIDAR_HESAI ? (float)wire_u8(p + L.off_intensity)
         : type == LV_LIDAR_OUSTER ? (float)wire_u16(p + L.off_intensity)
                                   : wire_f32(p + L.off_intensity);
}
/* Point.cpp:166-169: the driver's range for the ouster, |p| otherwise */
LV_HD float wire_range(lv_lidar_type type, const lv_cloud_layout& L, const uint8_t* p, float x, float y, float z) {
    return type == LV_LIDAR_OUSTER ? (float)wire_u32(p + L.off_range) : wire_norm(x, y, z);
}

/* temporal_downsample: keep point i (its index in the raw message) iff rate <= 1 or (i + 1) % rate == 0, and
 * min_dist < |p| (a strict <, the double against the fp32 norm; a NaN coordinate drops the point) */
LV_HD bool temporal_keep(int64_t i, int rate, double min_dist, float x, float y, float z) {
    return (rate <= 1 || (i + 1) % rate == 0) && min_dist < (double)wire_norm(x, y, z);
}

/* the bounds pcl::fromROSMsg takes from the message itself: a LiDAR type this reader knows, every field that type reads
 * inside point_step, and n points inside data_bytes.  NULL when the layout is usable, else what is wrong with it. */
inline const char* cloud_layout_error(lv_lidar_type type, const lv_cloud_layout& L, int64_t n, int64_t data_bytes) {
    if (type != LV_LIDAR_VELODYNE && type != LV_LIDAR_HESAI && type != LV_LIDAR_OUSTER && type != LV_LIDAR_CUSTOM) return "unknown LiDAR type";
    if (n < 0 || data_bytes < 0) return "negative point count or data length";
    if (L.point_step <= 0) return "point_step must be positive";
    const int tsz = type == LV_LIDAR_VELODYNE ? 4 : (type == LV_LIDAR_OUSTER ? 4 : 8);
    const int isz = type == LV_LIDAR_HESAI ? 1 : (type == LV_LIDAR_OUSTER ? 2 : 4);
    const int32_t offs[6] = {L.off_x, L.off_y, L.off_z, L.off_intensity, L.off_time, type == LV_LIDAR_OUSTER ? L.off_range : 0};
    const int32_t szs[6] = {4, 4, 4, isz, tsz, type == LV_LIDAR_OUSTER ? 4 : 0};
    for (int k = 0; k < 6; ++k)
        if (offs[k] < 0 || (int64_t)offs[k] + szs[k] > L.point_step) return "a field of the layout lies outside point_step";
    if (n > data_bytes / L.point_step) return "data_bytes is too short for n points of point_step bytes";
    return nullptr;
}

/* an absolute time in uint64 ns -> seconds as Conversions::nanosec2Sec (Utils.cpp:25-30) but with a 64-bit quotient: the
 * reference's int cast would truncate epoch seconds */
LV_HD double wire_ns_to_sec(uint64_t total) {
    const uint64_t order = 1000000000ull;
    return dadd((double)(int64_t)(total / order), dmul((double)(total % order), 1e-9));
}

/* ---- livox_ros_driver(2)/CustomMsg: one uint64 time base (ns) per message, then packed 19-byte records
 *   uint32 offset_time (ns after timebase) | float32 x | float32 y | float32 z | uint8 reflectivity | uint8 tag | uint8 line
 * A record starts at data + 19 i, at any address. */
enum { kLivoxRecord = 19 };
/* the largest time base whose sum with any uint32 offset still fits a uint64 */
constexpr uint64_t kLivoxTimebaseMax = 0xFFFFFFFF00000000ull;

LV_HD const uint8_t* livox_point(const uint8_t* data, int64_t i) { return data + (uint64_t)i * (uint64_t)kLivoxRecord; }
LV_HD uint32_t livox_tag(const uint8_t* p) { return wire_u8(p + 17); }
LV_HD float livox_reflectivity(const uint8_t* p) { return (float)wire_u8(p + 16); }
/* total = timebase + offset_time (ns, uint64), in seconds */
LV_HD double livox_time(uint64_t timebase, const uint8_t* p) { return wire_ns_to_sec(timebase + (uint64_t)wire_u32(p)); }
/* the tag filter of msg2points: bits of the tag set in the mask drop the point (0 keeps every point) */
LV_HD bool livox_tag_keep(const uint8_t* p, uint32_t tag_reject_mask) { return (livox_tag(p) & tag_reject_mask) == 0; }

/* NULL when n records fit data_bytes and the time base cannot wrap, else what is wrong */
inline const char* livox_layout_error(int64_t n, int64_t data_bytes, uint64_t timebase_ns) {
    if (n < 0 || data_bytes < 0) return "negative point count or data length";
    if (n > data_bytes / kLivoxRecord) return "data_bytes is too short for n records of 19 bytes";
    if (timebase_ns > kLivoxTimebaseMax) return "timebase above 2^64 - 2^32 ns (timebase + offset_time could wrap)";
    return nullptr;
}

/* ---- velodyne_msgs/VelodyneScan of a VLP-16 / Puck Hi-Res (include/limovelo_b200.h, "Velodyne packets"): packets of 1214 bytes
 *   uint32 stamp.sec | uint32 stamp.nsec | uint8[1206] data
 * at packets + 1214 k, any alignment.  data: 12 blocks of 100 bytes (uint16 flag 0xEEFF, uint16 azimuth in 0.01 deg, 32 x (uint16
 * distance in 2 mm, uint8 reflectivity)), then uint32 sensor us (unused), uint8 return mode, uint8 product id (unused).
 * Slot i of the message: packet k = i / 384, r = i % 384, block b = r / 32, firing f = (r % 32) / 16, laser l = r % 16. */
enum { kVelodynePacket = 1214, kVelodyneSlots = 384, kVelodyneLasers = 16, kVelodyneTable = 36000 };
enum : uint32_t { kVelodyneBlockFlag = 0xEEFFu, kVelodyneDualReturn = 0x39u };
constexpr int64_t kVelodyneMaxPackets = 0x7fffffff / kVelodyneSlots;   /* slot indices are int32 */

/* the calibration in the fp32 terms the point arithmetic reads (velodyne_calib), per laser */
struct VelodyneCalib {
    float cv[kVelodyneLasers], sv[kVelodyneLasers];   /* cos / sin of the vertical angle   */
    float cr[kVelodyneLasers], sr[kVelodyneLasers];   /* cos / sin of the rotational correction */
    float dist[kVelodyneLasers], vo[kVelodyneLasers], ho[kVelodyneLasers];
};

LV_HD const uint8_t* velodyne_packet(const uint8_t* packets, int64_t k) { return packets + (uint64_t)k * (uint64_t)kVelodynePacket; }
LV_HD const uint8_t* velodyne_block(const uint8_t* pkt, int b) { return pkt + 8 + 100 * b; }
LV_HD uint32_t velodyne_mode(const uint8_t* pkt) { return wire_u8(pkt + 8 + 1204); }
LV_HD const uint8_t* velodyne_channel(const uint8_t* pkt, int r) { return velodyne_block(pkt, r / 32) + 4 + 3 * (r % 32); }

/* msg2points: the packet is not a dual-return one, blocks 0 .. b all carry the flag and the slot has a return */
LV_HD bool velodyne_slot_valid(const uint8_t* pkt, int r) {
    if (velodyne_mode(pkt) == kVelodyneDualReturn) return false;
    for (int c = 0; c <= r / 32; ++c)
        if (wire_u16(velodyne_block(pkt, c)) != kVelodyneBlockFlag) return false;
    return wire_u16(velodyne_channel(pkt, r)) != 0;
}
/* the packet's stamp converts: nsec < 10^9 (with 32-bit seconds the ns sum below cannot wrap a uint64) */
LV_HD bool velodyne_stamp_ok(const uint8_t* pkt) { return wire_u32(pkt + 4) < 1000000000u; }

/* the table index of slot r's azimuth: A_b plus the part of the block's azimuth step its firing time covers, rounded to 0.01 deg */
LV_HD int velodyne_azimuth(const uint8_t* pkt, int r) {
    const int b = r / 32, f = (r % 32) / 16, l = r % 16;
    const int nb = b < 11 ? b + 1 : 11, pb = b < 11 ? b : 10;           /* block 11 takes block 10's step */
    const int a_b = (int)wire_u16(velodyne_block(pkt, b) + 2);
    int delta = ((int)wire_u16(velodyne_block(pkt, nb) + 2) + kVelodyneTable - (int)wire_u16(velodyne_block(pkt, pb) + 2)) % kVelodyneTable;
    if (delta < 0) delta += kVelodyneTable;                            /* a raw azimuth above 36000 (not a valid packet) */
    const float a = fadd((float)a_b, fdiv(fmul((float)delta, fadd(fmul((float)l, 2.304f), fmul((float)f, 55.296f))), 110.592f));
    return (int)(((int64_t)roundf(a)) % kVelodyneTable);              /* a >= 0: roundf is half away from zero */
}
/* the point of slot r (C, S: the cos / sin tables of velodyne_tables), in the ROS frame (x forward, y left, z up) */
LV_HD void velodyne_xyz(const uint8_t* pkt, int r, const float* C, const float* S, const VelodyneCalib& k, float& x, float& y, float& z) {
    const int l = r % 16, q = velodyne_azimuth(pkt, r);
    const float d = fadd(fmul((float)wire_u16(velodyne_channel(pkt, r)), 0.002f), k.dist[l]);
    const float c = C[q], s = S[q];
    const float cosr = fadd(fmul(c, k.cr[l]), fmul(s, k.sr[l])), sinr = fsub(fmul(s, k.cr[l]), fmul(c, k.sr[l]));
    const float xy = fsub(fmul(d, k.cv[l]), fmul(k.vo[l], k.sv[l]));
    const float X = fsub(fmul(xy, sinr), fmul(k.ho[l], cosr)), Y = fadd(fmul(xy, cosr), fmul(k.ho[l], sinr));
    x = Y;
    y = -X;
    z = fadd(fmul(d, k.sv[l]), fmul(k.vo[l], k.cv[l]));
}
LV_HD float velodyne_reflectivity(const uint8_t* pkt, int r) { return (float)wire_u8(velodyne_channel(pkt, r) + 2); }
/* the packet stamp is its first firing's time; firing sequence 2b + f starts 55.296 us after the previous, laser l fires 2.304 us
 * into it */
LV_HD double velodyne_time(const uint8_t* pkt, int r) {
    const int b = r / 32, f = (r % 32) / 16, l = r % 16;
    const uint64_t total = (uint64_t)wire_u32(pkt) * 1000000000ull + (uint64_t)wire_u32(pkt + 4) + (uint64_t)(2 * b + f) * 55296ull +
                           (uint64_t)l * 2304ull;
    return wire_ns_to_sec(total);
}

/* host code from here.  C[q] = cos(q 0.01 deg), S[q] = sin(q 0.01 deg) for q in [0, 36000): computed in double, rounded to float.  The host decoder and
 * the device tables both come from here, so both read the same bits */
inline void velodyne_tables(float* C, float* S) {
    for (int q = 0; q < kVelodyneTable; ++q) {
        const double a = (double)q * 0.01 * M_PI / 180.0;
        C[q] = (float)cos(a);
        S[q] = (float)sin(a);
    }
}
inline bool velodyne_calib_finite(const lv_velodyne_calibration& c) {
    for (int l = 0; l < kVelodyneLasers; ++l)
        if (!isfinite(c.vert_correction[l]) || !isfinite(c.rot_correction[l]) || !isfinite(c.dist_correction[l]) ||
            !isfinite(c.vert_offset_correction[l]) || !isfinite(c.horiz_offset_correction[l]))
            return false;
    return true;
}
inline VelodyneCalib velodyne_calib(const lv_velodyne_calibration& c) {
    VelodyneCalib k;
    for (int l = 0; l < kVelodyneLasers; ++l) {
        k.cv[l] = (float)cos(c.vert_correction[l]);
        k.sv[l] = (float)sin(c.vert_correction[l]);
        k.cr[l] = (float)cos(c.rot_correction[l]);
        k.sr[l] = (float)sin(c.rot_correction[l]);
        k.dist[l] = (float)c.dist_correction[l];
        k.vo[l] = (float)c.vert_offset_correction[l];
        k.ho[l] = (float)c.horiz_offset_correction[l];
    }
    return k;
}

/* NULL when n_packets is in range and its packets fit data_bytes, else what is wrong */
inline const char* velodyne_layout_error(int64_t n_packets, int64_t data_bytes) {
    if (n_packets < 0 || data_bytes < 0) return "negative packet count or data length";
    if (n_packets > kVelodyneMaxPackets) return "n_packets above (2^31 - 1) / 384 (slot indices are int32)";
    if (n_packets > data_bytes / kVelodynePacket) return "data_bytes is too short for n_packets packets of 1214 bytes";
    return nullptr;
}

/* ---- ouster_ros/PacketMsg of an OS0 / OS1 / OS2 (include/limovelo_b200.h, "Ouster packets"): packets of 16 columns in one of four
 * UDP profiles.  What differs between the profiles is data, an OusterFormat built on the host (ouster_format); one decoder reads
 * all four through it.
 *   LEGACY   packet: 16 columns of 20 + 12 H bytes
 *            column: uint64 timestamp (ns) | uint16 measurement_id m | uint16 frame_id | uint32 encoder | H x 12-byte pixels |
 *                    uint32 status
 *            pixel:  uint32 range word (low 20 bits: range in mm) | uint16 reflectivity | signal, noise
 *   others   packet: 32-byte header | 16 columns of 12 + s H bytes | 32-byte footer (header and footer not read)
 *            column: uint64 timestamp (ns) | uint16 measurement_id m | uint16 status | H x s-byte pixels
 *            pixel:  RNG19_RFL8_SIG16_NIR16        s = 12  range = u32 @0 & 0x7FFFF          reflectivity = u8 @4
 *                    RNG19_RFL8_SIG16_NIR16_DUAL   s = 16  range = u32 @0 & 0x7FFFF (first)  reflectivity = u8 @3 (first)
 *                    RNG15_RFL8_NIR8 (low data)    s = 4   range = (u16 @0 & 0x7FFF) << 3    reflectivity = u8 @2
 * Every profile keeps the timestamp at byte 0 and the measurement id at byte 8 of the column, and bit 0 of the status' first byte
 * says the column is valid.  The low-data range is read as u32 @0 under the mask, which gives the same bits as u16 @0.  Packet k
 * starts at packets + k packet bytes, any alignment.  Slot i of the message: column g = i / H (packet g / 16, column g % 16),
 * pixel p = i % H. */
enum { kOusterColumns = 16, kOusterMaxBeams = 128, kOusterTable = 2048 };

/* the calibration in the fp32 terms the point arithmetic reads (ouster_calib): per beam, cos / sin of the altitude and the azimuth */
struct OusterCalib {
    float ce[kOusterMaxBeams], se[kOusterMaxBeams];   /* cos / sin of the beam altitude  */
    float ca[kOusterMaxBeams], sa[kOusterMaxBeams];   /* cos / sin of the beam azimuth   */
    float nf;                                         /* lidar_origin_to_beam_origin in m */
    int32_t W, H;                                     /* columns per frame, pixels per column */
};

/* where a UDP profile keeps a packet's fields, for one H (ouster_format) */
struct OusterFormat {
    int32_t packet;            /* bytes per packet                                                  */
    int32_t header;            /* bytes before the first column (the packet header)                 */
    int32_t column;            /* bytes per column                                                  */
    int32_t pixels;            /* offset of pixel 0 in the column (the column header's bytes)       */
    int32_t stride;            /* bytes per pixel                                                   */
    int32_t status;            /* offset in the column of the status byte whose bit 0 is read       */
    uint32_t range_mask;       /* range = (u32 at the pixel's byte 0 & range_mask) << range_shift   */
    int32_t range_shift;
    int32_t refl;              /* offset of the reflectivity in the pixel                           */
    int32_t refl_bytes;        /* its width: 1 or 2                                                 */
};

LV_HD uint64_t wire_u64(const uint8_t* p) { return (uint64_t)wire_u32(p) | (uint64_t)wire_u32(p + 4) << 32; }
/* the column of slot i and its pixel p */
LV_HD const uint8_t* ouster_column(const OusterFormat& f, const uint8_t* packets, int64_t i, int H) {
    const uint64_t g = (uint64_t)(i / H);
    return packets + (g / kOusterColumns) * (uint64_t)f.packet + (uint64_t)f.header + (g % kOusterColumns) * (uint64_t)f.column;
}
LV_HD const uint8_t* ouster_pixel(const OusterFormat& f, const uint8_t* col, int p) { return col + f.pixels + f.stride * p; }
LV_HD uint32_t ouster_measurement_id(const uint8_t* col) { return wire_u16(col + 8); }
LV_HD uint32_t ouster_range_mm(const OusterFormat& f, const uint8_t* col, int p) {
    return (wire_u32(ouster_pixel(f, col, p)) & f.range_mask) << f.range_shift;
}

/* msg2points: the column's status has bit 0 set, its measurement id is a column of the frame, and the pixel has a return */
LV_HD bool ouster_slot_valid(const OusterFormat& f, const uint8_t* col, int p, int W) {
    return (wire_u8(col + f.status) & 1u) && ouster_measurement_id(col) < (uint32_t)W && ouster_range_mm(f, col, p) != 0;
}
/* the point of pixel p of a valid column (C, S: the column table of ouster_table), in the LiDAR frame (os_lidar), fp32, each
 * product and sum rounded, in the order of the header */
LV_HD void ouster_xyz(const OusterFormat& f, const uint8_t* col, int p, const float* C, const float* S, const OusterCalib& k, float& x,
                      float& y, float& z) {
    const int q = (int)ouster_measurement_id(col) * (kOusterTable / k.W);
    const float c = C[q], s = S[q];
    const float e = fsub(fmul((float)ouster_range_mm(f, col, p), 0.001f), k.nf);
    const float ch = fsub(fmul(c, k.ca[p]), fmul(s, k.sa[p])), sh = fadd(fmul(s, k.ca[p]), fmul(c, k.sa[p]));
    const float ee = fmul(e, k.ce[p]);
    x = fadd(fmul(ee, ch), fmul(k.nf, c));
    y = -fadd(fmul(ee, sh), fmul(k.nf, s));
    z = fmul(e, k.se[p]);
}
LV_HD float ouster_reflectivity(const OusterFormat& f, const uint8_t* col, int p) {
    const uint8_t* r = ouster_pixel(f, col, p) + f.refl;
    return (float)(f.refl_bytes == 2 ? wire_u16(r) : wire_u8(r));
}
LV_HD float ouster_range(const OusterFormat& f, const uint8_t* col, int p) { return (float)ouster_range_mm(f, col, p); }
/* the column's own timestamp, absolute */
LV_HD double ouster_time(const uint8_t* col) { return wire_ns_to_sec(wire_u64(col)); }

/* host code from here.  C[q] = cos(2 pi q / 2048), S[q] = sin(...) for q in [0, 2048): computed in double, rounded to float.  The host
 * decoder and the device table both come from here, so both read the same bits */
inline void ouster_table(float* C, float* S) {
    for (int q = 0; q < kOusterTable; ++q) {
        const double a = 2.0 * M_PI * (double)q / (double)kOusterTable;
        C[q] = (float)cos(a);
        S[q] = (float)sin(a);
    }
}
/* NULL when W and H are in their sets and the entries the decoder reads (the first H angles of each array, and n) are finite */
inline const char* ouster_calib_error(const lv_ouster_calibration& c) {
    const int W = c.columns_per_frame, H = c.pixels_per_column;
    if (W != 512 && W != 1024 && W != 2048) return "columns_per_frame is not 512, 1024 or 2048";
    if (H != 16 && H != 32 && H != 64 && H != 128) return "pixels_per_column is not 16, 32, 64 or 128";
    for (int p = 0; p < H; ++p)
        if (!isfinite(c.beam_altitude_angles[p]) || !isfinite(c.beam_azimuth_angles[p])) return "a calibration entry is not finite";
    return isfinite(c.lidar_origin_to_beam_origin_mm) ? nullptr : "a calibration entry is not finite";
}
/* the fp32 terms of a calibration ouster_calib_error accepts */
inline OusterCalib ouster_calib(const lv_ouster_calibration& c) {
    OusterCalib k = {};
    k.W = c.columns_per_frame;
    k.H = c.pixels_per_column;
    for (int p = 0; p < k.H; ++p) {
        const double alt = c.beam_altitude_angles[p] * M_PI / 180.0, az = c.beam_azimuth_angles[p] * M_PI / 180.0;
        k.ce[p] = (float)cos(alt);
        k.se[p] = (float)sin(alt);
        k.ca[p] = (float)cos(az);
        k.sa[p] = (float)sin(az);
    }
    k.nf = (float)(c.lidar_origin_to_beam_origin_mm * 0.001);
    return k;
}
/* the most packets whose slot indices fit an int32 */
inline int64_t ouster_max_packets(int H) { return 0x7fffffff / (kOusterColumns * (int64_t)H); }

/* the layout of a profile for H pixels per column; false for a value outside lv_ouster_profile (*f is then left as it was) */
inline bool ouster_format(int profile, int H, OusterFormat* f) {
    if (profile == LV_OUSTER_LEGACY) {
        const int32_t column = 20 + 12 * H;
        *f = {kOusterColumns * column, 0, column, 16, 12, 16 + 12 * H, 0xFFFFFu, 0, 4, 2};
        return true;
    }
    int32_t s, refl, shift = 0;
    uint32_t mask;
    switch (profile) {
        case LV_OUSTER_RNG19_RFL8_SIG16_NIR16: s = 12; mask = 0x7FFFFu; refl = 4; break;
        case LV_OUSTER_RNG19_RFL8_SIG16_NIR16_DUAL: s = 16; mask = 0x7FFFFu; refl = 3; break;
        case LV_OUSTER_RNG15_RFL8_NIR8: s = 4; mask = 0x7FFFu; shift = 3; refl = 2; break;
        default: return false;
    }
    const int32_t column = 12 + s * H;
    *f = {32 + kOusterColumns * column + 32, 32, column, 12, s, 10, mask, shift, refl, 1};
    return true;
}

/* NULL when n_packets is in range and its packets fit data_bytes (H from a calibration ouster_calib_error accepts, f its profile's
 * layout), else what is wrong */
inline const char* ouster_layout_error(const OusterFormat& f, int64_t n_packets, int64_t data_bytes, int H) {
    if (n_packets < 0 || data_bytes < 0) return "negative packet count or data length";
    if (n_packets > ouster_max_packets(H)) return "n_packets above (2^31 - 1) / (16 pixels_per_column) (slot indices are int32)";
    if (n_packets > data_bytes / f.packet) return "data_bytes is too short for n_packets packets of the profile";
    return nullptr;
}

}  // namespace lv
#endif
