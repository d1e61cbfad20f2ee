/*
 * lv_bag_host.cpp — a reader for rosbag files (format 2.0), the input side of the reference driver without ROS.
 *
 * Replaces what roscpp + rosbag play deliver to the node: the callbacks Accumulator::receive_lidar / receive_imu get
 * sensor_msgs::PointCloud2 and sensor_msgs::Imu messages (src/main.cpp:27-39, src/Modules/Accumulator.cpp:39-60,
 * src/Utils/PointCloudProcessor.cpp:24-33).  Here the bag file is read directly:
 *
 *   file      "#ROSBAG V2.0\n", then records  <u32 header_len><header><u32 data_len><data>
 *   header    fields <u32 len><name>=<value>; every record has `op` (1 byte)
 *   op 0x03   bag header (index_pos, conn_count, chunk_count; padded)                      -> skipped
 *   op 0x05   chunk: compression = none | bz2 | lz4, data = records (0x02, 0x07)           -> "none" is read, the
 *             compressed forms are refused with LV_ERR_IO (`rosbag decompress` first): no codec is linked here
 *   op 0x07   connection: conn id, topic; data = connection header (type, md5sum, ...)      -> topic / type table
 *   op 0x02   message data: conn id, time (u32 sec, u32 nsec); data = the serialised message
 *   op 0x04 / 0x06   index data / chunk info                                                -> skipped (sequential read)
 *
 * and the two message types the reference subscribes to are decoded from the ROS serialisation (little endian, strings
 * and arrays prefixed by a u32 length): sensor_msgs/PointCloud2 -> a view of the point bytes plus the byte offsets of the
 * fields the LiDAR's point struct uses (include/Headers/Common.hpp:109-221: velodyne x y z intensity time(f32); hesai
 * x y z intensity(u8) timestamp(f64); ouster x y z reflectivity(u16) t(u32) range(u32); custom like hesai with f32
 * intensity), ready for lv_pointcloud2_to_points; sensor_msgs/Imu -> stamp, orientation, angular velocity, acceleration.
 * Livox sensors publish livox_ros_driver/CustomMsg instead of PointCloud2: lv_bag_parse_livox -> a view of its 19-byte records.
 * A Velodyne driver that records packets publishes velodyne_msgs/VelodyneScan: lv_bag_parse_velodyne_scan -> a view of its packets.
 * An Ouster driver that records packets publishes ouster_ros/PacketMsg, one LiDAR or IMU packet each: lv_bag_parse_ouster_packet ->
 * a view of the packet; lv_ouster_imu_packet decodes an IMU packet into the sample sensor_msgs/Imu would give.
 * Everything is host code: a sweep is a few MB per 100 ms.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/limovelo_b200.h"
#include "../csrc/lv_wire.h"

namespace {

struct Conn { std::string topic, type; };

uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

/* walks the fields of a record header; returns false on a malformed header */
template <class F>
bool for_fields(const uint8_t* h, uint32_t len, F f) {
    uint32_t at = 0;
    while (at + 4 <= len) {
        const uint32_t fl = rd32(h + at);
        at += 4;
        if (fl > len - at) return false;
        const uint8_t* eq = (const uint8_t*)memchr(h + at, '=', fl);
        if (!eq) return false;
        f(std::string((const char*)h + at, (size_t)(eq - (h + at))), eq + 1, (uint32_t)(fl - (eq + 1 - (h + at))));
        at += fl;
    }
    return at == len;
}

}  // namespace

struct lv_bag {
    std::vector<uint8_t> file;
    std::map<uint32_t, Conn> conns;
    /* cursor: position in the top-level record stream and, inside an uncompressed chunk, the chunk's end */
    size_t pos = 0, chunk_end = 0;
    std::string error;
};

namespace {

/* reads one record at `at` (bounded by `end`): header span, data span, op; returns the position after it or 0 */
size_t read_record(const lv_bag* b, size_t at, size_t end, const uint8_t** hdr, uint32_t* hlen, const uint8_t** data, uint32_t* dlen,
                   int* op) {
    if (at + 4 > end) return 0;
    *hlen = rd32(&b->file[at]);
    if (*hlen > end - at - 4) return 0;
    *hdr = &b->file[at + 4];
    size_t p = at + 4 + *hlen;
    if (p + 4 > end) return 0;
    *dlen = rd32(&b->file[p]);
    if (*dlen > end - p - 4) return 0;
    *data = &b->file[p + 4];
    *op = -1;
    int o = -1;
    if (!for_fields(*hdr, *hlen, [&](const std::string& k, const uint8_t* v, uint32_t n) { if (k == "op" && n == 1) o = v[0]; })) return 0;
    *op = o;
    return p + 4 + *dlen;
}

bool add_connection(lv_bag* b, const uint8_t* hdr, uint32_t hlen, const uint8_t* data, uint32_t dlen) {
    uint32_t id = 0xFFFFFFFFu;
    Conn c;
    bool ok = for_fields(hdr, hlen, [&](const std::string& k, const uint8_t* v, uint32_t n) {
        if (k == "conn" && n == 4) id = rd32(v);
        else if (k == "topic") c.topic.assign((const char*)v, n);
    });
    ok = ok && for_fields(data, dlen, [&](const std::string& k, const uint8_t* v, uint32_t n) {
        if (k == "type") c.type.assign((const char*)v, n);
        else if (k == "topic" && c.topic.empty()) c.topic.assign((const char*)v, n);
    });
    if (!ok || id == 0xFFFFFFFFu) return false;
    b->conns[id] = c;
    return true;
}

/* first pass: collect every connection record (top level and inside uncompressed chunks), check the chunk codecs */
lv_status scan(lv_bag* b) {
    size_t at = 13;
    const size_t end = b->file.size();
    while (at < end) {
        const uint8_t *h, *d;
        uint32_t hl, dl;
        int op;
        const size_t next = read_record(b, at, end, &h, &hl, &d, &dl, &op);
        if (!next) { b->error = "malformed record"; return LV_ERR_IO; }
        if (op == 0x07) {
            if (!add_connection(b, h, hl, d, dl)) { b->error = "malformed connection record"; return LV_ERR_IO; }
        } else if (op == 0x05) {
            std::string comp;
            for_fields(h, hl, [&](const std::string& k, const uint8_t* v, uint32_t n) { if (k == "compression") comp.assign((const char*)v, n); });
            if (comp != "none") { b->error = "compressed chunk (" + comp + "): run `rosbag decompress` first"; return LV_ERR_IO; }
            size_t in = (size_t)(d - b->file.data());
            const size_t in_end = in + dl;
            while (in < in_end) {
                const uint8_t *h2, *d2;
                uint32_t hl2, dl2;
                int op2;
                const size_t n2 = read_record(b, in, in_end, &h2, &hl2, &d2, &dl2, &op2);
                if (!n2) { b->error = "malformed record inside a chunk"; return LV_ERR_IO; }
                if (op2 == 0x07 && !add_connection(b, h2, hl2, d2, dl2)) { b->error = "malformed connection record"; return LV_ERR_IO; }
                in = n2;
            }
        }
        at = next;
    }
    return LV_OK;
}

/* cursor over a serialised ROS message */
struct Rd {
    const uint8_t* p;
    int64_t n, at;
    bool ok;
    Rd(const uint8_t* p_, int64_t n_) : p(p_), n(n_), at(0), ok(true) {}
    const uint8_t* take(int64_t k) {
        if (!ok || k < 0 || k > n - at) { ok = false; return nullptr; }
        const uint8_t* r = p + at;
        at += k;
        return r;
    }
    uint32_t u32() { const uint8_t* r = take(4); return r ? rd32(r) : 0; }
    uint8_t u8() { const uint8_t* r = take(1); return r ? *r : 0; }
    double f64() { const uint8_t* r = take(8); double v = 0; if (r) memcpy(&v, r, 8); return v; }
    std::string str() { const uint32_t k = u32(); const uint8_t* r = take(k); return r ? std::string((const char*)r, k) : std::string(); }
};

}  // namespace

extern "C" {

lv_status lv_bag_open(const char* path, lv_bag** out) {
    if (!path || !out) return LV_ERR_ARG;
    *out = nullptr;
    FILE* f = fopen(path, "rb");
    if (!f) return LV_ERR_IO;
    lv_bag* b = new lv_bag();
    fseek(f, 0, SEEK_END);
    const long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (sz < 13) { fclose(f); delete b; return LV_ERR_IO; }
    b->file.resize((size_t)sz);
    const size_t got = fread(b->file.data(), 1, (size_t)sz, f);
    fclose(f);
    if (got != (size_t)sz || memcmp(b->file.data(), "#ROSBAG V2.0\n", 13) != 0) { delete b; return LV_ERR_IO; }
    const lv_status st = scan(b);
    if (st != LV_OK) { fprintf(stderr, "lv_bag_open(%s): %s\n", path, b->error.c_str()); delete b; return st; }
    b->pos = 13;
    b->chunk_end = 0;
    *out = b;
    return LV_OK;
}

void lv_bag_close(lv_bag* b) { delete b; }
void lv_bag_rewind(lv_bag* b) { if (b) { b->pos = 13; b->chunk_end = 0; } }
int32_t lv_bag_connection_count(const lv_bag* b) { return b ? (int32_t)b->conns.size() : 0; }

int lv_bag_next(lv_bag* b, lv_bag_message* msg) {
    if (!b || !msg) return -1;
    for (;;) {
        const size_t end = b->chunk_end ? b->chunk_end : b->file.size();
        if (b->pos >= end) {
            if (b->chunk_end) { b->chunk_end = 0; continue; }       /* end of a chunk: back to the top level */
            return 0;
        }
        const uint8_t *h, *d;
        uint32_t hl, dl;
        int op;
        const size_t next = read_record(b, b->pos, end, &h, &hl, &d, &dl, &op);
        if (!next) return -1;
        if (op == 0x05 && !b->chunk_end) {                          /* descend into the chunk's records */
            b->pos = (size_t)(d - b->file.data());
            b->chunk_end = b->pos + dl;
            continue;
        }
        b->pos = next;
        if (op != 0x02) continue;
        uint32_t id = 0xFFFFFFFFu, sec = 0, nsec = 0;
        for_fields(h, hl, [&](const std::string& k, const uint8_t* v, uint32_t n) {
            if (k == "conn" && n == 4) id = rd32(v);
            else if (k == "time" && n == 8) { sec = rd32(v); nsec = rd32(v + 4); }
        });
        const auto it = b->conns.find(id);
        msg->conn = (int32_t)id;
        msg->topic = it != b->conns.end() ? it->second.topic.c_str() : "";
        msg->type = it != b->conns.end() ? it->second.type.c_str() : "";
        msg->sec = sec;
        msg->nsec = nsec;
        msg->data = d;
        msg->size = dl;
        return 1;
    }
}

lv_status lv_bag_parse_pointcloud2(const uint8_t* data, int64_t size, lv_lidar_type type, lv_pointcloud2_view* out) {
    if (!data || !out || size < 0) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));
    Rd r(data, size);
    r.u32();                                          /* std_msgs/Header: seq, stamp, frame_id */
    out->stamp_sec = r.u32();
    out->stamp_nsec = r.u32();
    r.str();
    out->height = r.u32();
    out->width = r.u32();
    const uint32_t nf = r.u32();                      /* sensor_msgs/PointField[]: name, offset, datatype, count */
    if (!r.ok || nf > 4096) return LV_ERR_IO;
    const char* tname = type == LV_LIDAR_VELODYNE ? "time" : (type == LV_LIDAR_OUSTER ? "t" : "timestamp");
    const char* iname = type == LV_LIDAR_OUSTER ? "reflectivity" : "intensity";
    /* datatype codes of sensor_msgs/PointField: 2 UINT8, 4 UINT16, 6 UINT32, 7 FLOAT32, 8 FLOAT64 */
    const int t_dt = type == LV_LIDAR_VELODYNE ? 7 : (type == LV_LIDAR_OUSTER ? 6 : 8);
    const int i_dt = type == LV_LIDAR_HESAI ? 2 : (type == LV_LIDAR_OUSTER ? 4 : 7);
    int32_t ox = -1, oy = -1, oz = -1, oi = -1, ot = -1, orng = -1;
    for (uint32_t k = 0; k < nf; ++k) {
        const std::string name = r.str();
        const uint32_t off = r.u32();
        const uint8_t dt = r.u8();
        r.u32();
        if (!r.ok) return LV_ERR_IO;
        if (name == "x" && dt == 7) ox = (int32_t)off;
        else if (name == "y" && dt == 7) oy = (int32_t)off;
        else if (name == "z" && dt == 7) oz = (int32_t)off;
        else if (name == iname && dt == i_dt) oi = (int32_t)off;
        else if (name == tname && dt == t_dt) ot = (int32_t)off;
        else if (name == "range" && dt == 6) orng = (int32_t)off;
    }
    out->is_bigendian = r.u8();
    out->point_step = r.u32();
    out->row_step = r.u32();
    const uint32_t nbytes = r.u32();
    out->data = r.take(nbytes);
    out->data_bytes = nbytes;
    out->is_dense = r.u8();
    if (!r.ok || out->is_bigendian) return LV_ERR_IO;
    if (ox < 0 || oy < 0 || oz < 0 || oi < 0 || ot < 0 || (type == LV_LIDAR_OUSTER && orng < 0)) return LV_ERR_IO;   /* not this LiDAR's point struct */
    out->layout.point_step = (int32_t)out->point_step;
    out->layout.off_x = ox; out->layout.off_y = oy; out->layout.off_z = oz;
    out->layout.off_intensity = oi; out->layout.off_time = ot; out->layout.off_range = orng < 0 ? 0 : orng;
    out->n_points = (int64_t)out->height * (int64_t)out->width;
    if (out->point_step == 0 || (uint64_t)out->n_points * out->point_step > nbytes) return LV_ERR_IO;
    return LV_OK;
}

lv_status lv_bag_parse_imu(const uint8_t* data, int64_t size, lv_imu_sample* out) {
    if (!data || !out || size < 0) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));
    Rd r(data, size);
    r.u32();
    out->stamp_sec = r.u32();
    out->stamp_nsec = r.u32();
    r.str();
    for (int i = 0; i < 4; ++i) out->orientation[i] = r.f64();      /* geometry_msgs/Quaternion x y z w */
    r.take(72);
    for (int i = 0; i < 3; ++i) out->angular_velocity[i] = r.f64();
    r.take(72);
    for (int i = 0; i < 3; ++i) out->linear_acceleration[i] = r.f64();
    r.take(72);
    return r.ok ? LV_OK : LV_ERR_IO;
}

lv_status lv_bag_parse_livox(const uint8_t* data, int64_t size, lv_livox_view* out) {
    if (!data || !out || size < 0) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));
    Rd r(data, size);
    r.u32();                                          /* std_msgs/Header: seq, stamp, frame_id */
    const uint32_t sec = r.u32(), nsec = r.u32();
    r.str();
    const uint8_t* tb = r.take(8);
    const uint32_t point_num = r.u32();
    const uint8_t lidar_id = r.u8();
    r.take(3);                                        /* uint8[3] rsvd: a fixed-size array, no length prefix */
    const uint32_t count = r.u32();                   /* CustomPoint[] */
    const uint8_t* recs = r.take((int64_t)count * lv::kLivoxRecord);
    if (!r.ok || r.at != size || point_num != count) return LV_ERR_ARG;
    out->stamp_sec = sec;
    out->stamp_nsec = nsec;
    out->timebase = (uint64_t)rd32(tb) | (uint64_t)rd32(tb + 4) << 32;
    out->point_num = point_num;
    out->lidar_id = lidar_id;
    out->n_points = count;
    out->data = recs;
    out->data_bytes = (int64_t)count * lv::kLivoxRecord;
    return LV_OK;
}

lv_status lv_bag_parse_velodyne_scan(const uint8_t* data, int64_t size, lv_velodyne_view* out) {
    if (!data || !out || size < 0) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));
    Rd r(data, size);
    r.u32();                                          /* std_msgs/Header: seq, stamp, frame_id */
    const uint32_t sec = r.u32(), nsec = r.u32();
    r.str();
    const uint32_t count = r.u32();                   /* VelodynePacket[]: time stamp, uint8[1206] data (fixed, no length prefix) */
    const uint8_t* packets = r.take((int64_t)count * lv::kVelodynePacket);
    if (!r.ok || r.at != size) return LV_ERR_ARG;
    out->stamp_sec = sec;
    out->stamp_nsec = nsec;
    out->n_packets = count;
    out->packets = packets;
    out->data_bytes = (int64_t)count * lv::kVelodynePacket;
    return LV_OK;
}

lv_status lv_bag_parse_ouster_packet(const uint8_t* data, int64_t size, lv_ouster_packet_view* out) {
    if (!data || !out || size < 0) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));
    Rd r(data, size);
    const uint32_t bytes = r.u32();                   /* uint8[] buf */
    const uint8_t* buf = r.take(bytes);
    if (!r.ok || r.at != size) return LV_ERR_ARG;
    out->data = buf;
    out->bytes = bytes;
    return LV_OK;
}

lv_status lv_ouster_imu_packet(const uint8_t* pkt, int64_t bytes, lv_imu_sample* out) {
    if (!pkt || !out || bytes != 48) return LV_ERR_ARG;
    const uint64_t gyro_ts = lv::wire_u64(pkt + 16);
    if (gyro_ts / 1000000000ull > 0xFFFFFFFFull) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));                     /* orientation {0, 0, 0, 0}: none (IMU::has_orientation) */
    out->stamp_sec = (uint32_t)(gyro_ts / 1000000000ull);
    out->stamp_nsec = (uint32_t)(gyro_ts % 1000000000ull);
    for (int k = 0; k < 3; ++k) {
        out->linear_acceleration[k] = (double)lv::wire_f32(pkt + 24 + 4 * k) * 9.80665;     /* g -> m/s^2 */
        out->angular_velocity[k] = ((double)lv::wire_f32(pkt + 36 + 4 * k) * M_PI) / 180.0;  /* deg/s -> rad/s */
    }
    return LV_OK;
}

/* lv_pointcloud2_to_points with the bounds pcl::fromROSMsg gets from the message itself (lv::cloud_layout_error, which
 * lv_process_cloud_device applies as well) */
lv_status lv_pointcloud2_to_points_checked(lv_lidar_type type, const lv_cloud_layout* L, const uint8_t* data, int64_t data_bytes, int64_t n,
                                           uint64_t header_stamp_us, int stamp_beginning, int offset_beginning, double full_rotation_time,
                                           float* xyz, double* time, float* intensity, float* range) {
    if (!L || !data || lv::cloud_layout_error(type, *L, n, data_bytes)) return LV_ERR_ARG;
    return lv_pointcloud2_to_points(type, L, data, n, header_stamp_us, stamp_beginning, offset_beginning, full_rotation_time, xyz, time,
                                    intensity, range);
}

}  // extern "C"
