/*
 * lv_pcd_host.cpp — PCD map files (Point Cloud Library format v0.7), the map format of the reference's PCL stack
 * (pcl::io::savePCDFileBinary) and of most LiDAR SLAM tools.
 *
 *   header   one "KEY values" line per key, '#' lines are comments: VERSION, FIELDS, SIZE, TYPE, COUNT, WIDTH, HEIGHT,
 *            VIEWPOINT, POINTS, DATA (the last header line).  COUNT may be absent (all 1).
 *   data     ascii: one record per line, the values of every field (COUNT values each) separated by blanks;
 *            binary: POINTS packed records of sum(SIZE * COUNT) bytes, little endian;
 *            binary_compressed (LZF, field-major) is refused: no codec is linked here.
 *
 * The map needs x, y and z (TYPE F, SIZE 4, COUNT 1); any other field (intensity, rgb, timestamps, '_' padding) is skipped
 * by its size.  Host code: a 10 M point map is 120 MB of floats.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <sstream>
#include <string>
#include <vector>

#include "../../include/limovelo_b200.h"
#include "../csrc/lv_host.h"

namespace {

lv_status pcd_fail(const std::string& what) {
    lvh_set_error(("pcd: " + what).c_str());
    return LV_ERR_IO;
}

struct PcdField {
    std::string name;
    int size = 0;
    char type = 0;
    int64_t count = 1;
};

/* the bytes of the whole file (PCD maps are read once, at the start of a sequence) */
bool read_file(const char* path, std::vector<char>* buf) {
    FILE* f = fopen(path, "rb");
    if (!f) return false;
    bool ok = fseek(f, 0, SEEK_END) == 0;
    const long sz = ok ? ftell(f) : -1;
    ok = ok && sz >= 0 && fseek(f, 0, SEEK_SET) == 0;
    if (ok) {
        buf->resize((size_t)sz);
        ok = fread(buf->data(), 1, (size_t)sz, f) == (size_t)sz;
    }
    fclose(f);
    return ok;
}

std::vector<std::string> split(const std::string& line) {
    std::vector<std::string> out;
    std::istringstream is(line);
    std::string w;
    while (is >> w) out.push_back(w);
    return out;
}

bool to_i64(const std::string& s, int64_t* v) {
    char* end = nullptr;
    const long long x = strtoll(s.c_str(), &end, 10);
    if (end == s.c_str() || *end) return false;
    *v = (int64_t)x;
    return true;
}

}  // namespace

extern "C" {

lv_status lv_pcd_write(const char* path, const float* xyz, int64_t n) {
    if (!path || (!xyz && n > 0) || n < 0) { lvh_set_error("pcd write: null path or points, or n < 0"); return LV_ERR_ARG; }
    FILE* f = fopen(path, "wb");
    if (!f) return pcd_fail(std::string("cannot open ") + path + " for writing");
    char hdr[512];
    const int len = snprintf(hdr, sizeof(hdr),
                             "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\n"
                             "COUNT 1 1 1\nWIDTH %lld\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %lld\nDATA binary\n",
                             (long long)n, (long long)n);
    bool ok = fwrite(hdr, 1, (size_t)len, f) == (size_t)len;
    if (ok && n > 0) ok = fwrite(xyz, sizeof(float) * 3, (size_t)n, f) == (size_t)n;
    const bool closed = fclose(f) == 0;
    if (!ok) return pcd_fail(std::string("short write to ") + path);
    if (!closed) return pcd_fail(std::string("closing ") + path + " failed");
    return LV_OK;
}

lv_status lv_pcd_read(const char* path, float* xyz, int64_t cap, int64_t* n) {
    if (!path || !n || (xyz && cap < 0)) { lvh_set_error("pcd read: null path or count, or cap < 0"); return LV_ERR_ARG; }
    *n = 0;
    std::vector<char> buf;
    if (!read_file(path, &buf)) return pcd_fail(std::string("cannot read ") + path);
    /* header: lines up to and including DATA */
    size_t pos = 0;
    std::vector<PcdField> fields;
    bool have_count = false, have_size = false, have_type = false;
    int64_t width = -1, height = -1, points = -1;
    std::string data;
    while (pos < buf.size() && data.empty()) {
        size_t e = pos;
        while (e < buf.size() && buf[e] != '\n') ++e;
        std::string line(buf.data() + pos, e - pos);
        pos = e < buf.size() ? e + 1 : e;
        if (!line.empty() && line.back() == '\r') line.pop_back();
        const std::vector<std::string> w = split(line);
        if (w.empty() || w[0][0] == '#') continue;
        const std::string& key = w[0];
        const size_t nv = w.size() - 1;
        if (key == "VERSION") {
            if (nv != 1 || (w[1] != "0.7" && w[1] != ".7")) return pcd_fail("unsupported VERSION (0.7 is read)");
        } else if (key == "FIELDS") {
            fields.assign(nv, PcdField());
            for (size_t i = 0; i < nv; ++i) fields[i].name = w[1 + i];
        } else if (key == "SIZE" || key == "TYPE" || key == "COUNT") {
            if (nv != fields.size() || fields.empty()) return pcd_fail(key + " does not match FIELDS");
            for (size_t i = 0; i < nv; ++i) {
                if (key == "TYPE") {
                    if (w[1 + i].size() != 1 || !strchr("FIU", w[1 + i][0])) return pcd_fail("TYPE " + w[1 + i] + " is not F, I or U");
                    fields[i].type = w[1 + i][0];
                    continue;
                }
                int64_t v = 0;
                if (!to_i64(w[1 + i], &v)) return pcd_fail(key + " value " + w[1 + i] + " is not an integer");
                if (key == "SIZE") {
                    if (v != 1 && v != 2 && v != 4 && v != 8) return pcd_fail("SIZE " + w[1 + i] + " is not 1, 2, 4 or 8");
                    fields[i].size = (int)v;
                } else {
                    if (v < 1 || v > (1 << 20)) return pcd_fail("COUNT " + w[1 + i] + " outside [1, 2^20]");
                    fields[i].count = v;
                }
            }
            (key == "SIZE" ? have_size : key == "TYPE" ? have_type : have_count) = true;
        } else if (key == "WIDTH" || key == "HEIGHT" || key == "POINTS") {
            int64_t v = 0;
            if (nv != 1 || !to_i64(w[1], &v) || v < 0) return pcd_fail(key + " is not a non-negative integer");
            (key == "WIDTH" ? width : key == "HEIGHT" ? height : points) = v;
        } else if (key == "VIEWPOINT") {
            /* the sensor pose the cloud was taken from: a map is stored in the world frame, nothing to apply */
        } else if (key == "DATA") {
            if (nv != 1) return pcd_fail("malformed DATA line");
            data = w[1];
        } else {
            return pcd_fail("unknown header line '" + key + "'");
        }
    }
    if (data.empty()) return pcd_fail("no DATA line");
    if (data == "binary_compressed")
        return pcd_fail("DATA binary_compressed is not read: convert the file with pcl_convert_pcd_ascii_binary (binary mode 1)");
    if (data != "ascii" && data != "binary") return pcd_fail("DATA " + data + " is not ascii or binary");
    if (fields.empty() || !have_size || !have_type) return pcd_fail("FIELDS, SIZE or TYPE missing");
    (void)have_count;
    if (width < 0 || height < 0) return pcd_fail("WIDTH or HEIGHT missing");
    if (height > 0 && width > ((int64_t)1 << 40) / height) return pcd_fail("WIDTH x HEIGHT above 2^40");
    if (points < 0) points = width * height;
    if (points != width * height) return pcd_fail("POINTS " + std::to_string((long long)points) + " != WIDTH x HEIGHT " +
                                                  std::to_string((long long)(width * height)));
    int fx = -1, fy = -1, fz = -1;
    for (size_t i = 0; i < fields.size(); ++i) {
        if (fields[i].name == "x") fx = (int)i;
        if (fields[i].name == "y") fy = (int)i;
        if (fields[i].name == "z") fz = (int)i;
    }
    if (fx < 0 || fy < 0 || fz < 0) return pcd_fail("no x, y and z fields");
    for (int f : {fx, fy, fz})
        if (fields[f].type != 'F' || fields[f].size != 4 || fields[f].count != 1)
            return pcd_fail("field " + fields[f].name + " is not TYPE F, SIZE 4, COUNT 1");
    /* value offset of x, y, z within a record (in values for ascii, in bytes for binary) */
    int64_t rec_bytes = 0, rec_values = 0, bx = 0, by = 0, bz = 0, vx = 0, vy = 0, vz = 0;
    for (size_t i = 0; i < fields.size(); ++i) {
        if ((int)i == fx) { bx = rec_bytes; vx = rec_values; }
        if ((int)i == fy) { by = rec_bytes; vy = rec_values; }
        if ((int)i == fz) { bz = rec_bytes; vz = rec_values; }
        rec_bytes += (int64_t)fields[i].size * fields[i].count;
        rec_values += fields[i].count;
    }
    std::vector<float> kept;
    auto keep = [&](float x, float y, float z) {
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) return;
        kept.push_back(x); kept.push_back(y); kept.push_back(z);
    };
    if (data == "binary") {
        const uint64_t avail = buf.size() - pos;
        if ((uint64_t)points > avail / (uint64_t)rec_bytes)
            return pcd_fail("data section holds " + std::to_string((unsigned long long)(avail / (uint64_t)rec_bytes)) + " of " +
                            std::to_string((long long)points) + " POINTS records");
        kept.reserve(3 * (size_t)points);
        const char* d = buf.data() + pos;
        for (int64_t r = 0; r < points; ++r, d += rec_bytes) {
            float x, y, z;
            memcpy(&x, d + bx, 4); memcpy(&y, d + by, 4); memcpy(&z, d + bz, 4);
            keep(x, y, z);
        }
    } else {
        buf.push_back('\0');
        const char* s = buf.data() + pos;
        std::vector<float> rec((size_t)rec_values);
        for (int64_t r = 0; r < points; ++r) {
            while (*s == ' ' || *s == '\t' || *s == '\r' || *s == '\n') ++s;
            for (int64_t v = 0; v < rec_values; ++v) {
                while (*s == ' ' || *s == '\t') ++s;
                char* end = nullptr;
                const float val = strtof(s, &end);
                if (end == s) return pcd_fail("data section holds " + std::to_string((long long)r) + " of " + std::to_string((long long)points) +
                                              " POINTS records");
                rec[(size_t)v] = val;
                s = end;
            }
            keep(rec[(size_t)vx], rec[(size_t)vy], rec[(size_t)vz]);
        }
    }
    const int64_t m = (int64_t)(kept.size() / 3);
    *n = m;
    if (!xyz) return LV_OK;
    if (cap < m) {
        lvh_set_error(("pcd read: " + std::to_string((long long)m) + " points, more than cap " + std::to_string((long long)cap)).c_str());
        return LV_ERR_CAPACITY;
    }
    if (m) memcpy(xyz, kept.data(), sizeof(float) * 3 * (size_t)m);
    return LV_OK;
}

}  // extern "C"
