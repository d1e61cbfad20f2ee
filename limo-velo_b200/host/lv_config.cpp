/*
 * lv_config.cpp — configuration: defaults of fill_config (src/main.cpp:135-176) and a reader for the
 * reference's config/<name>.yaml files (the ROS parameter server of launch/run.launch:3 is replaced by
 * a plain file parser; same keys, same defaults, unknown keys ignored like rosparam does).
 */
#include <ctype.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/limovelo_b200.h"

extern "C" void lv_default_params(lv_params* p) {
    if (!p) return;
    memset(p, 0, sizeof(*p));
    p->MAX_NUM_ITERS = 3;                     /* main.cpp:144 */
    p->NUM_MATCH_POINTS = 5;                  /* main.cpp:146 */
    p->estimate_extrinsics = 0;               /* main.cpp:139 */
    p->print_degeneracy_values = 0;           /* main.cpp:156 */
    p->MAX_DIST_PLANE = 2.0;                  /* main.cpp:148 */
    p->PLANES_THRESHOLD = 0.1f;               /* main.cpp:149 */
    p->LiDAR_noise = 0.001;                   /* main.cpp:152 */
    p->degeneracy_threshold = 5.0;            /* main.cpp:155 */
    for (int i = 0; i < LV_DOF; ++i) p->LIMITS[i] = 0.001;   /* main.cpp:145 */
    p->covariance_gyroscope = 1e-4;           /* main.cpp:160-163 */
    p->covariance_acceleration = 1e-2;
    p->covariance_bias_gyroscope = 1e-5;
    p->covariance_bias_acceleration = 1e-4;
    p->initial_gravity[0] = 0.f; p->initial_gravity[1] = 0.f; p->initial_gravity[2] = -9.807f;   /* main.cpp:173 */
    /* I_Translation_L / I_Rotation_L default to zeros in the reference (main.cpp:174-175); a zero
     * rotation is unusable, identity is the neutral choice here */
    p->I_Rotation_L[0] = p->I_Rotation_L[4] = p->I_Rotation_L[8] = 1.f;
    p->map_downsample_size = 0.2f;            /* Mapper.cpp:65 */
    p->voxel_size = 0.4f;
    p->device = 0;
    p->max_map_points = 4 * 1024 * 1024;
    p->max_points = 512 * 1024;
    p->stream = NULL;
}

namespace {

std::string strip(const std::string& s) {
    size_t a = 0, b = s.size();
    while (a < b && isspace((unsigned char)s[a])) ++a;
    while (b > a && isspace((unsigned char)s[b - 1])) --b;
    return s.substr(a, b - a);
}
std::string strip_comment(const std::string& s) {
    bool in_q = false;
    for (size_t i = 0; i < s.size(); ++i) {
        if (s[i] == '"') in_q = !in_q;
        if (s[i] == '#' && !in_q) return s.substr(0, i);
    }
    return s;
}
/* YAML 1.1 floats as they appear in the reference configs: "5.", "5.e-2", "+9.807", "1.e-1" */
bool parse_number(const std::string& t, double* out) {
    std::string s = strip(t);
    if (s.empty()) return false;
    char* end = NULL;
    *out = strtod(s.c_str(), &end);
    return end && *end == '\0';
}
bool parse_bool(const std::string& t, int* out) {
    std::string s = strip(t);
    for (auto& c : s) c = (char)tolower((unsigned char)c);
    if (s == "true" || s == "yes" || s == "on") { *out = 1; return true; }
    if (s == "false" || s == "no" || s == "off") { *out = 0; return true; }
    return false;
}
std::vector<double> parse_list(const std::string& t) {
    std::vector<double> v;
    std::string s = t;
    size_t a = s.find('['), b = s.rfind(']');
    if (a == std::string::npos || b == std::string::npos || b <= a) return v;
    s = s.substr(a + 1, b - a - 1);
    size_t pos = 0;
    while (pos <= s.size()) {
        size_t c = s.find(',', pos);
        std::string item = s.substr(pos, c == std::string::npos ? std::string::npos : c - pos);
        double d;
        if (parse_number(item, &d)) v.push_back(d);
        if (c == std::string::npos) break;
        pos = c + 1;
    }
    return v;
}

}  // namespace

extern "C" lv_status lv_params_from_yaml(const char* path, lv_params* p) {
    if (!path || !p) return LV_ERR_ARG;
    FILE* f = fopen(path, "r");
    if (!f) return LV_ERR_IO;
    std::map<std::string, std::string> kv;   /* top-level scalars and (possibly multi-line) flow lists */
    char buf[4096];
    std::string pending_key, pending_val;
    int depth = 0;
    while (fgets(buf, sizeof(buf), f)) {
        std::string line = strip_comment(buf);
        if (depth > 0) {   /* continuation of a multi-line [ ... ] */
            pending_val += " " + line;
            for (char c : line) { if (c == '[') ++depth; else if (c == ']') --depth; }
            if (depth <= 0) { kv[pending_key] = pending_val; depth = 0; }
            continue;
        }
        if (strip(line).empty()) continue;
        const bool indented = isspace((unsigned char)line[0]);
        size_t colon = line.find(':');
        if (colon == std::string::npos) continue;
        std::string key = strip(line.substr(0, colon));
        std::string val = strip(line.substr(colon + 1));
        if (indented) continue;   /* nested maps (Initialization: times/deltas) are driver-side, not on the path */
        for (char c : val) { if (c == '[') ++depth; else if (c == ']') --depth; }
        if (depth > 0) { pending_key = key; pending_val = val; continue; }
        depth = 0;
        kv[key] = val;
    }
    fclose(f);

    auto num = [&](const char* k, double* dst) { auto it = kv.find(k); double d; if (it != kv.end() && parse_number(it->second, &d)) *dst = d; };
    auto numf = [&](const char* k, float* dst) { double d = *dst; num(k, &d); *dst = (float)d; };
    auto numi = [&](const char* k, int32_t* dst) { double d = *dst; num(k, &d); *dst = (int32_t)d; };
    auto boolean = [&](const char* k, int32_t* dst) { auto it = kv.find(k); int b; if (it != kv.end() && parse_bool(it->second, &b)) *dst = b; };
    auto listf = [&](const char* k, float* dst, size_t n) {
        auto it = kv.find(k);
        if (it == kv.end()) return;
        std::vector<double> v = parse_list(it->second);
        if (v.size() == n) for (size_t i = 0; i < n; ++i) dst[i] = (float)v[i];
    };
    numi("MAX_NUM_ITERS", &p->MAX_NUM_ITERS);
    numi("NUM_MATCH_POINTS", &p->NUM_MATCH_POINTS);
    boolean("estimate_extrinsics", &p->estimate_extrinsics);
    boolean("print_degeneracy_values", &p->print_degeneracy_values);
    num("MAX_DIST_PLANE", &p->MAX_DIST_PLANE);
    numf("PLANES_THRESHOLD", &p->PLANES_THRESHOLD);
    num("LiDAR_noise", &p->LiDAR_noise);
    num("degeneracy_threshold", &p->degeneracy_threshold);
    num("covariance_gyroscope", &p->covariance_gyroscope);
    num("covariance_acceleration", &p->covariance_acceleration);
    num("covariance_bias_gyroscope", &p->covariance_bias_gyroscope);
    num("covariance_bias_acceleration", &p->covariance_bias_acceleration);
    listf("initial_gravity", p->initial_gravity, 3);
    listf("I_Translation_L", p->I_Translation_L, 3);
    listf("I_Rotation_L", p->I_Rotation_L, 9);
    {
        auto it = kv.find("LIMITS");
        if (it != kv.end()) {
            std::vector<double> v = parse_list(it->second);
            if (v.size() == LV_DOF) for (int i = 0; i < LV_DOF; ++i) p->LIMITS[i] = v[i];
        }
    }
    /* device tuning keys are optional extensions */
    numf("voxel_size", &p->voxel_size);
    return LV_OK;
}

/* ---- the Ouster sensor metadata JSON (lv_ouster_calibration_from_json): a scanner for the few keys the decoder needs, not a JSON
 * library.  A key is a string followed by ':'; its value starts after the ':'.  Keys are taken at any depth, the first occurrence
 * counts, and string values are skipped whole, so text inside them is never read as a key. */
namespace {

struct JsonScan {
    const std::string& t;
    std::map<std::string, size_t> at;   /* key -> position of its value */
    explicit JsonScan(const std::string& text) : t(text) {
        size_t i = 0;
        while (i < t.size()) {
            if (t[i] != '"') { ++i; continue; }
            std::string key;
            if (!string_at(i, &key, &i)) return;
            size_t j = skip(i);
            if (j < t.size() && t[j] == ':' && !at.count(key)) at[key] = skip(j + 1);
        }
    }
    size_t skip(size_t i) const {
        while (i < t.size() && isspace((unsigned char)t[i])) ++i;
        return i;
    }
    /* the string starting at t[i] == '"' (escapes kept as written); *end = one past its closing quote */
    bool string_at(size_t i, std::string* out, size_t* end) const {
        if (i >= t.size() || t[i] != '"') return false;
        for (size_t j = i + 1; j < t.size(); ++j) {
            if (t[j] == '\\') { ++j; continue; }
            if (t[j] == '"') { *out = t.substr(i + 1, j - i - 1); *end = j + 1; return true; }
        }
        return false;
    }
    /* a finite JSON number at t[i]; *end = one past it */
    bool number_at(size_t i, double* out, size_t* end) const {
        if (i >= t.size() || !(t[i] == '-' || isdigit((unsigned char)t[i]))) return false;
        char* e = nullptr;
        *out = strtod(t.c_str() + i, &e);
        if (e == t.c_str() + i || !isfinite(*out)) return false;
        *end = (size_t)(e - t.c_str());
        return true;
    }
    bool has(const char* k) const { return at.count(k) != 0; }
    bool number(const char* k, double* out) const { size_t e; return has(k) && number_at(at.at(k), out, &e); }
    bool str(const char* k, std::string* out) const { size_t e; return has(k) && string_at(at.at(k), out, &e); }
    bool numbers(const char* k, std::vector<double>* out) const {
        if (!has(k)) return false;
        size_t i = at.at(k);
        if (i >= t.size() || t[i] != '[') return false;
        i = skip(i + 1);
        if (i < t.size() && t[i] == ']') return true;
        for (;;) {
            double d;
            if (!number_at(i, &d, &i)) return false;
            out->push_back(d);
            i = skip(i);
            if (i < t.size() && t[i] == ']') return true;
            if (i >= t.size() || t[i] != ',') return false;
            i = skip(i + 1);
        }
    }
};

/* "<W>x<rate>", e.g. "1024x10" -> W */
bool lidar_mode_columns(const std::string& mode, int32_t* W) {
    const size_t x = mode.find('x');
    if (x == 0 || x == std::string::npos || x + 1 == mode.size() || x > 4) return false;
    for (size_t i = 0; i < mode.size(); ++i)
        if (i != x && !isdigit((unsigned char)mode[i])) return false;
    *W = (int32_t)atoi(mode.substr(0, x).c_str());
    return true;
}

}  // namespace

/* the udp_profile_lidar strings the decoder reads, in lv_ouster_profile order */
static const char* const kOusterProfiles[] = {"LEGACY", "RNG19_RFL8_SIG16_NIR16", "RNG19_RFL8_SIG16_NIR16_DUAL", "RNG15_RFL8_NIR8"};

extern "C" lv_status lv_ouster_sensor_from_json(const char* text, int64_t len, lv_ouster_calibration* out, lv_ouster_profile* profile) {
    if (!text || len < 0 || !out || !profile) return LV_ERR_ARG;
    memset(out, 0, sizeof(*out));
    *profile = LV_OUSTER_LEGACY;
    const std::string t(text, (size_t)len);
    const JsonScan j(t);
    std::vector<double> alt, az;
    std::string mode, name;
    int32_t W = 0;
    if (!j.numbers("beam_altitude_angles", &alt) || !j.numbers("beam_azimuth_angles", &az) || alt.size() != az.size() ||
        !j.str("lidar_mode", &mode) || !lidar_mode_columns(mode, &W))
        return LV_ERR_ARG;
    const int32_t H = (int32_t)alt.size();
    if ((W != 512 && W != 1024 && W != 2048) || (H != 16 && H != 32 && H != 64 && H != 128)) return LV_ERR_ARG;
    double v = 0;
    if (j.has("pixels_per_column") && (!j.number("pixels_per_column", &v) || v != H)) return LV_ERR_ARG;
    if (j.has("columns_per_packet") && (!j.number("columns_per_packet", &v) || v != 16)) return LV_ERR_ARG;
    int kind = LV_OUSTER_LEGACY;                                  /* firmware 1.x has no udp_profile_lidar: LEGACY */
    if (j.has("udp_profile_lidar")) {
        if (!j.str("udp_profile_lidar", &name)) return LV_ERR_ARG;
        kind = -1;
        for (int k = 0; k < 4; ++k)
            if (name == kOusterProfiles[k]) kind = k;
        if (kind < 0) return LV_ERR_ARG;
    }
    double n = 0;
    if (j.has("lidar_origin_to_beam_origin_mm") && !j.number("lidar_origin_to_beam_origin_mm", &n)) return LV_ERR_ARG;
    out->columns_per_frame = W;
    out->pixels_per_column = H;
    for (int32_t p = 0; p < H; ++p) {
        out->beam_altitude_angles[p] = alt[p];
        out->beam_azimuth_angles[p] = az[p];
    }
    out->lidar_origin_to_beam_origin_mm = n;
    *profile = (lv_ouster_profile)kind;
    return LV_OK;
}

extern "C" lv_status lv_ouster_calibration_from_json(const char* text, int64_t len, lv_ouster_calibration* out) {
    lv_ouster_profile profile;
    const lv_status st = lv_ouster_sensor_from_json(text, len, out, &profile);
    if (st != LV_OK) return st;
    if (profile != LV_OUSTER_LEGACY) {
        memset(out, 0, sizeof(*out));
        return LV_ERR_ARG;
    }
    return LV_OK;
}
