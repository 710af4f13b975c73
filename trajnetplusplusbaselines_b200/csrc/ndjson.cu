// Host-side TrajNet++ ndjson codec of the batched evaluator path (SURVEY.md 8f rank 1: "ndjson reader/writer as the on-disk
// format either side"; reference: trajnetplusplustools.Reader / writers as used by evaluator/write_utils.py:42-81 and
// lstm/trajnet_evaluator.py:28-64).  No CUDA in this file: once the forward runs at > 10 k scenes/s the per-line
// json.loads / json.dumps of the Python path is what bounds the evaluator end to end, so the two text passes are native:
//
//   tb2_ndjson_parse   one pass over the file text -> column arrays of the track rows (frame, pedestrian, x, y in file order)
//                      and of the scene rows (id, pedestrian, start, end).  It understands exactly the objects the format
//                      holds ({"track": {...}} / {"scene": {...}}, any key order, any JSON whitespace) and REFUSES a line it
//                      is not sure about (escapes, a non-integer frame, unknown record types ...): the caller then takes the
//                      json.loads path for the whole file, so the result never depends on which parser ran.
//   tb2_ndjson_parse_meta  the same pass, plus the metadata the scorer reads: prediction_number / scene_id of the track
//                      rows and the tag of the scene rows (main type + sub-type bitmask), refusing anything unusual there.
//   tb2_ndjson_format  prediction records -> text, byte-identical to json.dumps of the reference writer's dictionaries:
//                      coordinates are round(x, 2) printed like repr(float) ("%.2f" is the same correctly rounded decimal;
//                      trailing zero stripped down to one decimal), NaN / Infinity spelled as json.dumps spells them.
#include <errno.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace tb2 {
namespace {

struct Cursor {
    const char* p;
    const char* end;
};

inline void skip_ws(Cursor& c) {
    while (c.p < c.end && (*c.p == ' ' || *c.p == '\t' || *c.p == '\r')) ++c.p;
}

// a JSON string without escapes; returns false on anything else
inline bool parse_key(Cursor& c, const char** s, size_t* n) {
    if (c.p >= c.end || *c.p != '"') return false;
    const char* b = ++c.p;
    while (c.p < c.end && *c.p != '"') {
        if (*c.p == '\\' || (unsigned char)*c.p < 0x20) return false;
        ++c.p;
    }
    if (c.p >= c.end) return false;
    *s = b;
    *n = (size_t)(c.p - b);
    ++c.p;
    return true;
}

enum ValueKind { V_INT, V_FLOAT, V_OTHER, V_BAD };

// one scalar JSON value; numbers as json.loads reads them (int literal -> int, otherwise float(str)); NaN / Infinity /
// -Infinity like json.loads; null / true / false / escape-free strings and (skipped) nested arrays / objects are V_OTHER
inline ValueKind parse_value(Cursor& c, long long* iv, double* dv) {
    if (c.p >= c.end) return V_BAD;
    const char ch = *c.p;
    if (ch == '"') {
        const char* s;
        size_t n;
        return parse_key(c, &s, &n) ? V_OTHER : V_BAD;
    }
    if (ch == '[' || ch == '{') {                   // a nested value of a key we do not read (e.g. "tag": [3, [2]]): skip it
        int depth = 0;
        while (c.p < c.end) {
            const char d = *c.p;
            if (d == '"') {
                const char* s;
                size_t n;
                if (!parse_key(c, &s, &n)) return V_BAD;
                continue;
            }
            if (d == '[' || d == '{') ++depth;
            else if (d == ']' || d == '}') {
                if (--depth == 0) { ++c.p; return V_OTHER; }
            }
            ++c.p;
        }
        return V_BAD;
    }
    auto lit = [&](const char* word) {
        const size_t n = strlen(word);
        if ((size_t)(c.end - c.p) >= n && memcmp(c.p, word, n) == 0) { c.p += n; return true; }
        return false;
    };
    if (ch == 'n') return lit("null") ? V_OTHER : V_BAD;
    if (ch == 't') return lit("true") ? V_OTHER : V_BAD;
    if (ch == 'f') return lit("false") ? V_OTHER : V_BAD;
    if (ch == 'N') { if (lit("NaN")) { *dv = NAN; return V_FLOAT; } return V_BAD; }
    if (ch == 'I') { if (lit("Infinity")) { *dv = INFINITY; return V_FLOAT; } return V_BAD; }
    if (ch == '-' && c.p + 1 < c.end && c.p[1] == 'I') {
        ++c.p;
        if (lit("Infinity")) { *dv = -INFINITY; return V_FLOAT; }
        return V_BAD;
    }
    // JSON number grammar: -? (0 | [1-9][0-9]*) (\.[0-9]+)? ([eE][+-]?[0-9]+)?
    const char* b = c.p;
    const char* q = b;
    if (q < c.end && *q == '-') ++q;
    if (q >= c.end) return V_BAD;
    if (*q == '0') ++q;
    else if (*q >= '1' && *q <= '9') { while (q < c.end && *q >= '0' && *q <= '9') ++q; }
    else return V_BAD;
    bool is_float = false;
    if (q < c.end && *q == '.') {
        ++q;
        if (q >= c.end || *q < '0' || *q > '9') return V_BAD;
        while (q < c.end && *q >= '0' && *q <= '9') ++q;
        is_float = true;
    }
    if (q < c.end && (*q == 'e' || *q == 'E')) {
        ++q;
        if (q < c.end && (*q == '+' || *q == '-')) ++q;
        if (q >= c.end || *q < '0' || *q > '9') return V_BAD;
        while (q < c.end && *q >= '0' && *q <= '9') ++q;
        is_float = true;
    }
    const size_t n = (size_t)(q - b);
    if (n == 0 || n >= 64) return V_BAD;            // longer literals go to the json.loads path
    if (is_float) {
        // Clinger's exact case: a decimal d x 10^-k with d < 2^53 and k <= 22 is ONE correctly rounded division of two
        // exactly representable doubles -- the same double strtod returns.  Covers the "%.2f"-style coordinates of
        // the DATA_BLOCK files; exponents, long mantissas and everything else go through strtod below.
        static const double kPow10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15,
                                          1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
        const char* t = b;
        const bool neg = *t == '-';
        if (neg) ++t;
        unsigned long long mant = 0;
        int digits = 0, frac = 0;
        bool seen_point = false, simple = true;
        for (; t < q; ++t) {
            if (*t == '.') { seen_point = true; continue; }
            if (*t < '0' || *t > '9') { simple = false; break; }          // an exponent part
            if (digits >= 15 && mant != 0) { simple = false; break; }    // keep the mantissa below 10^15 < 2^53
            mant = mant * 10 + (unsigned)(*t - '0');
            if (mant != 0) ++digits;
            if (seen_point) ++frac;
        }
        if (simple && frac <= 22) {
            const double v = (double)mant / kPow10[frac];
            *dv = neg ? -v : v;
            c.p = q;
            return V_FLOAT;
        }
    }
    char tok[64];
    memcpy(tok, b, n);
    tok[n] = 0;
    char* stop = nullptr;
    errno = 0;
    if (is_float) {
        *dv = strtod(tok, &stop);                   // correctly rounded, like float(str)
        if (stop != tok + n) return V_BAD;          // (overflow to inf is what float(str) returns too)
    } else {
        *iv = strtoll(tok, &stop, 10);
        if (stop != tok + n || errno == ERANGE) return V_BAD;      // beyond int64: Python keeps a big int
        *dv = (double)*iv;
    }
    c.p = q;
    return is_float ? V_FLOAT : V_INT;
}

inline bool key_is(const char* s, size_t n, const char* word) { return strlen(word) == n && memcmp(s, word, n) == 0; }

inline int format_uint(char* out, unsigned long long v) {
    char tmp[24];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    for (int i = 0; i < n; ++i) out[i] = tmp[n - 1 - i];
    return n;
}

// Correctly rounded "%.2f", trailing zero stripped to at least one decimal == repr(round(v, 2)) for |v| < 1e15.
inline int format_coord(char* out, double v) {
    if (isnan(v)) { memcpy(out, "NaN", 3); return 3; }
    if (isinf(v)) {
        if (v > 0) { memcpy(out, "Infinity", 8); return 8; }
        memcpy(out, "-Infinity", 9);
        return 9;
    }
    // fast path: c = round(v * 100) proven correct through the exact residual of the product (one fma); anything within
    // 1e-6 of a rounding tie, or large, takes the correctly rounded snprintf
    if (fabs(v) < 1e11) {
        const double c = nearbyint(v * 100.0);
        const double resid = fma(v, 100.0, -c);              // v * 100 - c, exact up to one rounding of a tiny number
        if (fabs(resid) < 0.5 - 1e-6) {
            unsigned long long q = (unsigned long long)fabs(c);
            const unsigned frac = (unsigned)(q % 100);
            q /= 100;
            int n = 0;
            if (signbit(v)) out[n++] = '-';
            n += format_uint(out + n, q);
            out[n++] = '.';
            out[n++] = (char)('0' + frac / 10);
            if (frac % 10) out[n++] = (char)('0' + frac % 10);
            return n;
        }
    }
    int n = snprintf(out, 40, "%.2f", v);
    if (out[n - 1] == '0') --n;
    return n;
}

inline int format_int(char* out, long long v) {
    if (v < 0) {
        out[0] = '-';
        return 1 + format_uint(out + 1, 0ull - (unsigned long long)v);
    }
    return format_uint(out, (unsigned long long)v);
}

inline int put(char* out, const char* lit) {
    const size_t n = strlen(lit);
    memcpy(out, lit, n);
    return (int)n;
}

// "tag" of a scene row as the TrajNet++ categorisation writes it: an integer, or [main, [sub, ...]] with sub-types 0..62
// (returned as bit `sub` of *subs).  Anything else is refused.
bool parse_tag(Cursor& c, long long* main_type, long long* subs) {
    long long iv = 0;
    double dv = 0.0;
    *subs = 0;
    if (c.p < c.end && *c.p != '[') {
        if (parse_value(c, &iv, &dv) != V_INT || iv < 0) return false;
        *main_type = iv;
        return true;
    }
    ++c.p;
    skip_ws(c);
    if (parse_value(c, &iv, &dv) != V_INT || iv < 0) return false;
    *main_type = iv;
    skip_ws(c);
    if (c.p >= c.end || *c.p != ',') return false;
    ++c.p;
    skip_ws(c);
    if (c.p >= c.end || *c.p != '[') return false;
    ++c.p;
    skip_ws(c);
    if (c.p < c.end && *c.p == ']') ++c.p;
    else
        for (;;) {
            skip_ws(c);
            if (parse_value(c, &iv, &dv) != V_INT || iv < 0 || iv > 62) return false;
            *subs |= 1ll << iv;
            skip_ws(c);
            if (c.p < c.end && *c.p == ',') { ++c.p; continue; }
            if (c.p < c.end && *c.p == ']') { ++c.p; break; }
            return false;
        }
    skip_ws(c);
    if (c.p >= c.end || *c.p != ']') return false;
    ++c.p;
    return true;
}

// The parse of tb2_ndjson_parse; with track_pn != nullptr also the metadata columns of tb2_ndjson_parse_meta.
int parse_rows(const char* text, size_t len, int64_t max_rows, int64_t* track_frame, int64_t* track_ped, double* track_x,
               double* track_y, int64_t* track_pn, int64_t* track_sid, int64_t* num_tracks_out, int64_t* scene_id,
               int64_t* scene_ped, int64_t* scene_start, int64_t* scene_end, int64_t* scene_tag, int64_t* scene_subs,
               int64_t* num_scenes_out, int64_t* refused_line_out) {
    const bool meta = track_pn != nullptr;
    int64_t nt = 0, ns = 0, line_no = 0;
    *refused_line_out = -1;
    const char* p = text;
    const char* const end = text + len;
    while (p < end) {
        const char* eol = (const char*)memchr(p, '\n', (size_t)(end - p));
        if (!eol) eol = end;
        Cursor c{p, eol};
        p = eol < end ? eol + 1 : end;
        const int64_t this_line = line_no++;
        skip_ws(c);
        if (c.p == c.end) continue;                                   // blank line
        bool ok = false;
        do {
            if (*c.p != '{') break;
            ++c.p;
            skip_ws(c);
            const char* k;
            size_t kn;
            if (!parse_key(c, &k, &kn)) break;
            const bool is_track = key_is(k, kn, "track"), is_scene = key_is(k, kn, "scene");
            if (!is_track && !is_scene) break;
            skip_ws(c);
            if (c.p >= c.end || *c.p != ':') break;
            ++c.p;
            skip_ws(c);
            if (c.p >= c.end || *c.p != '{') break;
            ++c.p;
            long long f0 = 0, f1 = 0, f2 = 0, f3 = 0;                  // track: f, p | scene: id, p, s, e
            long long m0 = -1, m1 = -1;                                // track: prediction_number, scene_id | scene: tag
            double x = 0.0, y = 0.0;
            unsigned have = 0;
            bool inner_ok = false;
            skip_ws(c);
            if (c.p < c.end && *c.p == '}') { ++c.p; inner_ok = true; }
            else
                for (;;) {
                    skip_ws(c);
                    if (!parse_key(c, &k, &kn)) break;
                    skip_ws(c);
                    if (c.p >= c.end || *c.p != ':') break;
                    ++c.p;
                    skip_ws(c);
                    long long iv = 0;
                    double dv = 0.0;
                    const bool tag = meta && !is_track && key_is(k, kn, "tag");
                    const ValueKind kind = tag ? (parse_tag(c, &m0, &m1) ? V_OTHER : V_BAD) : parse_value(c, &iv, &dv);
                    if (kind == V_BAD) break;
                    bool bad = false;
                    if (is_track) {
                        if (key_is(k, kn, "f")) { if (kind != V_INT) bad = true; f0 = iv; have |= 1; }
                        else if (key_is(k, kn, "p")) { if (kind != V_INT) bad = true; f1 = iv; have |= 2; }
                        else if (key_is(k, kn, "x")) { if (kind == V_OTHER) bad = true; x = dv; have |= 4; }
                        else if (key_is(k, kn, "y")) { if (kind == V_OTHER) bad = true; y = dv; have |= 8; }
                        else if (meta && key_is(k, kn, "prediction_number")) { if (kind != V_INT || iv < 0) bad = true; m0 = iv; }
                        else if (meta && key_is(k, kn, "scene_id")) { if (kind != V_INT || iv < 0) bad = true; m1 = iv; }
                    } else {
                        if (key_is(k, kn, "id")) { if (kind != V_INT) bad = true; f0 = iv; have |= 1; }
                        else if (key_is(k, kn, "p")) { if (kind != V_INT) bad = true; f1 = iv; have |= 2; }
                        else if (key_is(k, kn, "s")) { if (kind != V_INT) bad = true; f2 = iv; have |= 4; }
                        else if (key_is(k, kn, "e")) { if (kind != V_INT) bad = true; f3 = iv; have |= 8; }
                    }
                    if (bad) break;
                    skip_ws(c);
                    if (c.p < c.end && *c.p == ',') { ++c.p; continue; }
                    if (c.p < c.end && *c.p == '}') { ++c.p; inner_ok = true; }
                    break;
                }
            if (!inner_ok || have != 15) break;                       // a missing field raises in the Python path: let it
            skip_ws(c);
            if (c.p >= c.end || *c.p != '}') break;                    // a second top-level key: not ours to interpret
            ++c.p;
            skip_ws(c);
            if (c.p != c.end) break;
            if (is_track) {
                if (nt >= max_rows) break;
                track_frame[nt] = f0; track_ped[nt] = f1; track_x[nt] = x; track_y[nt] = y;
                if (meta) { track_pn[nt] = m0; track_sid[nt] = m1; }
                ++nt;
            } else {
                if (ns >= max_rows) break;
                scene_id[ns] = f0; scene_ped[ns] = f1; scene_start[ns] = f2; scene_end[ns] = f3;
                if (meta) { scene_tag[ns] = m0; scene_subs[ns] = m0 < 0 ? 0 : m1; }
                ++ns;
            }
            ok = true;
        } while (0);
        if (!ok) {
            *refused_line_out = this_line;
            break;
        }
    }
    *num_tracks_out = nt;
    *num_scenes_out = ns;
    return TB2_OK;
}

}  // namespace
}  // namespace tb2

using namespace tb2;

extern "C" {

int tb2_ndjson_parse(const char* text, size_t len, int64_t max_rows, int64_t* track_frame, int64_t* track_ped, double* track_x,
                     double* track_y, int64_t* num_tracks_out, int64_t* scene_id, int64_t* scene_ped, int64_t* scene_start,
                     int64_t* scene_end, int64_t* num_scenes_out, int64_t* refused_line_out) {
    TB2_REQUIRE(text || len == 0, "null text");
    TB2_REQUIRE(track_frame && track_ped && track_x && track_y && num_tracks_out && scene_id && scene_ped && scene_start &&
                    scene_end && num_scenes_out && refused_line_out,
                "null argument");
    return parse_rows(text, len, max_rows, track_frame, track_ped, track_x, track_y, nullptr, nullptr, num_tracks_out, scene_id,
                      scene_ped, scene_start, scene_end, nullptr, nullptr, num_scenes_out, refused_line_out);
}

int tb2_ndjson_parse_meta(const char* text, size_t len, int64_t max_rows, int64_t* track_frame, int64_t* track_ped,
                          double* track_x, double* track_y, int64_t* track_prediction_number, int64_t* track_scene_id,
                          int64_t* num_tracks_out, int64_t* scene_id, int64_t* scene_ped, int64_t* scene_start,
                          int64_t* scene_end, int64_t* scene_tag, int64_t* scene_sub_tags, int64_t* num_scenes_out,
                          int64_t* refused_line_out) {
    TB2_REQUIRE(text || len == 0, "null text");
    TB2_REQUIRE(track_frame && track_ped && track_x && track_y && track_prediction_number && track_scene_id && num_tracks_out &&
                    scene_id && scene_ped && scene_start && scene_end && scene_tag && scene_sub_tags && num_scenes_out &&
                    refused_line_out,
                "null argument");
    return parse_rows(text, len, max_rows, track_frame, track_ped, track_x, track_y, track_prediction_number, track_scene_id,
                      num_tracks_out, scene_id, scene_ped, scene_start, scene_end, scene_tag, scene_sub_tags, num_scenes_out,
                      refused_line_out);
}

// Text of the prediction records of `num_scenes` scenes, each = one scene line followed by its rows_per_scene[i] track
// lines (the caller lays the rows out in the writer's order).  Returns the number of bytes needed; writes only if
// capacity suffices (call once with capacity 0 to size the buffer, or pass an upper bound: 160 bytes per line).
int64_t tb2_ndjson_format(int64_t num_scenes, const int64_t* scene_id, const int64_t* scene_ped, const int64_t* scene_start,
                          const int64_t* scene_end, const int64_t* rows_per_scene, const int64_t* row_frame,
                          const int64_t* row_ped, const double* row_x, const double* row_y, const int64_t* row_mode, char* out,
                          int64_t capacity) {
    if (num_scenes < 0 || (num_scenes > 0 && !(scene_id && scene_ped && scene_start && scene_end && rows_per_scene))) {
        set_error("invalid argument: tb2_ndjson_format");
        return TB2_ERR_INVALID;
    }
    int64_t total_rows = 0;
    for (int64_t s = 0; s < num_scenes; ++s) total_rows += rows_per_scene[s];
    if (total_rows > 0 && !(row_frame && row_ped && row_x && row_y && row_mode)) {
        set_error("invalid argument: tb2_ndjson_format rows");
        return TB2_ERR_INVALID;
    }
    for (int64_t i = 0; i < total_rows; ++i)
        if (fabs(row_x[i]) >= 1e15 || fabs(row_y[i]) >= 1e15) {      // finite and huge: repr() switches to exponents at 1e16
            if (isinf(row_x[i]) || isinf(row_y[i])) continue;
            set_error("unsupported: coordinate magnitude >= 1e15 (use the json.dumps writer)");
            return TB2_ERR_UNSUPPORTED;
        }
    int64_t used = 0, r = 0;
    char line[320];
    for (int64_t s = 0; s < num_scenes; ++s) {
        int n = put(line, "{\"scene\": {\"id\": ");
        n += format_int(line + n, scene_id[s]);
        n += put(line + n, ", \"p\": ");
        n += format_int(line + n, scene_ped[s]);
        n += put(line + n, ", \"s\": ");
        n += format_int(line + n, scene_start[s]);
        n += put(line + n, ", \"e\": ");
        n += format_int(line + n, scene_end[s]);
        n += put(line + n, ", \"fps\": 2.5, \"tag\": 0}}\n");
        if (out && used + n <= capacity) memcpy(out + used, line, (size_t)n);
        used += n;
        for (int64_t k = 0; k < rows_per_scene[s]; ++k, ++r) {
            n = put(line, "{\"track\": {\"f\": ");
            n += format_int(line + n, row_frame[r]);
            n += put(line + n, ", \"p\": ");
            n += format_int(line + n, row_ped[r]);
            n += put(line + n, ", \"x\": ");
            n += format_coord(line + n, row_x[r]);
            n += put(line + n, ", \"y\": ");
            n += format_coord(line + n, row_y[r]);
            n += put(line + n, ", \"prediction_number\": ");
            n += format_int(line + n, row_mode[r]);
            n += put(line + n, ", \"scene_id\": ");
            n += format_int(line + n, scene_id[s]);
            n += put(line + n, "}}\n");
            if (out && used + n <= capacity) memcpy(out + used, line, (size_t)n);
            used += n;
        }
    }
    return used;
}

}  // extern "C"
