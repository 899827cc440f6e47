// inspect.hpp — `sylph-b200 inspect`: what a .syldb / .sylsp holds, as the YAML of sylph's `inspect`
// (src/inspect.rs).  The files are read field by field and the k-mer arrays are stepped over, so a
// database of many gigabytes is inspected in constant memory.
//
// The YAML restates what serde_yaml 0.9.34 (over unsafe-libyaml 0.2.11, floats by ryu 1.0.18) writes
// for these structs: block style without `---`, keys of a list item at two spaces, a nested list at
// its key's indentation, `[]` for an empty list, `true`/`false`/`null`, shortest round-trip floats in
// ryu's layout, and strings plain unless they would read back as another scalar or libyaml cannot
// write them plain.  One deviation: a string holding a line break (LF, U+2028, U+2029) is written
// double-quoted, where serde_yaml writes a literal block or a single-quoted scalar over several lines.
#pragma once
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "sketch_io.hpp"

namespace host {
namespace yaml {

// ---- which strings serde_yaml quotes because they would resolve to another type (serde_yaml src/de.rs) ----

// "0" followed by digits, after one optional sign: a string in YAML 1.2, quoted so that it stays one
inline bool digits_but_not_number(const std::string &s) {
    const std::string t = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? s.substr(1) : s;
    if (t.size() < 2 || t[0] != '0') return false;
    for (size_t i = 1; i < t.size(); i++) if (t[i] < '0' || t[i] > '9') return false;
    return true;
}

// Rust's from_str_radix on a digit string without its sign: every character a digit of `radix`, magnitude <= limit
inline bool digits_within(const std::string &d, unsigned radix, unsigned __int128 limit) {
    if (d.empty()) return false;
    unsigned __int128 v = 0;
    for (char ch : d) {
        unsigned x = ch >= '0' && ch <= '9' ? ch - '0' : ch >= 'a' && ch <= 'z' ? ch - 'a' + 10 : ch >= 'A' && ch <= 'Z' ? ch - 'A' + 10 : 99;
        if (x >= radix || v > (limit - x) / radix) return false;
        v = v * radix + x;
    }
    return true;
}

inline bool starts_with(const std::string &s, const char *p) { return s.compare(0, strlen(p), p) == 0; }
inline bool signed_start(const std::string &s) { return !s.empty() && (s[0] == '+' || s[0] == '-'); }

// parse_unsigned_int / parse_negative_int over u128 / i128 (the widest types serde_yaml tries)
inline bool is_int(const std::string &s) {
    const unsigned __int128 umax = ~(unsigned __int128)0, imin = (unsigned __int128)1 << 127;
    static const std::pair<const char *, unsigned> radix[] = {{"0x", 16}, {"0o", 8}, {"0b", 2}};
    const std::string u = s.compare(0, 1, "+") == 0 ? s.substr(1) : s;
    bool unsigned_ok = false, done = false;
    for (const auto &[p, r] : radix) {
        if (done || !starts_with(u, p)) continue;
        const std::string rest = u.substr(2);
        if (signed_start(rest)) { done = true; break; }
        if (digits_within(rest, r, umax)) { unsigned_ok = true; done = true; }
    }
    if (!done && !signed_start(u) && !digits_but_not_number(s)) unsigned_ok = digits_within(u, 10, umax);
    if (unsigned_ok) return true;
    for (const auto &[p, r] : radix) {
        const std::string np = std::string("-") + p;
        if (starts_with(s, np.c_str())) {
            const std::string rest = s.substr(3);
            if (!signed_start(rest) && digits_within(rest, r, imin)) return true;
        }
    }
    if (digits_but_not_number(s)) return false;
    if (s.empty()) return false;
    if (s[0] == '-') return digits_within(s.substr(1), 10, imin);
    if (s[0] == '+') return digits_within(s.substr(1), 10, imin - 1);
    return digits_within(s, 10, imin - 1);
}

// parse_f64: the YAML infinities and NaN, or Rust's f64 grammar ([+-]? digits with one optional '.', optional
// exponent) whose value is finite
inline bool is_float(const std::string &s) {
    std::string u = s;
    if (!s.empty() && s[0] == '+') {
        u = s.substr(1);
        if (signed_start(u)) return false;
    }
    if (u == ".inf" || u == ".Inf" || u == ".INF") return true;
    if (s == "-.inf" || s == "-.Inf" || s == "-.INF") return true;
    if (s == ".nan" || s == ".NaN" || s == ".NAN") return true;
    size_t i = signed_start(u) ? 1 : 0, digits = 0;
    while (i < u.size() && isdigit((unsigned char)u[i])) { i++; digits++; }
    if (i < u.size() && u[i] == '.') {
        i++;
        while (i < u.size() && isdigit((unsigned char)u[i])) { i++; digits++; }
    }
    if (!digits) return false;
    if (i < u.size() && (u[i] == 'e' || u[i] == 'E')) {
        i++;
        if (i < u.size() && (u[i] == '+' || u[i] == '-')) i++;
        size_t e = 0;
        while (i < u.size() && isdigit((unsigned char)u[i])) { i++; e++; }
        if (!e) return false;
    }
    if (i != u.size()) return false;
    return std::isfinite(strtod(u.c_str(), nullptr));
}

inline bool resolves_to_non_string(const std::string &s) {
    if (s.empty() || s == "null" || s == "Null" || s == "NULL" || s == "~") return true;
    if (s == "true" || s == "True" || s == "TRUE" || s == "false" || s == "False" || s == "FALSE") return true;
    return is_int(s) || digits_but_not_number(s) || is_float(s);
}

// ---- libyaml's scalar analysis (yaml_emitter_analyze_scalar) on UTF-8 bytes; past the end reads as NUL ----

struct Bytes {
    const std::string &s;
    unsigned char at(size_t i) const { return i < s.size() ? (unsigned char)s[i] : 0; }
    size_t width(size_t i) const {
        const unsigned char b = at(i);
        return (b & 0x80) == 0 ? 1 : (b & 0xE0) == 0xC0 ? 2 : (b & 0xF0) == 0xE0 ? 3 : (b & 0xF8) == 0xF0 ? 4 : 1;
    }
    bool is_break(size_t i) const {
        return at(i) == '\r' || at(i) == '\n' || (at(i) == 0xC2 && at(i + 1) == 0x85) ||
               (at(i) == 0xE2 && at(i + 1) == 0x80 && (at(i + 2) == 0xA8 || at(i + 2) == 0xA9));
    }
    bool is_blankz(size_t i) const { return at(i) == ' ' || at(i) == '\t' || is_break(i) || at(i) == 0; }
    bool is_printable(size_t i) const {
        const unsigned char b = at(i), n = at(i + 1), n2 = at(i + 2);
        return b == 0x0A || (b >= 0x20 && b <= 0x7E) || (b == 0xC2 && n >= 0xA0) || (b > 0xC2 && b < 0xED) ||
               (b == 0xED && n < 0xA0) || b == 0xEE ||
               (b == 0xEF && !(n == 0xBB && n2 == 0xBF) && !(n == 0xBF && (n2 == 0xBE || n2 == 0xBF)));
    }
};

struct Analysis { bool line_breaks = false, plain = true, single = true; };

inline Analysis analyze(const std::string &s) {
    Analysis a;
    const Bytes b{s};
    if (s.empty()) { a.single = true; return a; }
    bool block_ind = false, special = false, leading_space = false, leading_break = false, trailing_space = false,
         trailing_break = false, break_space = false, space_break = false, prev_space = false, prev_break = false;
    if (s.compare(0, 3, "---") == 0 || s.compare(0, 3, "...") == 0) block_ind = true;
    bool preceded_ws = true, followed_ws = b.is_blankz(b.width(0));
    for (size_t i = 0; i < s.size();) {
        const unsigned char c = b.at(i);
        const size_t w = b.width(i);
        if (i == 0) {
            if (strchr("#,[]{}&*!|>'\"%@`", c) && c) block_ind = true;
            if ((c == '?' || c == ':') && followed_ws) block_ind = true;
            if (c == '-' && followed_ws) block_ind = true;
        } else {
            if (c == ':' && followed_ws) block_ind = true;
            if (c == '#' && preceded_ws) block_ind = true;
        }
        if (!b.is_printable(i)) special = true;  // emitter->unicode is set: non-ASCII printables stay as they are
        if (b.is_break(i)) a.line_breaks = true;
        if (c == ' ') {
            if (i == 0) leading_space = true;
            if (i + w == s.size()) trailing_space = true;
            if (prev_break) break_space = true;
            prev_space = true; prev_break = false;
        } else if (b.is_break(i)) {
            if (i == 0) leading_break = true;
            if (i + w == s.size()) trailing_break = true;
            if (prev_space) space_break = true;
            prev_space = false; prev_break = true;
        } else {
            prev_space = prev_break = false;
        }
        preceded_ws = b.is_blankz(i);
        i += w;
        if (i < s.size()) followed_ws = b.is_blankz(i + b.width(i));
    }
    if (leading_space || leading_break || trailing_space || trailing_break) a.plain = false;
    if (break_space) a.plain = a.single = false;
    if (space_break || special) a.plain = a.single = false;
    if (a.line_breaks || block_ind) a.plain = false;
    return a;
}

inline std::string hex(unsigned v, int digits) {
    static const char *x = "0123456789ABCDEF";
    std::string o(digits, '0');
    for (int i = digits - 1; i >= 0; i--, v >>= 4) o[i] = x[v & 15];
    return o;
}

// yaml_emitter_write_double_quoted without line folding (serde_yaml sets the width to unlimited)
inline std::string double_quoted(const std::string &s) {
    const Bytes b{s};
    std::string o = "\"";
    for (size_t i = 0; i < s.size();) {
        const size_t w = b.width(i);
        const bool bom = b.at(i) == 0xEF && b.at(i + 1) == 0xBB && b.at(i + 2) == 0xBF;
        const unsigned char c = b.at(i);
        if (!b.is_printable(i) || bom || b.is_break(i) || c == '"' || c == '\\') {
            unsigned v = w == 1 ? c & 0x7F : w == 2 ? c & 0x1F : w == 3 ? c & 0x0F : c & 0x07;
            for (size_t k = 1; k < w; k++) v = (v << 6) + (b.at(i + k) & 0x3F);
            o += '\\';
            switch (v) {
                case 0x00: o += '0'; break;
                case 0x07: o += 'a'; break;
                case 0x08: o += 'b'; break;
                case 0x09: o += 't'; break;
                case 0x0A: o += 'n'; break;
                case 0x0B: o += 'v'; break;
                case 0x0C: o += 'f'; break;
                case 0x0D: o += 'r'; break;
                case 0x1B: o += 'e'; break;
                case 0x22: o += '"'; break;
                case 0x5C: o += '\\'; break;
                case 0x85: o += 'N'; break;
                case 0xA0: o += '_'; break;
                case 0x2028: o += 'L'; break;
                case 0x2029: o += 'P'; break;
                default: o += v <= 0xFF ? "x" + hex(v, 2) : v <= 0xFFFF ? "u" + hex(v, 4) : "U" + hex(v, 8);
            }
        } else {
            o.append(s, i, w);
        }
        i += w;
    }
    return o + "\"";
}

// a string value: serde_yaml picks single quotes for strings that resolve to another scalar, libyaml falls back
// from plain to single to double quotes as its analysis allows
inline std::string str(const std::string &s) {
    const Analysis a = analyze(s);
    if (a.line_breaks) return double_quoted(s);
    const bool want_single = resolves_to_non_string(s);
    if (!want_single && a.plain) return s;
    if (!a.single) return double_quoted(s);
    std::string o = "'";
    for (char c : s) { if (c == '\'') o += '\''; o += c; }
    return o + "'";
}

// ryu's layout of the shortest round-trip digits (std::to_chars finds them): plain decimal while the decimal point
// falls within `max_kk` digits, "0.000ddd" down to `min_kk` + 1, otherwise d.ddde<exp>; NaN and infinities as YAML
template <typename T>
inline std::string ryu(T v, int max_kk, int min_kk) {
    if (std::isnan(v)) return ".nan";
    if (std::isinf(v)) return v > 0 ? ".inf" : "-.inf";
    std::string out = std::signbit(v) ? "-" : "";
    if (v == 0) return out + "0.0";
    char buf[64];
    const std::to_chars_result r = std::to_chars(buf, buf + sizeof buf, std::fabs(v), std::chars_format::scientific);
    const std::string sci(buf, r.ptr);
    const size_t e = sci.find('e');
    std::string m = sci.substr(0, e);
    if (m.size() > 1) m.erase(1, 1);  // "d.ddd" -> "dddd"
    const int len = (int)m.size(), kk = std::stoi(sci.substr(e + 1)) + 1, k = kk - len;
    if (0 <= k && kk <= max_kk) return out + m + std::string(k, '0') + ".0";
    if (0 < kk && kk <= max_kk) return out + m.substr(0, kk) + "." + m.substr(kk);
    if (min_kk < kk && kk <= 0) return out + "0." + std::string(-kk, '0') + m;
    const std::string exp = "e" + std::to_string(kk - 1);
    if (len == 1) return out + m + exp;
    return out + m.substr(0, 1) + "." + m.substr(1) + exp;
}
inline std::string f32(float v) { return ryu(v, 13, -6); }
inline std::string f64(double v) { return ryu(v, 16, -5); }

}  // namespace yaml

// bincode rejects a String that is not UTF-8 (RFC 3629: no overlongs, surrogates or code points past U+10FFFF)
inline bool valid_utf8(const std::string &s) {
    for (size_t i = 0; i < s.size();) {
        const unsigned char c = s[i];
        const size_t n = c < 0x80 ? 0 : (c >> 5) == 6 ? 1 : (c >> 4) == 14 ? 2 : (c >> 3) == 30 ? 3 : 9;  // continuation bytes
        if (n == 9 || i + n >= s.size()) return false;
        uint32_t cp = n == 0 ? c : n == 1 ? c & 0x1F : n == 2 ? c & 0x0F : c & 0x07;
        for (size_t k = 1; k <= n; k++) {
            const unsigned char d = s[i + k];
            if ((d & 0xC0) != 0x80) return false;
            cp = (cp << 6) | (d & 0x3F);
        }
        if ((n == 1 && cp < 0x80) || (n == 2 && cp < 0x800) || (n == 3 && cp < 0x10000) || cp > 0x10FFFF ||
            (cp >= 0xD800 && cp <= 0xDFFF))
            return false;
        i += n + 1;
    }
    return true;
}

// ---- the summaries (src/inspect.rs:19-76) ----

struct GenomeInspect { std::string file_name, first_contig_name; uint64_t genome_kmers_num = 0, genome_size = 0; };
struct DatabaseInspect {  // a database without genomes is all defaults
    std::string database_file;
    uint64_t c = 0, k = 0, min_spacing_parameter = 0;  // of the first genome
    std::vector<GenomeInspect> genome_files;
};
struct SampleInspect {
    std::string file_name;
    uint64_t c = 0, k = 0, num_sketched_kmers = 0;
    float approximate_number_bases = 0.f;
    double mean_read_length = 0.;
    bool has_sample_name = false;
    std::string sample_name;
    bool paired = false;
};

inline std::string read_utf8(Reader &r) {
    std::string s = r.str();
    if (!valid_utf8(s)) r.bad();
    return s;
}
inline bool read_bool(Reader &r) {  // bincode: a bool or an Option tag is one byte, 0 or 1
    const uint8_t v = r.u8();
    if (v > 1) r.bad();
    return v == 1;
}
inline std::runtime_error invalid_sketch(const char *kind, const std::string &path) {
    return std::runtime_error(std::string("The ") + kind + " sketch `" + path +
                              "` is not a valid sketch. Perhaps it is an older, incompatible version ");
}

// -> false for a database without genomes
inline bool inspect_db(const std::string &path, DatabaseInspect &out) {
    Reader r(path);  // throws "The sketch `path` could not be opened. Exiting"
    out = DatabaseInspect();
    out.database_file = path;
    try {
        const uint64_t n = r.len();
        for (uint64_t i = 0; i < n; i++) {
            GenomeInspect g;
            g.genome_kmers_num = r.len();
            r.skip(g.genome_kmers_num * 8);
            if (read_bool(r)) r.skip(r.len() * 8);  // tracked k-mers
            g.file_name = read_utf8(r);
            g.first_contig_name = read_utf8(r);
            const uint64_t c = r.u64(), k = r.u64();
            g.genome_size = r.u64();
            const uint64_t ms = r.u64();
            if (i == 0) { out.c = c; out.k = k; out.min_spacing_parameter = ms; }
            out.genome_files.push_back(std::move(g));
        }
    } catch (const std::exception &) { throw invalid_sketch("database", path); }
    if (out.genome_files.empty()) out = DatabaseInspect();
    return !out.genome_files.empty();
}

inline SampleInspect inspect_sample(const std::string &path) {
    Reader r(path);
    SampleInspect s;
    try {
        s.num_sketched_kmers = r.len();
        r.skip(s.num_sketched_kmers * 12);  // (u64 hash, u32 count) entries
        s.c = r.u64();
        s.k = r.u64();
        s.file_name = read_utf8(r);
        s.has_sample_name = read_bool(r);
        if (s.has_sample_name) s.sample_name = read_utf8(r);
        s.paired = read_bool(r);
        s.mean_read_length = r.f64();
    } catch (const std::exception &) { throw invalid_sketch("sequence", path); }
    // f32 arithmetic in the reference's order (src/inspect.rs:40)
    s.approximate_number_bases = (float)(s.mean_read_length + (double)s.k - 1.) / (float)s.mean_read_length * (float)s.c *
                                 (float)s.num_sketched_kmers;
    return s;
}

inline std::string databases_yaml(const std::vector<DatabaseInspect> &dbs) {
    std::string o;
    for (const DatabaseInspect &d : dbs) {
        o += "- database_file: " + yaml::str(d.database_file) + "\n";
        o += "  c: " + std::to_string(d.c) + "\n";
        o += "  k: " + std::to_string(d.k) + "\n";
        o += "  min_spacing_parameter: " + std::to_string(d.min_spacing_parameter) + "\n";
        o += d.genome_files.empty() ? "  genome_files: []\n" : "  genome_files:\n";
        for (const GenomeInspect &g : d.genome_files) {
            o += "  - file_name: " + yaml::str(g.file_name) + "\n";
            o += "    genome_kmers_num: " + std::to_string(g.genome_kmers_num) + "\n";
            o += "    first_contig_name: " + yaml::str(g.first_contig_name) + "\n";
            o += "    genome_size: " + std::to_string(g.genome_size) + "\n";
        }
    }
    return o;
}

inline std::string samples_yaml(const std::vector<SampleInspect> &ss) {
    std::string o;
    for (const SampleInspect &s : ss) {
        o += "- file_name: " + yaml::str(s.file_name) + "\n";
        o += "  c: " + std::to_string(s.c) + "\n";
        o += "  k: " + std::to_string(s.k) + "\n";
        o += "  num_sketched_kmers: " + std::to_string(s.num_sketched_kmers) + "\n";
        o += "  approximate_number_bases: " + yaml::f32(s.approximate_number_bases) + "\n";
        o += "  mean_read_length: " + yaml::f64(s.mean_read_length) + "\n";
        o += "  sample_name: " + (s.has_sample_name ? yaml::str(s.sample_name) : std::string("null")) + "\n";
        o += std::string("  paired: ") + (s.paired ? "true" : "false") + "\n";
    }
    return o;
}

}  // namespace host
