// sketch_io.hpp — sylph's on-disk sketches (.syldb / .sylsp): bincode 1.3 default configuration
// (little-endian fixed-width ints, u64 length prefixes, usize as u64, Option = 1 tag byte,
// bool = 1 byte) of the structs in src/types.rs:145-173; writers src/sketch.rs:411,474,
// loaders src/contain.rs:492-499,554-561.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace host {

struct GenomeSketch {              // src/types.rs:163-173 (field order = serialisation order)
    std::vector<uint64_t> genome_kmers;
    bool has_tracked = false;      // Option<Vec<Kmer>>
    std::vector<uint64_t> tracked;
    std::string file_name, first_contig_name;
    uint64_t c = 200, k = 31, gn_size = 0, min_spacing = 30;
};

struct SequencesSketch {           // src/types.rs:145-155
    std::vector<uint64_t> hashes;  // kmer_counts serialised as a sequence of (u64, u32)
    std::vector<uint32_t> counts;
    uint64_t c = 200, k = 31;
    std::string file_name;
    bool has_sample_name = false;
    std::string sample_name;
    bool paired = false;
    double mean_read_length = 0.;
};

class Writer {
  public:
    explicit Writer(const std::string &path) : f_(fopen(path.c_str(), "wb")) {
        if (!f_) throw std::runtime_error(path + " path not valid; exiting.");
    }
    ~Writer() { if (f_) fclose(f_); }
    void u8(uint8_t v) { raw(&v, 1); }
    void u32(uint32_t v) { raw(&v, 4); }
    void u64(uint64_t v) { raw(&v, 8); }
    void f64(double v) { raw(&v, 8); }
    void str(const std::string &s) { u64(s.size()); raw(s.data(), s.size()); }
    void vec64(const std::vector<uint64_t> &v) { u64(v.size()); raw(v.data(), v.size() * 8); }
    void raw(const void *p, size_t n) { if (n && fwrite(p, 1, n, f_) != n) throw std::runtime_error("write failed"); }
  private:
    FILE *f_;
};

class Reader {
  public:
    explicit Reader(const std::string &path) : path_(path), f_(fopen(path.c_str(), "rb")) {
        if (!f_) throw std::runtime_error("The sketch `" + path + "` could not be opened. Exiting");
        setvbuf(f_, nullptr, _IOFBF, 10000000);
    }
    ~Reader() { if (f_) fclose(f_); }
    uint8_t u8() { uint8_t v; raw(&v, 1); return v; }
    uint32_t u32() { uint32_t v; raw(&v, 4); return v; }
    uint64_t u64() { uint64_t v; raw(&v, 8); return v; }
    double f64() { double v; raw(&v, 8); return v; }
    std::string str() { uint64_t n = len(); std::string s(n, '\0'); raw(&s[0], n); return s; }
    std::vector<uint64_t> vec64() { uint64_t n = len(); std::vector<uint64_t> v(n); raw(v.data(), n * 8); return v; }
    uint64_t len() {
        uint64_t n = u64();
        if (n > (1ull << 40)) bad();
        return n;
    }
    void raw(void *p, size_t n) { if (n && fread(p, 1, n, f_) != n) bad(); }
    // step over n bytes without reading them (k-mer arrays of a GTDB-scale .syldb run to gigabytes); the last byte is
    // read, so a file that ends inside the skipped range is invalid rather than silently short
    void skip(uint64_t n) {
        if (!n) return;
        if (n > (uint64_t)INT64_MAX || fseeko(f_, (off_t)(n - 1), SEEK_CUR) != 0) bad();
        uint8_t last;
        raw(&last, 1);
    }
    [[noreturn]] void bad() {
        throw std::runtime_error("The sketch `" + path_ + "` is not a valid sketch. Perhaps it is an older, incompatible version ");
    }
  private:
    std::string path_;
    FILE *f_;
};

inline void write_syldb(const std::string &path, const std::vector<GenomeSketch> &gs) {
    Writer w(path);
    w.u64(gs.size());
    for (const GenomeSketch &g : gs) {
        w.vec64(g.genome_kmers);
        w.u8(g.has_tracked ? 1 : 0);
        if (g.has_tracked) w.vec64(g.tracked);
        w.str(g.file_name);
        w.str(g.first_contig_name);
        w.u64(g.c); w.u64(g.k); w.u64(g.gn_size); w.u64(g.min_spacing);
    }
}

inline std::vector<GenomeSketch> read_syldb(const std::string &path) {
    Reader r(path);
    uint64_t n = r.len();
    std::vector<GenomeSketch> gs(n);
    for (GenomeSketch &g : gs) {
        g.genome_kmers = r.vec64();
        uint8_t tag = r.u8();
        if (tag > 1) r.bad();
        g.has_tracked = tag == 1;
        if (g.has_tracked) g.tracked = r.vec64();
        g.file_name = r.str();
        g.first_contig_name = r.str();
        g.c = r.u64(); g.k = r.u64(); g.gn_size = r.u64(); g.min_spacing = r.u64();
    }
    return gs;
}

inline void write_sylsp(const std::string &path, const SequencesSketch &s) {
    Writer w(path);
    w.u64(s.hashes.size());
    for (size_t i = 0; i < s.hashes.size(); i++) { w.u64(s.hashes[i]); w.u32(s.counts[i]); }
    w.u64(s.c); w.u64(s.k);
    w.str(s.file_name);
    w.u8(s.has_sample_name ? 1 : 0);
    if (s.has_sample_name) w.str(s.sample_name);
    w.u8(s.paired ? 1 : 0);
    w.f64(s.mean_read_length);
}

inline SequencesSketch read_sylsp(const std::string &path) {
    Reader r(path);
    SequencesSketch s;
    uint64_t n = r.len();
    s.hashes.resize(n); s.counts.resize(n);
    for (uint64_t i = 0; i < n; i++) { s.hashes[i] = r.u64(); s.counts[i] = r.u32(); }
    s.c = r.u64(); s.k = r.u64();
    s.file_name = r.str();
    uint8_t tag = r.u8();
    if (tag > 1) r.bad();
    s.has_sample_name = tag == 1;
    if (s.has_sample_name) s.sample_name = r.str();
    s.paired = r.u8() != 0;
    s.mean_read_length = r.f64();
    return s;
}

}  // namespace host
