// sylph-b200 — host driver over libsylph_b200.so mirroring sylph's `sketch`, `query`, `profile`, `inspect`
// (src/main.rs:25-30) for the in-scope paths: single-end reads, read pairs with the exact dedup set
// (-1/-2 --fpr 0) and genomes, k in {21,31}, with sample names (-S / --lS) and list inputs (-l --rl --gl --l1 --l2).
// Files are inflated and parsed by up to -t threads at a time (the reference parallelises per file with rayon,
// src/sketch.rs:313,371,428) while the GPU works.
// File classification, defaults and TSV output follow the reference (src/cmdline.rs,
// src/sketch.rs:95-127,276-479, src/contain.rs:18-94,115-351,461-480).  All compute goes through
// the C ABI; there is no CPU path.  --devices runs one context per listed device, each on its own worker thread.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <filesystem>
#include <future>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include <unistd.h>

#include "../include/sylph_b200.h"
#include "fastx.hpp"
#include "inspect.hpp"
#include "sketch_io.hpp"

using namespace host;

static void info(const std::string &m) { fprintf(stderr, "INFO  [sylph-b200] %s\n", m.c_str()); }
static void warn(const std::string &m) { fprintf(stderr, "WARN  [sylph-b200] %s\n", m.c_str()); }
// die() exits at once and is only called on the main thread; code that may run on a worker thread throws instead
// (fail, check), and main() prints the message and exits after every worker has stopped.
[[noreturn]] static void die(const std::string &m) { fprintf(stderr, "ERROR [sylph-b200] %s\n", m.c_str()); exit(1); }
[[noreturn]] static void fail(const std::string &m) { throw std::runtime_error(m); }
static void check(int rc, const char *what) {
    if (rc != SYL_OK) fail(std::string(what) + ": " + syl_last_error());
}
static bool ends_with(const std::string &s, const std::string &suf) {
    return s.size() >= suf.size() && s.compare(s.size() - suf.size(), suf.size(), suf) == 0;
}
// src/sketch.rs:95-121
static bool is_fastq(const std::string &f) {
    for (const char *e : {".fq", ".fnq", ".fastq", ".fq.gz", ".fnq.gz", ".fastq.gz"}) if (ends_with(f, e)) return true;
    return false;
}
static bool is_fasta(const std::string &f) {
    for (const char *e : {".fa", ".fna", ".fasta", ".fa.gz", ".fna.gz", ".fasta.gz"}) if (ends_with(f, e)) return true;
    return false;
}
static bool is_syldb(const std::string &f) { return ends_with(f, ".syldb") || ends_with(f, ".sylqueries"); }  // src/constants.rs:6-9
static bool is_sylsp(const std::string &f) { return ends_with(f, ".sylsp") || ends_with(f, ".sylsample"); }
static std::string basename_of(const std::string &p) {
    size_t i = p.find_last_of('/');
    return i == std::string::npos ? p : p.substr(i + 1);
}

// a single-end read file of `sketch` and the index of its sample name (-S / --lS), if any
struct ReadInput { std::string file; size_t name; };

struct Args {
    std::string cmd;
    std::vector<std::string> files, reads, genomes, first_pairs, second_pairs;
    size_t n_positional = 0;  // files[0, n_positional) are positional, the rest are lines of -l
    std::string read_list, genome_list, first_pair_list, second_pair_list, names_list;  // --rl --gl --l1 --l2 --lS
    std::vector<std::string> sample_names;  // -S, or the lines of --lS
    std::vector<ReadInput> sketch_reads;    // sketch: every single-end read file, in the order they are sketched
    std::vector<std::string> sketch_genomes;
    bool estimate_unknown = false;
    double read_seq_id = -1.;  // -I / --read-seq-id (percent)
    int threads = 3;       // src/cmdline.rs:61,100
    double fpr = 0.0001;   // src/constants.rs:16 (paired-end dedup; only 0 = the exact set is supported)
    uint64_t k = 31, c = 200, min_spacing = 30;
    bool individual = false, no_dedup = false, no_pseudotax = false, no_ci = false, no_adj = false, mean_cov = false;
    std::string db_out = "database", sample_dir = "./", out_file, list_file;
    double min_ani = -1., min_number_kmers = 50., min_count_correct = 3., redundant_ani = 99.;
    int device = 0;
    bool device_given = false;
    std::vector<int> devices;  // --devices: one context per entry (a device may repeat); empty = {device}
    // test hooks (INTEGRATION.md), read once from the environment: small values make the split paths run on small inputs
    uint64_t batch_bases = 1ull << 30;  // SYL_DRIVER_BATCH_BASES: a genome batch closes once it holds this many bases
    uint64_t samples_per_call = 0;      // SYL_DRIVER_SAMPLES_PER_CALL: cap on samples per host batch of query / profile (0 = none)
    uint64_t rows0 = 0;                 // SYL_DRIVER_ROWS: initial row-buffer length (0 = sized from the call)
    uint64_t shard_entries = 0;         // SYL_DRIVER_SHARD_ENTRIES: query / profile through db shards of this many entries
    uint64_t max_db_entries = 0;        // --max-db-entries: the same, as an option
    uint64_t max_sample_bytes = 0;      // --max-sample-bytes: host bytes of one batch of query / profile samples (0 = default)
};

static uint64_t env_u64(const char *name, uint64_t dflt) {
    const char *v = getenv(name);
    if (!v || !*v) return dflt;
    return std::max<uint64_t>(1, std::strtoull(v, nullptr, 10));
}

// the lines of a list file as BufRead::lines splits them ("\n", a trailing "\r" dropped)
static void read_list(const std::string &path, std::vector<std::string> &out, bool skip_empty) {
    LineReader lr(path);
    if (!lr.ok()) die("cannot open list file " + path);
    std::string line;
    while (lr.next(line)) if (!skip_empty || !line.empty()) out.push_back(line);
}

// sketch's inputs in sylph's order (src/sketch.rs:164-250): reads and genomes from -l then positional files, then -r / -g,
// then --rl / --gl; first mates -1 then --l1, second mates -2 then --l2.  Sample names go to the pairs, then to the
// reads in that order (src/sketch.rs:260-293).  The reads are sketched in the driver's own order (-r, positional,
// -l, --rl) and the genomes kept in it (-g, positional, -l, --gl), so runs without names write what they always did.
static void resolve_sketch_inputs(Args &a) {
    std::vector<std::string> pos_reads, list_reads;
    a.sketch_genomes = a.genomes;
    for (size_t i = 0; i < a.files.size(); i++) {
        const std::string &f = a.files[i];
        if (is_fasta(f)) a.sketch_genomes.push_back(f);
        else if (is_fastq(f)) (i < a.n_positional ? pos_reads : list_reads).push_back(f);
        else warn(f + " does not have a fasta/fastq/gzip type extension.");
    }
    std::vector<std::string> rl;
    if (!a.genome_list.empty()) read_list(a.genome_list, a.sketch_genomes, false);
    if (!a.read_list.empty()) read_list(a.read_list, rl, false);
    const size_t o_list = a.first_pairs.size(), o_pos = o_list + list_reads.size(), o_r = o_pos + pos_reads.size(),
                 o_rl = o_r + a.reads.size();
    for (size_t i = 0; i < a.reads.size(); i++) a.sketch_reads.push_back({a.reads[i], o_r + i});
    for (size_t i = 0; i < pos_reads.size(); i++) a.sketch_reads.push_back({pos_reads[i], o_pos + i});
    for (size_t i = 0; i < list_reads.size(); i++) a.sketch_reads.push_back({list_reads[i], o_list + i});
    for (size_t i = 0; i < rl.size(); i++) a.sketch_reads.push_back({rl[i], o_rl + i});
    if (!a.names_list.empty()) {  // --lS wins over -S
        a.sample_names.clear();
        read_list(a.names_list, a.sample_names, false);
    }
    const bool named = !a.names_list.empty() || !a.sample_names.empty();
    if (named && a.sample_names.size() != a.first_pairs.size() + a.sketch_reads.size())
        die("Sample name length is not equal to the number of reads. Exiting");
}

// --devices LIST: comma-separated CUDA device ordinals, each a plain decimal number
static std::vector<int> parse_devices(const std::string &list) {
    if (list.empty()) die("--devices: empty device list");
    std::vector<int> out;
    size_t i = 0;
    while (i <= list.size()) {
        size_t j = list.find(',', i);
        if (j == std::string::npos) j = list.size();
        const std::string t = list.substr(i, j - i);
        if (t.empty() || t.size() > 6 || t.find_first_not_of("0123456789") != std::string::npos)
            die("--devices " + list + ": `" + t + "` is not a device ordinal (a comma-separated list such as 0,1,2,3)");
        out.push_back(std::stoi(t));
        i = j + 1;
    }
    return out;
}

static Args parse(int argc, char **argv) {
    Args a;
    if (argc < 2) die("usage: sylph-b200 <sketch|query|profile|inspect> [options] files...");
    a.cmd = argv[1];
    auto need = [&](int &i) -> std::string { if (i + 1 >= argc) die(std::string("missing value for ") + argv[i]); return argv[++i]; };
    for (int i = 2; i < argc; i++) {
        std::string s = argv[i];
        if (s == "-k") a.k = std::stoull(need(i));
        else if (s == "-c") a.c = std::stoull(need(i));
        else if (s == "-t") a.threads = std::max(1, std::stoi(need(i)));          // files parsed concurrently
        else if (s == "-s" || s == "--sample-threads") need(i);
        else if (s == "--fpr") a.fpr = std::stod(need(i));
        else if (s == "-1" || s == "--first-pairs") { while (i + 1 < argc && argv[i + 1][0] != '-') a.first_pairs.push_back(argv[++i]); }
        else if (s == "-2" || s == "--second-pairs") { while (i + 1 < argc && argv[i + 1][0] != '-') a.second_pairs.push_back(argv[++i]); }
        else if (s == "--min-spacing") a.min_spacing = std::stoull(need(i));
        else if (s == "-i" || s == "--individual-records") a.individual = true;
        else if (s == "--no-dedup") a.no_dedup = true;
        else if (s == "--disable-profiling") a.no_pseudotax = true;
        else if (s == "-o" || s == "--out-name-db" || s == "--output-file") { if (a.cmd == "sketch") a.db_out = need(i); else a.out_file = need(i); }
        else if (s == "-d" || s == "--sample-output-directory") a.sample_dir = need(i);
        else if (s == "-l" || s == "--list") a.list_file = need(i);
        else if (s == "-r" || s == "--reads") { while (i + 1 < argc && argv[i + 1][0] != '-') a.reads.push_back(argv[++i]); }
        else if (s == "-g" || s == "--genomes") { while (i + 1 < argc && argv[i + 1][0] != '-') a.genomes.push_back(argv[++i]); }
        else if (s == "-m" || s == "--minimum-ani") a.min_ani = std::stod(need(i));
        else if (s == "-M" || s == "--min-number-kmers") a.min_number_kmers = std::stod(need(i));
        else if (s == "--min-count-correct") a.min_count_correct = std::stod(need(i));
        else if (s == "-R" || s == "--redundancy-threshold") a.redundant_ani = std::stod(need(i));
        else if (s == "--no-ci") a.no_ci = true;
        else if (s == "--no-adjust") a.no_adj = true;
        else if (s == "--mean-coverage") a.mean_cov = true;
        else if (s == "--device") { a.device = std::stoi(need(i)); a.device_given = true; }
        else if (s == "--devices") a.devices = parse_devices(need(i));  // driver-only
        else if (s == "-u" || s == "--estimate-unknown") a.estimate_unknown = true;
        else if (s == "-I" || s == "--read-seq-id") a.read_seq_id = std::stod(need(i));
        else if (s == "--max-db-entries") a.max_db_entries = std::max<uint64_t>(1, std::stoull(need(i)));  // driver-only
        else if (s == "--max-sample-bytes") {  // driver-only
            const std::string v = need(i);
            if (v.empty() || v.size() > 19 || v.find_first_not_of("0123456789") != std::string::npos || std::stoull(v) == 0)
                die("--max-sample-bytes " + v + ": not a positive number of bytes");
            a.max_sample_bytes = std::stoull(v);
        }
        else if (a.cmd == "sketch" && (s == "-S" || s == "--sample-names")) {
            while (i + 1 < argc && argv[i + 1][0] != '-') a.sample_names.push_back(argv[++i]);
        }
        else if (a.cmd == "sketch" && s == "--lS") a.names_list = need(i);
        else if (a.cmd == "sketch" && s == "--rl") a.read_list = need(i);
        else if (a.cmd == "sketch" && s == "--gl") a.genome_list = need(i);
        else if (a.cmd == "sketch" && s == "--l1") a.first_pair_list = need(i);
        else if (a.cmd == "sketch" && s == "--l2") a.second_pair_list = need(i);
        else if (!s.empty() && s[0] == '-') die("unknown option " + s);
        else a.files.push_back(s);
    }
    if (a.device_given && !a.devices.empty()) die("--device and --devices exclude each other; list every device in --devices");
    if (a.devices.empty()) a.devices.push_back(a.device);
    a.n_positional = a.files.size();
    if (!a.list_file.empty()) read_list(a.list_file, a.files, true);
    if (!(a.k == 21 || a.k == 31)) die("Only k = 21, 31 are currently supported");  // src/cmdline.rs:57
    if (a.fpr < 0. || a.fpr >= 1.) die("Invalid value for --fpr. Exiting.");             // src/sketch.rs:158-161
    if (a.first_pairs.size() != a.second_pairs.size()) die("Different number of paired sequences. Exiting.");  // :223-226
    if (!a.first_pair_list.empty()) read_list(a.first_pair_list, a.first_pairs, false);
    if (!a.second_pair_list.empty()) read_list(a.second_pair_list, a.second_pairs, false);
    if (a.first_pairs.size() != a.second_pairs.size()) die("Different number of paired sequences. Exiting.");  // :246-249
    if (a.cmd == "sketch") resolve_sketch_inputs(a);
    // the reference's query / profile sketch pairs with the approximate cuckoo filter (src/contain.rs:201-210,
    // DEFAULT_FPR), which is out of scope; an exact-set profile would silently differ from it
    if (!a.first_pairs.empty() && (a.cmd == "query" || a.cmd == "profile"))
        die("query/profile do not sketch read pairs (-1/-2) here: sylph sketches them with its approximate paired-end filter. "
            "Run `sylph-b200 sketch -1 ... -2 ... --fpr 0` and pass the *.paired.sylsp files instead. Exiting.");
    if (a.estimate_unknown && !(a.read_seq_id > 0.))
        die("-u needs -I/--read-seq-id here: sylph's automatic read-identity estimate depends on hash-map iteration order (DESIGN.md)");
    if (!a.first_pairs.empty() && a.fpr != 0.)
        die("paired-end reads need --fpr 0 (the exact dedup set); the default approximate cuckoo filter is not bit-reproducible and out of scope");
    a.batch_bases = env_u64("SYL_DRIVER_BATCH_BASES", a.batch_bases);
    a.samples_per_call = env_u64("SYL_DRIVER_SAMPLES_PER_CALL", 0);
    a.rows0 = env_u64("SYL_DRIVER_ROWS", 0);
    a.shard_entries = env_u64("SYL_DRIVER_SHARD_ENTRIES", 0);
    return a;
}

// ---- worker threads ------------------------------------------------------------------------------

// Set once a worker has failed: the others take no new work item.
static std::atomic<bool> g_abort{false};
struct Aborted : std::exception {
    const char *what() const noexcept override { return "aborted"; }
};
static void check_abort() {
    if (g_abort) throw Aborted();
}

// -t: files being parsed, or parsed and not yet used, across every worker and queue of the process
class ParseBudget {
  public:
    void reset(int n) { free_ = n; }
    void acquire() {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&]() { return free_ > 0 || g_abort; });
        if (g_abort) throw Aborted();
        free_--;
    }
    bool try_acquire() {
        std::lock_guard<std::mutex> lk(mu_);
        if (free_ <= 0) return false;
        free_--;
        return true;
    }
    void release() {
        { std::lock_guard<std::mutex> lk(mu_); free_++; }
        cv_.notify_one();
    }
    void wake() {
        { std::lock_guard<std::mutex> lk(mu_); }
        cv_.notify_all();
    }
  private:
    std::mutex mu_;
    std::condition_variable cv_;
    int free_ = 1;
};
static ParseBudget g_parse;

// Runs fn(w) for every worker w in [0, n), each on its own thread (on this one when n == 1), and joins them all.  The
// first exception is rethrown here once every worker has stopped, so that exit() never runs beside a worker.
template <typename F>
static void run_workers(size_t n, F fn) {
    if (n == 1) { fn(0); return; }
    std::mutex mu;
    std::exception_ptr first;
    std::vector<std::thread> th;
    for (size_t w = 0; w < n; w++)
        th.emplace_back([&, w]() {
            try {
                fn(w);
            } catch (...) {
                {
                    std::lock_guard<std::mutex> lk(mu);
                    if (!first) first = std::current_exception();
                }
                g_abort = true;
                g_parse.wake();
            }
        });
    for (std::thread &t : th) t.join();
    if (first) std::rethrow_exception(first);
}

// ---- sketching -----------------------------------------------------------------------------------

// Files inflated and parsed ahead of their use, handed out in order to whichever worker asks next: the next files are
// being read while the GPUs sketch the current ones.  Each file in flight holds one unit of g_parse until it is used.
struct Parsed { bool ok = false; FlatRecords recs; std::string first_id; };
struct ParsedFile {
    size_t i = 0;
    std::unique_ptr<Parsed> p;
    ParsedFile() = default;
    ParsedFile(const ParsedFile &) = delete;
    ParsedFile &operator=(const ParsedFile &) = delete;
    ~ParsedFile() { if (p) g_parse.release(); }
};
class ParseQueue {
  public:
    ParseQueue(const std::vector<std::string> &files, bool want_ids) : files_(files), want_ids_(want_ids), fut_(files.size()) {}
    // false once every file has been taken
    bool take(ParsedFile &out) {
        std::unique_lock<std::mutex> lk(mu_);
        if (taken_ == files_.size()) return false;
        const size_t i = taken_++;
        if (launched_ == i) {  // none of this queue's files is in flight: wait for a unit the other queues give back
            g_parse.acquire();
            launch();
        }
        while (launched_ < files_.size() && g_parse.try_acquire()) launch();
        lk.unlock();
        out.i = i;
        out.p = fut_[i].get();
        return true;
    }
  private:
    void launch() {
        const std::string f = files_[launched_];
        const bool ids = want_ids_;
        fut_[launched_++] = std::async(std::launch::async, [f, ids]() {
            std::unique_ptr<Parsed> p(new Parsed());
            p->ok = read_fastx(f, p->recs, ids, &p->first_id);
            return p;
        });
    }
    const std::vector<std::string> &files_;
    const bool want_ids_;
    std::mutex mu_;
    std::vector<std::future<std::unique_ptr<Parsed>>> fut_;
    size_t launched_ = 0, taken_ = 0;
};

static void store_sample(syl_ctx *ctx, syl_sample *s, const Args &a, const std::string &file, bool paired, SequencesSketch &out) {
    out.hashes.resize(syl_sample_size(s));
    out.counts.resize(out.hashes.size());
    check(syl_sample_download(ctx, s, out.hashes.data(), out.counts.data()), "syl_sample_download");
    out.c = a.c; out.k = a.k; out.file_name = file; out.paired = paired;
    out.mean_read_length = syl_sample_mean_read_length(s);
    syl_sample_free(s);
}

// src/sketch.rs:771-895 with --fpr 0
static bool sketch_pair_files(syl_ctx *ctx, const Args &a, const std::string &f1, const std::string &f2, SequencesSketch &out) {
    auto fut = std::async(std::launch::async, [&]() { std::unique_ptr<Parsed> p(new Parsed()); p->ok = read_fastx(f2, p->recs, false); return p; });
    FlatRecords r1;
    const bool ok1 = read_fastx(f1, r1, false);
    std::unique_ptr<Parsed> p2 = fut.get();
    if (!ok1 || !p2->ok) fail("Paired end reading failed for '" + f1 + "' and '" + f2 + "'. Make sure the files are present or the sequences are valid.");
    const uint64_t n_pairs = std::min(r1.n(), p2->recs.n());
    syl_sample *s = nullptr;
    check(syl_sketch_read_pairs(ctx, SYL_MEM_HOST, r1.bases.data(), r1.offsets[n_pairs], r1.offsets.data(), p2->recs.bases.data(),
                                p2->recs.offsets[n_pairs], p2->recs.offsets.data(), n_pairs, (int)a.k, a.c, a.no_dedup ? 1 : 0,
                                SYL_SEM_AVX2, &s), "syl_sketch_read_pairs");
    store_sample(ctx, s, a, f1, true, out);
    return true;
}

static bool sketch_reads_parsed(syl_ctx *ctx, const Args &a, const std::string &file, const Parsed &p, SequencesSketch &out) {
    if (!p.ok) { warn(file + " is not a valid fasta/fastq file; skipping."); return false; }
    syl_sample *s = nullptr;
    check(syl_sketch_reads(ctx, SYL_MEM_HOST, p.recs.bases.data(), p.recs.bases.size(), p.recs.offsets.data(), p.recs.n(), (int)a.k,
                           a.c, a.no_dedup ? 1 : 0, SYL_SEM_AVX2, &s), "syl_sketch_reads");
    store_sample(ctx, s, a, file, false, out);
    return true;
}

// Genome files in batches of <= batch_bases, one syl_sketch_genomes call per batch.  Batches are cut in file order
// (whichever worker asks next cuts the next one) and their sketches are collected in batch order, so the result does not
// depend on which context sketched which batch or when it finished.
class GenomeBatches {
  public:
    GenomeBatches(const Args &a, const std::vector<std::string> &files, bool pseudotax)
        : a_(a), files_(files), pseudotax_(pseudotax), queue_(files, a.individual) {}
    // cut the next batch and sketch it on ctx; false once every file has been used
    bool sketch_next(syl_ctx *ctx) {
        check_abort();
        FlatRecords recs;
        std::vector<uint64_t> genome_off{0};
        std::vector<std::string> names, first_ids;
        size_t b = 0;
        {
            std::lock_guard<std::mutex> lk(cut_mu_);
            if (done_) return false;
            while (recs.bases.size() < a_.batch_bases) {
                ParsedFile pf;
                if (!queue_.take(pf)) { done_ = true; break; }
                const std::string &f = files_[pf.i];
                const Parsed &p = *pf.p;
                // a file that fails half way contributes nothing (records are merged only after a complete parse)
                if (!p.ok) { warn(f + " is not a valid fasta/fastq file; skipping."); continue; }
                const FlatRecords &tmp = p.recs;
                const uint64_t base = recs.bases.size();
                recs.bases.insert(recs.bases.end(), tmp.bases.begin(), tmp.bases.end());
                for (size_t i = 1; i < tmp.offsets.size(); i++) recs.offsets.push_back(base + tmp.offsets[i]);
                if (!a_.individual) {
                    genome_off.push_back(recs.n());
                    names.push_back(f);
                    first_ids.push_back(p.first_id);
                } else {
                    for (size_t i = 0; i < tmp.n(); i++) { names.push_back(f); first_ids.push_back(tmp.ids[i]); }
                }
            }
            b = batches_.size();
            batches_.emplace_back();
        }
        const uint64_t G = a_.individual ? recs.n() : genome_off.size() - 1;
        if (G == 0) return true;
        syl_genomes *g = nullptr;
        check(syl_sketch_genomes(ctx, SYL_MEM_HOST, recs.bases.data(), recs.bases.size(), recs.offsets.data(), recs.n(),
                                 a_.individual ? nullptr : genome_off.data(), G, (int)a_.k, a_.c, a_.min_spacing, pseudotax_ ? 1 : 0,
                                 a_.individual ? 1 : 0, SYL_SEM_AVX2, &g), "syl_sketch_genomes");
        std::vector<uint64_t> kmers(syl_genomes_total_kmers(g)), koff(G + 1), tracked(syl_genomes_total_tracked(g)), toff(G + 1), gs(G);
        check(syl_genomes_download(ctx, g, kmers.data(), koff.data(), tracked.data(), toff.data(), gs.data()), "syl_genomes_download");
        syl_genomes_free(g);
        std::vector<GenomeSketch> out(G);
        for (uint64_t i = 0; i < G; i++) {
            GenomeSketch &s = out[i];
            s.genome_kmers.assign(kmers.begin() + koff[i], kmers.begin() + koff[i + 1]);
            s.has_tracked = pseudotax_;
            if (pseudotax_) s.tracked.assign(tracked.begin() + toff[i], tracked.begin() + toff[i + 1]);
            s.file_name = names[i];
            s.first_contig_name = first_ids[i];
            s.c = a_.c; s.k = a_.k; s.gn_size = gs[i]; s.min_spacing = a_.min_spacing;
        }
        std::lock_guard<std::mutex> lk(cut_mu_);
        n_done_ += G;
        batches_[b] = std::move(out);
        info(std::to_string(n_done_) + " genomes processed.");
        return true;
    }
    void collect(std::vector<GenomeSketch> &out) {
        for (std::vector<GenomeSketch> &v : batches_)
            for (GenomeSketch &g : v) out.push_back(std::move(g));
    }
  private:
    const Args &a_;
    const std::vector<std::string> &files_;
    const bool pseudotax_;
    ParseQueue queue_;
    std::mutex cut_mu_;
    bool done_ = false;
    std::vector<std::vector<GenomeSketch>> batches_;
    uint64_t n_done_ = 0;
};

static void sketch_genome_files(const std::vector<syl_ctx *> &ctxs, const Args &a, const std::vector<std::string> &files,
                                bool pseudotax, std::vector<GenomeSketch> &out) {
    GenomeBatches batches(a, files, pseudotax);
    run_workers(ctxs.size(), [&](size_t w) { while (batches.sketch_next(ctxs[w])) {} });
    batches.collect(out);
}

// Path::file_name of a sample name (src/sketch.rs:346,401): its last component, with empty and "." components ignored
static std::string name_file_component(const std::string &name) {
    std::string last;
    size_t i = 0;
    while (i <= name.size()) {
        size_t j = name.find('/', i);
        if (j == std::string::npos) j = name.size();
        const std::string c = name.substr(i, j - i);
        if (!c.empty() && c != ".") last = c;
        i = j + 1;
    }
    if (last.empty() || last == "..") fail("Sample name `" + name + "` does not end in a file name. Exiting");
    return last;
}

// Work items in this order: read pairs, single-end read files, genome batches; each idle context takes the next one.
static int cmd_sketch(const std::vector<syl_ctx *> &ctxs, const Args &a) {
    const std::string dir = a.sample_dir.empty() || a.sample_dir.back() == '/' ? a.sample_dir : a.sample_dir + "/";
    const bool named = !a.sample_names.empty();
    std::mutex dir_mu;
    // a named sketch carries its sample name and is written as <-d>/<file name of the sample name>[.paired].sylsp
    auto write_sample = [&](SequencesSketch &s, const std::string &file, size_t name, const char *suffix) {
        std::string stem = basename_of(file);
        if (named) {
            s.has_sample_name = true;
            s.sample_name = a.sample_names[name];
            stem = name_file_component(s.sample_name);
        }
        if (!dir.empty()) {
            std::lock_guard<std::mutex> lk(dir_mu);
            std::filesystem::create_directories(dir);
        }
        const std::string path = dir + stem + suffix;
        write_sylsp(path, s);
        info("Sketching " + path + " complete.");
    };
    std::vector<std::string> reads;
    for (const ReadInput &r : a.sketch_reads) reads.push_back(r.file);
    std::atomic<size_t> next_pair{0};
    ParseQueue read_queue(reads, false);
    GenomeBatches batches(a, a.sketch_genomes, !a.no_pseudotax);
    run_workers(ctxs.size(), [&](size_t w) {
        syl_ctx *ctx = ctxs[w];
        for (size_t i; (i = next_pair++) < a.first_pairs.size();) {  // src/sketch.rs:310-364
            check_abort();
            SequencesSketch s;
            if (!sketch_pair_files(ctx, a, a.first_pairs[i], a.second_pairs[i], s)) continue;
            write_sample(s, a.first_pairs[i], i, ".paired.sylsp");
        }
        for (;;) {
            check_abort();
            ParsedFile pf;
            if (!read_queue.take(pf)) break;
            SequencesSketch s;
            if (!sketch_reads_parsed(ctx, a, reads[pf.i], *pf.p, s)) continue;
            write_sample(s, reads[pf.i], a.sketch_reads[pf.i].name, ".sylsp");
        }
        while (batches.sketch_next(ctx)) {}
    });
    if (!a.sketch_genomes.empty()) {
        std::vector<GenomeSketch> gs;
        batches.collect(gs);
        if (gs.empty()) warn("No valid genomes to sketch; " + a.db_out + ".syldb is not output");
        else { write_syldb(a.db_out + ".syldb", gs); info("Wrote all genome sketches to " + a.db_out + ".syldb"); }
    }
    info("Finished.");
    return 0;
}

// ---- query / profile ---------------------------------------------------------------------------

// src/contain.rs:18-94
static void print_row(FILE *o, const syl_ani_row &r, bool pseudotax, const std::string &seq, const GenomeSketch &g) {
    char ani[64], lam[64], cia[96], cil[96];
    snprintf(ani, sizeof ani, "%.2f", std::min(r.final_est_ani * 100., 100.));
    if (r.lambda_status == SYL_LAMBDA_VALUE) snprintf(lam, sizeof lam, "%.3f", r.lambda);
    else snprintf(lam, sizeof lam, "%s", r.lambda_status == SYL_LAMBDA_HIGH ? "HIGH" : "LOW");
    if (!r.ci_valid) { snprintf(cia, sizeof cia, "NA-NA"); snprintf(cil, sizeof cil, "NA-NA"); }
    else { snprintf(cia, sizeof cia, "%.2f-%.2f", r.ci[0] * 100., r.ci[1] * 100.); snprintf(cil, sizeof cil, "%.2f-%.2f", r.ci[2], r.ci[3]); }
    if (!pseudotax)
        fprintf(o, "%s\t%s\t%s\t%.3f\t%s\t%s\t%s\t%.0f\t%.3f\t%llu/%llu\t%.2f\t%s\n", seq.c_str(), g.file_name.c_str(), ani,
                r.final_est_cov, cia, lam, cil, r.median_cov, r.mean_cov, (unsigned long long)r.contain, (unsigned long long)r.glen,
                r.naive_ani * 100., g.first_contig_name.c_str());
    else
        fprintf(o, "%s\t%s\t%.4f\t%.4f\t%s\t%.3f\t%s\t%s\t%s\t%.0f\t%.3f\t%llu/%llu\t%.2f\t%lld\t%s\n", seq.c_str(),
                g.file_name.c_str(), r.rel_abund, r.seq_abund, ani, r.final_est_cov, cia, lam, cil, r.median_cov, r.mean_cov,
                (unsigned long long)r.contain, (unsigned long long)r.glen, r.naive_ani * 100., (long long)r.kmers_lost,
                g.first_contig_name.c_str());
}

// Contiguous blocks of samples, one per context, balanced by weight: sample i goes to the block its weight's midpoint
// falls in, so every block holds at most total / n_blocks plus one sample's weight.  -> first sample of each block,
// and the end (n_blocks + 1 entries).
static std::vector<size_t> sample_blocks(const std::vector<uint64_t> &weight, size_t n_blocks) {
    long double total = 0;
    for (uint64_t w : weight) total += (long double)w;
    std::vector<size_t> first(n_blocks + 1, weight.size());
    long double before = 0;
    size_t blk = 0;
    first[0] = 0;
    for (size_t i = 0; i < weight.size(); i++) {
        // all weights 0: by count
        const long double mid = total > 0 ? (before + (long double)weight[i] / 2) / total : ((long double)i + 0.5L) / weight.size();
        const size_t b = std::min(n_blocks - 1, (size_t)(mid * n_blocks));
        while (blk < b) first[++blk] = i;
        before += (long double)weight[i];
    }
    return first;
}

// Sketch k-mers a sample is expected to bring, the weight of sample_blocks: a .sylsp's count from its header; raw reads
// from the file size (a FASTQ byte is about half a base, gzip inflates about 4x, one k-mer per c bases)
static uint64_t sample_weight(const std::string &f, bool sketched, uint64_t c) {
    std::error_code ec;
    const uint64_t bytes = std::filesystem::file_size(f, ec);
    if (ec) return 0;
    if (sketched) {
        try { Reader r(f); return r.u64(); } catch (const std::exception &) { return 0; }  // read again (and reported) by its worker
    }
    const uint64_t bases = ends_with(f, ".gz") ? bytes * 2 : bytes / 2;
    return bases / std::max<uint64_t>(c, 1);
}

// The rows of each sample printed in sample order, each sample as soon as it and every earlier one is done.
class RowPrinter {
  public:
    RowPrinter(FILE *o, bool pseudotax, const std::vector<std::string> &names, const std::vector<GenomeSketch> &gs)
        : o_(o), pseudotax_(pseudotax), names_(names), gs_(gs), rows_(names.size()), done_(names.size(), 0) {}
    // sample i's rows (in the library's order), or none with `valid` false (a skipped file: no rows, no line)
    void done(size_t i, std::vector<syl_ani_row> rows, bool valid) {
        std::lock_guard<std::mutex> lk(mu_);
        rows_[i] = std::move(rows);
        done_[i] = valid ? 1 : 2;
        for (; next_ < names_.size() && done_[next_]; next_++) {
            std::vector<syl_ani_row> &r = rows_[next_];
            if (!pseudotax_)  // src/contain.rs:332-334: stable sort by ANI descending
                std::stable_sort(r.begin(), r.end(), [](const syl_ani_row &x, const syl_ani_row &y) { return x.final_est_ani > y.final_est_ani; });
            for (const syl_ani_row &row : r) print_row(o_, row, pseudotax_, names_[next_], gs_[row.genome]);
            if (done_[next_] == 1) info("Finished sample " + names_[next_] + ".");
            std::vector<syl_ani_row>().swap(r);
        }
    }
  private:
    std::mutex mu_;
    FILE *o_;
    const bool pseudotax_;
    const std::vector<std::string> &names_;
    const std::vector<GenomeSketch> &gs_;
    std::vector<std::vector<syl_ani_row>> rows_;
    std::vector<uint8_t> done_;  // 0: pending, 1: rows, 2: skipped
    size_t next_ = 0;
};

// One context's index: the whole db, or shards over the shared host arrays.
struct ContextDb { syl_db *db = nullptr; syl_db_shards *shards = nullptr; };

static int cmd_contain(const std::vector<syl_ctx *> &ctxs, const Args &a, bool pseudotax) {
    std::vector<std::string> db_files, genome_files, sample_files, read_files = a.reads;
    for (const std::string &f : a.files) {  // src/contain.rs:167-199
        if (is_syldb(f)) db_files.push_back(f);
        else if (is_sylsp(f)) sample_files.push_back(f);
        else if (is_fasta(f)) genome_files.push_back(f);
        else if (is_fastq(f)) read_files.push_back(f);
        else warn(f + " file extension is not a sketch or a fasta/fastq file.");
    }
    if (db_files.empty() && genome_files.empty()) die("No genome files found; see sylph query/profile -h for help. Exiting");
    if (sample_files.empty() && read_files.empty()) die("No read files found; see sylph query/profile -h for help. Exiting");
    info("Obtaining sketches...");
    std::vector<GenomeSketch> gs;
    for (const std::string &f : db_files) {
        try { std::vector<GenomeSketch> v = read_syldb(f); for (auto &g : v) gs.push_back(std::move(g)); }
        catch (const std::exception &e) { die(e.what()); }
    }
    if (!gs.empty() && gs[0].k != a.k && !genome_files.empty()) die("-k is not equal to -k found in sketches.");
    if (!genome_files.empty()) sketch_genome_files(ctxs, a, genome_files, pseudotax, gs);
    if (gs.empty()) die("No genome sketches found; see sylph query/profile -h for help. Exiting");
    for (const GenomeSketch &g : gs) if (g.k != gs[0].k) die("Query sketches have inconsistent -k. Exiting.");
    if (pseudotax && !gs[0].has_tracked)
        die("Attempting profiling, but *.syldb was sketched with the --disable-profiling option. Exiting");  // src/contain.rs:231-234
    info("Finished obtaining genome sketches.");
    // index the db from flat CSR arrays; each sketch's k-mers are freed once appended, so host memory holds about one
    // copy of the sketches (only the names and gn_size are used afterwards)
    std::vector<uint64_t> kmers, koff{0}, tracked, toff{0}, gsz;
    uint64_t db_c = gs[0].c, nk = 0, nt = 0;
    for (const GenomeSketch &g : gs) { nk += g.genome_kmers.size(); nt += g.tracked.size(); }
    kmers.reserve(nk);
    tracked.reserve(nt);
    for (GenomeSketch &g : gs) {
        kmers.insert(kmers.end(), g.genome_kmers.begin(), g.genome_kmers.end());
        koff.push_back(kmers.size());
        tracked.insert(tracked.end(), g.tracked.begin(), g.tracked.end());
        toff.push_back(tracked.size());
        gsz.push_back(g.gn_size);
        db_c = std::min(db_c, g.c);
        std::vector<uint64_t>().swap(g.genome_kmers);
        std::vector<uint64_t>().swap(g.tracked);
    }
    const bool has_tr = gs[0].has_tracked;
    // samples: raw reads, then sketches, cut into one contiguous block per context
    if (!read_files.empty() && a.c > gs[0].c) {
        for (const std::string &f : read_files) warn(f + " error: value of -c for contain is greater than the smallest value of -c for a genome sketch. Continuing without sketching.");
        read_files.clear();
    }
    if (!read_files.empty() && a.k != gs[0].k) {  // src/contain.rs:578-584: raw reads are sketched with -k or not at all
        for (const std::string &f : read_files)
            warn(f + " -k " + std::to_string(a.k) + " is not equal to -k " + std::to_string(gs[0].k) + " found in sketches. Continuing without sketching.");
        read_files.clear();
    }
    const size_t n_reads = read_files.size(), n_samples = n_reads + sample_files.size();
    std::vector<uint64_t> weight(n_samples);
    for (size_t i = 0; i < n_samples; i++)
        weight[i] = i < n_reads ? sample_weight(read_files[i], false, a.c) : sample_weight(sample_files[i - n_reads], true, a.c);
    const std::vector<size_t> block = sample_blocks(weight, ctxs.size());
    // one index while the db fits one (fewer than 2^32-2 entries and 2^31-1 genomes) and no cap is set; otherwise db
    // shards that every query / profile call sweeps once, reading the flat arrays from host memory
    uint64_t shard_cap = a.max_db_entries;
    if (a.shard_entries) shard_cap = shard_cap ? std::min(shard_cap, a.shard_entries) : a.shard_entries;
    const bool sharded = shard_cap || nk + (has_tr ? nt : 0) >= 0xFFFFFFFEull || gs.size() >= 0x7FFFFFFFull;
    // a context whose block of samples the library would scan past the genome k-mers (syl_db_scan_plan) takes shards
    // too: its calls then build no index at all
    std::vector<char> scans(ctxs.size(), 0);
    for (size_t w = 0; w < ctxs.size() && !sharded; w++) {
        uint64_t sk = 0;
        for (size_t i = block[w]; i < block[w + 1]; i++) sk += weight[i];
        int scan = 0;
        check(syl_db_scan_plan(ctxs[w], nk, has_tr ? nt : 0, gs.size(), (uint32_t)(block[w + 1] - block[w]), sk, &scan), "syl_db_scan_plan");
        scans[w] = scan != 0;
    }
    const bool any_scan = std::count(scans.begin(), scans.end(), 1) > 0;
    // every context builds its own index (or shards) from the same host arrays, which stay alive until all have
    std::vector<ContextDb> dbs(ctxs.size());
    run_workers(ctxs.size(), [&](size_t w) {
        syl_ctx *ctx = ctxs[w];
        if (!sharded && !scans[w]) {
            check(syl_db_build_arrays(ctx, SYL_MEM_HOST, kmers.data(), koff.data(), has_tr ? tracked.data() : nullptr,
                                      has_tr ? toff.data() : nullptr, gsz.data(), gs.size(), (int)gs[0].k, db_c, 0, &dbs[w].db),
                  "syl_db_build_arrays");
            return;
        }
        auto create = [&](uint64_t cap) {
            check(syl_db_shards_create(ctx, kmers.data(), koff.data(), has_tr ? tracked.data() : nullptr, has_tr ? toff.data() : nullptr,
                                       gsz.data(), gs.size(), (int)gs[0].k, db_c, cap, &dbs[w].shards), "syl_db_shards_create");
        };
        create(shard_cap);
        // without a cap the library cuts shards to this device's free memory; contexts sharing the device split it:
        // each cuts again at its largest shard divided by the number of contexts on the device
        const size_t share = (size_t)std::count(a.devices.begin(), a.devices.end(), a.devices[w]);
        if (!shard_cap && share > 1) {
            uint64_t largest = 1;
            for (uint64_t i = 0; i < syl_db_shards_count(dbs[w].shards); i++) {
                uint64_t g0 = 0, ng = 0, ne = 0;
                check(syl_db_shards_range(dbs[w].shards, i, &g0, &ng, &ne), "syl_db_shards_range");
                largest = std::max(largest, ne);
            }
            syl_db_shards_free(dbs[w].shards);
            dbs[w].shards = nullptr;
            create(std::max<uint64_t>(1, largest / share));
        }
    });
    if (!sharded && !any_scan) {
        std::vector<uint64_t>().swap(kmers);
        std::vector<uint64_t>().swap(tracked);
    } else if (sharded) {
        const uint64_t n_shards = syl_db_shards_count(dbs[0].shards);
        for (uint64_t i = 0; i < n_shards; i++) {
            uint64_t g0 = 0, ng = 0, ne = 0;
            check(syl_db_shards_range(dbs[0].shards, i, &g0, &ng, &ne), "syl_db_shards_range");
            info("Database shard " + std::to_string(i + 1) + "/" + std::to_string(n_shards) + ": genomes " + std::to_string(g0) + ".." +
                 std::to_string(g0 + ng) + ", " + std::to_string(ne) + " index entries.");
        }
    }
    FILE *o = a.out_file.empty() ? stdout : fopen(a.out_file.c_str(), "w");
    if (!o) die("cannot open output file " + a.out_file);
    if (!pseudotax)  // src/contain.rs:461-480
        fprintf(o, "Sample_file\tGenome_file\tAdjusted_ANI\tEff_cov\tANI_5-95_percentile\tEff_lambda\tLambda_5-95_percentile\tMedian_cov\tMean_cov_geq1\tContainment_ind\tNaive_ANI\tContig_name\n");
    else  // with -u the coverage column holds the true coverage (src/contain.rs:469-475)
        fprintf(o, "Sample_file\tGenome_file\tTaxonomic_abundance\tSequence_abundance\tAdjusted_ANI\t%s\tANI_5-95_percentile\tEff_lambda\tLambda_5-95_percentile\tMedian_cov\tMean_cov_geq1\tContainment_ind\tNaive_ANI\tkmers_reassigned\tContig_name\n",
                a.estimate_unknown ? "True_cov" : "Eff_cov");
    syl_contain_params p;
    syl_contain_params_default(&p, (int)gs[0].k, pseudotax ? 1 : 0);
    p.no_ci = a.no_ci; p.no_adj = a.no_adj; p.mean_coverage = a.mean_cov;
    p.min_number_kmers = a.min_number_kmers; p.min_count_correct = a.min_count_correct;
    p.minimum_ani = a.min_ani; p.redundant_ani = a.redundant_ani;
    p.estimate_unknown = a.estimate_unknown ? 1 : 0; p.read_seq_id = a.read_seq_id;
    std::vector<std::string> names(n_samples);
    RowPrinter printer(o, pseudotax, names, gs);
    // Each context queries its block of samples in host batches of at most --max-sample-bytes (default: a quarter of
    // physical memory shared by the contexts), one syl_*_host_samples call per batch; the library stages each batch
    // through the device in pieces that fit it, so the device never holds more than one batch's share.  The reference
    // walks the samples in chunks too (src/contain.rs:239-263).
    uint64_t max_bytes = a.max_sample_bytes;
    if (!max_bytes) {
        const long pages = sysconf(_SC_PHYS_PAGES), page = sysconf(_SC_PAGE_SIZE);
        max_bytes = std::max<uint64_t>(1, (uint64_t)std::max(pages, 1L) * (uint64_t)std::max(page, 1L) / 4 / ctxs.size());
    }
    run_workers(ctxs.size(), [&](size_t w) {
        syl_ctx *ctx = ctxs[w];
        const ContextDb &db = dbs[w];
        const size_t s_begin = block[w], s_end = block[w + 1];
        // one host batch: the samples' pairs back to back, in the order they were added
        std::vector<uint64_t> hashes, off{0}, cs;
        std::vector<uint32_t> counts;
        std::vector<double> mrl;
        std::vector<size_t> ids;  // global index of each sample of the batch
        int batch_k = (int)gs[0].k;
        auto flush = [&]() {
            if (ids.empty()) return;
            check_abort();
            const syl_host_samples hs{hashes.data(), counts.data(), off.data(), cs.data(), mrl.data(), (uint32_t)ids.size(), batch_k};
            std::vector<syl_ani_row> rows(a.rows0 ? a.rows0 : std::max<size_t>(1024, std::min<size_t>(gs.size() * ids.size(), 1u << 22)));
            uint64_t n = 0;
            for (;;) {
                const int rc = (pseudotax ? syl_profile_host_samples : syl_query_host_samples)(ctx, db.db, db.shards, &hs, &p, rows.data(),
                                                                                                rows.size(), &n);
                if (rc == SYL_ERR_CAPACITY) { rows.resize(n); continue; }  // shards: the retry copies out the kept rows
                check(rc, pseudotax ? "syl_profile_host_samples" : "syl_query_host_samples");
                break;
            }
            rows.resize(n);
            size_t i = 0;
            for (uint32_t s = 0; s < ids.size(); s++) {
                size_t j = i;
                while (j < rows.size() && rows[j].sample == s) j++;
                printer.done(ids[s], std::vector<syl_ani_row>(rows.begin() + i, rows.begin() + j), true);
                i = j;
            }
            hashes.clear(); counts.clear(); off.assign(1, 0); cs.clear(); mrl.clear(); ids.clear();
        };
        // a sample joins the batch unless the batch holds samples and would pass the byte or sample cap with it
        auto add = [&](size_t id, const uint64_t *h, const uint32_t *c, uint64_t n, int k, uint64_t sc, double m) {
            const uint64_t bytes = 12 * (hashes.size() + n) + 24 * (ids.size() + 1);
            if (!ids.empty() && (bytes > max_bytes || k != batch_k || (a.samples_per_call && ids.size() >= a.samples_per_call))) flush();
            batch_k = k;
            hashes.insert(hashes.end(), h, h + n);
            counts.insert(counts.end(), c, c + n);
            off.push_back(hashes.size());
            cs.push_back(sc);
            mrl.push_back(m);
            ids.push_back(id);
        };
        // a raw read file is sketched on the context that queries it and copied out to the host batch
        std::vector<std::string> my_reads(read_files.begin() + std::min(s_begin, n_reads), read_files.begin() + std::min(s_end, n_reads));
        ParseQueue queue(my_reads, false);
        std::vector<uint64_t> h;
        std::vector<uint32_t> c;
        for (;;) {
            check_abort();
            ParsedFile pf;
            if (!queue.take(pf)) break;
            const size_t id = std::min(s_begin, n_reads) + pf.i;
            const std::string &f = read_files[id];
            names[id] = f;
            if (!pf.p->ok) { warn(f + " is not a valid fasta/fastq file; skipping."); printer.done(id, {}, false); continue; }
            const FlatRecords &r = pf.p->recs;
            syl_sample *s = nullptr;
            check(syl_sketch_reads(ctx, SYL_MEM_HOST, r.bases.data(), r.bases.size(), r.offsets.data(), r.n(), (int)gs[0].k, a.c, 0,
                                   SYL_SEM_AVX2, &s), "syl_sketch_reads");
            h.resize(syl_sample_size(s));
            c.resize(h.size());
            check(syl_sample_download(ctx, s, h.data(), c.data()), "syl_sample_download");
            const double m = syl_sample_mean_read_length(s);
            syl_sample_free(s);
            add(id, h.data(), c.data(), h.size(), (int)gs[0].k, a.c, m);
        }
        for (size_t id = std::max(s_begin, n_reads); id < s_end; id++) {
            check_abort();
            const std::string &f = sample_files[id - n_reads];
            SequencesSketch sk = read_sylsp(f);
            if (sk.c > gs[0].c) {
                warn(f + " value of -c is greater than the smallest value of -c for a genome sketch. Exiting.");
                printer.done(id, {}, false);
                continue;
            }
            names[id] = sk.has_sample_name ? sk.sample_name : sk.file_name;
            add(id, sk.hashes.data(), sk.counts.data(), sk.hashes.size(), (int)sk.k, sk.c, sk.mean_read_length);
        }
        flush();
    });
    if (o != stdout) fclose(o);
    for (ContextDb &db : dbs) {
        syl_db_free(db.db);
        syl_db_shards_free(db.shards);
    }
    info("sylph finished.");
    return 0;
}

// fastx-stats: parser self-check without a GPU (records, bases, first id, FNV-1a of all bases + lengths)
static int cmd_fastx_stats(const Args &a) {
    for (const std::string &f : a.files) {
        FlatRecords recs;
        std::string first;
        if (!read_fastx(f, recs, true, &first)) { printf("%s\tINVALID\n", f.c_str()); continue; }
        uint64_t h = 1469598103934665603ull;
        for (uint8_t b : recs.bases) { h ^= b; h *= 1099511628211ull; }
        for (size_t i = 0; i < recs.n(); i++) { h ^= recs.offsets[i + 1] - recs.offsets[i]; h *= 1099511628211ull; }
        for (const std::string &id : recs.ids) for (char c : id) { h ^= (uint8_t)c; h *= 1099511628211ull; }
        printf("%s\t%zu\t%zu\t%016llx\t%s\n", f.c_str(), recs.n(), recs.bases.size(), (unsigned long long)h, first.c_str());
    }
    return 0;
}

// sample-blocks: the split of samples of these weights over the --devices contexts, without a device
// (first sample, samples and total weight of each block)
static int cmd_sample_blocks(const Args &a) {
    std::vector<uint64_t> w;
    for (const std::string &f : a.files) w.push_back(std::stoull(f));
    const std::vector<size_t> first = sample_blocks(w, a.devices.size());
    for (size_t b = 0; b + 1 < first.size(); b++) {
        uint64_t sum = 0;
        for (size_t i = first[b]; i < first[b + 1]; i++) sum += w[i];
        printf("%zu\t%zu\t%llu\n", first[b], first[b + 1] - first[b], (unsigned long long)sum);
    }
    return 0;
}

// inspect (src/inspect.rs:117-182): databases first, then samples, each as one YAML list; no device is needed
static int cmd_inspect(const Args &a) {
    std::vector<std::string> db_files, sample_files;
    for (const std::string &f : a.files) {
        if (is_syldb(f)) db_files.push_back(f);
        else if (is_sylsp(f)) sample_files.push_back(f);
        else warn(f + " file is not a .sylsp or .syldb file. Skipping...");
    }
    FILE *o = a.out_file.empty() ? stdout : fopen(a.out_file.c_str(), "w");
    if (!o) die("cannot open output file " + a.out_file);
    auto put = [&](const std::string &text) {
        if (!text.empty() && fwrite(text.data(), 1, text.size(), o) != text.size()) die("write failed: " + a.out_file);
    };
    try {
        std::vector<DatabaseInspect> dbs(db_files.size());
        for (size_t i = 0; i < db_files.size(); i++) {
            if (inspect_db(db_files[i], dbs[i]))
                info("Database file " + db_files[i] + " processed with " + std::to_string(dbs[i].genome_files.size()) + " genomes");
            else
                warn("The database sketch `" + db_files[i] + "` is empty. Skipping...");
        }
        put(databases_yaml(dbs));
        std::vector<SampleInspect> samples;
        for (const std::string &f : sample_files) {
            samples.push_back(inspect_sample(f));
            info("Sequence file " + f + " processed");
        }
        put(samples_yaml(samples));
    } catch (const std::exception &e) { die(e.what()); }
    if (o != stdout && fclose(o) != 0) die("write failed: " + a.out_file);
    return 0;
}

int main(int argc, char **argv) {
    Args a = parse(argc, argv);
    host::inflate_threads() = std::max(1, a.threads);  // BGZF members of one file are inflated by this many threads
    if (a.cmd == "fastx-stats") return cmd_fastx_stats(a);
    if (a.cmd == "inspect") return cmd_inspect(a);
    if (a.cmd == "sample-blocks") return cmd_sample_blocks(a);
    g_parse.reset(a.threads);
    // every context exists before the first sketch call: a context's packer pool is sized by the live contexts
    std::vector<syl_ctx *> ctxs(a.devices.size(), nullptr);
    for (size_t i = 0; i < ctxs.size(); i++) {
        int rc = syl_ctx_create(a.devices[i], nullptr, &ctxs[i]);
        if (rc != SYL_OK) die(std::string("syl_ctx_create") + (a.devices.size() > 1 ? " (device " + std::to_string(a.devices[i]) + ")" : "") +
                              ": " + syl_last_error());
    }
    int rc;
    try {  // e.g. a sketch path that cannot be written, or a library error on any context: exit 1 with the message
        // contexts that share a device split its free memory for their read sketches (a sample that does not fit its share
        // is sketched in hash-range parts), as they split it for the database shards
        for (size_t i = 0; i < ctxs.size(); i++) {
            const size_t share = (size_t)std::count(a.devices.begin(), a.devices.end(), a.devices[i]);
            if (share < 2) continue;
            uint64_t free_b = 0;
            check(syl_ctx_sample_memory(ctxs[i], nullptr, &free_b), "syl_ctx_sample_memory");
            check(syl_ctx_set_sample_memory(ctxs[i], std::max<uint64_t>(1, free_b / share)), "syl_ctx_set_sample_memory");
        }
        if (a.cmd == "sketch") rc = cmd_sketch(ctxs, a);
        else if (a.cmd == "query") rc = cmd_contain(ctxs, a, false);
        else if (a.cmd == "profile") rc = cmd_contain(ctxs, a, true);
        else die("unknown command " + a.cmd + " (sketch | query | profile | inspect)");
    } catch (const std::exception &e) { die(e.what()); }
    for (syl_ctx *ctx : ctxs) syl_ctx_destroy(ctx);
    return rc;
}
