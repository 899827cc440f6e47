// sylph-b200 — host driver over libsylph_b200.so mirroring sylph's `sketch`, `query`, `profile`, `inspect`
// (src/main.rs:25-30) for the in-scope paths: single-end reads, read pairs with the exact dedup set
// (-1/-2 --fpr 0) and genomes, k in {21,31}, with sample names (-S / --lS) and list inputs (-l --rl --gl --l1 --l2).
// Files are inflated and parsed by up to -t threads at a time (the reference parallelises per file with rayon,
// src/sketch.rs:313,371,428) while the GPU works.
// File classification, defaults and TSV output follow the reference (src/cmdline.rs,
// src/sketch.rs:95-127,276-479, src/contain.rs:18-94,115-351,461-480).  All compute goes through
// the C ABI; there is no CPU path.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <future>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../include/sylph_b200.h"
#include "fastx.hpp"
#include "inspect.hpp"
#include "sketch_io.hpp"

using namespace host;

static void info(const std::string &m) { fprintf(stderr, "INFO  [sylph-b200] %s\n", m.c_str()); }
static void warn(const std::string &m) { fprintf(stderr, "WARN  [sylph-b200] %s\n", m.c_str()); }
[[noreturn]] static void die(const std::string &m) { fprintf(stderr, "ERROR [sylph-b200] %s\n", m.c_str()); exit(1); }
static void check(int rc, const char *what) {
    if (rc != SYL_OK) die(std::string(what) + ": " + syl_last_error());
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
    // test hooks (INTEGRATION.md), read once from the environment: small values make the split paths run on small inputs
    uint64_t batch_bases = 1ull << 30;  // SYL_DRIVER_BATCH_BASES: a genome batch closes once it holds this many bases
    uint64_t samples_per_call = 0;      // SYL_DRIVER_SAMPLES_PER_CALL: cap on samples per syl_query / syl_profile call (0 = none)
    uint64_t rows0 = 0;                 // SYL_DRIVER_ROWS: initial row-buffer length (0 = sized from the call)
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
        else if (s == "--device") a.device = std::stoi(need(i));
        else if (s == "-u" || s == "--estimate-unknown") a.estimate_unknown = true;
        else if (s == "-I" || s == "--read-seq-id") a.read_seq_id = std::stod(need(i));
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
    return a;
}

// ---- sketching -----------------------------------------------------------------------------------

// Inflate + parse `files` with up to `threads` of them in flight, handing them to `use` in order: the next files are
// being read while the GPU sketches the current one.
struct Parsed { bool ok = false; FlatRecords recs; std::string first_id; };
template <typename F>
static void parse_ahead(const std::vector<std::string> &files, int threads, bool want_ids, F use) {
    std::vector<std::future<std::unique_ptr<Parsed>>> inflight;
    size_t next = 0;
    auto launch = [&]() {
        const std::string f = files[next++];
        inflight.push_back(std::async(std::launch::async, [f, want_ids]() {
            std::unique_ptr<Parsed> p(new Parsed());
            p->ok = read_fastx(f, p->recs, want_ids, &p->first_id);
            return p;
        }));
    };
    for (size_t i = 0; i < files.size(); i++) {
        while (next < files.size() && inflight.size() - i < (size_t)threads) launch();
        std::unique_ptr<Parsed> p = inflight[i].get();
        use(files[i], *p);
    }
}

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
    if (!ok1 || !p2->ok) die("Paired end reading failed for '" + f1 + "' and '" + f2 + "'. Make sure the files are present or the sequences are valid.");
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

// sketches genome files in batches of <= ~1 Gbp through ONE syl_sketch_genomes call per batch
static void sketch_genome_files(syl_ctx *ctx, const Args &a, const std::vector<std::string> &files, bool pseudotax,
                                std::vector<GenomeSketch> &out) {
    // parse ahead (-t files in flight); batches of <= ~1 Gbp go through one syl_sketch_genomes call
    std::vector<std::unique_ptr<Parsed>> parsed(files.size());
    {
        size_t idx = 0;
        parse_ahead(files, a.threads, a.individual, [&](const std::string &, Parsed &p) { parsed[idx++].reset(new Parsed(std::move(p))); });
    }
    size_t fi = 0;
    while (fi < files.size()) {
        FlatRecords recs;
        std::vector<uint64_t> genome_off{0};
        std::vector<std::string> names, first_ids;
        while (fi < files.size() && recs.bases.size() < a.batch_bases) {
            const std::string &f = files[fi];
            Parsed &p = *parsed[fi++];
            // a file that fails half way contributes nothing (records are merged only after a complete parse)
            if (!p.ok) { warn(f + " is not a valid fasta/fastq file; skipping."); continue; }
            const FlatRecords &tmp = p.recs;
            const uint64_t base = recs.bases.size();
            recs.bases.insert(recs.bases.end(), tmp.bases.begin(), tmp.bases.end());
            for (size_t i = 1; i < tmp.offsets.size(); i++) recs.offsets.push_back(base + tmp.offsets[i]);
            if (!a.individual) {
                genome_off.push_back(recs.n());
                names.push_back(f);
                first_ids.push_back(p.first_id);
            } else {
                for (size_t i = 0; i < tmp.n(); i++) { names.push_back(f); first_ids.push_back(tmp.ids[i]); }
            }
            parsed[fi - 1].reset();
        }
        const uint64_t G = a.individual ? recs.n() : genome_off.size() - 1;
        if (G == 0) continue;
        syl_genomes *g = nullptr;
        check(syl_sketch_genomes(ctx, SYL_MEM_HOST, recs.bases.data(), recs.bases.size(), recs.offsets.data(), recs.n(),
                                 a.individual ? nullptr : genome_off.data(), G, (int)a.k, a.c, a.min_spacing, pseudotax ? 1 : 0,
                                 a.individual ? 1 : 0, SYL_SEM_AVX2, &g), "syl_sketch_genomes");
        std::vector<uint64_t> kmers(syl_genomes_total_kmers(g)), koff(G + 1), tracked(syl_genomes_total_tracked(g)), toff(G + 1), gs(G);
        check(syl_genomes_download(ctx, g, kmers.data(), koff.data(), tracked.data(), toff.data(), gs.data()), "syl_genomes_download");
        syl_genomes_free(g);
        for (uint64_t i = 0; i < G; i++) {
            GenomeSketch s;
            s.genome_kmers.assign(kmers.begin() + koff[i], kmers.begin() + koff[i + 1]);
            s.has_tracked = pseudotax;
            if (pseudotax) s.tracked.assign(tracked.begin() + toff[i], tracked.begin() + toff[i + 1]);
            s.file_name = names[i];
            s.first_contig_name = first_ids[i];
            s.c = a.c; s.k = a.k; s.gn_size = gs[i]; s.min_spacing = a.min_spacing;
            out.push_back(std::move(s));
        }
        info(std::to_string(out.size()) + " genomes processed.");
    }
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
    if (last.empty() || last == "..") die("Sample name `" + name + "` does not end in a file name. Exiting");
    return last;
}

static int cmd_sketch(syl_ctx *ctx, const Args &a) {
    const std::string dir = a.sample_dir.empty() || a.sample_dir.back() == '/' ? a.sample_dir : a.sample_dir + "/";
    const bool named = !a.sample_names.empty();
    // a named sketch carries its sample name and is written as <-d>/<file name of the sample name>[.paired].sylsp
    auto write_sample = [&](SequencesSketch &s, const std::string &file, size_t name, const char *suffix) {
        std::string stem = basename_of(file);
        if (named) {
            s.has_sample_name = true;
            s.sample_name = a.sample_names[name];
            stem = name_file_component(s.sample_name);
        }
        if (!dir.empty()) std::filesystem::create_directories(dir);
        const std::string path = dir + stem + suffix;
        write_sylsp(path, s);
        info("Sketching " + path + " complete.");
    };
    for (size_t i = 0; i < a.first_pairs.size(); i++) {  // src/sketch.rs:310-364
        SequencesSketch s;
        if (!sketch_pair_files(ctx, a, a.first_pairs[i], a.second_pairs[i], s)) continue;
        write_sample(s, a.first_pairs[i], i, ".paired.sylsp");
    }
    std::vector<std::string> reads;
    for (const ReadInput &r : a.sketch_reads) reads.push_back(r.file);
    size_t ri = 0;
    parse_ahead(reads, a.threads, false, [&](const std::string &f, Parsed &p) {
        const size_t name = a.sketch_reads[ri++].name;
        SequencesSketch s;
        if (!sketch_reads_parsed(ctx, a, f, p, s)) return;
        write_sample(s, f, name, ".sylsp");
    });
    const std::vector<std::string> &genomes = a.sketch_genomes;
    if (!genomes.empty()) {
        std::vector<GenomeSketch> gs;
        sketch_genome_files(ctx, a, genomes, !a.no_pseudotax, gs);
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

static int cmd_contain(syl_ctx *ctx, const Args &a, bool pseudotax) {
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
    if (!genome_files.empty()) sketch_genome_files(ctx, a, genome_files, pseudotax, gs);
    if (gs.empty()) die("No genome sketches found; see sylph query/profile -h for help. Exiting");
    for (const GenomeSketch &g : gs) if (g.k != gs[0].k) die("Query sketches have inconsistent -k. Exiting.");
    if (pseudotax && !gs[0].has_tracked)
        die("Attempting profiling, but *.syldb was sketched with the --disable-profiling option. Exiting");  // src/contain.rs:231-234
    info("Finished obtaining genome sketches.");
    // upload the db
    std::vector<uint64_t> kmers, koff{0}, tracked, toff{0}, gsz;
    uint64_t db_c = gs[0].c;
    for (const GenomeSketch &g : gs) {
        kmers.insert(kmers.end(), g.genome_kmers.begin(), g.genome_kmers.end());
        koff.push_back(kmers.size());
        tracked.insert(tracked.end(), g.tracked.begin(), g.tracked.end());
        toff.push_back(tracked.size());
        gsz.push_back(g.gn_size);
        db_c = std::min(db_c, g.c);
    }
    const bool has_tr = gs[0].has_tracked;
    syl_genomes *dg = nullptr;
    check(syl_genomes_upload(ctx, SYL_MEM_HOST, kmers.data(), koff.data(), has_tr ? tracked.data() : nullptr,
                             has_tr ? toff.data() : nullptr, gsz.data(), gs.size(), (int)gs[0].k, db_c, &dg), "syl_genomes_upload");
    syl_db *db = nullptr;
    check(syl_db_build(ctx, dg, 0, &db), "syl_db_build");
    // samples
    std::vector<syl_sample *> samples;
    std::vector<std::string> names;
    Args ra = a;
    ra.k = gs[0].k;
    if (!read_files.empty() && a.c > gs[0].c) {
        for (const std::string &f : read_files) warn(f + " error: value of -c for contain is greater than the smallest value of -c for a genome sketch. Continuing without sketching.");
        read_files.clear();
    }
    if (!read_files.empty() && a.k != gs[0].k) {  // src/contain.rs:578-584: raw reads are sketched with -k or not at all
        for (const std::string &f : read_files)
            warn(f + " -k " + std::to_string(a.k) + " is not equal to -k " + std::to_string(gs[0].k) + " found in sketches. Continuing without sketching.");
        read_files.clear();
    }
    parse_ahead(read_files, a.threads, false, [&](const std::string &f, Parsed &p) {
        if (!p.ok) { warn(f + " is not a valid fasta/fastq file; skipping."); return; }
        syl_sample *s = nullptr;
        check(syl_sketch_reads(ctx, SYL_MEM_HOST, p.recs.bases.data(), p.recs.bases.size(), p.recs.offsets.data(), p.recs.n(), (int)ra.k, a.c, 0,
                               SYL_SEM_AVX2, &s), "syl_sketch_reads");
        samples.push_back(s);
        names.push_back(f);
    });
    for (const std::string &f : sample_files) {
        SequencesSketch sk;
        try { sk = read_sylsp(f); } catch (const std::exception &e) { die(e.what()); }
        if (sk.c > gs[0].c) { warn(f + " value of -c is greater than the smallest value of -c for a genome sketch. Exiting."); continue; }
        syl_sample *s = nullptr;
        check(syl_sample_upload(ctx, SYL_MEM_HOST, sk.hashes.data(), sk.counts.data(), sk.hashes.size(), (int)sk.k, sk.c, &s), "syl_sample_upload");
        syl_sample_set_mean_read_length(s, sk.mean_read_length);
        samples.push_back(s);
        names.push_back(sk.has_sample_name ? sk.sample_name : sk.file_name);
    }
    FILE *o = a.out_file.empty() ? stdout : fopen(a.out_file.c_str(), "w");
    if (!o) die("cannot open output file " + a.out_file);
    if (!pseudotax)  // src/contain.rs:461-480
        fprintf(o, "Sample_file\tGenome_file\tAdjusted_ANI\tEff_cov\tANI_5-95_percentile\tEff_lambda\tLambda_5-95_percentile\tMedian_cov\tMean_cov_geq1\tContainment_ind\tNaive_ANI\tContig_name\n");
    else  // with -u the coverage column holds the true coverage (src/contain.rs:469-475)
        fprintf(o, "Sample_file\tGenome_file\tTaxonomic_abundance\tSequence_abundance\tAdjusted_ANI\t%s\tANI_5-95_percentile\tEff_lambda\tLambda_5-95_percentile\tMedian_cov\tMean_cov_geq1\tContainment_ind\tNaive_ANI\tkmers_reassigned\tContig_name\n",
                a.estimate_unknown ? "True_cov" : "Eff_cov");
    if (!samples.empty()) {
        syl_contain_params p;
        syl_contain_params_default(&p, (int)gs[0].k, pseudotax ? 1 : 0);
        p.no_ci = a.no_ci; p.no_adj = a.no_adj; p.mean_coverage = a.mean_cov;
        p.min_number_kmers = a.min_number_kmers; p.min_count_correct = a.min_count_correct;
        p.minimum_ani = a.min_ani; p.redundant_ani = a.redundant_ani;
        p.estimate_unknown = a.estimate_unknown ? 1 : 0; p.read_seq_id = a.read_seq_id;
        // sample batches sized so that samples x genomes stays below the library's per-call limits (2^31 pairs,
        // 8 GB of per-pair histograms = 2^23 pairs); the reference walks the samples in chunks too (src/contain.rs:239-263)
        size_t per_call = std::max<size_t>(1, std::min<size_t>(samples.size(), (size_t)((1ull << 22) / std::max<size_t>(gs.size(), 1))));
        if (a.samples_per_call) per_call = std::min<size_t>(per_call, a.samples_per_call);
        for (size_t s0 = 0; s0 < samples.size(); s0 += per_call) {
            const size_t ns = std::min(per_call, samples.size() - s0);
            std::vector<syl_ani_row> rows(a.rows0 ? a.rows0 : std::max<size_t>(1024, std::min<size_t>(gs.size() * ns, 1u << 22)));
            uint64_t n = 0;
            for (;;) {
                int rc = (pseudotax ? syl_profile : syl_query)(ctx, db, samples.data() + s0, (uint32_t)ns, &p, rows.data(), rows.size(), &n);
                if (rc == SYL_ERR_CAPACITY) { rows.resize(n); continue; }
                check(rc, pseudotax ? "syl_profile" : "syl_query");
                break;
            }
            rows.resize(n);
            size_t i = 0;
            for (uint32_t s = 0; s < ns; s++) {
                size_t j = i;
                while (j < rows.size() && rows[j].sample == s) j++;
                if (!pseudotax)  // src/contain.rs:332-334: stable sort by ANI descending
                    std::stable_sort(rows.begin() + i, rows.begin() + j,
                                     [](const syl_ani_row &x, const syl_ani_row &y) { return x.final_est_ani > y.final_est_ani; });
                for (size_t r = i; r < j; r++) print_row(o, rows[r], pseudotax, names[s0 + s], gs[rows[r].genome]);
                info("Finished sample " + names[s0 + s] + ".");
                i = j;
            }
        }
    }
    if (o != stdout) fclose(o);
    for (syl_sample *s : samples) syl_sample_free(s);
    syl_db_free(db);
    syl_genomes_free(dg);
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
    syl_ctx *ctx = nullptr;
    check(syl_ctx_create(a.device, nullptr, &ctx), "syl_ctx_create");
    int rc;
    try {  // e.g. a sketch path that cannot be written: exit 1 with the message instead of aborting
        if (a.cmd == "sketch") rc = cmd_sketch(ctx, a);
        else if (a.cmd == "query") rc = cmd_contain(ctx, a, false);
        else if (a.cmd == "profile") rc = cmd_contain(ctx, a, true);
        else die("unknown command " + a.cmd + " (sketch | query | profile | inspect)");
    } catch (const std::exception &e) { die(e.what()); }
    syl_ctx_destroy(ctx);
    return rc;
}
