// fastx.hpp — FASTA/FASTQ (+gzip via zlib, BGZF blocks inflated by several threads) reader with needletail 0.5.1's seq()/id() semantics
// as sylph uses them (src/sketch.rs:488,557,906): id = whole header line without the marker,
// seq = sequence with line endings stripped (multi-line FASTA joined), no case / alphabet
// normalisation. Records are appended to a flat base buffer + offsets, the layout the C ABI takes.
#pragma once
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace host {

struct FlatRecords {
    std::vector<uint8_t> bases;       // all sequences concatenated
    std::vector<uint64_t> offsets{0}; // n_records + 1
    std::vector<std::string> ids;     // header lines (only kept when want_ids)
    size_t n() const { return offsets.size() - 1; }
};

// Threads one file may use to inflate BGZF blocks (bgzip output: every gzip member carries its compressed size in a
// 'BC' extra field, so members can be cut out and inflated independently; src/sketch.rs:906 reads such files through
// needletail's single-threaded decoder).  Plain gzip has no such index and stays on zlib's gzread.
inline std::atomic<int> &inflate_threads() { static std::atomic<int> t{4}; return t; }

// Ordered, bounded pipeline: the consumer thread cuts blocks out of the file and hands them to worker threads; it
// takes the inflated blocks back in file order.
class BgzfSource {
  public:
    // nullptr unless the file starts with a well-formed BGZF block header
    static std::unique_ptr<BgzfSource> open(const std::string &path) {
        FILE *f = fopen(path.c_str(), "rb");
        if (!f) return nullptr;
        uint8_t h[18];
        const bool is_bgzf = fread(h, 1, 18, f) == 18 && block_size(h) > 0;
        if (!is_bgzf) { fclose(f); return nullptr; }
        fseek(f, 0, SEEK_SET);
        return std::unique_ptr<BgzfSource>(new BgzfSource(f));
    }
    ~BgzfSource() {
        { std::lock_guard<std::mutex> lk(mu_); stop_ = true; }
        cv_work_.notify_all();
        for (auto &t : workers_) t.join();
        fclose(f_);
    }
    // up to cap bytes of the inflated stream; 0 at the end of the file, -1 on a damaged block
    int read(char *buf, size_t cap) {
        for (;;) {
            if (cur_ && cur_pos_ < cur_->out.size()) {
                const size_t n = std::min(cap, cur_->out.size() - cur_pos_);
                memcpy(buf, cur_->out.data() + cur_pos_, n);
                cur_pos_ += n;
                return (int)n;
            }
            fill();
            if (inflight_.empty()) return failed_ ? -1 : 0;
            cur_ = inflight_.front();
            inflight_.pop_front();
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_done_.wait(lk, [&]() { return cur_->done; });
            }
            cur_pos_ = 0;
            if (!cur_->ok) { failed_ = true; drain(); return -1; }
        }
    }

  private:
    struct Block { std::vector<uint8_t> in; std::vector<uint8_t> out; bool done = false, ok = false; };
    // total size of the block whose first 18 bytes are h, 0 if this is not a BGZF header
    static size_t block_size(const uint8_t *h) {
        if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) return 0;
        const unsigned xlen = h[10] | (h[11] << 8);
        if (xlen < 6 || h[12] != 'B' || h[13] != 'C' || h[14] != 2 || h[15] != 0) return 0;  // bgzip writes BC first
        return (size_t)(h[16] | (h[17] << 8)) + 1;
    }
    explicit BgzfSource(FILE *f) : f_(f) {
        const int n = std::max(1, inflate_threads().load());
        for (int i = 0; i < n; i++) workers_.emplace_back([this]() { work(); });
        window_ = (size_t)n * 4;
    }
    void fill() {  // keep the window of blocks in flight full
        while (!eof_ && !failed_ && inflight_.size() < window_) {
            uint8_t h[18];
            const size_t got = fread(h, 1, 18, f_);
            if (got == 0) { eof_ = true; break; }
            const size_t bs = got == 18 ? block_size(h) : 0;
            if (bs < 26) { failed_ = true; break; }
            auto b = std::make_shared<Block>();
            b->in.resize(bs);
            memcpy(b->in.data(), h, 18);
            if (fread(b->in.data() + 18, 1, bs - 18, f_) != bs - 18) { failed_ = true; break; }
            inflight_.push_back(b);
            { std::lock_guard<std::mutex> lk(mu_); todo_.push_back(b); }
            cv_work_.notify_one();
        }
    }
    void drain() {
        std::unique_lock<std::mutex> lk(mu_);
        for (auto &b : inflight_) cv_done_.wait(lk, [&]() { return b->done; });
        inflight_.clear();
    }
    static bool inflate_block(Block &b) {
        const uint8_t *p = b.in.data();
        const size_t n = b.in.size();
        const unsigned xlen = p[10] | (p[11] << 8);
        if (n < 12u + xlen + 8u) return false;
        const uint8_t *tail = p + n - 8;
        const uint32_t crc = tail[0] | (tail[1] << 8) | (tail[2] << 16) | ((uint32_t)tail[3] << 24);
        const uint32_t isize = tail[4] | (tail[5] << 8) | (tail[6] << 16) | ((uint32_t)tail[7] << 24);
        if (isize > (1u << 16)) return false;  // BGZF blocks hold at most 64 KiB
        b.out.resize((size_t)isize + 1);  // one spare byte: the empty EOF block still needs a valid output pointer
        z_stream z;
        memset(&z, 0, sizeof z);
        if (inflateInit2(&z, -15) != Z_OK) return false;
        z.next_in = const_cast<Bytef *>(p + 12 + xlen);
        z.avail_in = (uInt)(n - 12 - xlen - 8);
        z.next_out = b.out.data();
        z.avail_out = isize + 1;
        const int rc = inflate(&z, Z_FINISH);
        const bool whole = rc == Z_STREAM_END && z.total_out == isize;
        inflateEnd(&z);
        b.out.resize(isize);
        return whole && crc32(crc32(0L, Z_NULL, 0), b.out.data(), isize) == crc;
    }
    void work() {
        for (;;) {
            std::shared_ptr<Block> b;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_work_.wait(lk, [&]() { return stop_ || !todo_.empty(); });
                if (todo_.empty()) return;
                b = todo_.front();
                todo_.pop_front();
            }
            const bool ok = inflate_block(*b);
            { std::lock_guard<std::mutex> lk(mu_); b->ok = ok; b->done = true; }
            cv_done_.notify_all();
        }
    }
    FILE *f_;
    std::vector<std::thread> workers_;
    std::mutex mu_;
    std::condition_variable cv_work_, cv_done_;
    std::deque<std::shared_ptr<Block>> todo_, inflight_;
    std::shared_ptr<Block> cur_;
    size_t cur_pos_ = 0, window_ = 4;
    bool stop_ = false, eof_ = false, failed_ = false;
};

class LineReader {
  public:
    explicit LineReader(const std::string &path) {
        if (inflate_threads().load() > 1) bgzf_ = BgzfSource::open(path);
        if (!bgzf_) {
            f_ = gzopen(path.c_str(), "rb");
            if (f_) gzbuffer(f_, 1 << 20);
        }
    }
    ~LineReader() { if (f_) gzclose(f_); }
    bool ok() const { return f_ != nullptr || bgzf_ != nullptr; }
    bool failed() const { return err_; }
    // next line without its terminator ("\n" or "\r\n"); false at EOF
    bool next(std::string &line) {
        line.clear();
        bool got = false;
        for (;;) {
            if (pos_ == len_) {
                const int n = read_some();
                if (n <= 0) {
                    if (got && !line.empty() && line.back() == '\r') line.pop_back();
                    return got;
                }
                len_ = (size_t)n;
                pos_ = 0;
            }
            got = true;
            const char *b = buf_ + pos_;
            const char *nl = (const char *)memchr(b, '\n', len_ - pos_);
            if (nl) {
                line.append(b, (size_t)(nl - b));
                pos_ += (size_t)(nl - b) + 1;
                if (!line.empty() && line.back() == '\r') line.pop_back();
                return true;
            }
            line.append(b, len_ - pos_);
            pos_ = len_;
        }
    }
    // first byte of the next line without consuming it; -1 at EOF
    int peek() {
        if (pos_ == len_ && !refill()) return -1;
        return (unsigned char)buf_[pos_];
    }
    // consume the next line, appending its bytes (without the terminator) to dst: no intermediate string.  false at EOF
    bool append_line(std::vector<uint8_t> &dst) {
        bool got = false;
        for (;;) {
            if (pos_ == len_ && !refill()) break;
            got = true;
            const char *b = buf_ + pos_;
            const char *nl = (const char *)memchr(b, '\n', len_ - pos_);
            const size_t n = nl ? (size_t)(nl - b) : len_ - pos_;
            dst.insert(dst.end(), (const uint8_t *)b, (const uint8_t *)b + n);
            pos_ += n + (nl ? 1 : 0);
            if (nl) { if (n_line_ + n > 0 && !dst.empty() && dst.back() == '\r') dst.pop_back(); n_line_ = 0; return true; }
            n_line_ += n;
        }
        if (got && n_line_ > 0 && !dst.empty() && dst.back() == '\r') dst.pop_back();
        n_line_ = 0;
        return got;
    }
    // consume the next line without keeping it; false at EOF
    bool skip_line() {
        bool got = false;
        for (;;) {
            if (pos_ == len_ && !refill()) return got;
            got = true;
            const char *b = buf_ + pos_;
            const char *nl = (const char *)memchr(b, '\n', len_ - pos_);
            if (nl) { pos_ += (size_t)(nl - b) + 1; return true; }
            pos_ = len_;
        }
    }
  private:
    // inflated bytes into buf_, 0 at the end of the file.  A damaged gzip stream / BGZF block makes the file invalid,
    // not merely shorter; so does a gzip stream cut short, which zlib reports only through gzerror's Z_BUF_ERROR
    int read_some() {
        int n = bgzf_ ? bgzf_->read(buf_, sizeof buf_) : gzread(f_, buf_, sizeof buf_);
        if (n == 0 && f_) {
            int e = Z_OK;
            gzerror(f_, &e);
            if (e == Z_BUF_ERROR) n = -1;
        }
        if (n < 0) err_ = true;
        return n;
    }
    bool refill() {
        const int n = read_some();
        if (n <= 0) return false;
        len_ = (size_t)n;
        pos_ = 0;
        return true;
    }
    size_t n_line_ = 0;  // bytes of the current line appended by earlier buffer fills (append_line)
    gzFile f_ = nullptr;
    std::unique_ptr<BgzfSource> bgzf_;
    char buf_[1 << 16];
    size_t pos_ = 0, len_ = 0;
    bool err_ = false;
};

// Appends every record of `path` to out. Returns false if the file cannot be opened or is not
// FASTA/FASTQ ("... is not a valid fasta/fastq file; skipping", src/sketch.rs:560-562).
inline bool read_fastx(const std::string &path, FlatRecords &out, bool want_ids, std::string *first_id = nullptr) {
    LineReader lr(path);
    if (!lr.ok()) return false;
    std::string line;
    if (!lr.next(line)) return false;
    while (line.empty()) if (!lr.next(line)) return false;
    bool first = true;
    if (line[0] == '>') {
        bool more = true;
        while (more) {
            if (line.empty() || line[0] != '>') return false;
            if (first && first_id) *first_id = line.substr(1);
            if (want_ids) out.ids.push_back(line.substr(1));
            first = false;
            more = false;
            for (int c0; (c0 = lr.peek()) >= 0;) {   // sequence lines go straight into the flat buffer
                if (c0 == '>') { more = lr.next(line); break; }
                lr.append_line(out.bases);
            }
            out.offsets.push_back(out.bases.size());
        }
        return !lr.failed();
    }
    if (line[0] == '@') {
        for (;;) {
            if (line.empty() || line[0] != '@') return false;
            if (first && first_id) *first_id = line.substr(1);
            if (want_ids) out.ids.push_back(line.substr(1));
            first = false;
            // a record without its sequence, '+' or quality line is an invalid file (needletail reports an
            // error for the record; sylph then drops the file, src/sketch.rs:909-915).  The sequence goes straight
            // into the flat buffer; the '+' and quality lines are skipped without being copied.
            if (!lr.append_line(out.bases) || lr.peek() != '+' || !lr.skip_line() || !lr.skip_line()) return false;
            out.offsets.push_back(out.bases.size());
            do { if (!lr.next(line)) return !lr.failed(); } while (line.empty());
        }
    }
    return false;
}

}  // namespace host
