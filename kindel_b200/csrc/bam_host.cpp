// bam_host.cpp -- host-side decode of a BAM file into the engine's flattened layout, in C++ threads.
//
// This replaces, for .bam input, the record materialisation the reference does through
// simplesam -> `samtools view` text -> one Python object per record (reference kindel/kindel.py:136-145).
// BAM's on-disk encodings (CIGAR as len<<4|op uint32, SEQ as 4-bit nibbles) are already the device layout
// described in include/kindel_b200.h, so nothing is ever turned into text:
//
//   kdl_bam_open     read the file, inflate its BGZF blocks in parallel (zlib, one block per task), parse the
//                    header (text + reference dictionary)
//   kdl_bam_prepare  index the records (the block_size chain), then in parallel: filter (kindel.py:43-46: mapped and
//                    len(seq) > 1), classify every kept record (simple / tile-eligible complex / hard, the rules of
//                    include/kindel_b200.h) and size the outputs per contig; contigs are ordered by first appearance
//                    over ALL records (kindel.py:143-151)
//   kdl_bam_fill     in parallel: write every kept record at its place -- start, lengths, CIGAR words, the packed
//                    bases byte-swapped into 32-bit words and, for complex reads, the inline block
//                    [n_ops][evt_off][ops...] behind them -- straight into caller-owned (e.g. pinned) buffers
//
// Extension: kdl_bam_set_filter (before prepare) excludes records by MAPQ / FLAG -- an excluded record is handled
// exactly like an unmapped one -- and masks bases below a Phred quality: they are written as N (nibble 15) before
// the read is classified, and kdl_bam_fill_mask lists them (the kdl_qmask of include/kindel_b200.h).  With every
// filter at 0 neither MAPQ nor QUAL is read.
//
// No GIL, no Python zlib, no numpy passes: Python only parses the @SQ text lines (the reference takes contig
// lengths from them, kindel.py:138-141) and wraps the arrays.  Ultra-long CIGARs stored in the CG:B,I tag
// (n_cigar == 2, `<l_seq>S<ref_len>N` placeholder; SAM spec 4.2.2) are taken from the tag, as samtools does.
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "../../include/kindel_b200.h"

namespace {

// KDL_BAM_TIMING=1: phase times of the decoder on stderr
struct PhaseTimer {
    const bool on = std::getenv("KDL_BAM_TIMING") != nullptr;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    void lap(const char* what) {
        if (!on) return;
        const auto t1 = std::chrono::steady_clock::now();
        std::fprintf(stderr, "[kdl_bam] %-28s %8.2f ms\n", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
        t0 = t1;
    }
};

inline int32_t rd_i32(const uint8_t* p) { int32_t v; std::memcpy(&v, p, 4); return v; }
inline uint32_t rd_u32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
inline uint16_t rd_u16(const uint8_t* p) { uint16_t v; std::memcpy(&v, p, 2); return v; }

// The decoder's worker threads live as long as the handle: the four parallel phases of one decode reuse them.
// (Spawning 64 threads per phase means ~60 stack mmaps and munmaps each time, which take the process's address-space
// lock away from the very page faults the workers are busy with.)  run(n, body): body(task_index, worker_index) for
// every task in [0, n), dynamic scheduling, the caller works too and returns when all tasks are done.
class Pool {
  public:
    explicit Pool(int threads) {
        const int extra = std::max(0, threads - 1);
        for (int t = 0; t < extra; ++t) workers_.emplace_back([this, t] { loop(t + 1); });
    }
    ~Pool() {
        {
            std::lock_guard<std::mutex> lk(m_);
            stop_ = true;
        }
        wake_.notify_all();
        for (auto& th : workers_) th.join();
    }
    Pool(const Pool&) = delete;
    Pool& operator=(const Pool&) = delete;
    int size() const { return (int)workers_.size() + 1; }

    template <class F>
    void run(int64_t n, int max_threads, F&& body) {
        if (n <= 0) return;
        const int helpers = (int)std::min<int64_t>(std::min<int64_t>((int64_t)workers_.size(), n - 1), std::max(0, max_threads - 1));
        if (helpers <= 0) {
            for (int64_t i = 0; i < n; ++i) body(i, 0);
            return;
        }
        {
            std::lock_guard<std::mutex> lk(m_);
            body_ = [&body](int64_t i, int t) { body(i, t); };
            n_ = n;
            next_.store(0, std::memory_order_relaxed);
            wanted_ = helpers;   // workers 1..helpers take part in this generation
            pending_ = helpers;
            ++gen_;
        }
        wake_.notify_all();
        drain(0);
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [this] { return pending_ == 0; });
        body_ = nullptr;
    }

  private:
    void drain(int t) {
        for (;;) {
            const int64_t i = next_.fetch_add(1, std::memory_order_relaxed);
            if (i >= n_) break;
            body_(i, t);
        }
    }
    void loop(int t) {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                wake_.wait(lk, [&] { return stop_ || (gen_ != seen && t <= wanted_); });
                if (stop_) return;
                seen = gen_;
            }
            drain(t);
            {
                std::lock_guard<std::mutex> lk(m_);
                if (--pending_ == 0) done_.notify_one();
            }
        }
    }
    std::vector<std::thread> workers_;
    std::mutex m_;
    std::condition_variable wake_, done_;
    std::function<void(int64_t, int)> body_;
    std::atomic<int64_t> next_{0};
    int64_t n_ = 0;
    uint64_t gen_ = 0;
    int wanted_ = 0, pending_ = 0;
    bool stop_ = false;
};

struct RecView {
    int32_t ref_id, pos, l_seq;
    uint32_t n_cigar, flag, mapq;
    const uint8_t* cigar;  // n_cigar uint32 words (unaligned)
    const uint8_t* seq;
    const uint8_t* qual;   // l_seq Phred bytes, nullptr if the record is too short to hold them
};

// the record filters of kdl_bam_set_filter (all 0: the reference's filter only)
struct Filter {
    uint32_t min_mapq = 0, exclude_flags = 0, min_bq = 0;
};

// Returns bytes consumed (4 + block_size) or 0 when the record is truncated / malformed.
inline int64_t parse_record(const uint8_t* p, int64_t avail, RecView* r) {
    if (avail < 36) return 0;
    const int32_t block_size = rd_i32(p);
    if (block_size < 32 || (int64_t)block_size + 4 > avail) return 0;
    const uint8_t* q = p + 4;
    r->ref_id = rd_i32(q);
    r->pos = rd_i32(q + 4);
    const uint32_t l_read_name = q[8];
    r->n_cigar = rd_u16(q + 12);
    r->flag = rd_u16(q + 14);
    r->l_seq = rd_i32(q + 16);
    if (r->l_seq < 0 || r->l_seq >= (1 << 30)) return 0;  // (the device word keeps two flag bits above the length)
    const int64_t fixed = 32 + (int64_t)l_read_name + 4ll * r->n_cigar + ((int64_t)r->l_seq + 1) / 2;
    if (fixed > block_size) return 0;
    r->mapq = q[9];
    r->cigar = q + 32 + l_read_name;
    r->seq = r->cigar + 4ll * r->n_cigar;
    r->qual = fixed + r->l_seq <= block_size ? r->seq + ((int64_t)r->l_seq + 1) / 2 : nullptr;
    // the real CIGAR of a read with more than 65535 ops lives in the CG:B,I tag behind the qualities
    if (r->n_cigar == 2) {
        const uint32_t c0 = rd_u32(r->cigar), c1 = rd_u32(r->cigar + 4);
        if ((c0 & 15u) == 4u && (int64_t)(c0 >> 4) == r->l_seq && (c1 & 15u) == 3u) {
            const uint8_t* a = r->seq + ((int64_t)r->l_seq + 1) / 2 + r->l_seq;  // aux data
            const uint8_t* end = q + block_size;
            while (a + 3 <= end) {
                const char t0 = (char)a[0], t1 = (char)a[1], ty = (char)a[2];
                a += 3;
                int64_t skip = -1;
                switch (ty) {
                    case 'A': case 'c': case 'C': skip = 1; break;
                    case 's': case 'S': skip = 2; break;
                    case 'i': case 'I': case 'f': skip = 4; break;
                    case 'Z': case 'H': { const uint8_t* z = a; while (z < end && *z) ++z; skip = (z - a) + 1; break; }
                    case 'B': {
                        if (a + 5 > end) return 4 + (int64_t)block_size;
                        const char sub = (char)a[0];
                        const uint32_t cnt = rd_u32(a + 1);
                        const int w = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
                        if (t0 == 'C' && t1 == 'G' && sub == 'I' && a + 5 + 4ll * cnt <= end) {
                            r->cigar = a + 5;
                            r->n_cigar = cnt;
                            return 4 + (int64_t)block_size;
                        }
                        skip = 5 + (int64_t)w * cnt;
                        break;
                    }
                    default: return 4 + (int64_t)block_size;  // unknown type: leave the placeholder
                }
                if (skip < 0) break;
                a += skip;
            }
        }
    }
    return 4 + (int64_t)block_size;
}

// kindel.py:43-46 (mapped and len(seq) > 1); a record the filters exclude is treated as unmapped
inline bool kept(const RecView& r, const Filter& f) {
    return !(r.flag & 0x4u) && r.l_seq > 1 && !(r.flag & f.exclude_flags) && r.mapq >= f.min_mapq;
}

// does base masking apply to this record: a threshold is set and the record has qualities (BAM: first byte != 0xff)
inline bool masks(const RecView& r, const Filter& f) { return f.min_bq > 0 && r.qual && r.l_seq > 0 && r.qual[0] != 0xff; }

// nibble mask (0xF per masked base, first base in the most significant nibble) of word k of the read's bases;
// *n += the number of masked bases
inline uint32_t qual_mask_word(const RecView& r, int64_t k, uint32_t min_bq, int64_t* n) {
    uint32_t m = 0;
    const int64_t b = 8 * k, e = std::min<int64_t>(b + 8, r.l_seq);
    for (int64_t q = b; q < e; ++q)
        if (r.qual[q] < min_bq) { m |= 0xF0000000u >> (4 * (q - b)); ++*n; }
    return m;
}

// one 32-bit word of packed bases (8 nibbles, first base in the most significant one) from BAM's byte order, with
// the nibbles of `masked` set to N; *bad |= nibbles that are not one of 1,2,4,8 (A,C,G,T) or 15 (N)
inline uint32_t seq_word(const uint8_t* seq, int64_t n_bytes_seq, int64_t k, int32_t l_seq, bool last, uint32_t* bad,
                         uint32_t masked = 0) {
    uint8_t b[4] = {0, 0, 0, 0};
    const int64_t left = n_bytes_seq - 4 * k;
    std::memcpy(b, seq + 4 * k, (size_t)(left < 4 ? left : 4));
    uint32_t v = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | b[3];
    if (last && (l_seq & 7)) v &= ~(0xFFFFFFFFu >> (4 * (l_seq & 7)));
    v |= masked;
    uint32_t chk = v;
    if (last && (l_seq & 7)) chk = v | ((0xFFFFFFFFu >> (4 * (l_seq & 7))) & 0x11111111u);  // padding counts as fine
    const uint32_t h = chk | (chk >> 1), pair = chk & (chk >> 1);
    const uint32_t two_plus = (pair | (pair >> 2) | (h & (h >> 2))) & 0x11111111u;
    const uint32_t all4 = pair & (pair >> 2) & 0x11111111u;
    const uint32_t zero = ~(h | (h >> 2)) & 0x11111111u;
    *bad |= (two_plus & ~all4) | zero;
    return v;
}

enum : uint8_t { CLS_DROP = 0, CLS_SIMPLE = 1, CLS_TILE = 2, CLS_HARD = 3 };

struct Class {
    uint8_t cls;
    uint8_t n_match;     // M/=/X ops (tile-eligible reads)
    uint16_t n_ins;      // I ops, saturating (only its sum over complex reads matters: recomputed in fill)
};

// the classification of include/kindel_b200.h (mirrors kindel_b200/bamio.py finalize), on the bases as masked by
// min_bq (0: no masking); *n_masked = masked bases
inline Class classify(const RecView& r, int64_t L, uint32_t min_bq, int64_t* reach_r, int64_t* reach_l, int64_t* aligned,
                      int64_t* n_masked) {
    Class c{CLS_HARD, 0, 0};
    const int64_t lseq = r.l_seq, start = r.pos;
    const int64_t n_bytes_seq = (lseq + 1) / 2, n_words = (lseq + 7) / 8;
    uint32_t bad = 0;
    *n_masked = 0;
    for (int64_t k = 0; k < n_words; ++k)
        seq_word(r.seq, n_bytes_seq, k, r.l_seq, k == n_words - 1, &bad, min_bq ? qual_mask_word(r, k, min_bq, n_masked) : 0);
    int64_t q_span = 0, r_span = 0, lead = 0, n_match = 0, al = 0;
    for (uint32_t o = 0; o < r.n_cigar; ++o) {
        const uint32_t cg = rd_u32(r.cigar + 4ull * o);
        const int64_t len = cg >> 4;
        const uint32_t op = cg & 15u;
        const bool m = op == 0 || op == 7 || op == 8;
        if (m) { ++n_match; al += len; }
        if (m || op == 1 || op == 4) q_span += len;
        if (m || op == 2 || (op == 4 && o > 0)) r_span += len;
        if (op == 4 && o == 0) lead = len;
    }
    *aligned = al;
    if (r.n_cigar == 1) {
        const uint32_t cg = rd_u32(r.cigar);
        const uint32_t op = cg & 15u;
        const int64_t len = cg >> 4;
        if ((op == 0 || op == 7 || op == 8) && len == lseq && start >= 0 && start + len <= L && len <= KDL_FAST_MAXLEN && !bad) {
            c.cls = CLS_SIMPLE;
            if (len > *reach_r) *reach_r = len;
            return c;
        }
    }
    const bool tile_ok = !bad && r.n_cigar <= KDL_TILE_MAXOPS && lseq <= KDL_FAST_MAXLEN && q_span <= lseq &&
                         start - lead - 1 >= 0 && start + r_span <= L - 1 && r_span + 1 <= KDL_TILE_MAXREACH &&
                         lead + 1 <= KDL_TILE_MAXREACH;
    if (tile_ok) {
        c.cls = CLS_TILE;
        c.n_match = (uint8_t)n_match;
        if (r_span + 1 > *reach_r) *reach_r = r_span + 1;
        if (lead + 1 > *reach_l) *reach_l = lead + 1;
    }
    return c;
}

// ---- SAM text -> the BAM record stream (in memory) -------------------------------------------------------------
// The reference reads SAM and BAM through the same reader (kindel.py:136-145), so the decoder takes text too: the
// lines are turned into BAM records by the worker threads and everything downstream -- filter, classification,
// layout -- is shared.  Anything this strict parser does not like (a field that is not a plain integer, an RNAME
// without @SQ line, a base outside the BAM alphabet in a read that would be used, more than 65535 CIGAR ops, header
// lines between records) makes it give up with an error; the Python caller then falls back to its own text reader,
// which raises exactly what the reference's path would.
struct SamRef { std::string name; int32_t len; };

// a carriage return inside a line (text mode would break the line there) or a non-ASCII byte (text mode would have
// to decode it): the Python reader's business
inline bool odd_bytes(const uint8_t* b, const uint8_t* e) {
    unsigned bad = 0;
    for (; b < e; ++b) bad |= (unsigned)(*b == '\r') | (unsigned)(*b >> 7);
    return bad != 0;
}

inline bool parse_int(const uint8_t* b, const uint8_t* e, int64_t* out) {
    if (b == e) return false;
    bool neg = false;
    if (*b == '+' || *b == '-') { neg = *b == '-'; ++b; }
    if (b == e || e - b > 18) return false;
    int64_t v = 0;
    for (; b < e; ++b) {
        if (*b < '0' || *b > '9') return false;
        v = v * 10 + (*b - '0');
    }
    *out = neg ? -v : v;
    return true;
}

// 255 = not a BAM base code
inline const uint8_t* base_codes() {
    static const struct Tab {
        uint8_t t[256];
        Tab() {
            std::memset(t, 255, sizeof t);
            const char* nib = "=ACMGRSVTWYHKDBN";
            for (int i = 0; i < 16; ++i) {
                t[(uint8_t)nib[i]] = (uint8_t)i;
                if (nib[i] >= 'A' && nib[i] <= 'Z') t[(uint8_t)(nib[i] + 32)] = (uint8_t)i;
            }
        }
    } tab;
    return tab.t;
}

bool looks_like_sam_text(const uint8_t* p, size_t n) {
    if (n == 0) return false;
    if (p[0] == '@') return n >= 3 && p[1] >= 'A' && p[1] <= 'Z' && p[2] >= 'A' && p[2] <= 'Z';
    const uint8_t* nl = (const uint8_t*)std::memchr(p, '\n', std::min<size_t>(n, 1 << 16));
    const uint8_t* end = nl ? nl : p + std::min<size_t>(n, 1 << 16);
    int tabs = 0;
    for (const uint8_t* q = p; q < end; ++q) {
        if (*q == '\t') ++tabs;
        else if (*q < 32 || *q > 126) return false;
    }
    return tabs >= 10;
}

// Returns KDL_OK and the BAM stream in `out`, or KDL_ERR_INVALID_ARG.  MAPQ and QUAL are carried over; a used
// record whose MAPQ is not a plain integer in 0..255 (written as 255) sets bit 0 of *odd, one whose QUAL is neither
// `*` nor one printable character per base (written as 0xff) bit 1: kdl_bam_set_filter then refuses the filters that
// would read them, and the caller's text reader decides.
int sam_text_to_bam(const uint8_t* p, size_t n, Pool& pool, int threads, std::vector<uint8_t>& out, int* odd) {
    // ---- header: the '@' lines at the top
    size_t body = 0;
    std::string text;
    std::vector<SamRef> refs;
    while (body < n && p[body] == '@') {
        const uint8_t* nl = (const uint8_t*)std::memchr(p + body, '\n', n - body);
        const size_t end = nl ? (size_t)(nl - p) : n;
        size_t le = end;
        if (le > body && p[le - 1] == '\r') --le;  // (text mode reading drops the \r of a CRLF file too)
        if (odd_bytes(p + body, p + le)) return KDL_ERR_INVALID_ARG;
        const std::string line((const char*)p + body, le - body);
        text += line;
        text += '\n';
        if (line.compare(0, 3, "@SQ") == 0) {
            std::string sn;
            int64_t ln = -1;
            bool have_sn = false;
            size_t f = line.find('\t');
            while (f != std::string::npos) {
                const size_t g = line.find('\t', f + 1);
                const std::string field = line.substr(f + 1, g == std::string::npos ? std::string::npos : g - f - 1);
                if (field.compare(0, 3, "SN:") == 0) { sn = field.substr(3); have_sn = true; }
                else if (field.compare(0, 3, "LN:") == 0) {
                    const uint8_t* b = (const uint8_t*)field.data() + 3;
                    if (!parse_int(b, (const uint8_t*)field.data() + field.size(), &ln) || ln < 0 || ln > INT32_MAX) return KDL_ERR_INVALID_ARG;
                }
                f = g;
            }
            if (have_sn && ln >= 0) {
                for (const SamRef& r : refs) if (r.name == sn) return KDL_ERR_INVALID_ARG;  // duplicate SN: not ours to resolve
                refs.push_back({sn, (int32_t)ln});
            }
        }
        body = nl ? end + 1 : n;
    }
    std::vector<std::pair<std::string, int32_t>> by_name;
    by_name.reserve(refs.size());
    for (size_t k = 0; k < refs.size(); ++k) by_name.emplace_back(refs[k].name, (int32_t)k);
    std::sort(by_name.begin(), by_name.end());
    auto ref_id_of = [&](const uint8_t* b, const uint8_t* e) -> int32_t {  // -1: '*', -2: unknown
        if (e - b == 1 && *b == '*') return -1;
        const std::string key((const char*)b, (size_t)(e - b));
        auto it = std::lower_bound(by_name.begin(), by_name.end(), std::make_pair(key, (int32_t)INT32_MIN));
        return (it != by_name.end() && it->first == key) ? it->second : -2;
    };
    // ---- records: byte ranges that end at line ends, one output vector per range
    if (threads < 1) threads = 1;
    const size_t len = n - body;
    int64_t n_tasks = std::min<int64_t>(std::max<int64_t>(1, (int64_t)(len / (256 << 10))), (int64_t)threads * 4);
    std::vector<size_t> cut((size_t)n_tasks + 1);
    cut[0] = body;
    for (int64_t t = 1; t < n_tasks; ++t) {
        size_t at = body + len * (size_t)t / (size_t)n_tasks;
        if (at < cut[(size_t)t - 1]) at = cut[(size_t)t - 1];
        const uint8_t* nl = at < n ? (const uint8_t*)std::memchr(p + at, '\n', n - at) : nullptr;
        cut[(size_t)t] = nl ? (size_t)(nl - p) + 1 : n;
    }
    cut[(size_t)n_tasks] = n;
    std::vector<std::vector<uint8_t>> part((size_t)n_tasks);
    std::atomic<int> failed{0}, odd_fields{0};
    const uint8_t* code = base_codes();
    pool.run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<uint8_t>& o = part[(size_t)t];
        o.reserve((cut[(size_t)t + 1] - cut[(size_t)t]) / 2 + 64);
        std::vector<uint32_t> ops;
        size_t at = cut[(size_t)t];
        const size_t stop = cut[(size_t)t + 1];
        while (at < stop) {
            const uint8_t* nl = (const uint8_t*)std::memchr(p + at, '\n', stop - at);
            size_t end = nl ? (size_t)(nl - p) : stop;
            const size_t next = nl ? end + 1 : stop;
            if (end > at && p[end - 1] == '\r') --end;
            if (odd_bytes(p + at, p + end)) { failed = 1; return; }
            if (end > at && p[at] == '@') { failed = 1; return; }  // a header line between records: the text reader's case
            const uint8_t* f[12];
            int nf = 0;
            f[nf++] = p + at;
            for (const uint8_t* q = p + at; q < p + end && nf < 12; ++q)
                if (*q == '\t') f[nf++] = q + 1;
            if (nf < 11) { at = next; continue; }  // not a record line (the text reader skips it too)
            auto fe = [&](int k) { return k + 1 < nf ? f[k + 1] - 1 : p + end; };  // end of field k (nf <= 12: field 11+ unused)
            int64_t flag, pos;
            if (!parse_int(f[1], fe(1), &flag) || !parse_int(f[3], fe(3), &pos) || flag < 0 || flag > 0xFFFF ||
                pos < INT32_MIN + 1ll || pos > INT32_MAX) { failed = 1; return; }
            const int32_t ref_id = ref_id_of(f[2], fe(2));
            if (ref_id == -2) { failed = 1; return; }  // RNAME without @SQ line: KeyError in the reference
            const uint8_t* sq = f[9];
            const int64_t slen = fe(9) - f[9];
            const bool used = ref_id >= 0 && !(flag & 4) && slen > 1;  // (kindel.py:43-46, :147-148)
            ops.clear();
            int64_t l_seq = 0;
            if (used) {
                const uint8_t* c = f[5];
                const uint8_t* ce = fe(5);
                if (!(ce - c == 1 && *c == '*')) {
                    int64_t num = 0;
                    for (; c < ce; ++c) {
                        if (*c >= '0' && *c <= '9') {
                            num = num * 10 + (*c - '0');
                            if (num >= (1ll << 28)) { failed = 1; return; }
                        } else {
                            if (*c >= 128) { failed = 1; return; }
                            const char* opc = "MIDNSHP=X";
                            const char* hit = (const char*)std::memchr(opc, *c, 9);
                            ops.push_back((uint32_t)(num << 4) | (hit ? (uint32_t)(hit - opc) : 15u));  // unknown op letters are no-ops
                            num = 0;
                        }
                    }
                }
                if (ops.size() > 65535) { failed = 1; return; }
                l_seq = slen;
            }
            int64_t mapq = 255;
            const uint8_t* qt = nullptr;  // QUAL text of a used record, nullptr for `*` or a malformed one
            if (used) {
                if (!parse_int(f[4], fe(4), &mapq) || mapq < 0 || mapq > 255) { mapq = 255; odd_fields |= 1; }
                const int64_t qlen = fe(10) - f[10];
                if (!(qlen == 1 && *f[10] == '*')) {
                    bool ok = qlen == l_seq;
                    for (const uint8_t* c = f[10]; ok && c < fe(10); ++c) ok = *c >= 33 && *c <= 126;
                    if (ok) qt = f[10];
                    else odd_fields |= 2;
                }
            }
            // QNAME, RNEXT and PNEXT travel as BAM keeps them (the mates of `--mask-overlaps` read them); an RNEXT
            // without @SQ line or a PNEXT that is no integer in 0..2^31-1 says "no mate on this contig": -1
            const int64_t l_name = fe(0) - f[0];
            if (l_name > 254) { failed = 1; return; }
            int32_t next_ref = -1, next_pos = -1;
            if (fe(6) - f[6] == 1 && *f[6] == '=') next_ref = ref_id;
            else if (ref_id_of(f[6], fe(6)) >= 0) next_ref = ref_id_of(f[6], fe(6));
            int64_t pnext;
            if (parse_int(f[7], fe(7), &pnext) && pnext >= 0 && pnext <= INT32_MAX) next_pos = (int32_t)(pnext - 1);
            const int64_t seq_bytes = (l_seq + 1) / 2;
            const int64_t block_size = 32 + (l_name + 1) + 4 * (int64_t)ops.size() + seq_bytes + l_seq;
            if (block_size > (1ll << 28)) { failed = 1; return; }
            const size_t base = o.size();
            o.resize(base + 4 + (size_t)block_size);
            uint8_t* w = o.data() + base;
            const int32_t bs32 = (int32_t)block_size, pos0 = (int32_t)(pos - 1), lseq32 = (int32_t)l_seq, zero = 0;
            const uint16_t ncig = (uint16_t)ops.size(), flag16 = (uint16_t)flag, bin = 4680;
            std::memcpy(w, &bs32, 4);
            std::memcpy(w + 4, &ref_id, 4);
            std::memcpy(w + 8, &pos0, 4);
            w[12] = (uint8_t)(l_name + 1); w[13] = (uint8_t)mapq;  // l_read_name (with its NUL), mapq
            std::memcpy(w + 14, &bin, 2);
            std::memcpy(w + 16, &ncig, 2);
            std::memcpy(w + 18, &flag16, 2);
            std::memcpy(w + 20, &lseq32, 4);
            std::memcpy(w + 24, &next_ref, 4);
            std::memcpy(w + 28, &next_pos, 4);
            std::memcpy(w + 32, &zero, 4);
            if (l_name) std::memcpy(w + 36, f[0], (size_t)l_name);
            w[36 + l_name] = 0;                                   // read name
            uint8_t* q = w + 37 + l_name;
            if (!ops.empty()) std::memcpy(q, ops.data(), 4 * ops.size());
            q += 4 * ops.size();
            for (int64_t k = 0; k < l_seq; k += 2) {
                const uint8_t hi = code[sq[k]], lo = k + 1 < l_seq ? code[sq[k + 1]] : 0;
                if (hi == 255 || lo == 255) { failed = 1; return; }  // cannot be packed in 4 bits: ValueError upstairs
                *q++ = (uint8_t)(hi << 4 | lo);
            }
            if (qt) for (int64_t k = 0; k < l_seq; ++k) q[k] = (uint8_t)(qt[k] - 33);
            else std::memset(q, 0xff, (size_t)l_seq);
            at = next;
        }
    });
    if (failed) return KDL_ERR_INVALID_ARG;
    *odd |= odd_fields.load();
    // ---- header + dictionary + the parts, back to back
    size_t total = 12 + text.size();
    for (const SamRef& r : refs) total += 8 + r.name.size() + 1;
    std::vector<size_t> at((size_t)n_tasks + 1);
    at[0] = total;
    for (int64_t t = 0; t < n_tasks; ++t) at[(size_t)t + 1] = at[(size_t)t] + part[(size_t)t].size();
    out.resize(at[(size_t)n_tasks]);
    uint8_t* w = out.data();
    std::memcpy(w, "BAM\1", 4);
    const int32_t l_text = (int32_t)text.size(), n_ref = (int32_t)refs.size();
    std::memcpy(w + 4, &l_text, 4);
    std::memcpy(w + 8, text.data(), text.size());
    w += 8 + text.size();
    std::memcpy(w, &n_ref, 4);
    w += 4;
    for (const SamRef& r : refs) {
        const int32_t l_name = (int32_t)r.name.size() + 1;
        std::memcpy(w, &l_name, 4);
        std::memcpy(w + 4, r.name.c_str(), (size_t)l_name);
        std::memcpy(w + 4 + l_name, &r.len, 4);
        w += 8 + l_name;
    }
    pool.run(n_tasks, threads, [&](int64_t t, int) {
        if (!part[(size_t)t].empty()) std::memcpy(out.data() + at[(size_t)t], part[(size_t)t].data(), part[(size_t)t].size());
    });
    return KDL_OK;
}

}  // namespace

struct kdl_bam {
    std::vector<uint8_t> data;          // the inflated BAM byte stream (plain gzip / uncompressed input) ...
    std::unique_ptr<uint8_t[]> big;     // ... or, for BGZF, an UNINITIALISED buffer the inflating threads first-touch
    const uint8_t* dptr = nullptr;
    int64_t dsize = 0;
    int64_t first_record = 0;
    std::string text;                   // header text
    std::vector<std::string> ref_name;
    std::vector<int32_t> ref_len;       // binary dictionary lengths (Python may override from the @SQ text)
    // after prepare
    std::vector<int64_t> rec_off;       // offset of every record (+ end)
    std::vector<Class> cls;             // per record
    std::vector<int32_t> order;         // contigs (ref ids) in first-seen order
    std::vector<int64_t> read_off, op_off, word_off;  // per ordered contig (+ total)
    std::vector<int64_t> chunk_lo;      // record ranges of the parallel tasks
    std::vector<int64_t> cur_read, cur_op, cur_word;   // [task][n_ref] start cursors
    Filter filter;                      // kdl_bam_set_filter
    int sam_odd = 0;                    // SAM text input: bit 0 odd MAPQ, bit 1 odd QUAL seen (sam_text_to_bam)
    std::vector<uint32_t> n_masked;     // per record, only when filter.min_bq > 0
    std::vector<int64_t> cur_mread, cur_mbase;  // [task][n_ref] start cursors of the mask list
    int64_t masked_bases = 0, masked_reads = 0;
    int64_t no_qual = 0;                // kept reads without qualities (BAM 0xff, SAM `*`)
    int64_t n_records = 0, n_kept = 0, n_complex = 0, n_hard = 0, aligned = 0, n_events = 0;
    int64_t reach_right = 0, reach_left = 0, max_simple = 0;
    int32_t reads_sorted = 1;
    bool prepared = false;
    std::unique_ptr<Pool> pool;         // the worker threads of this handle (created by kdl_bam_open)
};

extern "C" {

// Reads and inflates `path` (BGZF, plain gzip members, or an uncompressed BAM stream) with `threads` threads and
// parses the header.  Returns KDL_OK, KDL_ERR_INVALID_ARG for a file that is not a BAM.
int kdl_bam_open(const char* path, int threads, kdl_bam** out) {
    if (!path || !out) return KDL_ERR_INVALID_ARG;
    *out = nullptr;
    PhaseTimer pt;
    FILE* fh = std::fopen(path, "rb");
    if (!fh) return KDL_ERR_INVALID_ARG;
    std::vector<uint8_t> raw;
    {
        std::fseek(fh, 0, SEEK_END);
        const long sz = std::ftell(fh);
        std::fseek(fh, 0, SEEK_SET);
        if (sz < 0) { std::fclose(fh); return KDL_ERR_INVALID_ARG; }
        raw.resize((size_t)sz);
        if (sz && std::fread(raw.data(), 1, (size_t)sz, fh) != (size_t)sz) { std::fclose(fh); return KDL_ERR_INVALID_ARG; }
        std::fclose(fh);
    }
    pt.lap("open: read file");
    kdl_bam* h = new (std::nothrow) kdl_bam();
    if (!h) return KDL_ERR_INVALID_ARG;
    h->pool.reset(new Pool(threads < 1 ? 1 : threads));
    const size_t n = raw.size();
    if (n >= 4 && !std::memcmp(raw.data(), "BAM\1", 4)) {
        h->data.swap(raw);
    } else if (looks_like_sam_text(raw.data(), n)) {
        if (sam_text_to_bam(raw.data(), n, *h->pool, threads, h->data, &h->sam_odd) != KDL_OK) { delete h; return KDL_ERR_INVALID_ARG; }
        pt.lap("open: SAM text -> records");
    } else {
        // BGZF: gzip members with a BC extra field holding the block size; the chain of headers is walked
        // sequentially (cheap), the payloads are inflated in parallel at their prefix-summed offsets
        struct Blk { size_t pay, pay_len, out_off; uint32_t isize; };
        std::vector<Blk> blks;
        size_t off = 0, total = 0;
        bool bgzf = true;
        while (off < n) {
            if (n - off < 18 || raw[off] != 0x1f || raw[off + 1] != 0x8b || raw[off + 2] != 8 || !(raw[off + 3] & 4)) { bgzf = false; break; }
            const size_t xlen = rd_u16(&raw[off + 10]);
            size_t p = off + 12, end_x = off + 12 + xlen;
            long bsize = -1;
            if (end_x > n) { bgzf = false; break; }
            while (p + 4 <= end_x) {
                const uint8_t si1 = raw[p], si2 = raw[p + 1];
                const size_t slen = rd_u16(&raw[p + 2]);
                if (si1 == 66 && si2 == 67 && slen == 2 && p + 6 <= end_x) bsize = rd_u16(&raw[p + 4]);
                p += 4 + slen;
            }
            if (bsize < 0 || off + (size_t)bsize + 1 > n || (size_t)bsize + 1 < end_x - off + 8) { bgzf = false; break; }
            const size_t blk_end = off + (size_t)bsize + 1;
            const uint32_t isize = rd_u32(&raw[blk_end - 4]);
            blks.push_back({end_x, blk_end - 8 - end_x, total, isize});
            total += isize;
            off = blk_end;
        }
        if (!bgzf) {  // a plain gzip stream (or garbage): one sequential inflate
            z_stream zs;
            std::memset(&zs, 0, sizeof zs);
            if (inflateInit2(&zs, 15 + 32) != Z_OK) { delete h; return KDL_ERR_INVALID_ARG; }
            zs.next_in = raw.data();
            zs.avail_in = (uInt)n;
            std::vector<uint8_t> outb(std::max<size_t>(n * 4, 1 << 16));
            size_t have = 0;
            int rc = Z_OK;
            while (rc != Z_STREAM_END) {
                if (have == outb.size()) outb.resize(outb.size() * 2);
                zs.next_out = outb.data() + have;
                zs.avail_out = (uInt)std::min<size_t>(outb.size() - have, 1u << 30);
                const size_t before = zs.avail_out;
                rc = inflate(&zs, Z_NO_FLUSH);
                have += before - zs.avail_out;
                if (rc == Z_STREAM_END && zs.avail_in > 0) {  // concatenated members
                    if (inflateReset(&zs) != Z_OK) break;
                    rc = Z_OK;
                    continue;
                }
                if (rc != Z_OK && rc != Z_STREAM_END) break;
                if (rc == Z_OK && zs.avail_in == 0 && before == zs.avail_out) break;
            }
            inflateEnd(&zs);
            outb.resize(have);
            h->data.swap(outb);
        } else {
            pt.lap("open: BGZF header chain");
            h->big.reset(new (std::nothrow) uint8_t[total ? total : 1]);
            if (!h->big) { delete h; return KDL_ERR_INVALID_ARG; }
            h->dptr = h->big.get();
            h->dsize = (int64_t)total;
            std::atomic<int> failed{0};
            h->pool->run((int64_t)blks.size(), threads, [&](int64_t i, int) {
                const Blk& b = blks[(size_t)i];
                if (!b.isize) return;
                z_stream zs;
                std::memset(&zs, 0, sizeof zs);
                if (inflateInit2(&zs, -15) != Z_OK) { failed = 1; return; }
                zs.next_in = raw.data() + b.pay;
                zs.avail_in = (uInt)b.pay_len;
                zs.next_out = h->big.get() + b.out_off;
                zs.avail_out = b.isize;
                const int rc = inflate(&zs, Z_FINISH);
                if (rc != Z_STREAM_END || zs.avail_out != 0) failed = 1;
                inflateEnd(&zs);
            });
            if (failed) { delete h; return KDL_ERR_INVALID_ARG; }
            pt.lap("open: inflate (threads)");
        }
    }
    if (!h->dptr) { h->dptr = h->data.data(); h->dsize = (int64_t)h->data.size(); }
    if (h->dsize > 0 && std::memcmp(h->dptr, "BAM\1", h->dsize < 4 ? (size_t)h->dsize : 4) != 0 &&
        looks_like_sam_text(h->dptr, (size_t)h->dsize)) {  // gzip-compressed SAM text
        std::vector<uint8_t> conv;
        if (sam_text_to_bam(h->dptr, (size_t)h->dsize, *h->pool, threads, conv, &h->sam_odd) != KDL_OK) { delete h; return KDL_ERR_INVALID_ARG; }
        h->data.swap(conv);
        h->big.reset();
        h->dptr = h->data.data();
        h->dsize = (int64_t)h->data.size();
    }
    const uint8_t* d = h->dptr;
    const int64_t dn = h->dsize;
    if (dn < 12 || std::memcmp(d, "BAM\1", 4)) { delete h; return KDL_ERR_INVALID_ARG; }
    const int64_t l_text = rd_i32(&d[4]);
    if (l_text < 0 || 8 + l_text + 4 > dn) { delete h; return KDL_ERR_INVALID_ARG; }
    h->text.assign((const char*)&d[8], (size_t)l_text);
    const size_t nul = h->text.find('\0');
    if (nul != std::string::npos) h->text.resize(nul);
    int64_t off = 8 + l_text;
    const int64_t n_ref = rd_i32(&d[(size_t)off]);
    off += 4;
    if (n_ref < 0) { delete h; return KDL_ERR_INVALID_ARG; }
    for (int64_t k = 0; k < n_ref; ++k) {
        if (off + 4 > dn) { delete h; return KDL_ERR_INVALID_ARG; }
        const int64_t l_name = rd_i32(&d[(size_t)off]);
        if (l_name < 1 || off + 8 + l_name > dn) { delete h; return KDL_ERR_INVALID_ARG; }
        h->ref_name.emplace_back((const char*)&d[(size_t)off + 4], (size_t)l_name - 1);
        h->ref_len.push_back(rd_i32(&d[(size_t)(off + 4 + l_name)]));
        off += 8 + l_name;
    }
    h->first_record = off;
    *out = h;
    return KDL_OK;
}

void kdl_bam_close(kdl_bam* h) { delete h; }

const char* kdl_bam_header_text(const kdl_bam* h, int64_t* len) {
    if (!h) return nullptr;
    if (len) *len = (int64_t)h->text.size();
    return h->text.c_str();
}
int32_t kdl_bam_n_ref(const kdl_bam* h) { return h ? (int32_t)h->ref_name.size() : 0; }
const char* kdl_bam_ref_name(const kdl_bam* h, int32_t ref_id) {
    return (h && ref_id >= 0 && ref_id < (int32_t)h->ref_name.size()) ? h->ref_name[(size_t)ref_id].c_str() : nullptr;
}
int32_t kdl_bam_ref_len(const kdl_bam* h, int32_t ref_id) {
    return (h && ref_id >= 0 && ref_id < (int32_t)h->ref_len.size()) ? h->ref_len[(size_t)ref_id] : -1;
}

// Record / base filters for the next kdl_bam_prepare (extension; all 0 = the reference's filter only):
// MAPQ < min_mapq or FLAG & exclude_flags -> the record is treated as unmapped; Phred quality < min_base_quality ->
// the base is masked (N in seq4, listed by kdl_bam_fill_mask).  KDL_ERR_INVALID_ARG for values out of range, or when
// SAM text input had a MAPQ (QUAL) field this decoder could not carry and min_mapq (min_base_quality) is set.
int kdl_bam_set_filter(kdl_bam* h, int32_t min_mapq, int32_t exclude_flags, int32_t min_base_quality) {
    if (!h || min_mapq < 0 || min_mapq > 255 || exclude_flags < 0 || exclude_flags > 0xFFFF || min_base_quality < 0 ||
        min_base_quality > 255)
        return KDL_ERR_INVALID_ARG;
    if ((min_mapq > 0 && (h->sam_odd & 1)) || (min_base_quality > 0 && (h->sam_odd & 2))) return KDL_ERR_INVALID_ARG;
    h->filter.min_mapq = (uint32_t)min_mapq;
    h->filter.exclude_flags = (uint32_t)exclude_flags;
    h->filter.min_bq = (uint32_t)min_base_quality;
    h->prepared = false;
    return KDL_OK;
}

// ref_len[n_ref]: the contig lengths to classify against (the @SQ text's LN, as the reference uses; NULL = the binary
// dictionary's).  info[16] out: 0 records, 1 kept reads, 2 contigs seen, 3 CIGAR ops of kept reads, 4 words of the
// read stream, 5 complex reads, 6 hard reads, 7 aligned bases, 8 insertion events, 9 reach_right, 10 reach_left,
// 11 longest simple read, 12 reads_sorted (valid after kdl_bam_fill), 13 masked bases, 14 reads with masked bases,
// 15 kept reads without qualities.
int kdl_bam_prepare(kdl_bam* h, const int32_t* ref_len, int threads, int64_t* info) {
    if (!h || !info) return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int64_t n_bytes = h->dsize;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    if (ref_len) h->ref_len.assign(ref_len, ref_len + n_ref);
    PhaseTimer pt;
    // ---- records are found, filtered, classified and counted in ONE parallel pass over byte ranges of the stream.
    // The block_size chain is sequential by nature, so every task but the first GUESSES its first record boundary
    // (the first offset from which three consecutive plausible records follow); afterwards the chain is verified
    // task by task -- a task whose guess is not where its predecessor's walk ended is simply walked again from there
    // -- so the result never depends on the guess.  Tasks are byte ranges in file order, hence contiguous record
    // ranges: "file order inside a contig" is task order then record order.
    if (threads < 1) threads = 1;
    const int64_t body = n_bytes - h->first_record;
    if (body < 0) return KDL_ERR_INVALID_ARG;
    int64_t n_tasks = std::min<int64_t>(std::max<int64_t>(1, body / (256 << 10)), (int64_t)threads * 4);
    if ((int64_t)n_ref * n_tasks > (1ll << 24)) n_tasks = std::max<int64_t>(1, (1ll << 24) / std::max(1, n_ref));  // bound the cursor tables
    std::vector<int64_t> byte_lo((size_t)n_tasks + 1);
    for (int64_t t = 0; t <= n_tasks; ++t) byte_lo[(size_t)t] = h->first_record + body * t / n_tasks;
    struct Acc { int64_t kept = 0, ops = 0, words = 0, first = -1, mreads = 0, mbases = 0; };  // first: record index inside the task
    const size_t row = (size_t)std::max(1, n_ref);
    std::vector<Acc> acc((size_t)n_tasks * row);
    struct Tot { int64_t cx = 0, hard = 0, aligned = 0, rr = 0, rl = 0, ms = 0, noq = 0; };
    struct Task { std::vector<int64_t> off; std::vector<Class> cls; std::vector<uint32_t> nm; Tot tot; int64_t start = -1, end = -1; bool bad = false; };
    const Filter flt = h->filter;
    std::vector<Task> task((size_t)n_tasks);
    auto plausible = [&](int64_t off) -> int64_t {  // length of a believable record at `off`, 0 if none
        if (n_bytes - off < 36) return 0;
        const uint8_t* q = d + off + 4;
        const int64_t bs = rd_i32(d + off);
        if (bs < 32 || bs > (1 << 28) || off + 4 + bs > n_bytes) return 0;
        const int32_t ref_id = rd_i32(q), pos = rd_i32(q + 4), l_seq = rd_i32(q + 16), next_ref = rd_i32(q + 20), next_pos = rd_i32(q + 24);
        const int64_t l_name = q[8], n_cig = rd_u16(q + 12);
        if (ref_id < -1 || ref_id >= n_ref || pos < -1 || next_ref < -1 || next_ref >= n_ref || next_pos < -1 || l_seq < 0 || l_name < 1) return 0;
        if (32 + l_name + 4 * n_cig + ((int64_t)l_seq + 1) / 2 + l_seq > bs) return 0;
        if (q[32 + l_name - 1] != 0) return 0;  // the read name is NUL-terminated
        return 4 + bs;
    };
    auto guess = [&](int64_t lo, int64_t hi) -> int64_t {  // first offset in [lo, hi) that starts three plausible records
        for (int64_t o = lo; o < hi; ++o) {
            int64_t p = o;
            int k = 0;
            for (; k < 3 && p < n_bytes; ++k) {
                const int64_t len = plausible(p);
                if (!len) break;
                p += len;
            }
            if (k == 3 || (k > 0 && p == n_bytes)) return o;
        }
        return -1;
    };
    auto walk = [&](int64_t t, int64_t start) {  // the records that START in [start, byte_lo[t + 1])
        Task& tk = task[(size_t)t];
        Acc* a = acc.data() + (size_t)t * row;
        for (size_t c = 0; c < row; ++c) a[c] = Acc{};
        tk.off.clear(); tk.cls.clear(); tk.nm.clear(); tk.tot = Tot{}; tk.bad = false;
        tk.start = start;
        const int64_t stop = byte_lo[(size_t)t + 1];
        const int64_t expect = (stop - start) / 96 + 16;
        tk.off.reserve((size_t)expect); tk.cls.reserve((size_t)expect);
        RecView r;
        int64_t off = start;
        while (off < stop) {
            const int64_t used = parse_record(d + off, n_bytes - off, &r);
            if (!used || r.ref_id >= n_ref) { tk.bad = true; break; }
            Class c{CLS_DROP, 0, 0};
            int64_t nm = 0;
            if (r.ref_id >= 0) {  // rname '*' is dropped wholesale (kindel.py:147-148)
                Acc& ac = a[r.ref_id];
                if (ac.first < 0) ac.first = (int64_t)tk.off.size();
                if (kept(r, flt)) {
                    int64_t rr = 0, rl = 0, al = 0;
                    c = classify(r, h->ref_len[(size_t)r.ref_id], masks(r, flt) ? flt.min_bq : 0, &rr, &rl, &al, &nm);
                    ac.kept += 1;
                    if (nm) { ac.mreads += 1; ac.mbases += nm; }
                    ac.ops += r.n_cigar;
                    ac.words += ((int64_t)r.l_seq + 7) / 8 + (c.cls == CLS_SIMPLE ? 0 : 2 + (int64_t)r.n_cigar);
                    tk.tot.aligned += al;
                    if (!r.qual || r.qual[0] == 0xff) tk.tot.noq += 1;  // a kept read without qualities
                    if (c.cls != CLS_SIMPLE) tk.tot.cx += 1;
                    if (c.cls == CLS_HARD) tk.tot.hard += 1;
                    if (c.cls == CLS_SIMPLE && rr > tk.tot.ms) tk.tot.ms = rr;
                    if (c.cls != CLS_HARD) { tk.tot.rr = std::max(tk.tot.rr, rr); tk.tot.rl = std::max(tk.tot.rl, rl); }
                }
            }
            tk.off.push_back(off);
            tk.cls.push_back(c);
            if (flt.min_bq) tk.nm.push_back((uint32_t)nm);
            off += used;
        }
        tk.end = off;
    };
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        const int64_t start = t == 0 ? h->first_record : guess(byte_lo[(size_t)t], byte_lo[(size_t)t + 1]);
        if (start >= 0) walk(t, start);
    });
    pt.lap("prepare: walk + classify (threads)");
    {   // verify the chain; repair what was guessed wrong
        int64_t expected = h->first_record;
        for (int64_t t = 0; t < n_tasks; ++t) {
            Task& tk = task[(size_t)t];
            if (expected >= byte_lo[(size_t)t + 1]) {  // no record starts inside this range
                if (tk.start >= 0) walk(t, byte_lo[(size_t)t + 1]);  // (empties it)
                tk.start = tk.end = expected;
                continue;
            }
            if (tk.start != expected) walk(t, expected);
            if (tk.bad) return KDL_ERR_INVALID_ARG;
            expected = tk.end;
        }
        if (expected != n_bytes) return KDL_ERR_INVALID_ARG;
    }
    h->chunk_lo.assign((size_t)n_tasks + 1, 0);
    for (int64_t t = 0; t < n_tasks; ++t) h->chunk_lo[(size_t)t + 1] = h->chunk_lo[(size_t)t] + (int64_t)task[(size_t)t].off.size();
    const int64_t n_rec = h->chunk_lo[(size_t)n_tasks];
    h->n_records = n_rec;
    h->rec_off.resize((size_t)n_rec + 1);
    h->cls.resize((size_t)n_rec);
    h->n_masked.assign(flt.min_bq ? (size_t)n_rec : 0, 0);
    h->rec_off[(size_t)n_rec] = n_bytes;
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        const Task& tk = task[(size_t)t];
        const size_t base = (size_t)h->chunk_lo[(size_t)t];
        if (!tk.off.empty()) {
            std::memcpy(h->rec_off.data() + base, tk.off.data(), tk.off.size() * sizeof(int64_t));
            std::memcpy(h->cls.data() + base, tk.cls.data(), tk.cls.size() * sizeof(Class));
            if (flt.min_bq) std::memcpy(h->n_masked.data() + base, tk.nm.data(), tk.nm.size() * sizeof(uint32_t));
        }
        Acc* a = acc.data() + (size_t)t * row;
        for (size_t c = 0; c < row; ++c)
            if (a[c].first >= 0) a[c].first += (int64_t)base;  // -> index over all records
    });
    pt.lap("prepare: verify + gather");
    h->n_complex = h->n_hard = h->aligned = h->no_qual = 0;
    h->reach_right = h->reach_left = h->max_simple = 0;
    for (const Task& tk : task) {
        const Tot& tt = tk.tot;
        h->n_complex += tt.cx; h->n_hard += tt.hard; h->aligned += tt.aligned; h->no_qual += tt.noq;
        h->reach_right = std::max(h->reach_right, tt.rr); h->reach_left = std::max(h->reach_left, tt.rl);
        h->max_simple = std::max(h->max_simple, tt.ms);
    }
    // ---- contigs in first-seen order, sizes per contig, start cursors per (task, contig)
    std::vector<int64_t> first((size_t)std::max(1, n_ref), -1), kept_c((size_t)std::max(1, n_ref), 0),
        ops_c((size_t)std::max(1, n_ref), 0), words_c((size_t)std::max(1, n_ref), 0),
        mreads_c((size_t)std::max(1, n_ref), 0), mbases_c((size_t)std::max(1, n_ref), 0);
    for (int64_t t = 0; t < n_tasks; ++t)
        for (int32_t c = 0; c < n_ref; ++c) {
            const Acc& ac = acc[(size_t)t * (size_t)n_ref + (size_t)c];
            if (ac.first >= 0 && (first[(size_t)c] < 0 || ac.first < first[(size_t)c])) first[(size_t)c] = ac.first;
            kept_c[(size_t)c] += ac.kept; ops_c[(size_t)c] += ac.ops; words_c[(size_t)c] += ac.words;
            mreads_c[(size_t)c] += ac.mreads; mbases_c[(size_t)c] += ac.mbases;
        }
    h->order.clear();
    for (int32_t c = 0; c < n_ref; ++c) if (first[(size_t)c] >= 0) h->order.push_back(c);
    std::sort(h->order.begin(), h->order.end(), [&](int32_t a, int32_t b) { return first[(size_t)a] < first[(size_t)b]; });
    const size_t ns = h->order.size();
    h->read_off.assign(ns + 1, 0); h->op_off.assign(ns + 1, 0); h->word_off.assign(ns + 1, 0);
    for (size_t k = 0; k < ns; ++k) {
        const size_t c = (size_t)h->order[k];
        h->read_off[k + 1] = h->read_off[k] + kept_c[c];
        h->op_off[k + 1] = h->op_off[k] + ops_c[c];
        h->word_off[k + 1] = h->word_off[k] + words_c[c];
    }
    h->n_kept = h->read_off[ns];
    if (h->word_off[ns] >= (1ll << 32) || h->op_off[ns] >= (1ll << 32) || h->n_kept >= (1ll << 31)) return KDL_ERR_INVALID_ARG;
    const size_t tab = (size_t)n_tasks * (size_t)std::max(1, n_ref);
    h->cur_read.assign(tab, 0); h->cur_op.assign(tab, 0); h->cur_word.assign(tab, 0);
    h->cur_mread.assign(flt.min_bq ? tab : 0, 0); h->cur_mbase.assign(flt.min_bq ? tab : 0, 0);
    int64_t mr = 0, mb = 0;  // the mask list is in read order too
    for (size_t k = 0; k < ns; ++k) {
        const size_t c = (size_t)h->order[k];
        int64_t rr = h->read_off[k], oo = h->op_off[k], ww = h->word_off[k];
        for (int64_t t = 0; t < n_tasks; ++t) {
            const size_t ix = (size_t)t * (size_t)n_ref + c;
            h->cur_read[ix] = rr; h->cur_op[ix] = oo; h->cur_word[ix] = ww;
            rr += acc[ix].kept; oo += acc[ix].ops; ww += acc[ix].words;
            if (flt.min_bq) { h->cur_mread[ix] = mr; h->cur_mbase[ix] = mb; mr += acc[ix].mreads; mb += acc[ix].mbases; }
        }
    }
    h->masked_reads = mr;
    h->masked_bases = mb;
    if (mb >= (1ll << 32)) return KDL_ERR_INVALID_ARG;
    h->prepared = true;
    info[0] = n_rec; info[1] = h->n_kept; info[2] = (int64_t)ns; info[3] = h->op_off[ns]; info[4] = h->word_off[ns];
    info[5] = h->n_complex; info[6] = h->n_hard; info[7] = h->aligned; info[8] = 0;
    info[9] = std::max(h->reach_right, h->max_simple); info[10] = h->reach_left; info[11] = h->max_simple; info[12] = 1;
    info[13] = h->masked_bases; info[14] = h->masked_reads; info[15] = h->no_qual;
    return KDL_OK;
}

// order[n_seen]: ref ids in first-seen order; read_off[n_seen + 1]
int kdl_bam_contigs(const kdl_bam* h, int32_t* order, int64_t* read_off) {
    if (!h || !h->prepared || !order || !read_off) return KDL_ERR_INVALID_ARG;
    std::memcpy(order, h->order.data(), h->order.size() * sizeof(int32_t));
    std::memcpy(read_off, h->read_off.data(), h->read_off.size() * sizeof(int64_t));
    return KDL_OK;
}

// Caller-owned outputs (any memory, e.g. pinned): ref_start / seq_off / l_seq (device word) / seq_len [n_kept],
// cig_off [n_kept + 1], cigar [n_ops], stream [stream_words], complex_idx [n_complex], hard_idx [n_hard].
// contig_slot[n_seen]: the slot layout (for the coordinate-order check).  info[8] = insertion events,
// info[12] = reads_sorted are filled in.
int kdl_bam_fill(kdl_bam* h, int threads, const int64_t* contig_slot, int32_t* ref_start, uint32_t* seq_off,
                 int32_t* l_seq, int32_t* seq_len, uint32_t* cig_off, uint32_t* cigar, uint32_t* stream,
                 uint32_t* complex_idx, uint32_t* hard_idx, int64_t* info) {
    if (!h || !h->prepared || !ref_start || !seq_off || !l_seq || !seq_len || !cig_off || !stream || !info)
        return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    const int64_t n_tasks = (int64_t)h->chunk_lo.size() - 1;
    const int64_t n = h->n_kept;
    PhaseTimer pt;
    std::vector<uint32_t> ins_n((size_t)std::max<int64_t>(n, 1), 0);  // I ops per kept read (final order)
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<int64_t> cr(h->cur_read.begin() + t * n_ref, h->cur_read.begin() + (t + 1) * n_ref);
        std::vector<int64_t> co(h->cur_op.begin() + t * n_ref, h->cur_op.begin() + (t + 1) * n_ref);
        std::vector<int64_t> cw(h->cur_word.begin() + t * n_ref, h->cur_word.begin() + (t + 1) * n_ref);
        RecView r;
        for (int64_t i = h->chunk_lo[(size_t)t]; i < h->chunk_lo[(size_t)t + 1]; ++i) {
            const Class c = h->cls[(size_t)i];
            if (c.cls == CLS_DROP) continue;
            const int64_t off = h->rec_off[(size_t)i];
            parse_record(d + off, h->rec_off[(size_t)i + 1] - off, &r);
            const size_t ci = (size_t)r.ref_id;
            const int64_t k = cr[ci]++, o = co[ci], w = cw[ci];
            const int64_t n_words = ((int64_t)r.l_seq + 7) / 8, n_bytes_seq = ((int64_t)r.l_seq + 1) / 2;
            co[ci] += r.n_cigar;
            cw[ci] += n_words + (c.cls == CLS_SIMPLE ? 0 : 2 + (int64_t)r.n_cigar);
            ref_start[k] = r.pos;  // BAM pos is 0-based == SAM POS - 1 (kindel.py:42)
            seq_off[k] = (uint32_t)w;
            seq_len[k] = r.l_seq;
            cig_off[k] = (uint32_t)o;
            uint32_t lw;
            if (c.cls == CLS_SIMPLE) lw = (uint32_t)r.l_seq;
            else if (c.cls == CLS_TILE) lw = (uint32_t)r.l_seq | ((uint32_t)c.n_match << KDL_NM_SHIFT) | KDL_COMPLEX;
            else lw = (uint32_t)r.l_seq | KDL_COMPLEX | KDL_HARD;
            std::memcpy(&l_seq[k], &lw, 4);
            if (cigar && r.n_cigar) std::memcpy(cigar + o, r.cigar, 4ull * r.n_cigar);
            uint32_t bad = 0;
            if (!h->n_masked.empty() && h->n_masked[(size_t)i]) {
                int64_t nm = 0;
                for (int64_t q = 0; q < n_words; ++q)
                    stream[w + q] = seq_word(r.seq, n_bytes_seq, q, r.l_seq, q == n_words - 1, &bad,
                                             qual_mask_word(r, q, h->filter.min_bq, &nm));
            } else {
                for (int64_t q = 0; q < n_words; ++q) stream[w + q] = seq_word(r.seq, n_bytes_seq, q, r.l_seq, q == n_words - 1, &bad);
            }
            uint32_t ni = 0;
            for (uint32_t q = 0; q < r.n_cigar; ++q) ni += (rd_u32(r.cigar + 4ull * q) & 15u) == 1u;
            ins_n[(size_t)k] = ni;
            if (c.cls != CLS_SIMPLE) {
                stream[w + n_words] = r.n_cigar;
                stream[w + n_words + 1] = 0;  // evt_off: below
                std::memcpy(stream + w + n_words + 2, r.cigar, 4ull * r.n_cigar);
            }
        }
    });
    cig_off[n] = (uint32_t)h->op_off[h->order.size()];
    pt.lap("fill: records (threads)");
    // ---- insertion-event rows (exclusive prefix of the I-op counts in read order), the complex / hard lists and the
    // coordinate-order check: one cheap sequential pass over the per-read arrays
    int64_t evt = 0, ncx = 0, nh = 0;
    int32_t sorted_ok = 1;
    size_t contig = 0;
    long long prev_g = -(1ll << 62);
    for (int64_t k = 0; k < n; ++k) {
        while (contig + 1 < h->read_off.size() && k >= h->read_off[contig + 1]) ++contig;
        const long long g = (contig_slot ? contig_slot[contig] : 0) + (long long)ref_start[k];
        if (g < prev_g) sorted_ok = 0;
        prev_g = g;
        uint32_t lw;
        std::memcpy(&lw, &l_seq[k], 4);
        if (lw & KDL_COMPLEX) {
            stream[(size_t)seq_off[k] + (size_t)(((int64_t)seq_len[k] + 7) / 8) + 1] = (uint32_t)evt;
            if (complex_idx) complex_idx[ncx] = (uint32_t)k;
            ++ncx;
            if (lw & KDL_HARD) { if (hard_idx) hard_idx[nh] = (uint32_t)k; ++nh; }
        }
        evt += ins_n[(size_t)k];
    }
    pt.lap("fill: events, lists, order");
    h->n_events = evt;
    h->reads_sorted = sorted_ok;
    info[8] = evt;
    info[12] = sorted_ok;
    return KDL_OK;
}

// The mask list of the last prepare (info[14] reads, info[13] bases), in read order: read_idx[m] ascending kept-read
// indices, off[m + 1] their ranges in qpos, qpos[bases] the masked query offsets, ascending per read.
int kdl_bam_fill_mask(kdl_bam* h, int threads, uint32_t* read_idx, uint32_t* off, uint32_t* qpos) {
    if (!h || !h->prepared || !off) return KDL_ERR_INVALID_ARG;
    off[h->masked_reads] = (uint32_t)h->masked_bases;
    if (h->masked_reads == 0) return KDL_OK;
    if (!read_idx || !qpos || h->n_masked.empty()) return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    const int64_t n_tasks = (int64_t)h->chunk_lo.size() - 1;
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<int64_t> cr(h->cur_read.begin() + t * n_ref, h->cur_read.begin() + (t + 1) * n_ref);
        std::vector<int64_t> cm(h->cur_mread.begin() + t * n_ref, h->cur_mread.begin() + (t + 1) * n_ref);
        std::vector<int64_t> cb(h->cur_mbase.begin() + t * n_ref, h->cur_mbase.begin() + (t + 1) * n_ref);
        RecView r;
        for (int64_t i = h->chunk_lo[(size_t)t]; i < h->chunk_lo[(size_t)t + 1]; ++i) {
            if (h->cls[(size_t)i].cls == CLS_DROP) continue;
            const int64_t off_i = h->rec_off[(size_t)i];
            parse_record(d + off_i, h->rec_off[(size_t)i + 1] - off_i, &r);
            const size_t ci = (size_t)r.ref_id;
            const int64_t k = cr[ci]++;
            if (!h->n_masked[(size_t)i]) continue;
            const int64_t j = cm[ci]++;
            int64_t o = cb[ci];
            cb[ci] += h->n_masked[(size_t)i];
            read_idx[j] = (uint32_t)k;
            off[j] = (uint32_t)o;
            for (int64_t q = 0; q < r.l_seq; ++q)
                if (r.qual[q] < h->filter.min_bq) qpos[o++] = (uint32_t)q;
        }
    });
    return KDL_OK;
}

// The strand of the last prepare's kept reads, in read order: reverse[k] = 1 where FLAG & 0x10, else 0.
int kdl_bam_fill_strand(kdl_bam* h, int threads, uint8_t* reverse) {
    if (!h || !h->prepared || (h->n_kept > 0 && !reverse)) return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    const int64_t n_tasks = (int64_t)h->chunk_lo.size() - 1;
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<int64_t> cr(h->cur_read.begin() + t * n_ref, h->cur_read.begin() + (t + 1) * n_ref);
        RecView r;
        for (int64_t i = h->chunk_lo[(size_t)t]; i < h->chunk_lo[(size_t)t + 1]; ++i) {
            if (h->cls[(size_t)i].cls == CLS_DROP) continue;
            const int64_t off_i = h->rec_off[(size_t)i];
            parse_record(d + off_i, h->rec_off[(size_t)i + 1] - off_i, &r);
            reverse[cr[(size_t)r.ref_id]++] = (r.flag & 0x10u) ? 1 : 0;
        }
    });
    return KDL_OK;
}

// The mates of the last prepare's kept reads, in read order (K10, include/kindel_b200.h): name_hash[k] = 64-bit FNV-1a
// of QNAME (NUL excluded), mate_start[k] = PNEXT - 1 (BAM next_pos), pair_role[k] = 1 / 2 for a first / last mate of a
// pair whose FLAG has 0x1, none of 0x8 / 0x100 / 0x800, exactly one of 0x40 / 0x80 and next_refID == refID, else 0.
int kdl_bam_fill_mates(kdl_bam* h, int threads, uint64_t* name_hash, int32_t* mate_start, uint8_t* pair_role) {
    if (!h || !h->prepared || (h->n_kept > 0 && (!name_hash || !mate_start || !pair_role))) return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    const int64_t n_tasks = (int64_t)h->chunk_lo.size() - 1;
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<int64_t> cr(h->cur_read.begin() + t * n_ref, h->cur_read.begin() + (t + 1) * n_ref);
        RecView r;
        for (int64_t i = h->chunk_lo[(size_t)t]; i < h->chunk_lo[(size_t)t + 1]; ++i) {
            if (h->cls[(size_t)i].cls == CLS_DROP) continue;
            const int64_t off_i = h->rec_off[(size_t)i];
            parse_record(d + off_i, h->rec_off[(size_t)i + 1] - off_i, &r);
            const int64_t k = cr[(size_t)r.ref_id]++;
            const uint8_t* q = d + off_i + 4;  // the record behind block_size
            const uint32_t l_name = q[8];
            uint64_t hv = 0xcbf29ce484222325ull;
            for (uint32_t c = 0; c < l_name && q[32 + c]; ++c) hv = (hv ^ q[32 + c]) * 0x100000001b3ull;
            name_hash[k] = hv;
            mate_start[k] = rd_i32(q + 24);
            const uint32_t f = r.flag;
            const bool ends = ((f & 0x40u) != 0) != ((f & 0x80u) != 0);
            const bool ok = (f & 0x1u) && !(f & (0x8u | 0x100u | 0x800u)) && ends && rd_i32(q + 20) == r.ref_id;
            pair_role[k] = ok ? ((f & 0x40u) ? 1 : 2) : 0;
        }
    });
    return KDL_OK;
}

// The qualities of the last prepare's kept reads beside their bases (K11, include/kindel_b200.h): base k of kept read r
// at byte 8 * seq_off[r] + k of qual8 [8 * words], 0xff for the padding, a complex read's trailer words and every base of
// a read without qualities (prepare's info[15] counts those reads).
int kdl_bam_fill_qual(kdl_bam* h, int threads, uint8_t* qual8) {
    if (!h || !h->prepared || (h->n_kept > 0 && !qual8)) return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    const int64_t n_tasks = (int64_t)h->chunk_lo.size() - 1;
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<int64_t> cw(h->cur_word.begin() + t * n_ref, h->cur_word.begin() + (t + 1) * n_ref);
        RecView r;
        for (int64_t i = h->chunk_lo[(size_t)t]; i < h->chunk_lo[(size_t)t + 1]; ++i) {
            const Class c = h->cls[(size_t)i];
            if (c.cls == CLS_DROP) continue;
            const int64_t off_i = h->rec_off[(size_t)i];
            parse_record(d + off_i, h->rec_off[(size_t)i + 1] - off_i, &r);
            const size_t ci = (size_t)r.ref_id;
            const int64_t w = cw[ci], n_words = ((int64_t)r.l_seq + 7) / 8;
            const int64_t total = n_words + (c.cls == CLS_SIMPLE ? 0 : 2 + (int64_t)r.n_cigar);
            cw[ci] += total;
            uint8_t* out = qual8 + 8 * w;
            const bool has = r.qual && r.qual[0] != 0xff;
            if (has) std::memcpy(out, r.qual, (size_t)r.l_seq);
            std::memset(out + (has ? r.l_seq : 0), 0xff, (size_t)(8 * total - (has ? r.l_seq : 0)));
        }
    });
    return KDL_OK;
}

// The duplicate score of the last prepare's kept reads, in read order (K14, include/kindel_b200.h): -1 where FLAG has
// 0x100 or 0x800, else the sum of the Phred qualities >= 15 over all of SEQ (0 for a read without qualities),
// saturating at 2^31 - 1.  Summed here, while the record is at hand, so that no quality byte travels to the device.
// Refused for SAM text with a QUAL field the text parser could not carry: the caller's text reader decides.
int kdl_bam_fill_dup(kdl_bam* h, int threads, int32_t* dup_score) {
    if (!h || !h->prepared || (h->n_kept > 0 && !dup_score) || (h->sam_odd & 2)) return KDL_ERR_INVALID_ARG;
    const uint8_t* d = h->dptr;
    const int32_t n_ref = (int32_t)h->ref_name.size();
    const int64_t n_tasks = (int64_t)h->chunk_lo.size() - 1;
    h->pool->run(n_tasks, threads, [&](int64_t t, int) {
        std::vector<int64_t> cr(h->cur_read.begin() + t * n_ref, h->cur_read.begin() + (t + 1) * n_ref);
        RecView r;
        for (int64_t i = h->chunk_lo[(size_t)t]; i < h->chunk_lo[(size_t)t + 1]; ++i) {
            if (h->cls[(size_t)i].cls == CLS_DROP) continue;
            const int64_t off_i = h->rec_off[(size_t)i];
            parse_record(d + off_i, h->rec_off[(size_t)i + 1] - off_i, &r);
            const int64_t k = cr[(size_t)r.ref_id]++;
            if (r.flag & 0x900u) {
                dup_score[k] = -1;
                continue;
            }
            int64_t s = 0;
            if (r.qual && r.l_seq > 0 && r.qual[0] != 0xff)
                for (int32_t q = 0; q < r.l_seq; ++q) s += r.qual[q] >= 15 ? r.qual[q] : 0;
            dup_score[k] = s > 0x7fffffff ? 0x7fffffff : (int32_t)s;
        }
    });
    return KDL_OK;
}

}  // extern "C"
