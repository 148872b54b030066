// Host-side I/O of the cluster step, native so that the GPU path is not starved by Python:
//   * .pairs / .pairs.gz tokenizer with name -> id translation and the alignments.bed side product
//     (pairs_generator / pairs_generator_inter_ctgs, scripts/HapHiC_cluster.py:1539-1583), multi-threaded:
//     the text is cut at line boundaries and parsed by a pool of threads, BGZF-compressed input is inflated
//     block-parallel,
//   * BAM reader (bam_generator, 1586-1593),
//   * ultra-long read alignments for --ul (parse_ul_alignments, 1763-1869),
//   * paired_links.clm from the record stream (update_clm_dict 395-401 + output_clm 376-392), threaded.
// Pure C++ (no CUDA); part of libhaphic_b200.so, declared in include/haphic_b200.h.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/haphic_b200.h"

void hh_set_error(const char* fmt, ...);

static inline uint32_t le32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static inline uint16_t le16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }

static int hh_io_threads(int requested) {
    if (requested > 0) return requested;
    const unsigned hc = std::thread::hardware_concurrency();
    return (int)std::max(1u, std::min(16u, hc ? hc : 1u));
}

// ---------------------------------------------------------------------------------------------
// BGZF (blocked gzip: BAM, bgzipped .pairs): every block is an independent deflate stream with its
// compressed size in the gzip extra field and its uncompressed size in the trailer, so a batch of
// blocks inflates in parallel straight into its final place.
// ---------------------------------------------------------------------------------------------
struct hh_bgzf {
    FILE* f = nullptr;
    std::vector<uint8_t> comp;        // compressed bytes not yet consumed
    size_t comp_pos = 0, comp_len = 0;
    bool file_eof = false;
    std::vector<uint8_t> raw;         // decompressed bytes not yet consumed: [raw_pos, raw_len)
    size_t raw_pos = 0, raw_len = 0;
    int threads = 1;
};

struct hh_bgzf_block {
    size_t in_off, in_len;            // deflate payload inside comp
    size_t out_off;                   // destination offset inside raw
    uint32_t isize, crc;
};

// inflate the next batch of whole blocks (about target_bytes of compressed input); appends to raw.
// Returns 0 = appended something, 1 = end of file, <0 = error (message set).
static int bgzf_fill(hh_bgzf* r, size_t target_bytes) {
    if (r->comp_pos > 0) {
        memmove(r->comp.data(), r->comp.data() + r->comp_pos, r->comp_len - r->comp_pos);
        r->comp_len -= r->comp_pos;
        r->comp_pos = 0;
    }
    if (!r->file_eof && r->comp_len < target_bytes) {
        if (r->comp.size() < target_bytes + (1u << 16)) r->comp.resize(target_bytes + (1u << 16));
        const size_t got = fread(r->comp.data() + r->comp_len, 1, r->comp.size() - r->comp_len, r->f);
        if (got == 0) r->file_eof = true;
        r->comp_len += got;
    }
    if (r->comp_len == 0) return 1;
    std::vector<hh_bgzf_block> blocks;
    size_t p = 0, out_total = 0;
    while (p + 18 <= r->comp_len) {
        const uint8_t* h = r->comp.data() + p;
        if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) {
            hh_set_error("BGZF: bad block header (the file is corrupt or not blocked gzip)");
            return -1;
        }
        const size_t xlen = le16(h + 10);
        if (p + 12 + xlen > r->comp_len) break;
        size_t bsize = 0;
        for (size_t q = 0; q + 4 <= xlen;) {
            const uint8_t* sf = h + 12 + q;
            const size_t slen = le16(sf + 2);
            if (sf[0] == 'B' && sf[1] == 'C' && slen == 2) bsize = (size_t)le16(sf + 4) + 1;
            q += 4 + slen;
        }
        if (bsize == 0 || bsize < 12 + xlen + 8) {
            hh_set_error("BGZF: block without a valid BC subfield");
            return -1;
        }
        if (p + bsize > r->comp_len) break;          // incomplete block: wait for more input
        hh_bgzf_block b;
        b.in_off = p + 12 + xlen;
        b.in_len = bsize - 12 - xlen - 8;
        b.crc = le32(h + bsize - 8);
        b.isize = le32(h + bsize - 4);
        b.out_off = out_total;
        out_total += b.isize;
        blocks.push_back(b);
        p += bsize;
    }
    if (blocks.empty()) {
        if (r->file_eof) {
            hh_set_error("BGZF: truncated block at the end of the file");
            return -1;
        }
        return bgzf_fill(r, target_bytes * 2);       // blocks are <= 64 KiB: cannot recurse more than once
    }
    if (r->raw_pos > 0) {
        memmove(r->raw.data(), r->raw.data() + r->raw_pos, r->raw_len - r->raw_pos);
        r->raw_len -= r->raw_pos;
        r->raw_pos = 0;
    }
    if (r->raw.size() < r->raw_len + out_total) r->raw.resize(r->raw_len + out_total);
    uint8_t* out_base = r->raw.data() + r->raw_len;
    const uint8_t* in_base = r->comp.data();
    std::atomic<size_t> next(0);
    std::atomic<int> failed(0);
    auto work = [&]() {
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (inflateInit2(&zs, -15) != Z_OK) {
            failed = 1;
            return;
        }
        for (;;) {
            const size_t k = next.fetch_add(1);
            if (k >= blocks.size()) break;
            const hh_bgzf_block& b = blocks[k];
            inflateReset(&zs);
            zs.next_in = const_cast<Bytef*>(in_base + b.in_off);
            zs.avail_in = (uInt)b.in_len;
            zs.next_out = out_base + b.out_off;
            zs.avail_out = b.isize;
            const int rc = b.isize ? inflate(&zs, Z_FINISH) : Z_STREAM_END;
            if ((b.isize && rc != Z_STREAM_END) || zs.avail_out != 0 ||
                (uint32_t)crc32(crc32(0L, Z_NULL, 0), out_base + b.out_off, b.isize) != b.crc) {
                failed = 1;
                break;
            }
        }
        inflateEnd(&zs);
    };
    const int nt = (int)std::min<size_t>((size_t)std::max(1, r->threads), blocks.size());
    if (nt <= 1) {
        work();
    } else {
        std::vector<std::thread> pool;
        for (int t = 0; t < nt; ++t) pool.emplace_back(work);
        for (auto& t : pool) t.join();
    }
    if (failed) {
        hh_set_error("BGZF: a block failed to inflate (corrupt file)");
        return -1;
    }
    r->raw_len += out_total;
    r->comp_pos = p;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// contig name -> id: open addressing over the caller's NUL-separated name blob
// ---------------------------------------------------------------------------------------------
struct hh_name_table {
    struct slot {
        uint64_t hash;
        const char* s;
        uint32_t len;
        int32_t id;
    };
    std::vector<slot> slots;
    uint64_t mask = 0;
    std::string blob;                 // private copy: the caller's buffer need not outlive hh_*_open

    static inline uint64_t hash_of(const char* s, size_t n) {
        uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t)n;
        size_t i = 0;
        for (; i + 8 <= n; i += 8) {
            uint64_t w;
            memcpy(&w, s + i, 8);
            h = (h ^ w) * 0x9E3779B97F4A7C15ull;
            h ^= h >> 29;
        }
        uint64_t w = 0;
        memcpy(&w, s + i, n - i);
        h = (h ^ w) * 0x9E3779B97F4A7C15ull;
        h ^= h >> 32;
        return h | 1ull;              // 0 marks an empty slot
    }
    void build(const char* names_blob, int32_t n_names) {
        size_t total = 0;
        const char* p = names_blob;
        for (int32_t i = 0; i < n_names; ++i) {
            const size_t l = strlen(p);
            total += l + 1;
            p += l + 1;
        }
        blob.assign(names_blob, total);
        size_t cap = 16;
        while (cap < (size_t)n_names * 2 + 2) cap <<= 1;
        slots.assign(cap, slot{0, nullptr, 0, -1});
        mask = cap - 1;
        p = blob.data();
        for (int32_t i = 0; i < n_names; ++i) {
            const size_t l = strlen(p);
            const uint64_t h = hash_of(p, l);
            uint64_t k = h & mask;
            bool dup = false;
            while (slots[k].hash) {
                if (slots[k].hash == h && slots[k].len == l && memcmp(slots[k].s, p, l) == 0) {
                    dup = true;       // duplicate names: the first one wins, like a dict comprehension would not -- FASTA names are unique
                    break;
                }
                k = (k + 1) & mask;
            }
            if (!dup) slots[k] = slot{h, p, (uint32_t)l, i};
            p += l + 1;
        }
    }
    inline int32_t find(const char* s, size_t n) const {
        const uint64_t h = hash_of(s, n);
        uint64_t k = h & mask;
        while (slots[k].hash) {
            if (slots[k].hash == h && slots[k].len == n && memcmp(slots[k].s, s, n) == 0) return slots[k].id;
            k = (k + 1) & mask;
        }
        return -1;
    }
};

// ---------------------------------------------------------------------------------------------
// .pairs reader
// ---------------------------------------------------------------------------------------------
struct hh_bytes {                     // grow-only byte buffer without the zero fill of std::vector::resize
    char* data = nullptr;
    size_t len = 0, cap = 0;
    hh_bytes() = default;
    hh_bytes(const hh_bytes&) = delete;
    hh_bytes& operator=(const hh_bytes&) = delete;
    hh_bytes(hh_bytes&& o) noexcept : data(o.data), len(o.len), cap(o.cap) { o.data = nullptr; o.len = o.cap = 0; }
    hh_bytes& operator=(hh_bytes&& o) noexcept {
        if (this != &o) {
            free(data);
            data = o.data;
            len = o.len;
            cap = o.cap;
            o.data = nullptr;
            o.len = o.cap = 0;
        }
        return *this;
    }
    ~hh_bytes() { free(data); }
    inline char* room(size_t need) {
        if (len + need > cap) {
            size_t ncap = cap ? cap * 2 : (1u << 20);
            while (ncap < len + need) ncap *= 2;
            data = (char*)realloc(data, ncap);
            cap = ncap;
        }
        return data + len;
    }
    void release() {
        free(data);
        data = nullptr;
        len = cap = 0;
    }
};

struct hh_pairs_part {                // what one thread produced from its slice of a text window
    std::vector<int32_t> rec;
    hh_bytes bed;
    int64_t lines = 0;
    int64_t err_line = -1;            // first bad line (index inside the part), -1 = none
    int err_kind = 0;                 // 1 = fewer than 5 columns, 2 = position is not an integer
};

struct hh_pairs_reader {
    int mode = 0;                     // 0 plain text, 1 gzip stream (zlib), 2 BGZF
    FILE* f = nullptr;
    gzFile gz = nullptr;
    hh_bgzf bg;
    FILE* bed = nullptr;
    hh_name_table names;
    std::vector<uint8_t> text;        // undigested bytes of modes 0 / 1: [pos, len)
    size_t pos = 0, len = 0;
    bool eof = false;
    int inter_only = 1;
    int threads = 1;
    int64_t lines = 0;                // lines consumed by finished windows
    std::vector<hh_pairs_part> parts; // parsed, not yet handed out
    size_t part_k = 0, part_off = 0;
    // alignments.bed is written behind the parser by its own thread, slices in input order
    std::thread bed_writer;
    std::mutex bed_mu;
    std::condition_variable bed_cv;
    std::deque<hh_bytes> bed_queue;
    size_t bed_queued_bytes = 0;
    bool bed_done = false, bed_failed = false;
};

static void pairs_bed_writer(hh_pairs_reader* r) {
    for (;;) {
        hh_bytes buf;
        {
            std::unique_lock<std::mutex> lk(r->bed_mu);
            r->bed_cv.wait(lk, [&] { return r->bed_done || !r->bed_queue.empty(); });
            if (r->bed_queue.empty()) return;
            buf = std::move(r->bed_queue.front());
            r->bed_queue.pop_front();
        }
        if (fwrite(buf.data, 1, buf.len, r->bed) != buf.len) r->bed_failed = true;
        {
            std::lock_guard<std::mutex> lk(r->bed_mu);
            r->bed_queued_bytes -= buf.len;
        }
        r->bed_cv.notify_all();
    }
}

extern "C" int hh_pairs_open(const char* path, const char* names_blob, int32_t n_names, const char* bed_path, int inter_only,
                             int threads, hh_pairs_reader** out) {
    if (!path || !names_blob || !out || n_names < 0) {
        hh_set_error("hh_pairs_open: bad argument");
        return HH_ERR_ARG;
    }
    *out = nullptr;
    hh_pairs_reader* r = new hh_pairs_reader();
    r->threads = hh_io_threads(threads);
    r->f = fopen(path, "rb");
    if (!r->f) {
        hh_set_error("hh_pairs_open: cannot open %s", path);
        delete r;
        return HH_ERR_ARG;
    }
    // plain text, a gzip stream, or blocked gzip (bgzip): look at the first member's header
    uint8_t h[18];
    const size_t got = fread(h, 1, sizeof(h), r->f);
    if (got >= 4 && h[0] == 0x1f && h[1] == 0x8b) {
        r->mode = 1;
        if (got == 18 && h[2] == 8 && (h[3] & 4) && le16(h + 10) >= 6 && h[12] == 'B' && h[13] == 'C') r->mode = 2;
    }
    if (r->mode == 1) {
        fclose(r->f);
        r->f = nullptr;
        r->gz = gzopen(path, "rb");
        if (!r->gz) {
            hh_set_error("hh_pairs_open: cannot open %s", path);
            delete r;
            return HH_ERR_ARG;
        }
        gzbuffer(r->gz, 1 << 20);
    } else {
        fseek(r->f, 0, SEEK_SET);
        if (r->mode == 2) {
            r->bg.f = r->f;
            r->bg.threads = r->threads;
        }
    }
    if (bed_path && *bed_path) {
        r->bed = fopen(bed_path, "w");
        if (!r->bed) {
            hh_set_error("hh_pairs_open: cannot create %s", bed_path);
            if (r->gz) gzclose(r->gz);
            if (r->f) fclose(r->f);
            delete r;
            return HH_ERR_ARG;
        }
        setvbuf(r->bed, nullptr, _IONBF, 0);          // whole slices are written with one fwrite each
        r->bed_writer = std::thread(pairs_bed_writer, r);
    }
    r->names.build(names_blob, n_names);
    r->inter_only = inter_only;
    *out = r;
    return HH_OK;
}

static inline char* put_i64(char* p, int64_t v) {
    char tmp[24];
    int n = 0;
    uint64_t u = v < 0 ? (uint64_t)(-(v + 1)) + 1 : (uint64_t)v;
    do {
        tmp[n++] = (char)('0' + u % 10);
        u /= 10;
    } while (u);
    if (v < 0) *p++ = '-';
    while (n) *p++ = tmp[--n];
    return p;
}

static inline bool is_ws(char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; }

// parses a Python-int()-compatible decimal (optional sign, surrounding blanks already stripped)
static inline bool parse_int(const char* s, const char* e, int64_t* out) {
    if (s == e) return false;
    bool neg = false;
    if (*s == '+' || *s == '-') {
        neg = *s == '-';
        ++s;
    }
    if (s == e) return false;
    int64_t v = 0;
    for (; s < e; ++s) {
        if (*s == '_') continue;                 // int('1_000') is valid Python
        if (*s < '0' || *s > '9') return false;
        if (v > (INT64_MAX - 9) / 10) return false;     // does not fit: refuse instead of wrapping
        v = v * 10 + (*s - '0');
    }
    *out = neg ? -v : v;
    return true;
}

// one thread's share: whole lines in [s, e)
static void pairs_parse_slice(const hh_pairs_reader* r, const char* s, const char* e, hh_pairs_part* out) {
    const bool want_bed = r->bed != nullptr;
    const char* last_name[2] = {nullptr, nullptr};       // the previous line's contig names: Hi-C text is full of runs
    size_t last_len[2] = {0, 0};
    int32_t last_id[2] = {-1, -1};
    out->rec.reserve((size_t)(e - s) / 12);
    if (want_bed) out->bed.room((size_t)(e - s) * 2 + 256);
    while (s < e) {
        const char* nl = (const char*)memchr(s, '\n', (size_t)(e - s));
        const char* le = nl ? nl : e;
        const char* ls = s;
        s = nl ? nl + 1 : e;
        out->lines++;
        // `if not line.strip() or line.startswith('#'): continue`
        const char* t = ls;
        while (t < le && is_ws(*t)) ++t;
        if (t == le || *ls == '#') continue;
        // cols = line.split(): first five whitespace-separated tokens
        const char* tok[5];
        const char* tend[5];
        int k = 0;
        const char* c = t;
        while (k < 5 && c < le) {
            while (c < le && is_ws(*c)) ++c;
            if (c == le) break;
            tok[k] = c;
            while (c < le && !is_ws(*c)) ++c;
            tend[k] = c;
            ++k;
        }
        if (k < 5) {
            out->err_line = out->lines - 1;
            out->err_kind = 1;
            return;
        }
        int64_t p1, p2;
        if (!parse_int(tok[2], tend[2], &p1) || !parse_int(tok[4], tend[4], &p2)) {
            out->err_line = out->lines - 1;
            out->err_kind = 2;
            return;
        }
        p1 -= 1;                                    // pysam / BED are 0-based
        p2 -= 1;
        if (p1 < INT32_MIN || p1 > INT32_MAX || p2 < INT32_MIN || p2 > INT32_MAX) {     // records carry int32 positions
            out->err_line = out->lines - 1;
            out->err_kind = 2;
            return;
        }
        const size_t l1 = (size_t)(tend[1] - tok[1]), l3 = (size_t)(tend[3] - tok[3]);
        if (want_bed) {
            // '{ref}\t{pos}\t{pos}\t{readID}/1\t255\t.\n{mref}\t{mpos}\t{mpos}\t{readID}/2\t255\t.\n'  (1557, 1580)
            const size_t l0 = (size_t)(tend[0] - tok[0]);
            const size_t need = 2 * l0 + l1 + l3 + 128;
            char* q = out->bed.room(need);
            for (int side = 0; side < 2; ++side) {
                const char* cs = side ? tok[3] : tok[1];
                const size_t cl = side ? l3 : l1;
                const int64_t pv = side ? p2 : p1;
                memcpy(q, cs, cl);
                q += cl;
                *q++ = '\t';
                q = put_i64(q, pv);
                *q++ = '\t';
                q = put_i64(q, pv);
                *q++ = '\t';
                memcpy(q, tok[0], l0);
                q += l0;
                memcpy(q, side ? "/2\t255\t.\n" : "/1\t255\t.\n", 9);
                q += 9;
            }
            out->bed.len = (size_t)(q - out->bed.data);
        }
        if (r->inter_only && l1 == l3 && memcmp(tok[1], tok[3], l1) == 0) continue;    // ref != mref (1582)
        int32_t id[2];
        for (int side = 0; side < 2; ++side) {
            const char* cs = side ? tok[3] : tok[1];
            const size_t cl = side ? l3 : l1;
            if (last_name[side] && last_len[side] == cl && memcmp(last_name[side], cs, cl) == 0) {
                id[side] = last_id[side];
            } else {
                id[side] = r->names.find(cs, cl);
                last_name[side] = cs;
                last_len[side] = cl;
                last_id[side] = id[side];
            }
        }
        const int32_t four[4] = {id[0], (int32_t)p1, id[1], (int32_t)p2};
        out->rec.insert(out->rec.end(), four, four + 4);
    }
}

// read + parse the next window of text; 0 = parts ready, 1 = end of input, <0 error
static int pairs_next_window(hh_pairs_reader* r) {
    const size_t WINDOW = 64u << 20;
    const uint8_t* base = nullptr;
    size_t avail = 0;
    bool at_eof = false;
    if (r->mode == 2) {
        hh_bgzf* b = &r->bg;
        while (b->raw_len - b->raw_pos < WINDOW) {
            const int rc = bgzf_fill(b, 32u << 20);
            if (rc < 0) return -1;
            if (rc == 1) {
                at_eof = true;
                break;
            }
        }
        base = b->raw.data() + b->raw_pos;
        avail = b->raw_len - b->raw_pos;
    } else {
        if (r->pos > 0) {
            memmove(r->text.data(), r->text.data() + r->pos, r->len - r->pos);
            r->len -= r->pos;
            r->pos = 0;
        }
        while (!r->eof && r->len < WINDOW) {
            if (r->text.size() < r->len + (8u << 20)) r->text.resize(std::max(r->text.size() * 2, r->len + (16u << 20)));
            const size_t room = std::min(r->text.size() - r->len, (size_t)1 << 30);
            long got;
            if (r->mode == 1) {
                got = gzread(r->gz, r->text.data() + r->len, (unsigned)room);
                if (got < 0) {
                    hh_set_error("hh_pairs_next: read error (corrupt gzip stream)");
                    return -1;
                }
            } else {
                got = (long)fread(r->text.data() + r->len, 1, room, r->f);
            }
            if (got == 0) r->eof = true;
            r->len += (size_t)got;
        }
        at_eof = r->eof;
        base = r->text.data();
        avail = r->len;
    }
    if (avail == 0) return 1;
    // whole lines only (at the end of the input the last line may lack its newline)
    size_t use = avail;
    if (!at_eof) {
        const uint8_t* last = (const uint8_t*)memrchr(base, '\n', avail);
        if (!last) {
            hh_set_error("hh_pairs_next: a line longer than %zu MiB", WINDOW >> 20);
            return -1;
        }
        use = (size_t)(last - base) + 1;
    }
    // slices at line boundaries
    const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)r->threads, use / (1u << 20) + 1));
    std::vector<size_t> cut((size_t)nt + 1, use);
    cut[0] = 0;
    for (int t = 1; t < nt; ++t) {
        size_t c = use / (size_t)nt * (size_t)t;
        if (c < cut[(size_t)t - 1]) c = cut[(size_t)t - 1];
        const uint8_t* nl = (const uint8_t*)memchr(base + c, '\n', use - c);
        cut[(size_t)t] = nl ? (size_t)(nl - base) + 1 : use;
    }
    r->parts.clear();
    r->parts.resize((size_t)nt);
    r->part_k = 0;
    r->part_off = 0;
    if (nt == 1) {
        pairs_parse_slice(r, (const char*)base, (const char*)base + use, &r->parts[0]);
    } else {
        std::vector<std::thread> pool;
        for (int t = 0; t < nt; ++t)
            pool.emplace_back(pairs_parse_slice, r, (const char*)base + cut[(size_t)t], (const char*)base + cut[(size_t)t + 1],
                              &r->parts[(size_t)t]);
        for (auto& th : pool) th.join();
    }
    // errors in input order; BED in input order
    for (int t = 0; t < nt; ++t) {
        hh_pairs_part& p = r->parts[(size_t)t];
        if (r->bed && p.bed.len) {
            std::unique_lock<std::mutex> lk(r->bed_mu);
            r->bed_cv.wait(lk, [&] { return r->bed_queued_bytes < ((size_t)1 << 30); });     // bounded backlog
            r->bed_queued_bytes += p.bed.len;
            r->bed_queue.push_back(std::move(p.bed));
            lk.unlock();
            r->bed_cv.notify_all();
        }
        p.bed.release();
        if (p.err_line >= 0) {
            const long long line = (long long)(r->lines + p.err_line + 1);
            if (p.err_kind == 1) hh_set_error("hh_pairs_next: line %lld has fewer than 5 columns", line);
            else hh_set_error("hh_pairs_next: line %lld: position is not an integer", line);
            return -1;
        }
        r->lines += p.lines;
    }
    if (r->mode == 2) r->bg.raw_pos += use;
    else r->pos += use;
    if (r->bed_failed) {
        hh_set_error("hh_pairs_next: writing alignments.bed failed (disk full?)");
        return -1;
    }
    return 0;
}

extern "C" int hh_pairs_next(hh_pairs_reader* r, int32_t* rec, int64_t max_records, int64_t* n_out) {
    if (!r || !rec || !n_out || max_records <= 0) {
        hh_set_error("hh_pairs_next: bad argument");
        return HH_ERR_ARG;
    }
    int64_t n = 0;
    *n_out = 0;
    while (n < max_records) {
        if (r->part_k >= r->parts.size()) {
            const int rc = pairs_next_window(r);
            if (rc < 0) return HH_ERR_ARG;
            if (rc == 1) break;
            continue;
        }
        const std::vector<int32_t>& src = r->parts[r->part_k].rec;
        const size_t have = src.size() / 4 - r->part_off;
        if (have == 0) {
            std::vector<int32_t>().swap(r->parts[r->part_k].rec);
            r->part_k++;
            r->part_off = 0;
            continue;
        }
        const size_t take = std::min<size_t>(have, (size_t)(max_records - n));
        memcpy(rec + n * 4, src.data() + r->part_off * 4, take * 16);
        r->part_off += take;
        n += (int64_t)take;
    }
    *n_out = n;
    return HH_OK;
}

extern "C" int hh_pairs_close(hh_pairs_reader* r) {
    if (!r) return HH_OK;
    int rc = HH_OK;
    if (r->bed_writer.joinable()) {
        {
            std::lock_guard<std::mutex> lk(r->bed_mu);
            r->bed_done = true;
        }
        r->bed_cv.notify_all();
        r->bed_writer.join();
    }
    if (r->gz) gzclose(r->gz);
    if (r->f) fclose(r->f);
    if (r->bed && (fclose(r->bed) != 0 || r->bed_failed)) {
        hh_set_error("hh_pairs_close: writing alignments.bed failed (disk full?)");
        rc = HH_ERR_ARG;
    }
    delete r;
    return rc;
}

// ---------------------------------------------------------------------------------------------
// BAM reader (bam_generator, scripts/HapHiC_cluster.py:1586-1593, with the htslib filters of 2855 / 2862):
// BGZF blocks are inflated by a small thread pool (blocks are independent deflate streams), the
// records are walked in the decompressed stream and one int32 record per read1 alignment is produced:
// (id(reference_name), reference_start, id(next_reference_name), next_reference_start).
// ---------------------------------------------------------------------------------------------
struct hh_bam_reader {
    hh_bgzf z;
    std::string header_text;
    std::vector<int32_t> ref_to_id;   // BAM refID -> contig id (-1 = not in the FASTA)
    int inter_only = 1;
    int64_t n_records = 0;
};

// make sure `need` decompressed bytes are available at raw_pos; returns 0 ok, 1 clean EOF (nothing left), -1 error
static int bam_need(hh_bgzf* r, size_t need) {
    while (r->raw_len - r->raw_pos < need) {
        const int rc = bgzf_fill(r, 32u << 20);
        if (rc < 0) return -1;
        if (rc == 1) {
            if (r->raw_len == r->raw_pos) return 1;
            hh_set_error("hh_bam: truncated BAM record");
            return -1;
        }
    }
    return 0;
}

extern "C" int hh_bam_open(const char* path, const char* names_blob, int32_t n_names, int inter_only, int threads,
                           hh_bam_reader** out) {
    if (!path || !names_blob || !out || n_names < 0) {
        hh_set_error("hh_bam_open: bad argument");
        return HH_ERR_ARG;
    }
    *out = nullptr;
    hh_bam_reader* r = new hh_bam_reader();
    r->z.f = fopen(path, "rb");
    if (!r->z.f) {
        hh_set_error("hh_bam_open: cannot open %s", path);
        delete r;
        return HH_ERR_ARG;
    }
    r->inter_only = inter_only;
    r->z.threads = hh_io_threads(threads);
    auto fail = [&](const char* msg) {
        if (msg) hh_set_error("%s", msg);
        fclose(r->z.f);
        delete r;
        return HH_ERR_ARG;
    };
    if (bam_need(&r->z, 12) != 0) return fail(nullptr);
    const uint8_t* p = r->z.raw.data() + r->z.raw_pos;
    if (memcmp(p, "BAM\1", 4) != 0) return fail("hh_bam_open: not a BAM file");
    const size_t l_text = le32(p + 4);
    if (bam_need(&r->z, 12 + l_text) != 0) return fail(nullptr);
    p = r->z.raw.data() + r->z.raw_pos;
    r->header_text.assign(reinterpret_cast<const char*>(p + 8), l_text);
    while (!r->header_text.empty() && r->header_text.back() == '\0') r->header_text.pop_back();
    const int32_t n_ref = (int32_t)le32(p + 8 + l_text);
    r->z.raw_pos += 12 + l_text;
    hh_name_table ids;
    ids.build(names_blob, n_names);
    r->ref_to_id.assign((size_t)(n_ref > 0 ? n_ref : 0), -1);
    for (int32_t k = 0; k < n_ref; ++k) {
        if (bam_need(&r->z, 4) != 0) return fail("hh_bam_open: truncated BAM header");
        const size_t l_name = le32(r->z.raw.data() + r->z.raw_pos);
        if (bam_need(&r->z, 8 + l_name) != 0) return fail("hh_bam_open: truncated BAM header");
        const char* nm = reinterpret_cast<const char*>(r->z.raw.data() + r->z.raw_pos + 4);
        r->ref_to_id[(size_t)k] = ids.find(nm, l_name ? l_name - 1 : 0);
        r->z.raw_pos += 8 + l_name;
    }
    *out = r;
    return HH_OK;
}

extern "C" int hh_bam_header_text(hh_bam_reader* r, const char** text, int64_t* len) {
    if (!r || !text || !len) {
        hh_set_error("hh_bam_header_text: bad argument");
        return HH_ERR_ARG;
    }
    *text = r->header_text.data();
    *len = (int64_t)r->header_text.size();
    return HH_OK;
}

extern "C" int hh_bam_next(hh_bam_reader* r, int32_t* rec, int64_t max_records, int64_t* n_out) {
    if (!r || !rec || !n_out || max_records <= 0) {
        hh_set_error("hh_bam_next: bad argument");
        return HH_ERR_ARG;
    }
    int64_t n = 0;
    *n_out = 0;
    const int32_t n_ref = (int32_t)r->ref_to_id.size();
    while (n < max_records) {
        int rc = bam_need(&r->z, 4);
        if (rc == 1) break;
        if (rc < 0) return HH_ERR_ARG;
        const size_t bs = le32(r->z.raw.data() + r->z.raw_pos);
        if (bs < 32) {
            hh_set_error("hh_bam_next: corrupt BAM record (block_size %zu)", bs);
            return HH_ERR_ARG;
        }
        rc = bam_need(&r->z, 4 + bs);
        if (rc != 0) {
            if (rc == 1) hh_set_error("hh_bam_next: truncated BAM record");
            return HH_ERR_ARG;
        }
        const uint8_t* p = r->z.raw.data() + r->z.raw_pos + 4;
        r->z.raw_pos += 4 + bs;
        r->n_records++;
        const int32_t refid = (int32_t)le32(p), pos = (int32_t)le32(p + 4);
        const uint16_t flag = le16(p + 14);
        const int32_t mrefid = (int32_t)le32(p + 20), mpos = (int32_t)le32(p + 24);
        if (!(flag & 0x40)) continue;                              // flag.read1
        if (r->inter_only && refid == mrefid) continue;            // refid != mrefid (2862)
        int32_t* o = rec + n * 4;
        o[0] = (refid >= 0 && refid < n_ref) ? r->ref_to_id[(size_t)refid] : -1;
        o[1] = pos;
        o[2] = (mrefid >= 0 && mrefid < n_ref) ? r->ref_to_id[(size_t)mrefid] : -1;
        o[3] = mpos;
        ++n;
    }
    *n_out = n;
    return HH_OK;
}

extern "C" int hh_bam_close(hh_bam_reader* r) {
    if (!r) return HH_OK;
    if (r->z.f) fclose(r->z.f);
    delete r;
    return HH_OK;
}

// ---------------------------------------------------------------------------------------------
// Ultra-long read alignments (parse_ul_alignments, 1763-1869): one pass over the BAM with the htslib filter
// `!flag.unmap`, the MAPQ / length / end-distance filters, the primary / supplementary state machine and the best
// supplementary by AS.  What is kept is the header's references and one event per accepted (primary, supplementary)
// pair: the semi-contigs (2 * ref + 0 for `_H`, 1 for `_T`) of the inter-contig edge, the primary's reference and the
// supplementary's reference -- the three add_edge calls of parse_supplementary_aln_list, in file order.
// ---------------------------------------------------------------------------------------------
struct hh_ul_reader {
    std::string names;                // reference names, NUL-terminated, header order
    std::vector<int64_t> ref_len;
    std::vector<int32_t> events;      // [n][4]
    int64_t n_records = 0;
};

namespace {
struct ul_aln {
    int32_t ref;
    bool reverse;
    int64_t qs, qe;                   // query termini of get_query_alignment_termini
    bool has_as;
    int64_t as;
};

enum { CIG_M = 0, CIG_I = 1, CIG_D = 2, CIG_N = 3, CIG_S = 4, CIG_H = 5, CIG_EQ = 7, CIG_X = 8 };

// integer value of the aux tag `tag` (types c C s S i I); false when absent or not an integer
bool ul_aux_int(const uint8_t* p, const uint8_t* end, const char* tag, int64_t* v) {
    while (p + 3 <= end) {
        const bool hit = p[0] == (uint8_t)tag[0] && p[1] == (uint8_t)tag[1];
        const char t = (char)p[2];
        p += 3;
        size_t sz = 0;
        switch (t) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'd': sz = 8; break;
            case 'Z': case 'H': {
                const uint8_t* q = p;
                while (q < end && *q) ++q;
                sz = (size_t)(q - p) + 1;
                break;
            }
            case 'B': {
                if (p + 5 > end) return false;
                const char sub = (char)p[0];
                const size_t cnt = le32(p + 1);
                const size_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
                sz = 5 + cnt * es;
                break;
            }
            default: return false;
        }
        if (p + sz > end) return false;
        if (hit) {
            switch (t) {
                case 'c': *v = (int8_t)p[0]; return true;
                case 'C': *v = p[0]; return true;
                case 's': *v = (int16_t)le16(p); return true;
                case 'S': *v = le16(p); return true;
                case 'i': *v = (int32_t)le32(p); return true;
                case 'I': *v = le32(p); return true;
                default: return false;
            }
        }
        p += sz;
    }
    return false;
}
}  // namespace

extern "C" int hh_ul_open(const char* path, int threads, int32_t min_mapq, int64_t min_alignment_length, int64_t max_distance_to_end,
                          double max_overlap_ratio, int64_t max_gap_len, hh_ul_reader** out) {
    if (!path || !out) {
        hh_set_error("hh_ul_open: bad argument");
        return HH_ERR_ARG;
    }
    *out = nullptr;
    hh_bgzf z;
    z.f = fopen(path, "rb");
    if (!z.f) {
        hh_set_error("hh_ul_open: cannot open %s", path);
        return HH_ERR_ARG;
    }
    z.threads = hh_io_threads(threads);
    hh_ul_reader* r = new hh_ul_reader();
    const int rc = [&]() -> int {
        if (bam_need(&z, 12) != 0) {
            hh_set_error("hh_ul_open: %s is empty or not a BAM file", path);
            return HH_ERR_ARG;
        }
        const uint8_t* p = z.raw.data() + z.raw_pos;
        if (memcmp(p, "BAM\1", 4) != 0) {
            hh_set_error("hh_ul_open: %s is not a BAM file", path);
            return HH_ERR_ARG;
        }
        const size_t l_text = le32(p + 4);
        if (bam_need(&z, 12 + l_text) != 0) {
            hh_set_error("hh_ul_open: truncated BAM header in %s", path);
            return HH_ERR_ARG;
        }
        const int32_t n_ref = (int32_t)le32(z.raw.data() + z.raw_pos + 8 + l_text);
        z.raw_pos += 12 + l_text;
        for (int32_t k = 0; k < n_ref; ++k) {
            if (bam_need(&z, 4) != 0) {
                hh_set_error("hh_ul_open: truncated BAM header in %s", path);
                return HH_ERR_ARG;
            }
            const size_t l_name = le32(z.raw.data() + z.raw_pos);
            if (l_name == 0 || bam_need(&z, 8 + l_name) != 0) {
                hh_set_error("hh_ul_open: truncated BAM header");
                return HH_ERR_ARG;
            }
            const char* nm = reinterpret_cast<const char*>(z.raw.data() + z.raw_pos + 4);
            r->names.append(nm, strnlen(nm, l_name));
            r->names.push_back('\0');
            r->ref_len.push_back((int32_t)le32(z.raw.data() + z.raw_pos + 4 + l_name));
            z.raw_pos += 8 + l_name;
        }
        bool have_primary = false;
        ul_aln prim{};
        std::string prim_name;
        std::vector<ul_aln> supp;
        auto emit = [&]() -> int {
            // the best supplementary: stable sort by AS, descending (only when there is a choice)
            size_t best = 0;
            if (supp.size() > 1) {
                for (const ul_aln& s : supp)
                    if (!s.has_as) {
                        hh_set_error("hh_ul: supplementary alignment of %s without an integer AS tag", prim_name.c_str());
                        return HH_ERR_ARG;
                    }
                for (size_t k = 1; k < supp.size(); ++k)
                    if (supp[k].as > supp[best].as) best = k;
            }
            const ul_aln& s = supp[best];
            // the two semi-contig pairs in read order (stable: the primary first on a tie)
            const ul_aln& a = (s.qs < prim.qs) ? s : prim;
            const ul_aln& b = (s.qs < prim.qs) ? prim : s;
            const int32_t ev[4] = {2 * a.ref + (a.reverse ? 0 : 1), 2 * b.ref + (b.reverse ? 1 : 0), prim.ref, s.ref};
            r->events.insert(r->events.end(), ev, ev + 4);
            return HH_OK;
        };
        for (;;) {
            int need = bam_need(&z, 4);
            if (need == 1) break;
            if (need < 0) return HH_ERR_ARG;                      // bgzf_fill / bam_need set the message
            const size_t bs = le32(z.raw.data() + z.raw_pos);
            if (bs < 32 || bam_need(&z, 4 + bs) != 0) {
                hh_set_error("hh_ul: corrupt or truncated BAM record");
                return HH_ERR_ARG;
            }
            const uint8_t* p = z.raw.data() + z.raw_pos + 4;
            const uint8_t* end = p + bs;
            z.raw_pos += 4 + bs;
            r->n_records++;
            const int32_t refid = (int32_t)le32(p), pos = (int32_t)le32(p + 4);
            const uint8_t l_read_name = p[8], mapq = p[9];
            const uint16_t n_cigar = le16(p + 12), flag = le16(p + 14);
            const int32_t l_seq = (int32_t)le32(p + 16);
            if (flag & 0x4) continue;                                 // filter=!flag.unmap
            const uint8_t* name = p + 32;
            const uint8_t* cig = name + l_read_name;
            const uint8_t* aux = cig + 4 * (size_t)n_cigar + ((size_t)l_seq + 1) / 2 + (size_t)l_seq;
            if (aux > end || refid < 0 || refid >= n_ref) {
                hh_set_error("hh_ul: corrupt BAM record (mapped record without a reference, or fields past its end)");
                return HH_ERR_ARG;
            }
            if (n_cigar == 0) {
                hh_set_error("hh_ul: mapped record without a CIGAR (reference_length undefined)");
                return HH_ERR_ARG;
            }
            int64_t ref_span = 0, read_len = 0, qs = 0, qe = 0, qe_noseq = 0;
            bool lead = true;
            for (uint16_t k = 0; k < n_cigar; ++k) {
                const uint32_t c = le32(cig + 4 * k);
                const uint32_t op = c & 15, ln = c >> 4;
                if (op == CIG_M || op == CIG_D || op == CIG_N || op == CIG_EQ || op == CIG_X) ref_span += ln;
                if (op == CIG_M || op == CIG_I || op == CIG_S || op == CIG_EQ || op == CIG_X || op == CIG_H) read_len += ln;
                // pysam query_alignment_start: soft clips before the first aligned operation (hard clips skipped)
                if (lead) {
                    if (op == CIG_S) qs += ln;
                    else if (op != CIG_H) lead = false;
                }
                // pysam query_alignment_end without SEQ: M / I / = / X lengths plus a soft clip met while the sum is 0
                if (op == CIG_M || op == CIG_I || op == CIG_EQ || op == CIG_X || (op == CIG_S && qe_noseq == 0)) qe_noseq += ln;
            }
            if (l_seq == 0) {
                qe = qe_noseq;
            } else {
                // with SEQ: l_qseq less the trailing soft clips (hard clips skipped; the first operation is never examined)
                qe = l_seq;
                for (int k = (int)n_cigar - 1; k >= 1; --k) {
                    const uint32_t c = le32(cig + 4 * k);
                    const uint32_t op = c & 15;
                    if (op == CIG_S) qe -= c >> 4;
                    else if (op != CIG_H) break;
                }
            }
            if (mapq < min_mapq || ref_span < min_alignment_length) continue;
            if (pos > max_distance_to_end && r->ref_len[(size_t)refid] - (pos + ref_span) > max_distance_to_end) continue;
            ul_aln a;
            a.ref = refid;
            a.reverse = (flag & 0x10) != 0;
            if (!a.reverse) {
                const uint32_t c0 = le32(cig);
                const int64_t hc = ((c0 & 15) == CIG_H) ? (int64_t)(c0 >> 4) : 0;
                a.qs = qs + hc;
                a.qe = qe + hc;
            } else {
                const uint32_t cl = le32(cig + 4 * ((size_t)n_cigar - 1));
                const int64_t hc = ((cl & 15) == CIG_H) ? (int64_t)(cl >> 4) : 0;
                a.qs = read_len - qe + hc;
                a.qe = read_len - qs + hc;
            }
            a.has_as = ul_aux_int(aux, end, "AS", &a.as);
            const char* nm = reinterpret_cast<const char*>(name);
            const size_t nm_len = strnlen(nm, l_read_name);
            if (flag == 0 || flag == 16) {
                if (!supp.empty() && emit() != HH_OK) return HH_ERR_ARG;
                prim = a;
                prim_name.assign(nm, nm_len);
                have_primary = true;
                supp.clear();
            } else if ((flag & 0x800) && have_primary && prim_name.size() == nm_len && memcmp(prim_name.data(), nm, nm_len) == 0 &&
                       refid != prim.ref) {
                // query intervals closed(start + 1, end) of the primary and the supplementary
                const int64_t lo = std::max(prim.qs, a.qs) + 1, hi = std::min(prim.qe, a.qe);
                if (lo <= hi) {
                    const double ratio = (double)(hi - lo + 1) / (double)std::min(prim.qe - prim.qs, a.qe - a.qs);
                    if (ratio > max_overlap_ratio) continue;
                } else if (lo - hi + 1 > max_gap_len) {
                    continue;                                     // the open gap between them, measured as if closed
                }
                supp.push_back(a);
            }
        }
        if (!supp.empty() && emit() != HH_OK) return HH_ERR_ARG;
        return HH_OK;
    }();
    fclose(z.f);
    if (rc != HH_OK) {
        delete r;
        return rc;
    }
    *out = r;
    return HH_OK;
}

extern "C" int hh_ul_info(hh_ul_reader* r, int32_t* n_ref, int64_t* names_bytes, int64_t* n_events, int64_t* n_records) {
    if (!r) {
        hh_set_error("hh_ul_info: NULL handle");
        return HH_ERR_ARG;
    }
    if (n_ref) *n_ref = (int32_t)r->ref_len.size();
    if (names_bytes) *names_bytes = (int64_t)r->names.size();
    if (n_events) *n_events = (int64_t)(r->events.size() / 4);
    if (n_records) *n_records = r->n_records;
    return HH_OK;
}

extern "C" int hh_ul_fetch(hh_ul_reader* r, char* names, int64_t* ref_len, int32_t* events) {
    if (!r) {
        hh_set_error("hh_ul_fetch: NULL handle");
        return HH_ERR_ARG;
    }
    if (names && !r->names.empty()) memcpy(names, r->names.data(), r->names.size());
    if (ref_len && !r->ref_len.empty()) memcpy(ref_len, r->ref_len.data(), r->ref_len.size() * sizeof(int64_t));
    if (events && !r->events.empty()) memcpy(events, r->events.data(), r->events.size() * sizeof(int32_t));
    return HH_OK;
}

extern "C" int hh_ul_close(hh_ul_reader* r) {
    delete r;
    return HH_OK;
}

// ---------------------------------------------------------------------------------------------
// paired_links.clm straight from the record stream (update_clm_dict 395-401 + output_clm 376-392), threaded:
// records are partitioned by contig pair (stable, so stream order survives inside a pair), every partition is
// grouped by a stable sort, the pairs with >= 2 links are ordered by their first record (= dict insertion order),
// and slices of that list are turned into text by a pool of threads while one thread writes the slices in order.
// ---------------------------------------------------------------------------------------------
struct hh_clm_seg {
    uint32_t first;                   // stream index of the pair's first record
    uint32_t len;                     // links
    uint64_t start;                   // position of its (key, idx) run in the grouped array
};

extern "C" int hh_clm_from_records(const char* path, const char* names_blob, int32_t n_names, const int32_t* rec, int64_t n_rec,
                                   const int64_t* ctg_len, const int32_t* name_rank, int threads) {
    if (!path || !names_blob || !ctg_len || !name_rank || n_names <= 0 || n_rec < 0 || (n_rec > 0 && !rec)) {
        hh_set_error("hh_clm_from_records: bad argument");
        return HH_ERR_ARG;
    }
    if (n_rec > 0xFFFFFFFELL) {
        hh_set_error("hh_clm_from_records: more than 2^32 records");
        return HH_ERR_UNSUPPORTED;
    }
    const int T = hh_io_threads(threads);
    std::vector<const char*> name((size_t)n_names);
    std::vector<size_t> nlen((size_t)n_names);
    {
        const char* p = names_blob;
        for (int32_t i = 0; i < n_names; ++i) {
            name[(size_t)i] = p;
            nlen[(size_t)i] = strlen(p);
            p += nlen[(size_t)i] + 1;
        }
    }
    FILE* f = fopen(path, "w");
    if (!f) {
        hh_set_error("hh_clm_from_records: cannot create %s", path);
        return HH_ERR_ARG;
    }
    setvbuf(f, nullptr, _IONBF, 0);
    const uint64_t N = (uint64_t)n_names;
    // key of a record: (i, j) ordered by name rank; 0 = unusable (same contig / id outside the FASTA)
    auto key_of = [&](int64_t r, bool* swapped) -> uint64_t {
        const int32_t a = rec[4 * r], b = rec[4 * r + 2];
        if (a == b || (uint32_t)a >= (uint32_t)n_names || (uint32_t)b >= (uint32_t)n_names) return 0;
        const bool sw = name_rank[a] > name_rank[b];
        *swapped = sw;
        const uint64_t i = (uint64_t)(sw ? b : a), j = (uint64_t)(sw ? a : b);
        return i * N + j + 1;
    };
    auto mix = [](uint64_t k) {
        k ^= k >> 33;
        k *= 0xff51afd7ed558ccdull;
        k ^= k >> 33;
        return k;
    };
    auto run_pool = [&](int n_workers, const std::function<void(int)>& fn) {
        if (n_workers <= 1) {
            fn(0);
            return;
        }
        std::vector<std::thread> pool;
        for (int t = 0; t < n_workers; ++t) pool.emplace_back(fn, t);
        for (auto& th : pool) th.join();
    };
    // ---- A/B/C: stable partition of (key, idx) into buckets
    const int NB = 1024;
    const int64_t chunk = (n_rec + T - 1) / T;
    std::vector<std::vector<uint64_t>> cnt((size_t)T, std::vector<uint64_t>((size_t)NB, 0));
    run_pool(T, [&](int t) {
        const int64_t lo = std::min<int64_t>(n_rec, chunk * t), hi = std::min<int64_t>(n_rec, lo + chunk);
        bool sw;
        for (int64_t r = lo; r < hi; ++r) {
            const uint64_t k = key_of(r, &sw);
            if (k) cnt[(size_t)t][mix(k) & (NB - 1)]++;
        }
    });
    std::vector<uint64_t> bucket_start((size_t)NB + 1, 0);
    std::vector<std::vector<uint64_t>> cursor((size_t)T, std::vector<uint64_t>((size_t)NB, 0));
    {
        uint64_t acc = 0;
        for (int b = 0; b < NB; ++b) {
            bucket_start[(size_t)b] = acc;
            for (int t = 0; t < T; ++t) {
                cursor[(size_t)t][(size_t)b] = acc;        // thread t's share of bucket b starts here: idx ascending inside a bucket
                acc += cnt[(size_t)t][(size_t)b];
            }
        }
        bucket_start[(size_t)NB] = acc;
    }
    const uint64_t n_used = bucket_start[(size_t)NB];
    struct kv {
        uint64_t key;
        uint32_t idx;
    };
    std::vector<kv> items((size_t)n_used);
    run_pool(T, [&](int t) {
        const int64_t lo = std::min<int64_t>(n_rec, chunk * t), hi = std::min<int64_t>(n_rec, lo + chunk);
        bool sw;
        std::vector<uint64_t>& cur = cursor[(size_t)t];
        for (int64_t r = lo; r < hi; ++r) {
            const uint64_t k = key_of(r, &sw);
            if (k) items[(size_t)cur[mix(k) & (NB - 1)]++] = kv{k, (uint32_t)r};
        }
    });
    // ---- D: group every bucket; E: pairs with >= 2 links in first-seen order
    std::vector<std::vector<hh_clm_seg>> per_bucket((size_t)NB);
    std::atomic<int> next_bucket(0);
    run_pool(T, [&](int) {
        for (;;) {
            const int b = next_bucket.fetch_add(1);
            if (b >= NB) break;
            kv* s = items.data() + bucket_start[(size_t)b];
            kv* e = items.data() + bucket_start[(size_t)b + 1];
            std::stable_sort(s, e, [](const kv& x, const kv& y) { return x.key < y.key; });
            for (kv* p = s; p < e;) {
                kv* q = p + 1;
                while (q < e && q->key == p->key) ++q;
                if (q - p >= 2) per_bucket[(size_t)b].push_back(hh_clm_seg{p->idx, (uint32_t)(q - p), (uint64_t)(p - items.data())});
                p = q;
            }
        }
    });
    std::vector<hh_clm_seg> segs;
    {
        size_t total = 0;
        for (auto& v : per_bucket) total += v.size();
        segs.reserve(total);
        for (auto& v : per_bucket) {
            segs.insert(segs.end(), v.begin(), v.end());
            std::vector<hh_clm_seg>().swap(v);
        }
        std::sort(segs.begin(), segs.end(), [](const hh_clm_seg& x, const hh_clm_seg& y) { return x.first < y.first; });
    }
    // ---- F: text.  Slices of ~256k links; formatted by the pool, written in order by this thread.
    std::vector<size_t> slice_start{0};
    {
        uint64_t acc = 0;
        for (size_t k = 0; k < segs.size(); ++k) {
            acc += segs[k].len;
            if (acc >= (1u << 18)) {
                slice_start.push_back(k + 1);
                acc = 0;
            }
        }
        if (slice_start.back() != segs.size()) slice_start.push_back(segs.size());
    }
    const size_t n_slices = slice_start.size() - 1;
    std::vector<hh_bytes> text(n_slices);
    std::vector<char> ready(n_slices, 0);
    std::mutex mu;
    std::condition_variable cv;
    std::atomic<size_t> next_slice(0);
    size_t written = 0;                // slices already on disk (guarded by mu)
    const size_t max_ahead = (size_t)T * 4;
    bool failed = false;
    static const char sg[4][2] = {{'+', '+'}, {'+', '-'}, {'-', '+'}, {'-', '-'}};
    auto format_slices = [&](int) {
        std::vector<int64_t> d[4];
        for (;;) {
            const size_t sidx = next_slice.fetch_add(1);
            if (sidx >= n_slices) break;
            {
                std::unique_lock<std::mutex> lk(mu);          // do not run too far ahead of the writer
                cv.wait(lk, [&] { return sidx < written + max_ahead; });
            }
            hh_bytes& out = text[sidx];
            for (size_t k = slice_start[sidx]; k < slice_start[sidx + 1]; ++k) {
                const hh_clm_seg& sgm = segs[k];
                const kv* it = items.data() + sgm.start;
                const uint64_t key = it->key - 1;
                const int32_t ci = (int32_t)(key / N), cj = (int32_t)(key % N);
                const int64_t li = ctg_len[ci], lj = ctg_len[cj];
                for (int o = 0; o < 4; ++o) d[o].resize(sgm.len);
                for (uint32_t t = 0; t < sgm.len; ++t) {
                    const int32_t* r = rec + 4 * (int64_t)it[t].idx;
                    const bool sw = r[0] != ci;                 // the record names the pair as (j, i)
                    const int64_t a0 = sw ? r[3] : r[1], b0 = sw ? r[1] : r[3];
                    d[0][t] = li - a0 + b0;                     // ++  (395-401)
                    d[1][t] = li - a0 + lj - b0;                // +-
                    d[2][t] = a0 + b0;                          // -+
                    d[3][t] = a0 + lj - b0;                     // --
                }
                const size_t per_line = nlen[(size_t)ci] + nlen[(size_t)cj] + 64 + (size_t)sgm.len * 2 * 21;
                for (int o = 0; o < 4; ++o) {
                    std::sort(d[o].begin(), d[o].end());
                    char* q = out.room(per_line);
                    memcpy(q, name[(size_t)ci], nlen[(size_t)ci]);
                    q += nlen[(size_t)ci];
                    *q++ = sg[o][0];
                    *q++ = ' ';
                    memcpy(q, name[(size_t)cj], nlen[(size_t)cj]);
                    q += nlen[(size_t)cj];
                    *q++ = sg[o][1];
                    *q++ = '\t';
                    q = put_i64(q, (int64_t)sgm.len * 2);
                    *q++ = '\t';
                    for (uint32_t t = 0; t < sgm.len; ++t) {
                        if (t) *q++ = ' ';
                        q = put_i64(q, d[o][t]);
                        *q++ = ' ';
                        q = put_i64(q, d[o][t]);
                    }
                    *q++ = '\n';
                    out.len = (size_t)(q - out.data);
                }
            }
            {
                std::lock_guard<std::mutex> lk(mu);
                ready[sidx] = 1;
            }
            cv.notify_all();
        }
    };
    std::vector<std::thread> pool;
    for (int t = 0; t < T; ++t) pool.emplace_back(format_slices, t);
    for (size_t sidx = 0; sidx < n_slices; ++sidx) {
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return ready[sidx] != 0; });
        }
        if (text[sidx].len && fwrite(text[sidx].data, 1, text[sidx].len, f) != text[sidx].len) failed = true;
        text[sidx].release();
        {
            std::lock_guard<std::mutex> lk(mu);
            written = sidx + 1;
        }
        cv.notify_all();
    }
    for (auto& th : pool) th.join();
    if (fclose(f) != 0 || failed) {
        hh_set_error("hh_clm_from_records: write to %s failed", path);
        return HH_ERR_ARG;
    }
    return HH_OK;
}

// ---------------------------------------------------------------------------------------------
// full_links.pkl / HT_links.pkl (output_pickle, 710-715) without building the Python dicts: a pickle stream
// (protocol 3 opcodes) that loads as `defaultdict(int, {(name_i, name_j): value, ...})` in entry order.
// Strings are memoised like pickle does, so the loaded keys share one str object per contig.
//   mode 0: one entry per pair, value = values_i64[e] (or values_f64[e] when given; with is_float, entry e is a float
//           when is_float[e] and the int (int64_t)values_f64[e] otherwise -- the mixed dict of a fractional phasing weight);
//   mode 1: HT_link_dict -- ht[e][4] = {HH, HT, TH, TT}; non-zero counters become the keys
//           (name_i + '_H'|'_T', name_j + '_H'|'_T') (update_HT_link_dict, 404-416).
// ---------------------------------------------------------------------------------------------
namespace {
struct pickle_out {
    FILE* f;
    std::vector<char> buf;
    bool failed = false;
    explicit pickle_out(FILE* fp) : f(fp) { buf.reserve(1u << 22); }
    inline void flush_if(size_t need) {
        if (buf.size() + need > (1u << 22)) flush();
    }
    void flush() {
        if (!buf.empty() && fwrite(buf.data(), 1, buf.size(), f) != buf.size()) failed = true;
        buf.clear();
    }
    inline void byte(uint8_t b) { buf.push_back((char)b); }
    inline void raw(const void* p, size_t n) { buf.insert(buf.end(), (const char*)p, (const char*)p + n); }
    inline void u32(uint32_t v) {
        const uint8_t b[4] = {(uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16), (uint8_t)(v >> 24)};
        raw(b, 4);
    }
    inline void put(uint32_t memo) {          // BINPUT / LONG_BINPUT
        if (memo < 256) {
            byte('q');
            byte((uint8_t)memo);
        } else {
            byte('r');
            u32(memo);
        }
    }
    inline void get(uint32_t memo) {          // BINGET / LONG_BINGET
        if (memo < 256) {
            byte('h');
            byte((uint8_t)memo);
        } else {
            byte('j');
            u32(memo);
        }
    }
    inline void integer(int64_t v) {
        if (v >= 0 && v < 256) {
            byte('K');
            byte((uint8_t)v);
        } else if (v >= 0 && v < 65536) {
            byte('M');
            byte((uint8_t)v);
            byte((uint8_t)(v >> 8));
        } else if (v >= -2147483648LL && v <= 2147483647LL) {
            byte('J');
            u32((uint32_t)(int32_t)v);
        } else {                              // LONG1, 8 bytes little-endian two's complement
            byte(0x8a);
            byte(8);
            for (int k = 0; k < 8; ++k) byte((uint8_t)((uint64_t)v >> (8 * k)));
        }
    }
    inline void real(double d) {              // BINFLOAT: big-endian IEEE double
        uint64_t u;
        memcpy(&u, &d, 8);
        byte('G');
        for (int k = 7; k >= 0; --k) byte((uint8_t)(u >> (8 * k)));
    }
};
}   // namespace

static int pickle_links(const char* path, const char* names_blob, int32_t n_names, const int32_t* key_i, const int32_t* key_j,
                        int64_t n_entries, const int64_t* values_i64, const double* values_f64, const uint8_t* is_float,
                        const uint32_t* ht) {
    if (!path || !names_blob || n_names <= 0 || n_entries < 0 || (n_entries > 0 && (!key_i || !key_j)) ||
        (n_entries > 0 && !values_i64 && !values_f64 && !ht)) {
        hh_set_error("hh_pickle_links: bad argument");
        return HH_ERR_ARG;
    }
    std::vector<const char*> name((size_t)n_names);
    std::vector<uint32_t> nlen((size_t)n_names);
    {
        const char* p = names_blob;
        for (int32_t i = 0; i < n_names; ++i) {
            name[(size_t)i] = p;
            nlen[(size_t)i] = (uint32_t)strlen(p);
            p += nlen[(size_t)i] + 1;
        }
    }
    FILE* f = fopen(path, "wb");
    if (!f) {
        hh_set_error("hh_pickle_links: cannot create %s", path);
        return HH_ERR_ARG;
    }
    pickle_out o(f);
    // defaultdict.__reduce__ -> (defaultdict, (int,), None, None, items): GLOBAL GLOBAL TUPLE1 REDUCE, then SETITEMS batches
    o.byte(0x80);
    o.byte(3);
    static const char g1[] = "ccollections\ndefaultdict\n";
    static const char g2[] = "cbuiltins\nint\n";
    o.raw(g1, sizeof(g1) - 1);
    o.put(0);
    o.raw(g2, sizeof(g2) - 1);
    o.put(1);
    o.byte(0x85);
    o.put(2);
    o.byte('R');
    o.put(3);
    uint32_t next_memo = 4;
    const int variants = ht ? 2 : 1;            // HT mode: name_H and name_T are different strings
    std::vector<uint32_t> memo((size_t)n_names * (size_t)variants, 0);
    auto key_string = [&](int32_t c, int suffix) {   // suffix: -1 none, 0 '_H', 1 '_T'
        uint32_t& m = memo[(size_t)c * (size_t)variants + (size_t)(suffix < 0 ? 0 : suffix)];
        if (m) {
            o.get(m);
            return;
        }
        const uint32_t l = nlen[(size_t)c] + (suffix < 0 ? 0u : 2u);
        o.byte('X');
        o.u32(l);
        o.raw(name[(size_t)c], nlen[(size_t)c]);
        if (suffix >= 0) o.raw(suffix ? "_T" : "_H", 2);
        m = next_memo++;
        o.put(m);
    };
    int in_batch = 0;
    auto open_batch = [&]() {
        if (in_batch == 0) o.byte('(');
    };
    auto close_batch = [&](bool force) {
        if (in_batch > 0 && (force || in_batch >= 1000)) {
            o.byte('u');
            in_batch = 0;
        }
    };
    for (int64_t e = 0; e < n_entries; ++e) {
        const int32_t a = key_i[e], b = key_j[e];
        if ((uint32_t)a >= (uint32_t)n_names || (uint32_t)b >= (uint32_t)n_names) {
            fclose(f);
            hh_set_error("hh_pickle_links: entry %lld names a contig outside [0, %d)", (long long)e, n_names);
            return HH_ERR_ARG;
        }
        o.flush_if((size_t)nlen[(size_t)a] + nlen[(size_t)b] + 256);
        if (!ht) {
            open_batch();
            key_string(a, -1);
            key_string(b, -1);
            o.byte(0x86);
            if (values_f64 && (!is_float || is_float[e])) o.real(values_f64[e]);
            else o.integer(values_f64 ? (int64_t)values_f64[e] : values_i64[e]);
            ++in_batch;
            close_batch(false);
        } else {
            for (int c = 0; c < 4; ++c) {
                const uint32_t v = ht[e * 4 + c];
                if (!v) continue;
                open_batch();
                key_string(a, c >> 1);
                key_string(b, c & 1);
                o.byte(0x86);
                o.integer((int64_t)v);
                ++in_batch;
                close_batch(false);
            }
        }
    }
    close_batch(true);
    o.byte('.');
    o.flush();
    if (fclose(f) != 0 || o.failed) {
        hh_set_error("hh_pickle_links: write to %s failed", path);
        return HH_ERR_ARG;
    }
    return HH_OK;
}

extern "C" int hh_pickle_links(const char* path, const char* names_blob, int32_t n_names, const int32_t* key_i, const int32_t* key_j,
                               int64_t n_entries, const int64_t* values_i64, const double* values_f64, const uint32_t* ht) {
    return pickle_links(path, names_blob, n_names, key_i, key_j, n_entries, values_i64, values_f64, nullptr, ht);
}

extern "C" int hh_pickle_links_mixed(const char* path, const char* names_blob, int32_t n_names, const int32_t* key_i,
                                     const int32_t* key_j, int64_t n_entries, const double* values, const uint8_t* is_float) {
    if (n_entries > 0 && (!values || !is_float)) {
        hh_set_error("hh_pickle_links_mixed: bad argument");
        return HH_ERR_ARG;
    }
    return pickle_links(path, names_blob, n_names, key_i, key_j, n_entries, nullptr, values, is_float, nullptr);
}

// ---------------------------------------------------------------------------------------------------------------------
// .pairs writer: the inverse of hh_pairs_next for fixtures and benchmarks (4DN .pairs text, 1-based positions, seven
// columns `r{index} chr1 pos1 chr2 pos2 + -`).  Slices of the records are formatted on `threads` host threads and
// written in order.
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int hh_pairs_write(const char* path, const char* names_blob, int32_t n_names, const int32_t* rec, int64_t n_rec,
                              int64_t first_index, int append, int threads) {
    if (!(path && names_blob && (rec || n_rec == 0))) {
        hh_set_error("hh_pairs_write: NULL argument");
        return HH_ERR_ARG;
    }
    std::vector<const char*> nm((size_t)n_names);
    std::vector<uint32_t> nl((size_t)n_names);
    {
        const char* q = names_blob;
        for (int32_t k = 0; k < n_names; ++k) {
            nm[(size_t)k] = q;
            nl[(size_t)k] = (uint32_t)strlen(q);
            q += nl[(size_t)k] + 1;
        }
    }
    FILE* f = fopen(path, append ? "ab" : "wb");
    if (!f) {
        hh_set_error("hh_pairs_write: cannot open %s", path);
        return HH_ERR_ARG;
    }
    if (!append) fputs("## pairs format v1.0\n#columns: readID chr1 pos1 chr2 pos2 strand1 strand2\n", f);
    const int T = hh_io_threads(threads);
    const int64_t SL = 1 << 18;                 // records per slice
    std::vector<std::vector<char>> buf((size_t)T);
    int rc = HH_OK;
    for (int64_t base = 0; base < n_rec && rc == HH_OK; base += SL * T) {
        std::vector<std::thread> pool;
        for (int t = 0; t < T; ++t) {
            const int64_t lo = base + (int64_t)t * SL, hi = std::min(n_rec, lo + SL);
            buf[(size_t)t].clear();
            if (lo >= hi) continue;
            pool.emplace_back([&, t, lo, hi]() {
                std::vector<char>& b = buf[(size_t)t];
                b.resize((size_t)(hi - lo) * 160);
                char* q = b.data();
                for (int64_t i = lo; i < hi; ++i) {
                    const int32_t* r = rec + i * 4;
                    if ((size_t)(q - b.data()) + 2 * 64 + 512 > b.size()) {
                        const size_t used = (size_t)(q - b.data());
                        b.resize(b.size() * 2);
                        q = b.data() + used;
                    }
                    *q++ = 'r';
                    q = put_i64(q, first_index + i);
                    for (int side = 0; side < 2; ++side) {
                        const int32_t c = r[2 * side];
                        *q++ = '\t';
                        if (c >= 0 && c < n_names) {
                            memcpy(q, nm[(size_t)c], nl[(size_t)c]);
                            q += nl[(size_t)c];
                        } else {
                            *q++ = '*';
                        }
                        *q++ = '\t';
                        q = put_i64(q, (int64_t)r[2 * side + 1] + 1);
                    }
                    memcpy(q, "\t+\t-\n", 5);
                    q += 5;
                }
                b.resize((size_t)(q - b.data()));
            });
        }
        for (auto& th : pool) th.join();
        for (int t = 0; t < T; ++t)
            if (!buf[(size_t)t].empty() && fwrite(buf[(size_t)t].data(), 1, buf[(size_t)t].size(), f) != buf[(size_t)t].size()) rc = HH_ERR_ARG;
    }
    fclose(f);
    if (rc != HH_OK) hh_set_error("hh_pairs_write: write to %s failed", path);
    return rc;
}
