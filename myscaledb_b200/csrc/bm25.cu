// bm25.cu -- K8: BM25 posting-list scorer behind TextSearch()/HybridSearch().
//
// Replaces TANTIVY::ffi_bm25_search / ffi_get_doc_freq / ffi_get_total_num_docs /
// ffi_get_total_num_tokens / ffi_index_multi_column_docs as called from
// TantivyIndexStore (reference: src/Storages/MergeTree/TantivyIndexStore.cpp:742, :900-998) and
// driven by MergeTreeTextSearchManager::textSearch
// (src/VectorIndex/Storages/MergeTreeTextSearchManager.cpp:69-279).
//
// The Rust crate (tantivy_search 0.1.0 over tantivy 0.21.1) is not in the reference tree; the
// scoring formula is tantivy's published BM25 (k1 1.2, b 0.75, fp32 idf, 1-byte field-norm code),
// the tokenizer is tantivy's "default" (alphanumeric runs, <= 40 bytes, lowercased).
//
// Layout (one index per part, resident in HBM): postings as two flat arrays (doc ordinal u32,
// term frequency u32) concatenated term after term, each list sorted by doc; one field-norm code
// byte per (field, doc); row id per doc.  The dictionary (term -> list) stays on the host: a
// query touches a handful of terms.
// Kernel: bm25_score_kernel, grid (slices, queries).  A thread takes one posting of one clause
// (field, term) of its query; the doc is OWNED by the first clause that contains it (binary
// search in the earlier lists), the owner adds the other clauses' contributions in clause order
// (binary search in the later lists) so sums are deterministic and equal the reference's
// term-at-a-time order; dead rows (alive bitmap) are skipped; survivors go through the same
// warp-cooperative top-k as the vector scan (key = -score, tie -> smaller doc).
// HBM-bound: sum over clauses of df * (8 B posting + 1 B field norm).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

constexpr float kBm25K1 = 1.2f;
constexpr float kBm25B = 0.75f;
constexpr int kMaxClauses = 64;

static uint32_t g_fieldnorm[256];
static std::once_flag g_fieldnorm_once;
static void init_fieldnorm() {
    std::call_once(g_fieldnorm_once, [] {
        for (int i = 0; i < 40; i++) g_fieldnorm[i] = (uint32_t)i;
        uint64_t v = 40;
        for (int i = 40; i < 256; i++) {
            g_fieldnorm[i] = v > 0xffffffffull ? 0xffffffffu : (uint32_t)v;
            const int shift = (i - 40) / 8 + 1;
            v += shift >= 40 ? (1ull << 40) : (1ull << shift);
        }
    });
}
static uint8_t fieldnorm_to_id(uint32_t n) {
    int lo = 0, hi = 255;
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (g_fieldnorm[mid] <= n) lo = mid; else hi = mid - 1;
    }
    return (uint8_t)lo;
}

// tantivy 0.21 "default" analyzer: SimpleTokenizer (maximal runs of char::is_alphanumeric) -> RemoveLongFilter::limit(40)
// (a token is kept when it has FEWER than 40 bytes) -> LowerCaser (Unicode).  UTF-8 is decoded; the Unicode classes are
// carried for the blocks that matter in practice: Latin-1 signs, General Punctuation, currency, arrows / technical / box /
// dingbat symbols, CJK and full-width punctuation separate tokens; Latin-1, Latin Extended-A, Greek, Cyrillic and
// full-width capitals are lowercased; any other non-ASCII code point counts as a letter.
static size_t utf8_decode(const unsigned char *s, size_t n, uint32_t &cp) {
    if (s[0] < 0x80) { cp = s[0]; return 1; }
    if ((s[0] & 0xE0) == 0xC0 && n >= 2 && (s[1] & 0xC0) == 0x80) { cp = ((s[0] & 0x1Fu) << 6) | (s[1] & 0x3Fu); return 2; }
    if ((s[0] & 0xF0) == 0xE0 && n >= 3 && (s[1] & 0xC0) == 0x80 && (s[2] & 0xC0) == 0x80) {
        cp = ((s[0] & 0x0Fu) << 12) | ((s[1] & 0x3Fu) << 6) | (s[2] & 0x3Fu);
        return 3;
    }
    if ((s[0] & 0xF8) == 0xF0 && n >= 4 && (s[1] & 0xC0) == 0x80 && (s[2] & 0xC0) == 0x80 && (s[3] & 0xC0) == 0x80) {
        cp = ((s[0] & 0x07u) << 18) | ((s[1] & 0x3Fu) << 12) | ((s[2] & 0x3Fu) << 6) | (s[3] & 0x3Fu);
        return 4;
    }
    cp = 0xFFFD;  // invalid byte: treated as a letter, one byte consumed
    return 1;
}
static void utf8_append(uint32_t cp, std::string &out) {
    if (cp < 0x80) out.push_back((char)cp);
    else if (cp < 0x800) { out.push_back((char)(0xC0 | (cp >> 6))); out.push_back((char)(0x80 | (cp & 0x3F))); }
    else if (cp < 0x10000) { out.push_back((char)(0xE0 | (cp >> 12))); out.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); out.push_back((char)(0x80 | (cp & 0x3F))); }
    else { out.push_back((char)(0xF0 | (cp >> 18))); out.push_back((char)(0x80 | ((cp >> 12) & 0x3F))); out.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); out.push_back((char)(0x80 | (cp & 0x3F))); }
}
static bool cp_is_alnum(uint32_t c) {
    if (c < 0x80) return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z');
    if (c <= 0xBF) return c == 0xAA || c == 0xB2 || c == 0xB3 || c == 0xB5 || c == 0xB9 || c == 0xBA || c == 0xBC || c == 0xBD || c == 0xBE;
    if (c == 0xD7 || c == 0xF7) return false;
    if (c >= 0x2000 && c <= 0x206F) return false;
    if (c >= 0x20A0 && c <= 0x20CF) return false;
    if (c >= 0x2190 && c <= 0x245F) return false;
    if (c >= 0x2500 && c <= 0x2BFF) return false;
    if (c >= 0x2E00 && c <= 0x2E7F) return false;
    if ((c >= 0x3000 && c <= 0x3004) || (c >= 0x3008 && c <= 0x3020) || c == 0x3030 || (c >= 0x303D && c <= 0x303F)) return false;
    if ((c >= 0xFE10 && c <= 0xFE1F) || (c >= 0xFE30 && c <= 0xFE6F)) return false;
    if ((c >= 0xFF00 && c <= 0xFF0F) || (c >= 0xFF1A && c <= 0xFF20) || (c >= 0xFF3B && c <= 0xFF40) || (c >= 0xFF5B && c <= 0xFF65) ||
        (c >= 0xFFE0 && c <= 0xFFEF))
        return false;
    return true;
}
static uint32_t cp_lower(uint32_t c) {
    if (c < 0x80) return (c >= 'A' && c <= 'Z') ? c + 32 : c;
    if (c >= 0xC0 && c <= 0xDE && c != 0xD7) return c + 0x20;
    if (c >= 0x100 && c <= 0x137) return (c & 1) ? c : c + 1;
    if (c >= 0x139 && c <= 0x148) return (c & 1) ? c + 1 : c;
    if (c >= 0x14A && c <= 0x177) return (c & 1) ? c : c + 1;
    if (c == 0x178) return 0xFF;
    if (c >= 0x179 && c <= 0x17E) return (c & 1) ? c + 1 : c;
    if (c >= 0x391 && c <= 0x3A9 && c != 0x3A2) return c + 0x20;
    if (c >= 0x410 && c <= 0x42F) return c + 0x20;
    if (c >= 0x400 && c <= 0x40F) return c + 0x50;
    if (c >= 0xFF21 && c <= 0xFF3A) return c + 0x20;
    return c;
}
template <typename F>
static void tokenize_default(const char *text, F &&emit) {
    const unsigned char *t = reinterpret_cast<const unsigned char *>(text);
    const size_t n = strlen(text);
    size_t i = 0;
    std::string tok;
    while (i < n) {
        uint32_t cp;
        size_t adv = utf8_decode(t + i, n - i, cp);
        if (!cp_is_alnum(cp)) {
            i += adv;
            continue;
        }
        const size_t s = i;
        tok.clear();
        while (i < n) {
            adv = utf8_decode(t + i, n - i, cp);
            if (!cp_is_alnum(cp)) break;
            if (tok.size() < 160) utf8_append(cp_lower(cp), tok);
            i += adv;
        }
        if (i - s >= 40) continue;  // RemoveLongFilter::limit(40) keeps len < 40
        emit(tok);
    }
}

struct TermList {
    std::vector<uint32_t> docs, tfs;
    uint64_t offset = 0;  // into the device arrays after commit
};

struct Clause {  // device-side description of one (field, term) of one query
    uint64_t offset;
    uint32_t df;
    float weight;
    uint32_t field;
    uint32_t cache;  // index of the 256-entry norm table (high bits: term index << 24)
};
__host__ __device__ static inline uint32_t clause_cache(const Clause &c) { return c.cache & 0xffffffu; }
__host__ __device__ static inline uint32_t clause_term(const Clause &c) { return c.cache >> 24; }

struct Bm25ScoreParams {
    const uint32_t *post_docs;
    const uint32_t *post_tfs;
    const uint8_t *fieldnorm;  // [n_fields][n_docs]
    const uint32_t *row_id;    // [n_docs]
    const uint8_t *alive;      // LSB-first over row ids, or null
    const Clause *clauses;     // all queries
    const uint32_t *clause_begin;  // [nq + 1]
    const uint64_t *term_mask;     // [nq] AND: bit per query term that must be matched (in any searched field)
    const float *caches;       // [n_caches][256]
    float *part_keys;          // [nq][gridDim.x][k]
    uint32_t *part_ids;
    uint32_t n_docs;
    uint32_t q_begin;          // query of blockIdx.y == 0: a batch launches in slices of at most 65535 queries (gridDim.y)
    int k;
    int operator_or;
};

// first index in docs[0..n) whose value is >= key, found by the whole warp: every round the 32 lanes probe 32 evenly
// spaced splitters of the remaining range (one ballot narrows it 33x), the last <= 32 entries are read side by side
__device__ __forceinline__ uint32_t warp_lower_bound(const uint32_t *docs, uint32_t n, uint32_t key, int lane) {
    uint32_t lo = 0, hi = n;  // the answer lies in [lo, hi]
    while (hi - lo > 32) {
        const uint64_t span = hi - lo;
        const uint32_t idx = lo + (uint32_t)(span * (uint32_t)(lane + 1) / 33);  // lo < idx < hi, ascending with the lane
        const unsigned less = __ballot_sync(0xffffffffu, docs[idx] < key);        // a prefix mask: the list is sorted
        const uint32_t cnt = __popc(less);
        const uint32_t nlo = cnt ? lo + (uint32_t)(span * cnt / 33) + 1 : lo;
        const uint32_t nhi = cnt < 32 ? lo + (uint32_t)(span * (cnt + 1) / 33) : hi;
        lo = nlo;
        hi = nhi;
    }
    const uint32_t j = lo + (uint32_t)lane;
    const unsigned less = __ballot_sync(0xffffffffu, j < hi && docs[j] < key);
    return lo + __popc(less);
}
// [wlo, whi): the positions in docs[0..n) of every value in [dmin, dmax]
__device__ __forceinline__ void warp_window(const uint32_t *docs, uint32_t n, uint32_t dmin, uint32_t dmax, int lane,
                                            uint32_t &wlo, uint32_t &whi) {
    wlo = warp_lower_bound(docs, n, dmin, lane);
    whi = wlo + warp_lower_bound(docs + wlo, n - wlo, dmax + 1u, lane);  // doc ordinals stay far below 2^32 - 1
}
// private binary search of one lane inside the warp's window
__device__ __forceinline__ bool window_find(const uint32_t *docs, uint32_t lo, uint32_t hi, uint32_t doc, uint32_t &pos) {
    const uint32_t end = hi;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (docs[mid] < doc) lo = mid + 1; else hi = mid;
    }
    pos = lo;
    return lo < end && docs[lo] == doc;
}

__global__ void __launch_bounds__(256) bm25_score_kernel(const Bm25ScoreParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *lk = reinterpret_cast<float *>(smem_raw);
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + 8 * p.k);
    __shared__ Clause cl[kMaxClauses];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t q = p.q_begin + blockIdx.y;
    const uint32_t c0 = p.clause_begin[q], nc = p.clause_begin[q + 1] - c0;
    for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) cl[i] = p.clauses[c0 + i];
    WarpTopK list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncthreads();

    for (uint32_t c = 0; c < nc; c++) {
        const uint32_t df = cl[c].df;
        const uint32_t *docs = p.post_docs + cl[c].offset;
        const uint32_t *tfs = p.post_tfs + cl[c].offset;
        // warp-uniform trip count
        for (uint32_t base = (blockIdx.x * 8 + warp) * 32; base < df; base += gridDim.x * 256) {
            const uint32_t i = base + lane;
            const bool valid = i < df;
            bool cand = false;
            float key = FLT_MAX;
            // the 32 postings of this step are consecutive in a sorted list: their counterparts in another clause's
            // list lie in one narrow window, which the warp brackets together (32-ary search, 3 probes for 32 K
            // postings) before each lane finishes with a short private binary search inside it
            const uint32_t doc = valid ? docs[i] : 0u;
            const uint32_t n_valid = min(32u, df - base);
            const uint32_t dmin = __shfl_sync(0xffffffffu, doc, 0);
            const uint32_t dmax = __shfl_sync(0xffffffffu, doc, (int)n_valid - 1);
            bool active = valid;  // no earlier clause owns this document
            uint32_t pos;
            for (uint32_t e = 0; e < c; e++) {
                if (!cl[e].df) continue;
                const uint32_t *od = p.post_docs + cl[e].offset;
                uint32_t wlo, whi;
                warp_window(od, cl[e].df, dmin, dmax, lane, wlo, whi);
                if (active && window_find(od, wlo, whi, doc, pos)) active = false;
            }
            // The first clause (in clause order) that contains a document owns it and sums every clause's contribution in
            // clause order.  AND = every query TERM matched in at least one searched field (tantivy's QueryParser: AND over
            // terms of OR over fields): the owner collects a bit per matched term.
            bool all = active;
            uint64_t seen = 1ull << clause_term(cl[c]);
            float score = 0.f;
            if (all) {
                const float tf = (float)tfs[i];
                const float norm = p.caches[(size_t)clause_cache(cl[c]) * 256 + p.fieldnorm[(size_t)cl[c].field * p.n_docs + doc]];
                // explicit rn ops: no FMA contraction, so sums equal the reference's fp32 arithmetic bit for bit
                score = __fmul_rn(cl[c].weight, __fdiv_rn(tf, __fadd_rn(tf, norm)));
            }
            for (uint32_t e = c + 1; e < nc; e++) {
                if (!__any_sync(0xffffffffu, all)) break;
                if (!cl[e].df) continue;
                const uint32_t *od = p.post_docs + cl[e].offset;
                uint32_t wlo, whi;
                warp_window(od, cl[e].df, dmin, dmax, lane, wlo, whi);
                if (all && window_find(od, wlo, whi, doc, pos)) {
                    const float tf2 = (float)p.post_tfs[cl[e].offset + pos];
                    const float n2 = p.caches[(size_t)clause_cache(cl[e]) * 256 + p.fieldnorm[(size_t)cl[e].field * p.n_docs + doc]];
                    score = __fadd_rn(score, __fmul_rn(cl[e].weight, __fdiv_rn(tf2, __fadd_rn(tf2, n2))));
                    seen |= 1ull << clause_term(cl[e]);
                }
            }
            if (all && !p.operator_or && seen != p.term_mask[q]) all = false;
            if (all) {
                const uint32_t rid = p.row_id[doc];
                const bool live = !p.alive || ((p.alive[rid >> 3] >> (rid & 7)) & 1);
                key = -score;
                cand = live && list.passes(key, doc);
            }
            unsigned m = __ballot_sync(0xffffffffu, cand);
            while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, doc, src));
            }
        }
    }
    __syncthreads();
    block_rank_merge(lk, li, 8, p.k, p.k, p.part_keys + ((size_t)q * gridDim.x + blockIdx.x) * p.k,
                     p.part_ids + ((size_t)q * gridDim.x + blockIdx.x) * p.k);
}

// ------------------------------------------------------------------------------------
// Document-at-a-time inside doc RANGES.  The kernel above scores posting by posting and searches every other
// clause's list for each group of 32 postings (a small fraction of the HBM bandwidth).  Here a warp owns a CONTIGUOUS run of
// doc ranges of one query; for a range [r W, (r + 1) W) it
//   1. advances one cursor per clause (lanes = clauses) to the range end by a galloping + binary search from the previous
//      cursor (lists are sorted by doc: the cursors only move forward, every posting is read exactly once, coalesced),
//   2. accumulates the postings of the range clause after clause into a per-warp open-addressing table in shared memory keyed
//      by doc (score added with explicit rn ops in clause order -> bit-identical to the term-at-a-time sums; a bit per matched
//      query term for AND),
//   3. sweeps the table: AND mask, alive bitmap, warp-cooperative top-k.
// W is chosen per query on the host so that a range holds ~192 postings of its clauses together; a range that turns out
// denser than the table can hold is halved on the fly.
// ------------------------------------------------------------------------------------
constexpr int kDaatSlots = 512;           // per warp: doc u32 + score f32 + mask u64 = 8 KB (+ the list of occupied slots)
constexpr int kDaatFill = 352;            // postings a table takes in one go (load factor ~0.69)
constexpr int kDaatTarget = 192;          // postings per range the host aims for
// bytes of shared memory per warp: the table and the u16 list of occupied slots (the sweep visits only those).  1024-slot
// tables (16 KB per warp, 1 CTA per SM) swept in full leave the kernel bound by dependent-load latency at 8 warps per SM;
// 8.7 KB per warp keeps 3 CTAs resident.  The table size was chosen on an earlier GPU and is not re-measured on the H100.
constexpr int kDaatWarpBytes = kDaatSlots * 16 + ((kDaatFill * 2 + 15) / 16) * 16;
constexpr uint32_t kDaatEmpty = 0xffffffffu;

struct Bm25DaatParams {
    Bm25ScoreParams base;
    const uint32_t *range_log2;   // [nq] log2 of the range width W of each query
};

// first index i in docs[from, n) with docs[i] >= key (galloping from `from`, then binary search)
__device__ __forceinline__ uint32_t gallop_lower_bound(const uint32_t *docs, uint32_t from, uint32_t n, uint64_t key) {
    uint32_t lo = from, step = 32;
    if (lo >= n || docs[lo] >= key) return lo;
    uint32_t hi = lo + step;
    while (hi < n && docs[hi] < key) {   // docs[lo] < key always holds
        lo = hi;
        step <<= 1;
        hi = lo + step;
    }
    if (hi > n) hi = n;
    lo++;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (docs[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) bm25_daat_kernel(const Bm25DaatParams dp) {
    const Bm25ScoreParams &p = dp.base;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *lk = reinterpret_cast<float *>(smem_raw);                       // [8][k]
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + 8 * p.k);             // [8][k]
    unsigned char *tables = reinterpret_cast<unsigned char *>(li + 8 * p.k);
    tables = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(tables) + 15) & ~(uintptr_t)15);
    __shared__ Clause cl[kMaxClauses];
    __shared__ uint32_t cur_s[8][kMaxClauses], end_s[8][kMaxClauses];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t *t_doc = reinterpret_cast<uint32_t *>(tables + (size_t)warp * kDaatWarpBytes);
    float *t_score = reinterpret_cast<float *>(t_doc + kDaatSlots);
    unsigned long long *t_mask = reinterpret_cast<unsigned long long *>(t_score + kDaatSlots);
    unsigned short *t_occ = reinterpret_cast<unsigned short *>(t_mask + kDaatSlots);   // slots claimed in the current range
    __shared__ uint32_t n_occ_s[8];
    const uint32_t q = p.q_begin + blockIdx.y;
    const uint32_t c0 = p.clause_begin[q], nc = p.clause_begin[q + 1] - c0;
    for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) cl[i] = p.clauses[c0 + i];
    WarpTopK list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncthreads();
    if (nc) {
        const uint32_t lg = dp.range_log2[q];
        const uint64_t W = 1ull << lg;
        const uint64_t n_ranges = ((uint64_t)p.n_docs + W - 1) >> lg;
        // this warp's contiguous run of ranges
        const uint64_t warps_total = (uint64_t)gridDim.x * 8, wid = (uint64_t)blockIdx.x * 8 + warp;
        const uint64_t per = (n_ranges + warps_total - 1) / warps_total;
        const uint64_t r_begin = wid * per, r_end = r_begin + per < n_ranges ? r_begin + per : n_ranges;
        const unsigned long long full_mask = p.term_mask[q];
        if (r_begin < r_end) {
            // cursors at the start of the first range
            for (uint32_t c = lane; c < nc; c += 32)
                cur_s[warp][c] = gallop_lower_bound(p.post_docs + cl[c].offset, 0, cl[c].df, r_begin << lg);
            for (int i = lane; i < kDaatSlots; i += 32) t_doc[i] = kDaatEmpty;   // once: the sweep leaves the table empty
            if (lane == 0) n_occ_s[warp] = 0;
            __syncwarp();
            uint64_t d_lo = r_begin << lg;
            const uint64_t d_stop = (r_end << lg) < (uint64_t)p.n_docs ? (r_end << lg) : (uint64_t)p.n_docs;
            uint64_t width = W;
            while (d_lo < d_stop) {
                uint64_t d_hi = d_lo + width < d_stop ? d_lo + width : d_stop;
                // ---- 1. range ends per clause; shrink the range until its postings fit the table
                uint32_t total;
                for (;;) {
                    uint32_t mine = 0;
                    for (uint32_t c = lane; c < nc; c += 32) {
                        const uint32_t e = gallop_lower_bound(p.post_docs + cl[c].offset, cur_s[warp][c], cl[c].df, d_hi);
                        end_s[warp][c] = e;
                        mine += e - cur_s[warp][c];
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
                    total = mine;
                    if (total <= (uint32_t)kDaatFill || d_hi - d_lo <= 1) break;
                    width = (d_hi - d_lo + 1) >> 1;   // halve and retry (a single doc always fits: <= 64 clauses)
                    d_hi = d_lo + width;
                }
                __syncwarp();
                if (total) {
                    // ---- 2. accumulate clause after clause
                    for (uint32_t c = 0; c < nc; c++) {
                        const uint32_t b = cur_s[warp][c], e = end_s[warp][c];
                        const uint32_t *docs = p.post_docs + cl[c].offset;
                        const uint32_t *tfs = p.post_tfs + cl[c].offset;
                        const unsigned long long bit = 1ull << clause_term(cl[c]);
                        for (uint32_t i0 = b; i0 < e; i0 += 32) {
                            const uint32_t i = i0 + lane;
                            if (i < e) {
                                const uint32_t doc = docs[i];
                                const float tf = (float)tfs[i];
                                const float norm = p.caches[(size_t)clause_cache(cl[c]) * 256 + p.fieldnorm[(size_t)cl[c].field * p.n_docs + doc]];
                                const float contrib = __fmul_rn(cl[c].weight, __fdiv_rn(tf, __fadd_rn(tf, norm)));
                                uint32_t slot = (doc * 2654435761u) >> 23;   // 9 bits
                                for (;;) {
                                    const uint32_t prev = atomicCAS(&t_doc[slot], kDaatEmpty, doc);
                                    if (prev == kDaatEmpty) {   // first clause that contains this doc
                                        t_score[slot] = contrib;
                                        t_mask[slot] = bit;
                                        t_occ[atomicAdd(&n_occ_s[warp], 1u)] = (unsigned short)slot;
                                        break;
                                    }
                                    if (prev == doc) {          // an earlier clause owns the slot: add in clause order
                                        t_score[slot] = __fadd_rn(t_score[slot], contrib);
                                        t_mask[slot] |= bit;
                                        break;
                                    }
                                    slot = (slot + 1) & (kDaatSlots - 1);
                                }
                            }
                        }
                        __syncwarp();   // clause c is complete (and visible) before clause c + 1 touches the same docs
                    }
                    // ---- 3. sweep
                    const int n_occ = (int)n_occ_s[warp];
                    for (int i0 = 0; i0 < n_occ; i0 += 32) {
                        const int i = i0 + lane < n_occ ? (int)t_occ[i0 + lane] : -1;
                        uint32_t doc = kDaatEmpty;
                        bool cand = i >= 0;
                        float key = FLT_MAX;
                        if (cand) {
                            doc = t_doc[i];
                            t_doc[i] = kDaatEmpty;   // leave the table empty for the next range
                            if (!p.operator_or && t_mask[i] != full_mask) cand = false;
                        }
                        if (cand) {
                            const uint32_t rid = p.row_id[doc];
                            cand = !p.alive || ((p.alive[rid >> 3] >> (rid & 7)) & 1);
                            key = -t_score[i];
                            cand = cand && list.passes(key, doc);
                        }
                        unsigned m = __ballot_sync(0xffffffffu, cand);
                        while (m) {
                            const int src = __ffs(m) - 1;
                            m &= m - 1;
                            list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, doc, src));
                        }
                    }
                    if (lane == 0) n_occ_s[warp] = 0;
                    __syncwarp();
                }
                for (uint32_t c = lane; c < nc; c += 32) cur_s[warp][c] = end_s[warp][c];
                __syncwarp();
                d_lo = d_hi;
                if (width < W && total <= (uint32_t)kDaatFill / 4) width <<= 1;   // dense spot passed: widen again
            }
        }
    }
    __syncthreads();
    block_rank_merge(lk, li, 8, p.k, p.k, p.part_keys + ((size_t)q * gridDim.x + blockIdx.x) * p.k,
                     p.part_ids + ((size_t)q * gridDim.x + blockIdx.x) * p.k);
}

// doc ordinal -> row id on the merged result
__global__ void bm25_finish_kernel(const float *dis, const int64_t *docs, const uint32_t *row_id, int64_t n, float *out_score,
                                   uint64_t *out_row, uint32_t *out_count, int k) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t d = docs[i];
    out_score[i] = d >= 0 ? dis[i] : 0.f;
    out_row[i] = d >= 0 ? (uint64_t)row_id[d] : ~0ull;
    if (d >= 0) atomicAdd(&out_count[i / k], 1u);
}

}  // namespace b200

using namespace b200;

struct b200_bm25 {
    uint32_t n_fields = 1;
    std::vector<std::unordered_map<std::string, uint32_t>> dict;  // per field: term -> list index
    std::vector<TermList> lists;
    std::vector<std::vector<uint32_t>> doc_len;  // [field][doc]
    std::vector<uint64_t> row_ids;
    std::vector<uint64_t> total_tokens;
    bool committed = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // around the scoring kernel of the last batch
    double last_call_ms = 0;                     // wall time of the last b200_bm25_search_batch inside the library
    uint64_t last_postings = 0;                  // postings the scoring kernel walked (sum of df over the batch's clauses)
    int device = 0;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    DevMem d_docs, d_tfs, d_fn, d_rows, d_clauses, d_begin, d_caches, d_pk, d_pi, d_alive, d_odis, d_oids, d_score, d_row64, d_cnt, d_masks, d_ranges;
};

static int bm25_device_ok() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(B200_ERR_NO_DEVICE, "no CUDA device visible; libb200search has no CPU fallback");
    }
    return B200_OK;
}

extern "C" int b200_bm25_create(uint32_t n_fields, b200_bm25 **out) {
    if (!out || n_fields == 0 || n_fields > 64) return fail(B200_ERR_INVALID, "bad arguments");
    *out = nullptr;
    B200_TRY(bm25_device_ok());
    init_fieldnorm();
    b200_bm25 *ix = new b200_bm25();
    ix->n_fields = n_fields;
    ix->dict.resize(n_fields);
    ix->doc_len.resize(n_fields);
    ix->total_tokens.assign(n_fields, 0);
    cudaGetDevice(&ix->device);
    if (cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ix;
        return fail(B200_ERR_CUDA, "cudaStreamCreate failed");
    }
    *out = ix;
    return B200_OK;
}

extern "C" int b200_bm25_free(b200_bm25 *ix) {
    if (!ix) return B200_OK;
    cudaSetDevice(ix->device);
    if (ix->ev0) cudaEventDestroy(ix->ev0);
    if (ix->ev1) cudaEventDestroy(ix->ev1);
    if (ix->stream) cudaStreamDestroy(ix->stream);
    delete ix;
    return B200_OK;
}

// roofline inputs of the last batch: scoring-kernel milliseconds (CUDA events), wall milliseconds of the whole C call, postings walked
extern "C" int b200_bm25_last_timing(b200_bm25 *ix, double *kernel_ms, double *call_ms, uint64_t *postings) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    float ms = 0;
    if (ix->ev0 && cudaEventElapsedTime(&ms, ix->ev0, ix->ev1) != cudaSuccess) {
        cudaGetLastError();
        ms = 0;
    }
    if (kernel_ms) *kernel_ms = ms;
    if (call_ms) *call_ms = ix->last_call_ms;
    if (postings) *postings = ix->last_postings;
    return B200_OK;
}

// ffi_index_multi_column_docs(path, row_id, column_names, column_docs): one call per row;
// texts[f] may be null; call b200_bm25_add_text again for further values of an Array(String) column.
extern "C" int b200_bm25_add_doc(b200_bm25 *ix, uint64_t row_id) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    if (ix->committed) return fail(B200_ERR_INVALID, "index already committed");
    if (row_id >= 0xffffffffull) return fail(B200_ERR_UNSUPPORTED, "row ids are UInt32 part offsets");
    ix->row_ids.push_back(row_id);
    for (auto &dl : ix->doc_len) dl.push_back(0);
    return B200_OK;
}

extern "C" int b200_bm25_add_text(b200_bm25 *ix, uint32_t field, const char *text) {
    if (!ix || !text || field >= ix->n_fields) return fail(B200_ERR_INVALID, "bad arguments");
    if (ix->committed || ix->row_ids.empty()) return fail(B200_ERR_INVALID, "add_doc first / index already committed");
    const uint32_t doc = (uint32_t)ix->row_ids.size() - 1;
    tokenize_default(text, [&](const std::string &tok) {
        auto it = ix->dict[field].find(tok);
        uint32_t li;
        if (it == ix->dict[field].end()) {
            li = (uint32_t)ix->lists.size();
            ix->dict[field].emplace(tok, li);
            ix->lists.emplace_back();
        } else {
            li = it->second;
        }
        TermList &tl = ix->lists[li];
        if (!tl.docs.empty() && tl.docs.back() == doc) tl.tfs.back()++;
        else {
            tl.docs.push_back(doc);
            tl.tfs.push_back(1);
        }
        ix->doc_len[field][doc]++;
        ix->total_tokens[field]++;
    });
    return B200_OK;
}

// ffi_index_writer_commit: freeze and upload to HBM
extern "C" int b200_bm25_commit(b200_bm25 *ix) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (ix->committed) return B200_OK;
    B200_CUDA_OK(cudaSetDevice(ix->device));
    uint64_t total = 0;
    for (auto &tl : ix->lists) {
        tl.offset = total;
        total += tl.docs.size();
    }
    const size_t nd = ix->row_ids.size();
    std::vector<uint32_t> docs(total ? total : 1), tfs(total ? total : 1);
    for (auto &tl : ix->lists) {
        std::copy(tl.docs.begin(), tl.docs.end(), docs.begin() + tl.offset);
        std::copy(tl.tfs.begin(), tl.tfs.end(), tfs.begin() + tl.offset);
    }
    std::vector<uint8_t> fn((size_t)ix->n_fields * (nd ? nd : 1));
    for (uint32_t f = 0; f < ix->n_fields; f++)
        for (size_t d = 0; d < nd; d++) fn[(size_t)f * nd + d] = fieldnorm_to_id(ix->doc_len[f][d]);
    std::vector<uint32_t> rows(nd ? nd : 1);
    for (size_t d = 0; d < nd; d++) rows[d] = (uint32_t)ix->row_ids[d];
    B200_TRY(ix->d_docs.alloc(docs.size() * 4 + 256));
    B200_TRY(ix->d_tfs.alloc(tfs.size() * 4 + 256));
    B200_TRY(ix->d_fn.alloc(fn.size() + 256));
    B200_TRY(ix->d_rows.alloc(rows.size() * 4 + 256));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_docs.p, docs.data(), docs.size() * 4, cudaMemcpyHostToDevice, ix->stream));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_tfs.p, tfs.data(), tfs.size() * 4, cudaMemcpyHostToDevice, ix->stream));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_fn.p, fn.data(), fn.size(), cudaMemcpyHostToDevice, ix->stream));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_rows.p, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, ix->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ix->stream));
    for (auto &tl : ix->lists) {  // host copies of the postings are no longer needed (df stays)
        tl.tfs.clear();
        tl.tfs.shrink_to_fit();
    }
    ix->committed = true;
    return B200_OK;
}

extern "C" int b200_bm25_total_docs(const b200_bm25 *ix, uint64_t *out) {  // ffi_get_total_num_docs
    if (!ix || !out) return fail(B200_ERR_INVALID, "null argument");
    *out = ix->row_ids.size();
    return B200_OK;
}
extern "C" int b200_bm25_total_tokens(const b200_bm25 *ix, uint32_t field, uint64_t *out) {  // ffi_get_total_num_tokens
    if (!ix || !out || field >= ix->n_fields) return fail(B200_ERR_INVALID, "bad arguments");
    *out = ix->total_tokens[field];
    return B200_OK;
}
extern "C" int b200_bm25_doc_freq(const b200_bm25 *ix, uint32_t field, const char *term, uint64_t *out) {  // ffi_get_doc_freq
    if (!ix || !out || !term || field >= ix->n_fields) return fail(B200_ERR_INVALID, "bad arguments");
    auto it = ix->dict[field].find(term);
    *out = it == ix->dict[field].end() ? 0 : ix->lists[it->second].docs.size();
    return B200_OK;
}

// Tokenise a sentence into distinct lowercase terms, written NUL-separated into buf.
extern "C" int b200_bm25_query_terms(const char *sentence, char *buf, size_t buf_len, uint32_t *out_n) {
    if (!sentence || !buf || !out_n) return fail(B200_ERR_INVALID, "null argument");
    std::vector<std::string> terms;
    tokenize_default(sentence, [&](const std::string &t) {
        if (std::find(terms.begin(), terms.end(), t) == terms.end()) terms.push_back(t);
    });
    size_t off = 0;
    for (auto &t : terms) {
        if (off + t.size() + 1 > buf_len) return fail(B200_ERR_INVALID, "buffer too small");
        memcpy(buf + off, t.c_str(), t.size() + 1);
        off += t.size() + 1;
    }
    *out_n = (uint32_t)terms.size();
    return B200_OK;
}

// Batched ffi_bm25_search.  sentences[nq]; fields[n_fields_q] searched for every query.
// stats (nullable): table-wide statistics -- total_docs, total_tokens[n_fields] and, per query,
// doc_freq[q][fq * 64 + term] for its distinct terms in tokenisation order (up to 64 per query).
// Output per query: out_rows/out_scores [nq][topk] (score descending, ties -> smaller doc),
// out_counts[nq].
extern "C" int b200_bm25_search_batch(b200_bm25 *ix, const char *const *sentences, int64_t nq, const uint32_t *fields,
                                      uint32_t n_fields_q, uint32_t topk, const uint8_t *alive_bits, int use_filter,
                                      int operator_or, uint64_t stat_total_docs, const uint64_t *stat_total_tokens,
                                      const uint64_t *stat_doc_freq, uint64_t *out_rows, float *out_scores,
                                      uint32_t *out_counts) {
    if (!ix || !sentences || !fields || !out_rows || !out_scores || !out_counts || nq < 0 || n_fields_q == 0)
        return fail(B200_ERR_INVALID, "bad arguments");
    if (topk == 0 || topk > 2048) return fail(B200_ERR_UNSUPPORTED, "topk must be in 1..2048");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (!ix->committed) return fail(B200_ERR_INVALID, "commit the index before searching");
    if (nq == 0) return B200_OK;
    const auto t_call0 = std::chrono::steady_clock::now();
    B200_CUDA_OK(cudaSetDevice(ix->device));
    cudaStream_t s = ix->stream;
    const size_t nd = ix->row_ids.size();
    for (int64_t q = 0; q < nq; q++) out_counts[q] = 0;
    if (nd == 0) return B200_OK;

    // ---- host: tokenise, resolve terms, BM25 weights and norm tables (fp32, tantivy order of ops)
    std::vector<Clause> clauses;
    std::vector<uint32_t> begin(nq + 1, 0);
    std::vector<float> caches;
    std::vector<uint64_t> term_masks(nq, 0);
    for (int64_t q = 0; q < nq; q++) {
        begin[q] = (uint32_t)clauses.size();
        std::vector<std::string> terms;
        tokenize_default(sentences[q], [&](const std::string &t) {
            if (terms.size() < 64 && std::find(terms.begin(), terms.end(), t) == terms.end()) terms.push_back(t);
        });
        std::vector<Clause> mine;
        uint64_t known = 0;  // terms found in at least one searched field
        for (uint32_t fq = 0; fq < n_fields_q; fq++) {
            const uint32_t f = fields[fq];
            if (f >= ix->n_fields) return fail(B200_ERR_INVALID, "field out of range");
            const uint64_t N = stat_total_docs ? stat_total_docs : nd;
            const uint64_t T = stat_total_docs ? stat_total_tokens[f] : ix->total_tokens[f];
            const float avgdl = (float)T / (float)N;
            const uint32_t cache_idx = (uint32_t)(caches.size() / 256);
            for (int c = 0; c < 256; c++) caches.push_back(kBm25K1 * (1.0f - kBm25B + kBm25B * (float)g_fieldnorm[c] / avgdl));
            for (size_t t = 0; t < terms.size(); t++) {
                auto it = ix->dict[f].find(terms[t]);
                if (it == ix->dict[f].end()) continue;
                known |= 1ull << t;
                const TermList &tl = ix->lists[it->second];
                const uint64_t n = stat_total_docs ? stat_doc_freq[(size_t)q * n_fields_q * 64 + fq * 64 + t] : tl.docs.size();
                const float x = ((float)(N - n) + 0.5f) / ((float)n + 0.5f);
                const float idf = logf(1.0f + x);
                Clause cl;
                cl.offset = tl.offset;
                cl.df = (uint32_t)tl.docs.size();
                cl.weight = idf * (1.0f + kBm25K1);
                cl.field = f;
                cl.cache = cache_idx | ((uint32_t)t << 24);
                mine.push_back(cl);
            }
        }
        const uint64_t all_terms = terms.size() >= 64 ? ~0ull : ((1ull << terms.size()) - 1);
        term_masks[q] = all_terms;
        // AND with a term that no searched field knows matches nothing
        const bool dead = !operator_or && (terms.empty() || known != all_terms);
        if (!dead) {
            if (mine.size() > (size_t)kMaxClauses) return fail(B200_ERR_UNSUPPORTED, "more than 64 (field, term) clauses in one query");
            clauses.insert(clauses.end(), mine.begin(), mine.end());
        }
    }
    begin[nq] = (uint32_t)clauses.size();
    if (clauses.empty()) return B200_OK;

    // ---- device
    const int k = (int)topk;
    uint32_t max_df = 1;
    for (auto &c : clauses) max_df = std::max(max_df, c.df);
    int bx = (int)std::min<int64_t>(std::max<int64_t>(1, ceil_div(max_df, 256 * 4)), std::max<int64_t>(1, 592 / std::max<int64_t>(1, std::min<int64_t>(nq, 592))));
    B200_TRY(ix->d_clauses.reserve(clauses.size() * sizeof(Clause)));
    B200_TRY(ix->d_begin.reserve(begin.size() * 4));
    B200_TRY(ix->d_caches.reserve(caches.size() * 4));
    B200_TRY(ix->d_masks.reserve(term_masks.size() * 8));
    if (caches.size() / 256 >= (1u << 24)) return fail(B200_ERR_UNSUPPORTED, "too many (query, field) norm tables in one batch");
    B200_TRY(ix->d_pk.reserve((size_t)nq * bx * k * 4));
    B200_TRY(ix->d_pi.reserve((size_t)nq * bx * k * 4));
    B200_TRY(ix->d_odis.reserve((size_t)nq * k * 4));
    B200_TRY(ix->d_oids.reserve((size_t)nq * k * 8));
    B200_TRY(ix->d_score.reserve((size_t)nq * k * 4));
    B200_TRY(ix->d_row64.reserve((size_t)nq * k * 8));
    B200_TRY(ix->d_cnt.reserve((size_t)nq * 4));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_clauses.p, clauses.data(), clauses.size() * sizeof(Clause), cudaMemcpyHostToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_begin.p, begin.data(), begin.size() * 4, cudaMemcpyHostToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_caches.p, caches.data(), caches.size() * 4, cudaMemcpyHostToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(ix->d_masks.p, term_masks.data(), term_masks.size() * 8, cudaMemcpyHostToDevice, s));
    const uint8_t *d_alive = nullptr;
    if (use_filter && alive_bits) {
        uint64_t max_row = 0;
        for (auto r : ix->row_ids) max_row = std::max(max_row, r);
        const size_t ab = (size_t)(max_row / 8 + 1);
        B200_TRY(ix->d_alive.reserve(ab));
        B200_CUDA_OK(cudaMemcpyAsync(ix->d_alive.p, alive_bits, ab, cudaMemcpyHostToDevice, s));
        d_alive = reinterpret_cast<const uint8_t *>(ix->d_alive.p);
    }
    Bm25ScoreParams sp{};
    sp.post_docs = reinterpret_cast<const uint32_t *>(ix->d_docs.p);
    sp.post_tfs = reinterpret_cast<const uint32_t *>(ix->d_tfs.p);
    sp.fieldnorm = reinterpret_cast<const uint8_t *>(ix->d_fn.p);
    sp.row_id = reinterpret_cast<const uint32_t *>(ix->d_rows.p);
    sp.alive = d_alive;
    sp.clauses = reinterpret_cast<const Clause *>(ix->d_clauses.p);
    sp.clause_begin = reinterpret_cast<const uint32_t *>(ix->d_begin.p);
    sp.caches = reinterpret_cast<const float *>(ix->d_caches.p);
    sp.term_mask = reinterpret_cast<const uint64_t *>(ix->d_masks.p);
    sp.part_keys = reinterpret_cast<float *>(ix->d_pk.p);
    sp.part_ids = reinterpret_cast<uint32_t *>(ix->d_pi.p);
    sp.n_docs = (uint32_t)nd;
    sp.k = k;
    sp.operator_or = operator_or;
    if (!ix->ev0) {
        cudaEventCreate(&ix->ev0);
        cudaEventCreate(&ix->ev1);
    }
    ix->last_postings = 0;
    for (auto &c : clauses) ix->last_postings += c.df;
    cudaEventRecord(ix->ev0, s);
    static const int use_taat = getenv("B200_BM25_TAAT") ? atoi(getenv("B200_BM25_TAAT")) : 0;   // A/B: the round-1 kernel
    constexpr int64_t kMaxGridY = 65535;   // queries ride on gridDim.y: larger batches launch slice after slice
    if (use_taat) {
        const size_t smem = (size_t)8 * k * 8;
        B200_CUDA_OK(cudaFuncSetAttribute(bm25_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        for (int64_t q0 = 0; q0 < nq; q0 += kMaxGridY) {
            sp.q_begin = (uint32_t)q0;
            bm25_score_kernel<<<dim3(bx, (unsigned)std::min(nq - q0, kMaxGridY)), 256, smem, s>>>(sp);
        }
    } else {
        // range width per query: ~kDaatTarget postings of all its clauses per range
        std::vector<uint32_t> range_log2(nq, 8);
        for (int64_t q = 0; q < nq; q++) {
            uint64_t m_q = 0;
            for (uint32_t c = begin[q]; c < begin[q + 1]; c++) m_q += clauses[c].df;
            const double w = m_q ? (double)kDaatTarget * (double)nd / (double)m_q : (double)nd;
            uint32_t lg = 8;
            while (lg < 31 && (double)(1ull << (lg + 1)) <= w) lg++;
            range_log2[q] = lg;
        }
        B200_TRY(ix->d_ranges.reserve((size_t)nq * 4));
        B200_CUDA_OK(cudaMemcpyAsync(ix->d_ranges.p, range_log2.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
        Bm25DaatParams dpp{};
        dpp.base = sp;
        dpp.range_log2 = reinterpret_cast<const uint32_t *>(ix->d_ranges.p);
        const size_t smem = (size_t)8 * k * 8 + 16 + (size_t)8 * kDaatWarpBytes;
        B200_CUDA_OK(cudaFuncSetAttribute(bm25_daat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        for (int64_t q0 = 0; q0 < nq; q0 += kMaxGridY) {
            dpp.base.q_begin = (uint32_t)q0;
            bm25_daat_kernel<<<dim3(bx, (unsigned)std::min(nq - q0, kMaxGridY)), 256, smem, s>>>(dpp);
        }
    }
    cudaEventRecord(ix->ev1, s);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    MergeParams mp{};
    mp.in_keys = sp.part_keys;
    mp.in_ids = sp.part_ids;
    mp.list_stride = k;
    mp.q_stride = (int64_t)bx * k;
    mp.n_lists = bx;
    mp.k_in = k;
    mp.k = k;
    mp.nq = nq;
    mp.out_mode = kOutNeg;
    mp.out_dis = reinterpret_cast<float *>(ix->d_odis.p);
    mp.out_ids = reinterpret_cast<int64_t *>(ix->d_oids.p);
    B200_CUDA_OK(launch_topk_merge(mp, false, s));
    B200_CUDA_OK(cudaMemsetAsync(ix->d_cnt.p, 0, (size_t)nq * 4, s));
    const int64_t tot = nq * k;
    bm25_finish_kernel<<<(unsigned)ceil_div(tot, 256), 256, 0, s>>>(mp.out_dis, mp.out_ids, sp.row_id, tot,
                                                                   reinterpret_cast<float *>(ix->d_score.p),
                                                                   reinterpret_cast<uint64_t *>(ix->d_row64.p),
                                                                   reinterpret_cast<uint32_t *>(ix->d_cnt.p), k);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaMemcpyAsync(out_scores, ix->d_score.p, (size_t)tot * 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_rows, ix->d_row64.p, (size_t)tot * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_counts, ix->d_cnt.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    ix->last_call_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_call0).count();
    return B200_OK;
}

extern "C" int b200_bm25_search(b200_bm25 *ix, const char *sentence, const uint32_t *fields, uint32_t n_fields_q,
                                uint32_t topk, const uint8_t *alive_bits, int use_filter, int operator_or,
                                uint64_t stat_total_docs, const uint64_t *stat_total_tokens, const uint64_t *stat_doc_freq,
                                uint64_t *out_rows, float *out_scores, uint32_t *out_n) {
    const char *one[1] = {sentence};
    return b200_bm25_search_batch(ix, one, 1, fields, n_fields_q, topk, alive_bits, use_filter, operator_or, stat_total_docs,
                                  stat_total_tokens, stat_doc_freq, out_rows, out_scores, out_n);
}

// ------------------------------------------------------------------------------------
// persistence: the reference keeps a tantivy directory per part and (re)loads it with ffi_load_index_reader
// (TantivyIndexStore.cpp:646-686, with retries when the cache directory is damaged).  tantivy's segment files are not
// reproducible without the crate, so this is our own single file ("B2TX" v1): statistics, dictionary, postings.
// Loading validates every size before it allocates and uploads to HBM.
// ------------------------------------------------------------------------------------
namespace {
struct TxHeader {
    char magic[4];
    uint32_t version, n_fields;
    uint64_t n_docs, n_lists, n_postings;
};
bool fw(FILE *f, const void *p, size_t b) { return b == 0 || fwrite(p, 1, b, f) == b; }
bool fr(FILE *f, void *p, size_t b) { return b == 0 || fread(p, 1, b, f) == b; }
}  // namespace

extern "C" int b200_bm25_save(b200_bm25 *ix, const char *path) {
    if (!ix || !path) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (!ix->committed) return fail(B200_ERR_INVALID, "commit the index before saving it");
    B200_CUDA_OK(cudaSetDevice(ix->device));
    uint64_t total = 0;
    for (auto &tl : ix->lists) total += tl.docs.size();
    std::vector<uint32_t> tfs(total ? total : 1);
    if (total) B200_CUDA_OK(cudaMemcpy(tfs.data(), ix->d_tfs.p, total * 4, cudaMemcpyDeviceToHost));
    FILE *f = fopen(path, "wb");
    if (!f) return fail(B200_ERR_INVALID, std::string("cannot open ") + path);
    TxHeader h{};
    memcpy(h.magic, "B2TX", 4);
    h.version = 1;
    h.n_fields = ix->n_fields;
    h.n_docs = ix->row_ids.size();
    h.n_lists = ix->lists.size();
    h.n_postings = total;
    bool ok = fw(f, &h, sizeof(h)) && fw(f, ix->row_ids.data(), h.n_docs * 8) && fw(f, ix->total_tokens.data(), (size_t)h.n_fields * 8);
    for (uint32_t fld = 0; ok && fld < ix->n_fields; fld++) ok = fw(f, ix->doc_len[fld].data(), h.n_docs * 4);
    for (uint32_t fld = 0; ok && fld < ix->n_fields; fld++) {
        const uint64_t nt = ix->dict[fld].size();
        ok = fw(f, &nt, 8);
        for (auto &kv : ix->dict[fld]) {
            const uint32_t len = (uint32_t)kv.first.size(), li = kv.second;
            if (!(ok = ok && fw(f, &len, 4) && fw(f, kv.first.data(), len) && fw(f, &li, 4))) break;
        }
    }
    for (auto &tl : ix->lists) {
        const uint64_t df = tl.docs.size();
        if (!(ok = ok && fw(f, &df, 8) && fw(f, tl.docs.data(), df * 4) && fw(f, tfs.data() + tl.offset, df * 4))) break;
    }
    ok = (fclose(f) == 0) && ok;
    return ok ? B200_OK : fail(B200_ERR_INVALID, std::string("write failed: ") + path);
}

extern "C" int b200_bm25_load(const char *path, b200_bm25 **out) {
    if (!path || !out) return fail(B200_ERR_INVALID, "bad arguments");
    *out = nullptr;
    FILE *f = fopen(path, "rb");
    if (!f) return fail(B200_ERR_INVALID, std::string("cannot open ") + path);
    fseek(f, 0, SEEK_END);
    const uint64_t file_bytes = (uint64_t)ftell(f);
    fseek(f, 0, SEEK_SET);
    TxHeader h{};
    b200_bm25 *ix = nullptr;
    auto bail = [&](const std::string &msg) {
        fclose(f);
        if (ix) b200_bm25_free(ix);
        return fail(B200_ERR_INVALID, msg);
    };
    if (!fr(f, &h, sizeof(h)) || memcmp(h.magic, "B2TX", 4) != 0 || h.version != 1) return bail("not a B2TX v1 text index file");
    // nothing below may allocate more than the file can back
    if (h.n_fields == 0 || h.n_fields > 64 || h.n_docs >= 0xffffffffull || h.n_docs * 8 > file_bytes || h.n_postings * 8 > file_bytes ||
        h.n_lists > file_bytes / 8 + 1)
        return bail("corrupt text index header");
    if (b200_bm25_create(h.n_fields, &ix) != B200_OK) {
        fclose(f);
        return B200_ERR_NO_DEVICE;
    }
    try {
        ix->row_ids.resize(h.n_docs);
        if (!fr(f, ix->row_ids.data(), h.n_docs * 8) || !fr(f, ix->total_tokens.data(), (size_t)h.n_fields * 8)) return bail("truncated text index (rows)");
        for (uint32_t fld = 0; fld < h.n_fields; fld++) {
            ix->doc_len[fld].resize(h.n_docs);
            if (!fr(f, ix->doc_len[fld].data(), h.n_docs * 4)) return bail("truncated text index (field norms)");
        }
        ix->lists.resize(h.n_lists);
        for (uint32_t fld = 0; fld < h.n_fields; fld++) {
            uint64_t nt = 0;
            if (!fr(f, &nt, 8) || nt > h.n_lists) return bail("corrupt text index (dictionary)");
            std::string term;
            for (uint64_t t = 0; t < nt; t++) {
                uint32_t len = 0, li = 0;
                if (!fr(f, &len, 4) || len > 65536) return bail("corrupt text index (term)");
                term.resize(len);
                if (!fr(f, &term[0], len) || !fr(f, &li, 4) || li >= h.n_lists) return bail("corrupt text index (term)");
                ix->dict[fld].emplace(term, li);
            }
        }
        uint64_t total = 0;
        std::vector<uint32_t> tfs(h.n_postings ? h.n_postings : 1);
        for (auto &tl : ix->lists) {
            uint64_t df = 0;
            if (!fr(f, &df, 8) || total + df > h.n_postings) return bail("corrupt text index (postings)");
            tl.docs.resize(df);
            if (!fr(f, tl.docs.data(), df * 4) || !fr(f, tfs.data() + total, df * 4)) return bail("truncated text index (postings)");
            for (uint64_t i = 0; i < df; i++)
                if (tl.docs[i] >= h.n_docs || (i && tl.docs[i] <= tl.docs[i - 1])) return bail("corrupt text index (doc ordinals)");
            tl.tfs.assign(tfs.begin() + total, tfs.begin() + total + df);
            total += df;
        }
        if (total != h.n_postings) return bail("corrupt text index (posting count)");
    } catch (const std::bad_alloc &) {
        return bail("out of host memory while loading the text index");
    }
    fclose(f);
    const int rc = b200_bm25_commit(ix);
    if (rc != B200_OK) {
        b200_bm25_free(ix);
        return rc;
    }
    *out = ix;
    return B200_OK;
}
