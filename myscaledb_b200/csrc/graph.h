// graph.h -- fixed-degree neighbour graph of an HNSWFLAT, MSTG or BINARYMSTG index (graph_degree=D): build steps and the graph
// search, one CTA per query or one W-CTA cluster per query (search_width=W) (graph_sm90.cu).  The host side (candidates from
// the index's own list search, persistence, the search entry) lives in ivf.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

constexpr int kGraphThreads = 256;
// visited set of one query: open addressing (linear probing) over kGraphVisitedSlots u32 in shared memory (64 KB).  The
// iteration cap keeps it at most half full, so a lookup always ends at an empty slot and the set is exact.
constexpr int kGraphVisitedLog2 = 14;
constexpr int kGraphVisitedSlots = 1 << kGraphVisitedLog2;
constexpr int kGraphMaxSeeds = 32;     // seeds per query: the best min(ef_s, 32) ids of the list path's first stage at nprobe 1
constexpr int kGraphMaxWidth = 8;      // parents expanded per iteration (search_width=W): 1, 2, 4 or 8, one CTA of a cluster each
constexpr int kGraphMaxDegree = 64;
constexpr int kGraphMaxEf = 1024;

// Iterations one query may run: every iteration inserts at most width x D ids into the visited table and the seeds at most
// kGraphMaxSeeds, so the table never holds more than kGraphVisitedSlots / 2 ids.  W = 1, D = 16 / 32 / 64: 510 / 255 / 127;
// W = 8, D = 64: 15.
__host__ __device__ constexpr int graph_iteration_cap(int degree, int width = 1) {
    return (kGraphVisitedSlots / 2 - kGraphMaxSeeds) / (width * degree);
}

inline bool graph_degree_ok(int d) { return d == 16 || d == 32 || d == 64; }
inline bool graph_width_ok(int w) { return w == 1 || w == 2 || w == 4 || w == 8; }

// ids [m][K + 1] of the list search of rows row0 .. row0 + m - 1 (negative = none) -> cand [m][K] u32: the row's own id
// dropped (or, when it is absent, the last entry), negative ids as 0xFFFFFFFF.  A row in no list (row_slot 0xFFFFFFFF) gets
// none, so no edge leaves it; the list searches never return it, so none reaches it.
int graph_candidates(const int64_t *d_ids, const uint32_t *d_row_slot, int64_t m, int64_t row0, int K, uint32_t *d_cand, cudaStream_t s);
// rank-based pruning (CAGRA): cand [n][2D] -> pruned [n][D], per node the D candidates with the smallest (detour count, rank)
int graph_prune(const uint32_t *d_cand, int64_t n, int D, uint32_t *d_pruned, cudaStream_t s);
// reverse edges and merge: pruned [n][D] -> graph [n][D].  Allocates and frees its own scratch (2 x n x D x 12 B + the sort's).
int graph_merge(const uint32_t *d_pruned, int64_t n, int D, uint32_t *d_graph, cudaStream_t s);

// id -> pool slot map row_slot[n] of a finalized inverted-file index, from its page chains (one CTA per list); the caller fills
// it with 0xFFFFFFFF first, which stays the slot of a row in no list
int graph_row_slots(const uint32_t *d_list_len, const uint32_t *d_list_page_off, const uint32_t *d_list_pages, const uint32_t *d_row_ids, int nlist,
                    uint32_t *d_row_slot, cudaStream_t s);
// out [m][d] fp32 = the bf16 page rows of ids row0 .. row0 + m - 1 (pool: [page][d_pad64 / 64][256][64] bf16); zeros for a row
// in no list
int graph_page_rows(const void *d_pool, const uint32_t *d_row_slot, int64_t row0, int64_t m, int d, int d_pad64, float *d_out, cudaStream_t s);
// out [m][row_bytes] bytes = the binary page rows of ids row0 .. row0 + m - 1 (pool: [page][row_pad / kb_w][256][kb_w] bytes);
// zeros for a row in no list
int graph_bin_page_rows(const void *d_pool, const uint32_t *d_row_slot, int64_t row0, int64_t m, int row_bytes, int row_pad, int kb_w, uint8_t *d_out,
                        cudaStream_t s);

struct GraphSearchParams {
    const float *queries;      // [nq][d_pad], prepared (cosine: unit)
    const float *rows;         // [n][d_pad] fp32 (HNSWFLAT)
    const void *pages;         // MSTG, else null: the bf16 list pool [page][d_pad64 / 64][256][64] (cosine: unit rows) ...
    const uint32_t *row_slot;  // ... and row v's slot in it
    const uint32_t *graph;     // [n][degree], 0xFFFFFFFF = empty slot
    const int64_t *seeds;      // [nq][nseeds], negative = none
    const uint8_t *alive;      // nullable: bit r of byte r / 8 keeps row r
    float *out_dis;            // [nq][k]
    int64_t *out_ids;
    unsigned long long *rows_scored;   // += rows scored by every query
    int64_t n, id_offset;
    int d_pad, d_pad64, degree, nseeds, ef, k, max_iters;   // k: entries returned per query
    int l2;                    // else inner product (distance -key)
};

// BINARYMSTG: the walk over the binary list pages.  g.pages is the pool [page][row_pad / kb_w][256][kb_w] bytes, g.row_slot
// row v's slot in it, g.queries unused, g.l2 = 1 (the key is the distance), g.d_pad / g.d_pad64 unused.
struct GraphB1Params {
    GraphSearchParams g;
    const uint8_t *queries;    // [nq][row_bytes]
    const float *row_popc;     // [pool rows] popcount of the row at a slot (an exact float)
    int row_bytes, row_pad, kb_w;
    int jaccard;               // else Hamming
};

// dynamic shared memory of each CTA of a query; q_len = d_pad (fp32 rows), d_pad64 (bf16 pages) or row_pad / 4 (binary pages)
size_t graph_search_smem(int q_len, int ef, int k, bool filtered, int width);
// graph_search_kernel over the fp32 rows, or graph_search_bf16_kernel when p.pages is set; at width = W > 1 (W parents per
// iteration, graph_width_ok) their cluster forms, nq x W CTAs in clusters of W.  B200_ERR_UNSUPPORTED when the shared memory
// does not fit or a cluster cannot be resident.
int graph_search(const GraphSearchParams &p, int64_t nq, int width, cudaStream_t s);
// graph_search_b1_kernel over the binary list pages (BINARYMSTG), or its cluster forms at width = W > 1; errors as graph_search
int graph_search_b1(const GraphB1Params &p, int64_t nq, int width, cudaStream_t s);

}  // namespace b200
