// graph.h -- fixed-degree neighbour graph of an HNSWFLAT index (graph_degree=D): build steps and the one-CTA-per-query
// search (graph_sm90.cu).  The host side (candidates from the index's own list search, persistence, the search entry)
// lives in ivf.cu.
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
constexpr int kGraphWidth = 1;         // parents expanded per iteration
constexpr int kGraphMaxDegree = 64;
constexpr int kGraphMaxEf = 1024;

// Iterations one query may run: every iteration inserts at most kGraphWidth x D ids into the visited table and the seeds at
// most kGraphMaxSeeds, so the table never holds more than kGraphVisitedSlots / 2 ids.  D = 16 / 32 / 64: 510 / 255 / 127.
__host__ __device__ constexpr int graph_iteration_cap(int degree) {
    return (kGraphVisitedSlots / 2 - kGraphMaxSeeds) / (kGraphWidth * degree);
}

inline bool graph_degree_ok(int d) { return d == 16 || d == 32 || d == 64; }

// ids [m][K + 1] of the list search of rows row0 .. row0 + m - 1 (negative = none) -> cand [m][K] u32: the row's own id
// dropped (or, when it is absent, the last entry), negative ids as 0xFFFFFFFF
int graph_candidates(const int64_t *d_ids, int64_t m, int64_t row0, int K, uint32_t *d_cand, cudaStream_t s);
// rank-based pruning (CAGRA): cand [n][2D] -> pruned [n][D], per node the D candidates with the smallest (detour count, rank)
int graph_prune(const uint32_t *d_cand, int64_t n, int D, uint32_t *d_pruned, cudaStream_t s);
// reverse edges and merge: pruned [n][D] -> graph [n][D].  Allocates and frees its own scratch (2 x n x D x 12 B + the sort's).
int graph_merge(const uint32_t *d_pruned, int64_t n, int D, uint32_t *d_graph, cudaStream_t s);

struct GraphSearchParams {
    const float *queries;      // [nq][d_pad], prepared (cosine: unit)
    const float *rows;         // [n][d_pad] fp32
    const uint32_t *graph;     // [n][degree], 0xFFFFFFFF = empty slot
    const int64_t *seeds;      // [nq][nseeds], negative = none
    const uint8_t *alive;      // nullable: bit r of byte r / 8 keeps row r
    float *out_dis;            // [nq][k]
    int64_t *out_ids;
    unsigned long long *rows_scored;   // += rows scored by every query
    int64_t n, id_offset;
    int d_pad, degree, nseeds, ef, k, max_iters;
    int l2;                    // else inner product (distance -key)
};

size_t graph_search_smem(int d_pad, int ef, int k, bool filtered);
int graph_search(const GraphSearchParams &p, int64_t nq, cudaStream_t s);

}  // namespace b200
