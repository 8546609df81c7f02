// comm.cu -- multi-GPU as a product feature: a communicator below the C ABI so that a C++ host (one process per GPU, or
// one ClickHouse worker per device) runs "shard search -> all-gather of the per-shard top-k -> merge" without Python.
//
// Replaces, across GPUs, what MergeTreeBaseSearchManager::getTotalTopSearchResultImpl does across parts (reference:
// src/VectorIndex/Storages/MergeTreeBaseSearchManager.cpp:207-299) and the table-wide statistics sum of
// ReadWithHybridSearch::getStatisticForTextSearch (src/VectorIndex/Processors/ReadWithHybridSearch.cpp:89-209).
// The only data-path collective of the vector side is ONE ncclAllGather of the packed record
// {float dis[nq * k]; padding to 8 bytes; int64 id[nq * k]} per rank and batch (122 KB at nq = 1024, k = 10: latency-bound over NVSwitch),
// followed by the merge kernel (b200_topk_merge_device_ex); BM25 adds one ncclAllReduce(sum) of a few uint64 counters.
// NCCL is resolved at run time (dlopen of the libnccl.so.2 the process already carries, e.g. PyTorch's): the library has no
// link-time dependency on it and single-GPU users never touch it.
#include <dlfcn.h>

#include <cstring>
#include <string>

#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace {

typedef struct ncclComm *ncclComm_t;
struct ncclUniqueId { char internal[128]; };
enum { ncclUint8 = 1, ncclUint64 = 5 };
enum { ncclSum = 0 };

struct NcclApi {
    void *handle = nullptr;
    int (*GetUniqueId)(ncclUniqueId *) = nullptr;
    int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    std::string error;
};

NcclApi &nccl_api(const char *path_hint) {
    static NcclApi api;
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    if (api.handle) return api;
    const char *env = getenv("B200_NCCL_LIB");
    for (const char *cand : {path_hint, env, "libnccl.so.2", "libnccl.so"}) {
        if (!cand || !*cand) continue;
        api.handle = dlopen(cand, RTLD_NOW | RTLD_GLOBAL);
        if (api.handle) break;
    }
    if (!api.handle) {
        api.error = std::string("libnccl.so.2 not found (pass its path or set B200_NCCL_LIB): ") + (dlerror() ? dlerror() : "");
        return api;
    }
    auto sym = [&](const char *n) { return dlsym(api.handle, n); };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(sym("ncclAllReduce"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather || !api.AllReduce) {
        api.error = "libnccl lacks an expected symbol";
        dlclose(api.handle);
        api.handle = nullptr;
    }
    return api;
}

}  // namespace

using namespace b200;

struct b200_comm {
    ncclComm_t comm = nullptr;
    NcclApi *api = nullptr;
    int rank = 0, world = 1, device = 0;
    DevMem send, recv;                       // packed records: one / world of them
    DevMem d_counters;                       // uint64 all-reduce scratch
    DevMem d_host_out;                       // merged result of the host-buffer gather
    std::mutex mu;
    // CUDA graphs of whole sharded search steps, keyed by the corpus' serial number and the call's arguments; the corpus'
    // state epoch at capture says whether the rows, side arrays, path and workspaces the nodes point at are still current
    struct Graph {
        cudaGraphExec_t exec = nullptr;
        uint64_t epoch = 0;
        int64_t launches = 0;   // kernels / collectives one replay stands for (launch accounting)
    };
    std::map<std::tuple<uint64_t, const void *, int64_t, int, const void *, int64_t, void *, void *, void *>, Graph> graphs;
    int64_t graph_captures = 0, graph_replays = 0;
    DevMem host_stage;                                   // device staging of the host-buffer entry point
};

// The packed record of one rank: dis [nq * k] fp32, padded to a multiple of 8 bytes, then ids [nq * k] int64.  The record
// size is a multiple of 8, so the ids of every gathered record are 8-byte aligned.
static size_t record_dis_bytes(int64_t nq, int k) { return round_up((size_t)nq * k * 4, 8); }
static size_t record_bytes(int64_t nq, int k) { return record_dis_bytes(nq, k) + (size_t)nq * k * 8; }
static int64_t *record_ids(void *rec, int64_t nq, int k) {
    return reinterpret_cast<int64_t *>(reinterpret_cast<char *>(rec) + record_dis_bytes(nq, k));
}

static void drop_graphs(b200_comm *c) {
    for (auto &kv : c->graphs) cudaGraphExecDestroy(kv.second.exec);
    c->graphs.clear();
}

#define B200_NCCL_OK(c, expr)                                                                                              \
    do {                                                                                                                   \
        int _r = (expr);                                                                                                   \
        if (_r != 0)                                                                                                       \
            return fail(B200_ERR_CUDA, std::string(#expr) + ": " + ((c)->api->GetErrorString ? (c)->api->GetErrorString(_r) : "NCCL error")); \
    } while (0)

extern "C" int b200_comm_unique_id(const char *nccl_lib_path, void *out_id_128_bytes) {
    if (!out_id_128_bytes) return fail(B200_ERR_INVALID, "null output");
    NcclApi &api = nccl_api(nccl_lib_path);
    if (!api.handle) return fail(B200_ERR_UNSUPPORTED, api.error);
    ncclUniqueId id;
    const int r = api.GetUniqueId(&id);
    if (r != 0) return fail(B200_ERR_CUDA, std::string("ncclGetUniqueId: ") + (api.GetErrorString ? api.GetErrorString(r) : "error"));
    memcpy(out_id_128_bytes, id.internal, 128);
    return B200_OK;
}

extern "C" int b200_comm_create(const char *nccl_lib_path, const void *unique_id_128_bytes, int rank, int world, b200_comm **out) {
    if (!out || !unique_id_128_bytes || world < 1 || rank < 0 || rank >= world) return fail(B200_ERR_INVALID, "bad arguments");
    *out = nullptr;
    NcclApi &api = nccl_api(nccl_lib_path);
    if (!api.handle) return fail(B200_ERR_UNSUPPORTED, api.error);
    b200_comm *c = new b200_comm();
    c->api = &api;
    c->rank = rank;
    c->world = world;
    B200_CUDA_OK(cudaGetDevice(&c->device));
    ncclUniqueId id;
    memcpy(id.internal, unique_id_128_bytes, 128);
    const int r = api.CommInitRank(&c->comm, world, id, rank);
    if (r != 0) {
        delete c;
        return fail(B200_ERR_CUDA, std::string("ncclCommInitRank: ") + (api.GetErrorString ? api.GetErrorString(r) : "error"));
    }
    *out = c;
    return B200_OK;
}

extern "C" int b200_comm_free(b200_comm *c) {
    if (!c) return B200_OK;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    drop_graphs(c);
    if (c->comm) c->api->CommDestroy(c->comm);
    delete c;
    return B200_OK;
}

extern "C" int b200_comm_info(const b200_comm *c, int *rank, int *world) {
    if (!c) return fail(B200_ERR_INVALID, "null communicator");
    if (rank) *rank = c->rank;
    if (world) *world = c->world;
    return B200_OK;
}

static int comm_reserve(b200_comm *c, int64_t nq, int k) {
    const size_t rec = record_bytes(nq, k);
    if (rec > c->send.size()) {
        c->send.reset();
        c->recv.reset();
        drop_graphs(c);   // captured pointers are gone
        if (c->send.reserve(rec) != B200_OK || c->recv.alloc(c->send.size() * c->world) != B200_OK) {
            c->send.reset();
            return fail(B200_ERR_NOMEM, "cudaMalloc of the all-gather buffers failed");
        }
    }
    return B200_OK;
}

// where a shard search should write its [nq][k] result so that no pack step is needed before the all-gather
extern "C" int b200_comm_local_buffers(b200_comm *c, int64_t nq, int k, float **d_dis, int64_t **d_ids) {
    if (!c || !d_dis || !d_ids || nq < 0 || k <= 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    B200_TRY(comm_reserve(c, std::max<int64_t>(nq, 1), k));
    *d_dis = c->send.as<float>();
    *d_ids = record_ids(c->send.p, nq, k);
    return B200_OK;
}

// all-gather of the records written at b200_comm_local_buffers(nq, k) + merge -> the global top-k on every rank
extern "C" int b200_comm_gather_merge(b200_comm *c, int64_t nq, int k, int descending, float *d_out_dis, int64_t *d_out_ids, void *stream) {
    if (!c || !d_out_dis || !d_out_ids || nq < 0 || k <= 0) return fail(B200_ERR_INVALID, "bad arguments");
    // every refusal comes before the collective: a rank that returns early must not leave the others inside the all-gather
    if (k > 2048) return fail(B200_ERR_UNSUPPORTED, "k > 2048 not supported by the merge kernel");
    if (nq == 0) return B200_OK;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t rec = record_bytes(nq, k);
    if (rec > c->send.size()) return fail(B200_ERR_INVALID, "call b200_comm_local_buffers(nq, k) first");
    if (c->world == 1) {
        B200_CUDA_OK(cudaMemcpyAsync(d_out_dis, c->send.p, (size_t)nq * k * 4, cudaMemcpyDeviceToDevice, s));
        B200_CUDA_OK(cudaMemcpyAsync(d_out_ids, record_ids(c->send.p, nq, k), (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, s));
        return B200_OK;
    }
    B200_NCCL_OK(c, c->api->AllGather(c->send.p, c->recv.p, rec, ncclUint8, c->comm, s));
    g_launches++;
    // list l of the gathered buffer: dis at recv + l * rec, ids record_dis_bytes further; rec is a multiple of 8, so the
    // strides are whole elements of both types
    return b200_topk_merge_device_ex(c->recv.as<const float>(), record_ids(c->recv.p, nq, k), c->world, (int64_t)(rec / 4),
                                     (int64_t)(rec / 8), nq, k, k, descending, 0, d_out_dis, d_out_ids, nullptr, stream ? stream : nullptr);
}

// Host-buffer form for lists that are produced on the host (the per-shard BM25 top-k of b200_bm25_search_batch): uploads
// this rank's [nq][k] scores / ids (unused slots: score -inf (descending) or +inf, id -1), all-gathers + merges, and
// returns the table-wide top-k to the host.  Synchronous.
extern "C" int b200_comm_gather_merge_host(b200_comm *c, const float *h_dis, const int64_t *h_ids, int64_t nq, int k, int descending,
                                           float *h_out_dis, int64_t *h_out_ids) {
    if (!c || !h_dis || !h_ids || !h_out_dis || !h_out_ids || nq < 0 || k <= 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (nq == 0) return B200_OK;
    if (c->world == 1) {
        if (h_out_dis != h_dis) memcpy(h_out_dis, h_dis, (size_t)nq * k * 4);
        if (h_out_ids != h_ids) memcpy(h_out_ids, h_ids, (size_t)nq * k * 8);
        return B200_OK;
    }
    float *d_dis = nullptr;
    int64_t *d_ids = nullptr;
    B200_TRY(b200_comm_local_buffers(c, nq, k, &d_dis, &d_ids));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t nd = (size_t)nq * k * 4, ni = (size_t)nq * k * 8;
    if (nd + ni > c->d_host_out.size()) B200_TRY(c->d_host_out.alloc(nd + ni + 256));
    float *o_dis = c->d_host_out.as<float>();
    int64_t *o_ids = reinterpret_cast<int64_t *>(c->d_host_out.as<char>() + ((nd + 7) & ~(size_t)7));
    B200_CUDA_OK(cudaMemcpyAsync(d_dis, h_dis, nd, cudaMemcpyHostToDevice, nullptr));
    B200_CUDA_OK(cudaMemcpyAsync(d_ids, h_ids, ni, cudaMemcpyHostToDevice, nullptr));
    B200_TRY(b200_comm_gather_merge(c, nq, k, descending, o_dis, o_ids, nullptr));
    B200_CUDA_OK(cudaMemcpyAsync(h_out_dis, o_dis, nd, cudaMemcpyDeviceToHost, nullptr));
    B200_CUDA_OK(cudaMemcpyAsync(h_out_ids, o_ids, ni, cudaMemcpyDeviceToHost, nullptr));
    B200_CUDA_OK(cudaStreamSynchronize(nullptr));
    return B200_OK;
}

// table-wide statistics: in-place sum over the ranks of n uint64 counters held on the host
// (total_docs, total_tokens[field], doc_freq[(field, term)]; getStatisticForTextSearch)
extern "C" int b200_comm_allreduce_sum_u64(b200_comm *c, uint64_t *host_counters, int64_t n) {
    if (!c || (!host_counters && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (n == 0 || c->world == 1) return B200_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    if ((size_t)n * 8 > c->d_counters.size()) B200_TRY(c->d_counters.alloc((size_t)n * 8 + 256));
    B200_CUDA_OK(cudaMemcpy(c->d_counters.p, host_counters, (size_t)n * 8, cudaMemcpyHostToDevice));
    B200_NCCL_OK(c, c->api->AllReduce(c->d_counters.p, c->d_counters.p, (size_t)n, ncclUint64, ncclSum, c->comm, nullptr));
    g_launches++;
    B200_CUDA_OK(cudaStreamSynchronize(nullptr));
    B200_CUDA_OK(cudaMemcpy(host_counters, c->d_counters.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return B200_OK;
}

// ------------------------------------------------------------------------------------
// whole sharded steps
// ------------------------------------------------------------------------------------
extern "C" int b200_corpus_search_device(b200_corpus *c, const float *d_queries, int64_t nq, int k, const uint8_t *d_alive_bits,
                                         int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, void *stream);
extern "C" int b200_index_search_device(b200_index *ix, const float *d_queries, int64_t nq, int k, const char *params, int first_stage_only,
                                        const uint8_t *d_alive_bits, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, void *stream);
namespace b200 {
int corpus_metric(const b200_corpus *c);
bool corpus_timing_enabled(const b200_corpus *c);
int corpus_dim(const b200_corpus *c);
int64_t corpus_query_row_bytes(const b200_corpus *c);
uint64_t corpus_serial(const b200_corpus *c);
uint64_t corpus_state_epoch(b200_corpus *c);
int index_metric(const b200_index *ix);
}

static int sharded_corpus_step(b200_comm *cm, b200_corpus *corpus, const float *d_queries, int64_t nq, int k, const uint8_t *d_alive,
                               int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    float *l_dis = cm->send.as<float>();
    int64_t *l_ids = record_ids(cm->send.p, nq, k);
    B200_TRY(b200_corpus_search_device(corpus, d_queries, nq, k, d_alive, id_offset, l_dis, l_ids, s));
    return b200_comm_gather_merge(cm, nq, k, corpus_metric(corpus) == B200_METRIC_IP ? 1 : 0, d_out_dis, d_out_ids, s);
}

// FLAT corpus sharded by rows over the communicator's GPUs: this rank scans its shard (ids + id_offset), the per-shard
// top-k lists are all-gathered and merged; every rank ends with the global answer in d_out_*.  Asynchronous on `stream`
// (must be a real stream, not NULL).  use_graph: replay the whole step (query conversion, scan, all-gather, merge) as
// ONE CUDA graph after the first call with the same arguments -- the step is launch-latency-bound at 8 GPUs.
extern "C" int b200_sharded_corpus_search(b200_comm *cm, b200_corpus *corpus, const float *d_queries, int64_t nq, int k,
                                          const uint8_t *d_alive_bits, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, void *stream,
                                          int use_graph) {
    if (!cm || !corpus || (!d_queries && nq > 0) || !d_out_dis || !d_out_ids || nq < 0 || k <= 0 || !stream)
        return fail(B200_ERR_INVALID, "bad arguments (a non-NULL stream is required)");
    if (nq == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(cm->mu);
    B200_CUDA_OK(cudaSetDevice(cm->device));
    B200_TRY(comm_reserve(cm, nq, k));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (!use_graph || corpus_timing_enabled(corpus))
        return sharded_corpus_step(cm, corpus, d_queries, nq, k, d_alive_bits, id_offset, d_out_dis, d_out_ids, s);
    const auto key = std::make_tuple(corpus_serial(corpus), (const void *)d_queries, nq, k, (const void *)d_alive_bits, id_offset,
                                     (void *)d_out_dis, (void *)d_out_ids, (void *)s);
    auto it = cm->graphs.find(key);
    if (it != cm->graphs.end() && it->second.epoch != corpus_state_epoch(corpus)) {
        // the corpus grew, moved, changed path or reallocated a workspace since the capture: the nodes point at old state
        B200_CUDA_OK(cudaStreamSynchronize(s));
        cudaGraphExecDestroy(it->second.exec);
        cm->graphs.erase(it);
        it = cm->graphs.end();
    }
    if (it == cm->graphs.end()) {
        // first call: run eagerly once (sizes every workspace), then capture the identical sequence
        B200_TRY(sharded_corpus_step(cm, corpus, d_queries, nq, k, d_alive_bits, id_offset, d_out_dis, d_out_ids, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        cudaGraph_t g = nullptr;
        B200_CUDA_OK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        const int64_t launches_before = g_launches;
        int rc = sharded_corpus_step(cm, corpus, d_queries, nq, k, d_alive_bits, id_offset, d_out_dis, d_out_ids, s);
        const int64_t per_step = g_launches - launches_before;
        cudaError_t e = cudaStreamEndCapture(s, &g);
        if (rc != B200_OK || e != cudaSuccess || !g) {
            cudaGetLastError();
            if (g) cudaGraphDestroy(g);
            if (rc != B200_OK) return rc;
            return fail(B200_ERR_CUDA, std::string("stream capture of the sharded step failed: ") + cudaGetErrorString(e));
        }
        cudaGraphExec_t exec = nullptr;
        e = cudaGraphInstantiate(&exec, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return fail(B200_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
        b200_comm::Graph gr;
        gr.exec = exec;
        gr.epoch = corpus_state_epoch(corpus);
        gr.launches = per_step;
        it = cm->graphs.emplace(key, gr).first;
        cm->graph_captures++;
        g_launches = launches_before;   // the captured pass launched nothing
    }
    B200_CUDA_OK(cudaGraphLaunch(it->second.exec, s));
    cm->graph_replays++;
    g_launches += it->second.launches;
    return B200_OK;
}

// CUDA graphs this communicator captured and replayed (b200_sharded_corpus_search with use_graph)
extern "C" int b200_comm_graph_stats(b200_comm *c, int64_t *captures, int64_t *replays) {
    if (!c) return fail(B200_ERR_INVALID, "null communicator");
    std::lock_guard<std::mutex> lk(c->mu);
    if (captures) *captures = c->graph_captures;
    if (replays) *replays = c->graph_replays;
    return B200_OK;
}

// the same through host buffers (what a ClickHouse worker holds): pinned or pageable queries in, the global top-k out on
// every rank; H2D, scan, all-gather, merge, D2H and the synchronise are all inside
extern "C" int b200_sharded_corpus_search_host(b200_comm *cm, b200_corpus *corpus, const float *queries, int64_t nq, int d, int k,
                                               int64_t id_offset, float *out_dis, int64_t *out_ids, void *stream, int use_graph) {
    if (!cm || !corpus || (!queries && nq > 0) || !out_dis || !out_ids || nq < 0 || k <= 0 || d <= 0 || !stream)
        return fail(B200_ERR_INVALID, "bad arguments (a non-NULL stream is required)");
    if (d != corpus_dim(corpus)) return fail(B200_ERR_INVALID, "d differs from the corpus' dimension");
    if (nq == 0) return B200_OK;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t q_bytes = (size_t)nq * corpus_query_row_bytes(corpus);   // binary corpora: d / 8 bytes per query
    {
        std::lock_guard<std::mutex> lk(cm->mu);
        B200_CUDA_OK(cudaSetDevice(cm->device));
        const size_t need = round_up(q_bytes, 16) + round_up((size_t)nq * k * 4, 16) + (size_t)nq * k * 8;
        if (need > cm->host_stage.size()) {
            drop_graphs(cm);   // captured pointers are about to go
            B200_TRY(cm->host_stage.alloc(need + need / 4));
        }
    }
    float *d_q = cm->host_stage.as<float>();
    float *d_od = reinterpret_cast<float *>(cm->host_stage.as<char>() + round_up(q_bytes, 16));
    int64_t *d_oi = reinterpret_cast<int64_t *>(reinterpret_cast<char *>(d_od) + round_up((size_t)nq * k * 4, 16));
    B200_CUDA_OK(cudaMemcpyAsync(d_q, queries, q_bytes, cudaMemcpyHostToDevice, s));
    B200_TRY(b200_sharded_corpus_search(cm, corpus, d_q, nq, k, nullptr, id_offset, d_od, d_oi, stream, use_graph));
    B200_CUDA_OK(cudaMemcpyAsync(out_dis, d_od, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_ids, d_oi, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// a vector index sharded by rows (every rank built its own index over its rows): search + all-gather + merge
extern "C" int b200_sharded_index_search(b200_comm *cm, b200_index *ix, int metric, const float *d_queries, int64_t nq, int k, const char *params,
                                         const uint8_t *d_alive_bits, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, void *stream) {
    if (!cm || !ix || (!d_queries && nq > 0) || !d_out_dis || !d_out_ids || nq < 0 || k <= 0 || !stream)
        return fail(B200_ERR_INVALID, "bad arguments (a non-NULL stream is required)");
    if (metric != index_metric(ix)) return fail(B200_ERR_INVALID, "metric differs from the index' metric");
    if (nq == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(cm->mu);
    B200_CUDA_OK(cudaSetDevice(cm->device));
    B200_TRY(comm_reserve(cm, nq, k));
    float *l_dis = cm->send.as<float>();
    int64_t *l_ids = record_ids(cm->send.p, nq, k);
    B200_TRY(b200_index_search_device(ix, d_queries, nq, k, params, 0, d_alive_bits, id_offset, l_dis, l_ids, stream));
    return b200_comm_gather_merge(cm, nq, k, metric == B200_METRIC_IP ? 1 : 0, d_out_dis, d_out_ids, stream);
}
