// capi.cu -- the C ABI of libb200search.so (declared in include/b200_search.h) and the host
// orchestration under it: device-resident corpora, path selection (memory-bound scan vs
// wgmma GEMM), query staging, partial-list merge.
//
// There is deliberately no CPU compute path in this file: every entry point either runs
// CUDA kernels on an sm_90 device or fails with B200_ERR_NO_DEVICE / B200_ERR_CUDA.
#include <algorithm>
#include <array>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

thread_local std::string g_error;
thread_local int64_t g_launches = 0;
// rows the last corpus search launched on this thread scored (b200_thread_last_rows_scored)
static thread_local int64_t t_last_rows_scored = 0;

void set_error(const std::string &msg) { g_error = msg; }
int fail(int code, const std::string &msg) {
    g_error = msg;
    return code;
}

static int ensure_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(B200_ERR_NO_DEVICE, std::string("no CUDA device visible (") +
                                            (e != cudaSuccess ? cudaGetErrorString(e) : "count = 0") +
                                            "); libb200search has no CPU fallback");
    }
    int dev = 0;
    B200_CUDA_OK(cudaGetDevice(&dev));
    int major = 0;
    B200_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    if (major != 9)
        return fail(B200_ERR_NO_DEVICE, "device compute capability major is " + std::to_string(major) +
                                            "; this library carries sm_90a code only");
    return B200_OK;
}

static int num_sms() {
    int dev = 0, n = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}

}  // namespace b200

using namespace b200;

struct b200_corpus {
    int metric = 0, dtype = 0, d = 0, d_pad = 0;
    int64_t cap = 0, n = 0;
    int64_t row_bytes = 0;
    DevMem owned_rows;           // the rows, when the corpus allocated them
    void *data = nullptr;        // the rows: owned_rows, or device rows the caller adopted in and still owns
    int64_t side_cap_rows = 0;   // rows the row_scale / row_bias arrays can hold
    DevMem row_scale;            // float [rows]; cosine: -1/||y||
    DevMem row_bias;             // float [rows]; L2: ||y||^2 (GEMM path); binary: popcount of the row (tensor-core path)
    int device = 0;
    int path = 0;
    int sms = 132;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    // CUDA graphs of sharded steps (comm.cu) bake in the rows, the row count, the side arrays, the path and the workspace
    // pointers: `serial` names this corpus for the whole process (an address can be reused after a free), `epoch` moves
    // whenever one of those changes except the workspaces, whose reallocations corpus_state_epoch adds
    uint64_t serial = 0;
    uint64_t epoch = 0;
    // workspaces
    DevMem w_raw, w_q32, w_qbf, w_qlo, w_qnorm, w_pk, w_pi, w_lk, w_li, w_alive, w_odis, w_oids, w_stage, w_prog, w_qb;
    // pre-filtered search (prefilter.cu): kept row ids, compaction scratch, compact rows (+ a row of slack), their side arrays
    DevMem w_pf_ids, w_pf_tmp, w_pf_rows, w_pf_side;
    std::array<DevMem *, 19> workspaces() {
        return {&w_raw, &w_q32, &w_qbf, &w_qlo, &w_qnorm, &w_pk, &w_pi, &w_lk, &w_li, &w_alive, &w_odis, &w_oids, &w_stage, &w_prog,
                &w_qb, &w_pf_ids, &w_pf_tmp, &w_pf_rows, &w_pf_side};
    }
    int prefilter = 0;             // b200_corpus_set_prefilter: 0 auto | 1 never | 2 whenever the compact copy fits the budget
    int64_t last_rows_scored = 0;  // rows the last search scored: n after a full scan, the kept rows after a gathered one
    // fused single-launch path of the host entry point (small batches, scan kernel): mapped pinned staging + counters
    void *h_pin = nullptr;         // [queries 8 * d fp32 | dis 8 * k | ids 8 * k | flag]
    size_t h_pin_bytes = 0;
    DevMem d_tickets;              // uint32 [8] + tiles_done, then (at +64 bytes) the device copy of the staged queries
    unsigned int fused_seq = 0;
    int d_tickets_d = 0;           // row length the query staging behind d_tickets was sized for
    int fused_enabled = 1;         // B200_FUSED_SCAN=0 disables (A/B)
    int rescore_l2 = 1;      // tensor-core L2: re-score the k winners exactly (B200_GEMM_RESCORE_L2=0 disables, A/B only)
    // what the last launch really was (tests assert on it): kernel id, CTAs per MMA and per operand fetch (1 on sm_90), grid
    int last_cg = 0, last_mc = 0, last_grid = 0, last_kernel = 0;
    // optional CUDA-event timing of the dominant kernel (scan or GEMM) for the roofline report
    bool timing = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_used, ev_free;
    double timed_ms = 0;
    int64_t timed_launches = 0;
};

static void timing_begin(b200_corpus *c, cudaStream_t s, std::pair<cudaEvent_t, cudaEvent_t> &ev) {
    if (!c->timing) return;
    if (c->ev_free.empty()) {
        cudaEventCreate(&ev.first);
        cudaEventCreate(&ev.second);
    } else {
        ev = c->ev_free.back();
        c->ev_free.pop_back();
    }
    cudaEventRecord(ev.first, s);
}
// fold the recorded event pairs into the running totals (waits for them) and recycle the events
static void timing_drain(b200_corpus *c) {
    for (auto &ev : c->ev_used) {
        float ms = 0;
        if (cudaEventSynchronize(ev.second) == cudaSuccess && cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) {
            c->timed_ms += ms;
            c->timed_launches++;
        }
        c->ev_free.push_back(ev);
    }
    c->ev_used.clear();
}
static void timing_end(b200_corpus *c, cudaStream_t s, std::pair<cudaEvent_t, cudaEvent_t> &ev) {
    if (!c->timing) return;
    cudaEventRecord(ev.second, s);
    c->ev_used.push_back(ev);
    if (c->ev_used.size() >= 1024) timing_drain(c);  // nobody asked for the totals for a while: keep the list bounded
}

static int corpus_alloc(b200_corpus *c, int64_t rows);
static int corpus_norms(b200_corpus *c, int64_t first, int64_t n);

namespace b200 {
// hooks for comm.cu
int corpus_metric(const b200_corpus *c) { return c->metric; }
bool corpus_timing_enabled(const b200_corpus *c) { return c->timing; }
int corpus_dim(const b200_corpus *c) { return c->d; }
// bytes of one query row as the device entry points read it: fp32 [d], binary corpora [d / 8]
int64_t corpus_query_row_bytes(const b200_corpus *c) { return c->dtype == B200_DTYPE_BIN ? c->d_pad : (int64_t)c->d * 4; }
uint64_t corpus_serial(const b200_corpus *c) { return c->serial; }
// changes whenever something a captured search baked in changes: rows, row count, side arrays, path, workspace pointers
uint64_t corpus_state_epoch(b200_corpus *c) {
    std::lock_guard<std::mutex> lk(c->mu);
    uint64_t e = c->epoch;
    for (DevMem *b : c->workspaces()) e += b->reallocs;
    return e;
}
// hooks for the index layer (ivf.cu): device view of the rows / in-place row normalisation
const void *corpus_device_rows(const b200_corpus *c) { return c->data; }
// append fp32 rows [n][d] (binary corpora: bytes [n][d / 8]) that already live on the device (index build, centroid tables);
// asynchronous on s except for a reallocation, synchronised before returning so that the caller may reuse d_rows
int corpus_append_device(b200_corpus *c, const float *d_rows, int64_t n, cudaStream_t s) {
    if (!c || (!d_rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (n == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    B200_TRY(corpus_alloc(c, std::max(c->n + n, c->cap)));
    char *dst = reinterpret_cast<char *>(c->data) + c->n * c->row_bytes;
    if (c->dtype == B200_DTYPE_BIN) B200_CUDA_OK(cudaMemcpyAsync(dst, d_rows, (size_t)n * c->row_bytes, cudaMemcpyDeviceToDevice, s));
    else if (c->dtype == B200_DTYPE_BF16) B200_CUDA_OK(launch_f32_to_bf16_rows(d_rows, c->d, dst, c->d_pad, n, s));
    else B200_CUDA_OK(launch_pad_rows_f32(d_rows, c->d, reinterpret_cast<float *>(dst), c->d_pad, n, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    B200_TRY(corpus_norms(c, c->n, n));
    B200_CUDA_OK(cudaStreamSynchronize(c->stream));
    c->n += n;
    c->epoch++;
    return B200_OK;
}
int corpus_normalize_rows(b200_corpus *c) {
    if (c->dtype != B200_DTYPE_F32) return fail(B200_ERR_UNSUPPORTED, "normalise: fp32 corpora only");
    B200_CUDA_OK(cudaSetDevice(c->device));
    B200_CUDA_OK(launch_normalize_rows_f32(reinterpret_cast<float *>(c->data), c->d_pad, c->n, c->stream));
    B200_CUDA_OK(cudaStreamSynchronize(c->stream));
    return B200_OK;
}
}  // namespace b200

static bool is_float_metric(int m) { return m == B200_METRIC_L2 || m == B200_METRIC_IP || m == B200_METRIC_COSINE; }
static bool is_bin_metric(int m) { return m == B200_METRIC_HAMMING || m == B200_METRIC_JACCARD; }

static int pad_for(int dtype, int d) {
    if (dtype == B200_DTYPE_BF16) return (int)round_up(d, 64);  // 128-byte TMA/UMMA swizzle rows
    if (dtype == B200_DTYPE_F32) return (int)round_up(d, 4);    // 16-byte vector loads
    return d / 8;                                                // binary: bytes
}

extern "C" const char *b200_last_error(void) { return g_error.c_str(); }
extern "C" const char *b200_version(void) { return "b200search 0.1 (sm_90a)"; }

extern "C" int b200_device_count(int *out_n) {
    if (!out_n) return fail(B200_ERR_INVALID, "out_n is null");
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    *out_n = n;
    return B200_OK;
}

extern "C" int b200_set_device(int device) {
    B200_TRY(ensure_device());
    B200_CUDA_OK(cudaSetDevice(device));
    return B200_OK;
}

extern "C" int64_t b200_device_bytes(void) { return g_device_bytes; }

extern "C" int64_t b200_launch_count(int reset) {
    int64_t v = g_launches;
    if (reset) g_launches = 0;
    return v;
}

extern "C" int b200_corpus_create(int metric, int dtype, int d, int64_t capacity_rows, b200_corpus **out) {
    if (!out) return fail(B200_ERR_INVALID, "out is null");
    *out = nullptr;
    if (d <= 0 || capacity_rows < 0) return fail(B200_ERR_INVALID, "bad d / capacity");
    if (dtype == B200_DTYPE_BIN) {
        if (!is_bin_metric(metric)) return fail(B200_ERR_INVALID, "binary corpus needs HAMMING or JACCARD");
        if (d % 8) return fail(B200_ERR_INVALID, "binary dimension must be a multiple of 8 bits");
    } else if (dtype == B200_DTYPE_F32 || dtype == B200_DTYPE_BF16) {
        if (!is_float_metric(metric)) return fail(B200_ERR_INVALID, "float corpus needs L2, IP or COSINE");
    } else {
        return fail(B200_ERR_INVALID, "unknown dtype");
    }
    B200_TRY(ensure_device());
    b200_corpus *c = new b200_corpus();
    c->metric = metric;
    c->dtype = dtype;
    c->d = d;
    c->d_pad = pad_for(dtype, d);
    c->row_bytes = dtype == B200_DTYPE_BIN ? c->d_pad : (int64_t)c->d_pad * (dtype == B200_DTYPE_BF16 ? 2 : 4);
    c->cap = capacity_rows;
    static std::atomic<uint64_t> next_serial{0};
    c->serial = ++next_serial;
    cudaGetDevice(&c->device);
    c->sms = num_sms();
    if (const char *ev = getenv("B200_GEMM_RESCORE_L2")) c->rescore_l2 = atoi(ev);
    if (const char *ev = getenv("B200_FUSED_SCAN")) c->fused_enabled = atoi(ev);
    cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        delete c;
        return fail(B200_ERR_CUDA, std::string("cudaStreamCreate: ") + cudaGetErrorString(e));
    }
    *out = c;
    return B200_OK;
}

static int corpus_alloc(b200_corpus *c, int64_t rows) {
    if (c->data && !c->owned_rows) return fail(B200_ERR_INVALID, "corpus adopted device memory; cannot append");
    // +1 row of slack so that 16-byte vector loads of the last row never leave the allocation
    const size_t need = (size_t)(rows + 1) * c->row_bytes + 256;
    const bool want_scale = c->metric == B200_METRIC_COSINE, want_bias = c->metric == B200_METRIC_L2 || is_bin_metric(c->metric);
    if (!c->data || c->owned_rows.size() < need) {
        DevMem nd;   // the rows held so far are copied over before the old allocation goes
        B200_TRY(nd.alloc(need));
        if (c->data && c->n) {
            cudaMemcpyAsync(nd.p, c->data, (size_t)c->n * c->row_bytes, cudaMemcpyDeviceToDevice, c->stream);
            cudaStreamSynchronize(c->stream);
        }
        c->owned_rows = std::move(nd);
        c->data = c->owned_rows.p;
    }
    if ((want_scale && (!c->row_scale || c->side_cap_rows < rows)) || (want_bias && (!c->row_bias || c->side_cap_rows < rows))) {
        DevMem ns, nb;
        if (want_scale) B200_TRY(ns.alloc((size_t)rows * 4 + 256));
        if (want_bias) B200_TRY(nb.alloc((size_t)rows * 4 + 256));
        if (c->n) {
            if (ns && c->row_scale) cudaMemcpyAsync(ns.p, c->row_scale.p, (size_t)c->n * 4, cudaMemcpyDeviceToDevice, c->stream);
            if (nb && c->row_bias) cudaMemcpyAsync(nb.p, c->row_bias.p, (size_t)c->n * 4, cudaMemcpyDeviceToDevice, c->stream);
            cudaStreamSynchronize(c->stream);
        }
        c->row_scale = std::move(ns);
        c->row_bias = std::move(nb);
        c->side_cap_rows = rows;
    }
    c->cap = std::max(c->cap, rows);
    c->epoch++;
    return B200_OK;
}

static int corpus_norms(b200_corpus *c, int64_t first, int64_t n) {
    const char *rows = reinterpret_cast<const char *>(c->data) + first * c->row_bytes;
    if (c->dtype == B200_DTYPE_BIN)
        B200_CUDA_OK(launch_popc_rows(reinterpret_cast<const uint8_t *>(rows), c->row_bytes, n, c->row_bias.as<float>() + first, c->stream));
    if (c->metric == B200_METRIC_COSINE)
        B200_CUDA_OK(launch_row_norms(rows, c->dtype == B200_DTYPE_BF16, c->d_pad, n, 1, c->row_scale.as<float>() + first, c->stream));
    if (c->metric == B200_METRIC_L2)
        B200_CUDA_OK(launch_row_norms(rows, c->dtype == B200_DTYPE_BF16, c->d_pad, n, 0, c->row_bias.as<float>() + first, c->stream));
    return B200_OK;
}

extern "C" int b200_corpus_append(b200_corpus *c, const void *rows, int64_t n) {
    if (!c || (!rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (n == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    B200_TRY(corpus_alloc(c, std::max(c->n + n, c->cap)));
    char *dst = reinterpret_cast<char *>(c->data) + c->n * c->row_bytes;
    if (c->dtype == B200_DTYPE_BIN || (c->dtype == B200_DTYPE_F32 && c->d == c->d_pad)) {
        // rows already have the HBM layout: pageable host memory -> device through the pinned ring (ingest.cu)
        B200_TRY(staged_h2d(dst, rows, (size_t)n * c->row_bytes, c->device, c->stream));
    } else {
        // stage raw fp32 rows in chunks, then pad / convert on device
        const int64_t chunk = std::max<int64_t>(1, (int64_t)(256ll << 20) / ((int64_t)c->d * 4));
        for (int64_t off = 0; off < n; off += chunk) {
            const int64_t m = std::min(chunk, n - off);
            B200_TRY(c->w_raw.reserve((size_t)m * c->d * 4));
            B200_TRY(staged_h2d(c->w_raw.p, reinterpret_cast<const float *>(rows) + off * c->d, (size_t)m * c->d * 4, c->device,
                                c->stream));
            char *dd = dst + off * c->row_bytes;
            if (c->dtype == B200_DTYPE_BF16)
                B200_CUDA_OK(launch_f32_to_bf16_rows(c->w_raw.as<float>(), c->d, dd, c->d_pad, m, c->stream));
            else
                B200_CUDA_OK(launch_pad_rows_f32(c->w_raw.as<float>(), c->d, reinterpret_cast<float *>(dd), c->d_pad, m, c->stream));
            B200_CUDA_OK(cudaStreamSynchronize(c->stream));  // w_raw is reused
        }
    }
    B200_TRY(corpus_norms(c, c->n, n));
    B200_CUDA_OK(cudaStreamSynchronize(c->stream));
    c->n += n;
    c->epoch++;
    return B200_OK;
}

extern "C" int b200_corpus_memory_bytes(const b200_corpus *c, uint64_t *out_bytes) {
    if (!c || !out_bytes) return fail(B200_ERR_INVALID, "bad arguments");
    // rows (as allocated; adopted rows belong to the caller but still occupy HBM) + per-row side arrays
    uint64_t b = c->owned_rows ? (uint64_t)c->owned_rows.size() : (uint64_t)c->n * (uint64_t)c->row_bytes;
    if (c->row_scale) b += (uint64_t)std::max(c->side_cap_rows, c->n) * 4;
    if (c->row_bias) b += (uint64_t)std::max(c->side_cap_rows, c->n) * 4;
    *out_bytes = b;
    return B200_OK;
}

extern "C" int b200_corpus_adopt_device(b200_corpus *c, const void *device_rows, int64_t n) {
    if (!c || !device_rows || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->data) return fail(B200_ERR_INVALID, "corpus already holds data");
    if (c->dtype != B200_DTYPE_BIN && c->d != c->d_pad)
        return fail(B200_ERR_INVALID, "adopted rows must already be padded (d % 64 == 0 for bf16, d % 4 == 0 for f32)");
    B200_CUDA_OK(cudaSetDevice(c->device));
    if (c->metric == B200_METRIC_COSINE) B200_TRY(c->row_scale.alloc((size_t)n * 4 + 256));
    if (c->metric == B200_METRIC_L2 || c->dtype == B200_DTYPE_BIN) B200_TRY(c->row_bias.alloc((size_t)n * 4 + 256));
    c->data = const_cast<void *>(device_rows);
    c->n = n;
    c->cap = n;
    c->side_cap_rows = n;
    c->epoch++;
    B200_TRY(corpus_norms(c, 0, n));
    B200_CUDA_OK(cudaStreamSynchronize(c->stream));
    return B200_OK;
}

extern "C" int b200_corpus_size(const b200_corpus *c, int64_t *out_rows) {
    if (!c || !out_rows) return fail(B200_ERR_INVALID, "null argument");
    *out_rows = c->n;
    return B200_OK;
}

extern "C" int b200_corpus_set_path(b200_corpus *c, int path) {
    if (!c || path < 0 || path > 7) return fail(B200_ERR_INVALID, "path must be 0..7");
    std::lock_guard<std::mutex> lk(c->mu);
    // 0 auto | 1 scan | 2 tensor cores (binary corpora too: the b1 kernel).  3..7 named the tensor-core instantiations of an
    // earlier target (CTA pairs, multicast clusters, queries in tensor memory); sm_90 has one tensor-core kernel per operand
    // type, so they select it.
    c->path = path >= 2 ? 2 : path;
    c->epoch++;
    return B200_OK;
}

extern "C" int b200_corpus_last_variant(b200_corpus *c, int *kernel, int *cta_group, int *pairs_per_cluster, int *grid) {
    if (!c) return fail(B200_ERR_INVALID, "null corpus");
    std::lock_guard<std::mutex> lk(c->mu);
    if (kernel) *kernel = c->last_kernel;
    if (cta_group) *cta_group = c->last_cg;
    if (pairs_per_cluster) *pairs_per_cluster = c->last_mc;
    if (grid) *grid = c->last_grid;
    return B200_OK;
}

extern "C" int b200_corpus_enable_timing(b200_corpus *c, int on) {
    if (!c) return fail(B200_ERR_INVALID, "null corpus");
    std::lock_guard<std::mutex> lk(c->mu);
    c->timing = on != 0;
    return B200_OK;
}

extern "C" int b200_corpus_kernel_time(b200_corpus *c, int reset, double *out_total_ms, int64_t *out_launches) {
    if (!c || !out_total_ms || !out_launches) return fail(B200_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    timing_drain(c);
    *out_total_ms = c->timed_ms;
    *out_launches = c->timed_launches;
    if (reset) {
        c->timed_ms = 0;
        c->timed_launches = 0;
    }
    return B200_OK;
}

extern "C" int b200_corpus_free(b200_corpus *c) {
    if (!c) return B200_OK;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->h_pin) cudaFreeHost(c->h_pin);
    for (auto *v : {&c->ev_used, &c->ev_free})
        for (auto &ev : *v) {
            cudaEventDestroy(ev.first);
            cudaEventDestroy(ev.second);
        }
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
    return B200_OK;
}

// Auto path of a binary corpus: the tensor cores (gemm_topk_kernel<B1>) from ceil(kBinaryTensorMinQB2 / row_bytes^2) queries
// per batch, the scan below.  Up to 16 queries the tensor kernel costs about one 128-query tile pass (1.5 - 1.9 ms per 10 M
// rows at 256 and at 1024 bits); the scan costs one pass per query, and that pass grew 9.6x from 32- to 128-byte rows.
// Measured with tools/bench_aux.py binary on an H100 80GB HBM3 at a 400 W power limit (10 M rows, k = 10; DESIGN.md
// section 7): the curves cross between 1 and 2 queries at 1024 bits and between 8 and 16 at 256 bits.  20480 / row_bytes^2
// gives 2 and 20 queries (at 256 bits and 16 queries the scan is 10 % slower than the tensor path); other widths are
// extrapolated, not measured.
constexpr int64_t kBinaryTensorMinQB2 = 20480;

// corpus tiles a CTA of gemm_topk_kernel may run ahead of the slowest CTA that streams the same tiles for another query tile
constexpr int kGemmSyncSlack = 2;

// One launch of gemm_topk_kernel over a chunk of <= 1024 staged queries (gp: operands, side arrays, rows, d_pad and alive set),
// then the merge of the CTAs' partial lists into rows of k of d_out_dis / d_out_ids.  kernel: B200_KERNEL_GEMM_*.
static int gemm_chunk(b200_corpus *c, GemmTopkParams &gp, int64_t nq_c, int k, int kernel, int out_mode, const float *q_add,
                      int ip_min_quirk, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    const int nq_pad = (int)round_up(nq_c, 128);
    const int q_tiles = nq_pad / 128;
    int grid = gemm_topk_grid(q_tiles, gp.n, c->sms);
    grid = (grid / q_tiles) * q_tiles;
    if (grid < q_tiles) grid = q_tiles;
    // every consumer warpgroup of a CTA keeps and publishes its own per-query lists
    const size_t producers = (size_t)grid * gemm_consumer_warpgroups(kernel == B200_KERNEL_GEMM_TF32X3);
    B200_TRY(c->w_pk.reserve(producers * 128 * k * 4));
    B200_TRY(c->w_pi.reserve(producers * 128 * k * 4));
    gp.part_keys = c->w_pk.as<float>();
    gp.part_ids = c->w_pi.as<uint32_t>();
    {  // global scratch for the per-thread lists, used when they do not fit in shared memory (large k)
        B200_TRY(c->w_lk.reserve(producers * 128 * list_cap_for(k) * 4));
        B200_TRY(c->w_li.reserve(producers * 128 * list_cap_for(k) * 4));
        gp.list_keys_gmem = c->w_lk.as<float>();
        gp.list_ids_gmem = c->w_li.as<uint32_t>();
    }
    gp.nq_pad = nq_pad;
    gp.nq_valid = (int)nq_c;
    gp.k = k;
    gp.q_tiles = q_tiles;
    B200_TRY(c->w_qb.reserve((size_t)nq_pad * 4));
    B200_CUDA_OK(cudaMemsetAsync(c->w_qb.p, 0xff, (size_t)nq_pad * 4, s));   // no bound yet
    gp.query_bound = c->w_qb.as<uint32_t>();
    if (q_tiles > 1) {
        B200_TRY(c->w_prog.reserve((size_t)grid * 4));
        B200_CUDA_OK(cudaMemsetAsync(c->w_prog.p, 0, (size_t)grid * 4, s));
        gp.progress = c->w_prog.as<int>();
        gp.sync_slack = kGemmSyncSlack;
    }
    const char *detail = nullptr;
    std::pair<cudaEvent_t, cudaEvent_t> ev;
    timing_begin(c, s, ev);
    cudaError_t e = kernel == B200_KERNEL_GEMM_TF32X3 ? launch_gemm3_topk(gp, grid, s, &detail)
                    : kernel == B200_KERNEL_GEMM_B1  ? launch_gemm_b1_topk(gp, grid, s, &detail)
                                                     : launch_gemm_topk(gp, grid, s, &detail);
    timing_end(c, s, ev);
    c->last_kernel = kernel;
    c->last_cg = 1; c->last_mc = 1; c->last_grid = grid;
    if (e != cudaSuccess)
        return fail(B200_ERR_CUDA, std::string("gemm_topk launch: ") + (detail ? detail : cudaGetErrorString(e)));
    MergeParams mp{};
    mp.in_keys = gp.part_keys;
    mp.in_ids = gp.part_ids;
    mp.list_stride = (int64_t)nq_pad * k;
    mp.q_stride = k;
    mp.n_lists = (int)(producers / q_tiles);
    mp.k_in = k;
    mp.k = k;
    mp.nq = nq_c;
    mp.out_mode = out_mode;
    mp.q_add = q_add;
    mp.ip_min_quirk = ip_min_quirk;
    mp.id_offset = id_offset;
    mp.out_dis = d_out_dis;
    mp.out_ids = d_out_ids;
    B200_CUDA_OK(launch_topk_merge(mp, false, s));
    return B200_OK;
}

// The path a search of nq queries at this k takes (1 scan, 2 tensor cores) before the empty-corpus and limit checks:
// the forced one, else the auto choice.
//
// Auto on float corpora: when the batch goes to the tensor cores (bf16 rows: bf16 wgmma GEMM; fp32 rows: 3xTF32 split
// GEMM, same accuracy class as the fp32 FMA scan).  A <= 128-query tensor-core pass reads the corpus once, the scan reads
// it once per few queries, so the tensor cores take bf16 batches from 2 queries and fp32 batches from 5.  These crossovers
// were chosen on an earlier GPU and are not re-measured on the H100.  L2 keeps faiss' own switch: below
// distance_compute_blas_threshold = 20 queries the reference sums exact differences, from 20 up it uses
// ||x||^2 + ||y||^2 - 2xy like the GEMM kernels do (which cancels badly for far-from-origin data), so L2 batches move to
// the tensor cores at 20.  Very large k stays on the scan path, whose lists are warp-cooperative.
static int resolved_path(const b200_corpus *c, int64_t nq, int k) {
    if (c->path != 0) return c->path;
    if (c->dtype == B200_DTYPE_BIN) {
        // The tensor-core path loads rows with TMA (16-byte row stride) and keeps AND counts and keys exact in fp32 (< 2^24 bits).
        const bool tc_rows = c->row_bytes % 16 == 0, tc_exact = c->d < (1 << 24);
        return (tc_rows && tc_exact && nq >= ceil_div(kBinaryTensorMinQB2, c->row_bytes * c->row_bytes)) ? 2 : 1;
    }
    const int64_t min_nq = c->metric == B200_METRIC_L2 ? 20 : (c->dtype == B200_DTYPE_BF16 ? 2 : 5);
    return (nq >= min_nq && k <= (c->dtype == B200_DTYPE_BF16 ? 1024 : 256)) ? 2 : 1;
}

// The rows a search scores: the corpus itself, or the compact copy of the rows a filter keeps (search_gathered).
struct RowsView {
    const void *data;
    int64_t n;
    const float *row_scale, *row_bias;
};
static RowsView full_rows(const b200_corpus *c) { return {c->data, c->n, c->row_scale.as<float>(), c->row_bias.as<float>()}; }

// ------------------------------------------------------------------------------------
// search core: everything on device, asynchronous on `s`
// d_queries: raw device fp32 [nq][d] (or bytes [nq][d/8] for binary corpora); rows: what is scored (r.n rows of the
// corpus' dtype and layout); ids are row indices of r plus id_offset
// ------------------------------------------------------------------------------------
static int search_core(b200_corpus *c, const RowsView &r, const void *d_queries, int64_t nq, int k, const uint8_t *d_alive,
                       int64_t id_offset, int ip_min_quirk, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    if (k <= 0) return fail(B200_ERR_INVALID, "k must be positive");
    if (nq == 0) return B200_OK;
    if (r.n >= (int64_t)0xffffffffll) return fail(B200_ERR_UNSUPPORTED, "corpus shards are limited to 2^32 - 1 rows");
    const int sms = c->sms;
    c->last_rows_scored = t_last_rows_scored = r.n;

    if (c->dtype == B200_DTYPE_BIN) {
        if (k > 1024) return fail(B200_ERR_UNSUPPORTED, "k > 1024 not supported on the binary scan path");
        const bool tc_rows = c->row_bytes % 16 == 0, tc_exact = c->d < (1 << 24);
        int path = resolved_path(c, nq, k);
        if (path == 2 && !tc_rows)
            return fail(B200_ERR_UNSUPPORTED, "binary tensor-core path needs rows of a multiple of 16 bytes (d % 128 == 0 bits); "
                                              "this corpus has " + std::to_string(c->row_bytes) + "-byte rows");
        if (path == 2 && !tc_exact) return fail(B200_ERR_UNSUPPORTED, "binary tensor-core path needs d < 2^24 bits");
        if (r.n == 0) path = 1;
        const bool jaccard = c->metric == B200_METRIC_JACCARD;
        if (path == 1) {
            int blocks_x = (int)std::min<int64_t>(std::max<int64_t>(1, ceil_div(r.n, 256)), std::max<int64_t>(1, (2 * sms) / std::max<int64_t>(1, std::min<int64_t>(nq, 2 * sms))));
            B200_TRY(c->w_pk.reserve((size_t)nq * blocks_x * k * 4));
            B200_TRY(c->w_pi.reserve((size_t)nq * blocks_x * k * 4));
            BinaryScanParams bp{};
            bp.corpus = reinterpret_cast<const uint8_t *>(r.data);
            bp.queries = reinterpret_cast<const uint8_t *>(d_queries);
            bp.alive = d_alive;
            bp.part_keys = c->w_pk.as<float>();
            bp.part_ids = c->w_pi.as<uint32_t>();
            bp.n = r.n;
            bp.nq = nq;
            bp.nbytes = c->d_pad;
            bp.k = k;
            bp.jaccard = jaccard;
            std::pair<cudaEvent_t, cudaEvent_t> ev;
            timing_begin(c, s, ev);
            B200_CUDA_OK(launch_binary_scan(bp, blocks_x, s));
            timing_end(c, s, ev);
            c->last_kernel = B200_KERNEL_SCAN; c->last_cg = 0; c->last_mc = 0; c->last_grid = blocks_x;
            MergeParams mp{};
            mp.in_keys = bp.part_keys;
            mp.in_ids = bp.part_ids;
            mp.list_stride = k;
            mp.q_stride = (int64_t)blocks_x * k;
            mp.n_lists = blocks_x;
            mp.k_in = k;
            mp.k = k;
            mp.nq = nq;
            mp.out_mode = kOutKey;
            mp.id_offset = id_offset;
            mp.out_dis = d_out_dis;
            mp.out_ids = d_out_ids;
            B200_CUDA_OK(launch_topk_merge(mp, false, s));
            return B200_OK;
        }
        // ---- path 2: wgmma .b1 AND + popcount with fused top-k, <= 1024 queries per launch.  Hamming ranks popc(y) - 2 and
        // (popc(q) is added at the merge), Jaccard is keyed in the kernel; both exactly as binary_scan_kernel keys them.
        const int64_t QCHUNK = 1024;
        for (int64_t qb = 0; qb < nq; qb += QCHUNK) {
            const int64_t nq_c = std::min(QCHUNK, nq - qb);
            const int64_t nq_pad = round_up(nq_c, 128);
            // queries zero-padded to whole 128-query tiles, 16-byte aligned for TMA
            B200_TRY(c->w_qbf.reserve((size_t)nq_pad * c->row_bytes));
            B200_CUDA_OK(cudaMemsetAsync(c->w_qbf.p, 0, (size_t)nq_pad * c->row_bytes, s));
            B200_CUDA_OK(cudaMemcpyAsync(c->w_qbf.p, reinterpret_cast<const uint8_t *>(d_queries) + qb * c->row_bytes,
                                         (size_t)nq_c * c->row_bytes, cudaMemcpyDeviceToDevice, s));
            B200_TRY(c->w_qnorm.reserve((size_t)nq_pad * 4));
            B200_CUDA_OK(launch_popc_rows(c->w_qbf.as<uint8_t>(), c->row_bytes, nq_c, c->w_qnorm.as<float>(), s));
            GemmTopkParams gp{};
            gp.corpus_bf16 = r.data;
            gp.queries_bf16 = c->w_qbf.p;
            gp.row_bias = r.row_bias;
            gp.n = r.n;
            gp.scale_const = jaccard ? 1.f : -2.f;
            gp.alive = d_alive;
            gp.q_popc = jaccard ? c->w_qnorm.as<float>() : nullptr;
            gp.jaccard = jaccard;
            gp.d_pad = (int)c->row_bytes;
            B200_TRY(gemm_chunk(c, gp, nq_c, k, B200_KERNEL_GEMM_B1, jaccard ? kOutKey : kOutAddQ, jaccard ? nullptr : c->w_qnorm.as<float>(),
                                0, id_offset, d_out_dis + qb * k, d_out_ids + qb * k, s));
        }
        return B200_OK;
    }

    int path = resolved_path(c, nq, k);
    if (r.n == 0) path = 1;  // nothing to tile: the scan kernel exits at once and the merge emits the empty result
    // refuse out-of-limit requests before anything is launched
    if (path == 1 && k > 2048) return fail(B200_ERR_UNSUPPORTED, "k > 2048 not supported on the scan path");
    if (path == 2 && k > 1024) return fail(B200_ERR_UNSUPPORTED, "k > 1024 not supported on the GEMM path");
    // ---- stage queries: pad to d_pad fp32, cosine -> normalise (VIWithDataPart.h:354-360)
    B200_TRY(c->w_q32.reserve((size_t)nq * c->d_pad * 4));
    float *q32 = c->w_q32.as<float>();
    B200_CUDA_OK(launch_pad_rows_f32(reinterpret_cast<const float *>(d_queries), c->d, q32, c->d_pad, nq, s));
    // scan path: queries normalised in fp32 like the reference.  GEMM path: the bf16 operand
    // keeps the caller's values (normalising first would add a bf16 rounding of the unit
    // vector); the positive per-query factor 1/||q|| is applied when the result is emitted.
    if (c->metric == B200_METRIC_COSINE && path == 1) B200_CUDA_OK(launch_normalize_rows_f32(q32, c->d_pad, nq, s));

    const int out_mode_scan = c->metric == B200_METRIC_L2 ? kOutKey : c->metric == B200_METRIC_IP ? kOutNeg : kOutOnePlus;

    if (path == 1) {
        int qt = nq == 1 ? 1 : nq <= 4 ? 4 : 8;
        while (qt > 1 && scan_smem_bytes(qt, c->d_pad, k) > 100 * 1024) qt = qt == 8 ? 4 : 1;
        if (scan_smem_bytes(qt, c->d_pad, k) > 200 * 1024)
            return fail(B200_ERR_UNSUPPORTED, "d * 4 + 64 * k exceeds the shared-memory budget of the scan kernel");
        const int elems = c->dtype == B200_DTYPE_BF16 ? 8 : 4;
        const int chunks = c->d_pad / elems;
        int group = 1;
        while (group < 32 && group < chunks) group <<= 1;
        const int64_t y_tiles = ceil_div(nq, qt);
        const int64_t rows_per_block_step = 8 * (32 / group);
        int64_t bx = std::max<int64_t>(1, (2 * sms) / std::min<int64_t>(y_tiles, 2 * sms));
        bx = std::min<int64_t>(bx, std::max<int64_t>(1, ceil_div(r.n, rows_per_block_step)));
        const int blocks_x = (int)bx;
        B200_TRY(c->w_pk.reserve((size_t)nq * blocks_x * k * 4));
        B200_TRY(c->w_pi.reserve((size_t)nq * blocks_x * k * 4));
        ScanParams sp{};
        sp.corpus = r.data;
        sp.queries = q32;
        sp.row_scale = c->metric == B200_METRIC_COSINE ? r.row_scale : nullptr;
        sp.alive = d_alive;
        sp.part_keys = c->w_pk.as<float>();
        sp.part_ids = c->w_pi.as<uint32_t>();
        sp.n = r.n;
        sp.nq = nq;
        sp.row_bytes = c->row_bytes;
        sp.d_pad = c->d_pad;
        sp.k = k;
        sp.group = group;
        sp.l2 = c->metric == B200_METRIC_L2;
        sp.bf16 = c->dtype == B200_DTYPE_BF16;
        std::pair<cudaEvent_t, cudaEvent_t> ev;
        timing_begin(c, s, ev);
        B200_CUDA_OK(launch_flat_scan(sp, qt, blocks_x, s));
        timing_end(c, s, ev);
        c->last_kernel = B200_KERNEL_SCAN; c->last_cg = 0; c->last_mc = 0; c->last_grid = blocks_x;
        MergeParams mp{};
        mp.in_keys = sp.part_keys;
        mp.in_ids = sp.part_ids;
        mp.list_stride = k;
        mp.q_stride = (int64_t)blocks_x * k;
        mp.n_lists = blocks_x;
        mp.k_in = k;
        mp.k = k;
        mp.nq = nq;
        mp.out_mode = out_mode_scan;
        mp.ip_min_quirk = ip_min_quirk && c->metric == B200_METRIC_IP;
        mp.id_offset = id_offset;
        mp.out_dis = d_out_dis;
        mp.out_ids = d_out_ids;
        B200_CUDA_OK(launch_topk_merge(mp, false, s));
        return B200_OK;
    }

    // ---- path 2: wgmma GEMM with fused top-k, <= 1024 queries (8 query tiles) per launch
    const int64_t QCHUNK = 1024;
    for (int64_t qb = 0; qb < nq; qb += QCHUNK) {
        const int64_t nq_c = std::min(QCHUNK, nq - qb);
        const bool f32 = c->dtype == B200_DTYPE_F32;
        const int nq_pad = (int)round_up(nq_c, 128);
        if (f32) {
            // fp32 rows: queries split once per batch into TF32 hi / lo planes (ip_gemm_sm90.cu)
            B200_TRY(c->w_qbf.reserve((size_t)nq_pad * c->d_pad * 4));
            B200_TRY(c->w_qlo.reserve((size_t)nq_pad * c->d_pad * 4));
            B200_CUDA_OK(launch_split_tf32(q32 + qb * c->d_pad, nq_c, c->d_pad, c->w_qbf.as<float>(), c->w_qlo.as<float>(), nq_pad, s));
        } else {
            B200_TRY(c->w_qbf.reserve((size_t)nq_pad * c->d_pad * 2));
            B200_CUDA_OK(cudaMemsetAsync(c->w_qbf.p, 0, (size_t)nq_pad * c->d_pad * 2, s));
            B200_CUDA_OK(launch_f32_to_bf16_rows(q32 + qb * c->d_pad, c->d_pad, c->w_qbf.p, c->d_pad, nq_c, s));
        }
        const float *q_add = nullptr;
        if (c->metric == B200_METRIC_L2 || c->metric == B200_METRIC_COSINE) {
            // L2: ||q||^2 of the operand the MMA sees (bf16-rounded / fp32); cosine: -(1/||q||) (mode 1 stores the negative)
            B200_TRY(c->w_qnorm.reserve((size_t)nq_pad * 4));
            if (f32)
                B200_CUDA_OK(launch_row_norms(q32 + qb * c->d_pad, 0, c->d_pad, nq_c, c->metric == B200_METRIC_L2 ? 0 : 1,
                                              c->w_qnorm.as<float>(), s));
            else
                B200_CUDA_OK(launch_row_norms(c->w_qbf.p, 1, c->d_pad, nq_c, c->metric == B200_METRIC_L2 ? 0 : 1,
                                              c->w_qnorm.as<float>(), s));
            q_add = c->w_qnorm.as<float>();
        }
        GemmTopkParams gp{};
        gp.corpus_bf16 = r.data;
        gp.queries_bf16 = c->w_qbf.p;
        gp.queries_lo = f32 ? c->w_qlo.p : nullptr;
        gp.row_scale = c->metric == B200_METRIC_COSINE ? r.row_scale : nullptr;
        gp.scale_const = c->metric == B200_METRIC_L2 ? -2.f : -1.f;
        gp.row_bias = c->metric == B200_METRIC_L2 ? r.row_bias : nullptr;
        gp.n = r.n;
        gp.alive = d_alive;
        gp.d_pad = c->d_pad;
        const int out_mode = c->metric == B200_METRIC_L2 ? kOutAddQ : c->metric == B200_METRIC_IP ? kOutNeg : kOutCosQ;
        B200_TRY(gemm_chunk(c, gp, nq_c, k, f32 ? B200_KERNEL_GEMM_TF32X3 : B200_KERNEL_GEMM_BF16, out_mode, q_add,
                            ip_min_quirk && c->metric == B200_METRIC_IP, id_offset, d_out_dis + qb * k, d_out_ids + qb * k, s));
        // L2: the winners' distances from the direct difference form (the expanded form above only RANKS; it cancels for
        // data far from the origin).  The query operand is what the caller passed (fp32), the rows what is stored.
        if (c->metric == B200_METRIC_L2 && k <= 1024 && c->rescore_l2)
            B200_CUDA_OK(launch_rescore_l2(r.data, c->dtype == B200_DTYPE_BF16, c->row_bytes, c->d_pad, q32 + qb * c->d_pad, nq_c, id_offset, k,
                                           d_out_dis + qb * k, d_out_ids + qb * k, s));
    }
    return B200_OK;
}

extern "C" int b200_corpus_search_device(b200_corpus *c, const float *d_queries, int64_t nq, int k,
                                         const uint8_t *d_alive_bits, int64_t id_offset, float *d_out_dis,
                                         int64_t *d_out_ids, void *stream) {
    if (!c || (!d_queries && nq > 0) || !d_out_dis || !d_out_ids || nq < 0)
        return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? reinterpret_cast<cudaStream_t>(stream) : c->stream;
    B200_TRY(search_core(c, full_rows(c), d_queries, nq, k, d_alive_bits, id_offset, 0, d_out_dis, d_out_ids, s));
    if (!stream) B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// ------------------------------------------------------------------------------------
// Pre-filtered exact search (prefilter.cu).  When the host holds the filter bitmap, its set bits are counted first; a
// filter that keeps few enough rows has them compacted and copied to the corpus' scratch, the unchanged kernels score that
// compact corpus, and the ids are mapped back.  The answer is the full scan's, byte for byte; only the rows read change.
// ------------------------------------------------------------------------------------
// Measured with tools/bench_aux.py prefilter on an H100 80GB HBM3 at a 400 W power limit, 2026-10-16 (k = 10, call time of
// the gathered path against the full masked scan of the same search; DESIGN.md section 7).
// Auto takes the gathered path when the filter keeps at most this share of the rows.  Scan path (float rows, nq = 1): 2.5x
// faster at a 5 % share on 10 M x 768 bf16 rows and 1.6 - 1.7x on 2 M x 768 fp32 rows; 1.0 - 1.1x at 10 % (fp32; the bf16
// copy is over the budget there).  The crossover lies above 5 %; auto stops there.
constexpr double kPrefilterMaxShareScan = 0.05;
// Tensor-core path (bf16, 3xTF32 and b1 kernels): faster at every measured share that fits the budget below (2.3x for
// 10 M x 1024-bit rows at nq = 16 and 10 %, 7.5 - 7.6x for 2 M x 768 fp32 at nq = 1024 and 10 %), so the budget decides.
constexpr double kPrefilterMaxShareTensor = 0.125;
// The binary scan kernel tests the alive bit before it loads a row, so its full scan already reads little of a sparse
// filter's corpus: the gathered path was 0.65 - 0.95x as fast at 11 of the 12 measured points (10 M x 1024 bits, nq = 1;
// 1.16x at one).  Auto leaves that path alone.
// Corpora below this many row bytes are not pre-filtered by auto: at 768-d fp32 and nq = 1 the gathered path was 0.6 - 0.7x as
// fast at 65 536 rows (201 MB) and 1.1 - 1.3x faster at 262 144 rows (805 MB) for 0.1 - 1 % shares; the limit lies between.
constexpr int64_t kPrefilterMinCorpusBytes = 512ll << 20;
// Every mode takes the gathered path only when the compact copy fits the scratch budget: 1/8 of the corpus' row bytes and
// at most 1 GiB.  The budget bounds the extra HBM, and with it the compact rows always go through search_core in one piece.
constexpr int64_t kPrefilterMaxBytes = 1ll << 30;

// The largest number of kept rows for which a search of nq queries at this k takes the gathered path; -1 = never.
static int64_t prefilter_limit(const b200_corpus *c, int mode, int64_t nq, int k) {
    if (mode == 1 || c->n == 0) return -1;
    int64_t lim = std::min<int64_t>(c->n / 8, kPrefilterMaxBytes / c->row_bytes);
    if (mode == 0) {
        const int path = resolved_path(c, nq, k);
        if (c->n * c->row_bytes < kPrefilterMinCorpusBytes || (path != 2 && c->dtype == B200_DTYPE_BIN)) return -1;
        const double share = path == 2 ? kPrefilterMaxShareTensor : kPrefilterMaxShareScan;
        lim = std::min<int64_t>(lim, (int64_t)((double)c->n * share));
    }
    return lim;
}

// Set bits among the first n of an LSB-first host bitmap (bits past n in the last byte are ignored).  Stops once the
// count passes `limit`, so a dense filter costs a few cache lines; the result is then some value > limit.
template <typename Popc>
static inline __attribute__((always_inline)) int64_t count_alive_with(const uint8_t *bits, int64_t n, int64_t limit, Popc popc) {
    const int64_t full = n / 8;
    int64_t cnt = 0, b = 0;
    for (; b + 64 <= full; b += 64) {
        for (int j = 0; j < 64; j += 8) {
            uint64_t w;
            memcpy(&w, bits + b + j, 8);
            cnt += popc(w);
        }
        if (cnt > limit) return cnt;
    }
    for (; b < full; b++) cnt += popc(bits[b]);
    if (n % 8) cnt += popc(bits[full] & ((1u << (n % 8)) - 1u));
    return cnt;
}
#if defined(__x86_64__)
// The default x86-64 target has no POPCNT instruction (__builtin_popcountll becomes a library call, several times slower
// on a 10 M-bit bitmap); this copy uses it on the CPUs that have it.
__attribute__((target("popcnt"))) static int64_t count_alive_popcnt(const uint8_t *bits, int64_t n, int64_t limit) {
    return count_alive_with(bits, n, limit, [](uint64_t w) { return (int64_t)__builtin_popcountll(w); });
}
#endif
static int64_t count_alive(const uint8_t *bits, int64_t n, int64_t limit) {
#if defined(__x86_64__)
    if (__builtin_cpu_supports("popcnt")) return count_alive_popcnt(bits, n, limit);
#endif
    return count_alive_with(bits, n, limit, [](uint64_t w) { return (int64_t)__builtin_popcountll(w); });
}

// Scores the `alive` rows the device bitmap keeps (counted on the host) through a compact copy, then maps the ids back to
// row ids + id_offset.  Asynchronous on s.  The kernels index the compact rows until the map-back, which runs last (after
// the L2 re-score, which reads the winners' rows by id).
static int search_gathered(b200_corpus *c, const void *d_queries, int64_t nq, int k, const uint8_t *d_alive, int64_t alive,
                           int64_t id_offset, int ip_min_quirk, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    B200_TRY(c->w_pf_ids.reserve((size_t)alive * 4 + 16));
    B200_TRY(c->w_pf_tmp.reserve(prefilter_compact_temp_bytes(c->n)));
    B200_CUDA_OK(launch_prefilter_compact(d_alive, c->n, c->w_pf_ids.as<uint32_t>(), c->w_pf_tmp.p, s));
    // same layout as the corpus: d_pad rows, 256-byte aligned base (TMA wants 16), a row of slack behind the last row
    B200_TRY(c->w_pf_rows.reserve((size_t)(alive + 1) * c->row_bytes + 256));
    const int64_t side_stride = round_up(alive + 1, 64);
    B200_TRY(c->w_pf_side.reserve((size_t)side_stride * 2 * 4));
    // only the side arrays search_core reads for this metric: a re-dimensioned per-thread scratch corpus may still hold
    // arrays of another metric, sized for an earlier, smaller part
    const float *scale = c->metric == B200_METRIC_COSINE ? c->row_scale.as<float>() : nullptr;
    const float *bias = c->metric == B200_METRIC_L2 || c->dtype == B200_DTYPE_BIN ? c->row_bias.as<float>() : nullptr;
    float *cscale = scale ? c->w_pf_side.as<float>() : nullptr, *cbias = bias ? c->w_pf_side.as<float>() + side_stride : nullptr;
    B200_CUDA_OK(launch_prefilter_gather(c->data, c->row_bytes, scale, bias, c->w_pf_ids.as<uint32_t>(), alive, c->w_pf_rows.p,
                                         cscale, cbias, s));
    const RowsView r{c->w_pf_rows.p, alive, cscale, cbias};
    B200_TRY(search_core(c, r, d_queries, nq, k, nullptr, 0, ip_min_quirk, d_out_dis, d_out_ids, s));
    B200_CUDA_OK(launch_prefilter_map_ids(c->w_pf_ids.as<uint32_t>(), id_offset, d_out_ids, nq * k, s));
    return B200_OK;
}

namespace b200 {
// Exact search of a resident corpus for the index layer (FLAT, BINARYFLAT, the small-part fallback, exact_batch=1): as
// b200_corpus_search_device on the stream s, plus the host copy of the bitmap (nullable) and a prefilter mode, so that the
// gathered path can be chosen.
int corpus_search_exact(b200_corpus *c, const void *d_queries, int64_t nq, int k, const uint8_t *d_alive, const uint8_t *h_alive,
                        int prefilter_mode, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    const int64_t limit = h_alive && d_alive ? prefilter_limit(c, prefilter_mode, nq, k) : -1;
    const int64_t alive = limit >= 0 ? count_alive(h_alive, c->n, limit) : -1;
    if (alive >= 0 && alive <= limit) return search_gathered(c, d_queries, nq, k, d_alive, alive, id_offset, 0, d_out_dis, d_out_ids, s);
    return search_core(c, full_rows(c), d_queries, nq, k, d_alive, id_offset, 0, d_out_dis, d_out_ids, s);
}

// the host count above, for the index layer's filter_probe rule (stops past limit, as count_alive does)
int64_t host_count_alive(const uint8_t *bits, int64_t n, int64_t limit) { return count_alive(bits, n, limit); }
// the most kept rows for which corpus_search_exact takes the gathered path (-1: never), for the same filter_probe rule
int64_t corpus_prefilter_limit(const b200_corpus *c, int mode, int64_t nq, int k) { return prefilter_limit(c, mode, nq, k); }
}  // namespace b200

extern "C" int b200_corpus_set_prefilter(b200_corpus *c, int mode) {
    if (!c || mode < 0 || mode > 2) return fail(B200_ERR_INVALID, "prefilter mode must be 0 (auto), 1 (never) or 2 (always)");
    std::lock_guard<std::mutex> lk(c->mu);
    c->prefilter = mode;
    return B200_OK;
}

extern "C" int b200_corpus_last_rows_scored(b200_corpus *c, int64_t *rows) {
    if (!c || !rows) return fail(B200_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(c->mu);
    *rows = c->last_rows_scored;
    return B200_OK;
}

extern "C" int b200_thread_last_rows_scored(int64_t *rows) {
    if (!rows) return fail(B200_ERR_INVALID, "null argument");
    *rows = t_last_rows_scored;
    return B200_OK;
}

// One launch per call for small batches that go to the scan kernel (the reference's usual shape: one query x many parts from a
// ThreadPool, MergeTreeSelectWithHybridSearchProcessor.cpp:1212-1241).  The query is written to mapped pinned memory and
// read by the kernel directly, the last block to finish merges the partial lists and writes the result to mapped pinned
// memory, the host waits on a flag in that memory: no pad / merge launches, no H2D / D2H copies, no stream synchronise
// (the staged form spends most of a resident call on those).
static int search_host_fused(b200_corpus *c, const float *queries, int64_t nq, int k, const uint8_t *alive_bits, int ip_min_quirk,
                             float *out_dis, int64_t *out_ids, bool *done) {
    *done = false;
    if (!c->fused_enabled || c->dtype == B200_DTYPE_BIN || nq > 8 || k > 1024 || c->n == 0) return B200_OK;
    int path = c->path;
    if (path == 0) {
        const int64_t min_nq = c->metric == B200_METRIC_L2 ? 20 : (c->dtype == B200_DTYPE_BF16 ? 2 : 5);
        path = (nq >= min_nq) ? 2 : 1;
    }
    if (path != 1) return B200_OK;
    int qt = nq == 1 ? 1 : nq <= 4 ? 4 : 8;
    while (qt > 1 && scan_smem_bytes(qt, c->d_pad, k) > 100 * 1024) qt = qt == 8 ? 4 : 1;
    if (scan_smem_bytes(qt, c->d_pad, k) > 200 * 1024) return B200_OK;   // the staged path reports the error
    cudaStream_t s = c->stream;
    const size_t need = (size_t)8 * c->d * 4 + (size_t)8 * k * 12 + 64;
    if (need > c->h_pin_bytes) {
        if (c->h_pin) cudaFreeHost(c->h_pin);
        c->h_pin = nullptr;
        c->h_pin_bytes = 0;
        if (cudaHostAlloc(&c->h_pin, need, cudaHostAllocMapped) != cudaSuccess) {
            cudaGetLastError();
            return B200_OK;   // no pinned memory: the staged path still works
        }
        c->h_pin_bytes = need;
    }
    if (!c->d_tickets || c->d_tickets_d != c->d) {
        B200_TRY(c->d_tickets.alloc(64 + (size_t)8 * c->d * 4));
        B200_CUDA_OK(cudaMemsetAsync(c->d_tickets.p, 0, 64, s));
        c->d_tickets_d = c->d;
    }
    float *d_q = reinterpret_cast<float *>(c->d_tickets.as<char>() + 64);
    char *hp = reinterpret_cast<char *>(c->h_pin);
    float *h_q = reinterpret_cast<float *>(hp);
    float *h_dis = reinterpret_cast<float *>(hp + (size_t)8 * c->d * 4);
    int64_t *h_ids = reinterpret_cast<int64_t *>(hp + (size_t)8 * c->d * 4 + (size_t)round_up(8 * k * 4, 8));
    volatile unsigned int *h_flag = reinterpret_cast<volatile unsigned int *>(hp + need - 16);
    void *dp = nullptr;
    B200_CUDA_OK(cudaHostGetDevicePointer(&dp, c->h_pin, 0));
    char *dpc = reinterpret_cast<char *>(dp);
    // the query goes pinned -> device with one small async copy (reading it from the kernel over PCIe, 4 bytes per thread and
    // block, would cost most of the kernel); the RESULT is written to mapped host memory by one block
    const bool q_inline = nq * c->d <= 256;   // small queries ride in the kernel parameters: no copy at all
    if (!q_inline) {
        memcpy(h_q, queries, (size_t)nq * c->d * 4);
        B200_CUDA_OK(cudaMemcpyAsync(d_q, h_q, (size_t)nq * c->d * 4, cudaMemcpyHostToDevice, s));
    }
    const uint8_t *d_alive = nullptr;
    if (alive_bits) {
        const size_t ab = (size_t)ceil_div(c->n, 8);
        B200_TRY(c->w_alive.reserve(ab + 16));
        B200_CUDA_OK(cudaMemcpyAsync(c->w_alive.p, alive_bits, ab, cudaMemcpyHostToDevice, s));
        d_alive = c->w_alive.as<uint8_t>();
    }
    const int elems = c->dtype == B200_DTYPE_BF16 ? 8 : 4;
    const int chunks = c->d_pad / elems;
    int group = 1;
    while (group < 32 && group < chunks) group <<= 1;
    const int64_t y_tiles = ceil_div(nq, qt);
    const int64_t rows_per_block_step = 8 * (32 / group);
    int64_t bx = std::max<int64_t>(1, (2 * c->sms) / std::min<int64_t>(y_tiles, 2 * c->sms));
    bx = std::min<int64_t>(bx, std::max<int64_t>(1, ceil_div(c->n, rows_per_block_step)));
    const int blocks_x = (int)bx;
    B200_TRY(c->w_pk.reserve((size_t)nq * blocks_x * k * 4));
    B200_TRY(c->w_pi.reserve((size_t)nq * blocks_x * k * 4));
    ScanParams sp{};
    sp.corpus = c->data;
    sp.queries = d_q;
    sp.row_scale = c->metric == B200_METRIC_COSINE ? c->row_scale.as<float>() : nullptr;
    sp.alive = d_alive;
    sp.part_keys = c->w_pk.as<float>();
    sp.part_ids = c->w_pi.as<uint32_t>();
    sp.n = c->n;
    sp.nq = nq;
    sp.row_bytes = c->row_bytes;
    sp.d_pad = c->d_pad;
    sp.k = k;
    sp.group = group;
    sp.l2 = c->metric == B200_METRIC_L2;
    sp.bf16 = c->dtype == B200_DTYPE_BF16;
    sp.fused = 1;
    sp.q_dim = c->d;
    sp.cosine = c->metric == B200_METRIC_COSINE;
    sp.out_mode = c->metric == B200_METRIC_L2 ? kOutKey : c->metric == B200_METRIC_IP ? kOutNeg : kOutOnePlus;
    sp.ip_min_quirk = ip_min_quirk && c->metric == B200_METRIC_IP;
    sp.id_offset = 0;
    sp.tickets = c->d_tickets.as<unsigned int>();
    sp.tiles_done = c->d_tickets.as<unsigned int>() + 8;
    sp.out_dis = reinterpret_cast<float *>(dpc + (reinterpret_cast<char *>(h_dis) - hp));
    sp.out_ids = reinterpret_cast<int64_t *>(dpc + (reinterpret_cast<char *>(h_ids) - hp));
    sp.done_flag = reinterpret_cast<volatile unsigned int *>(dpc + need - 16);
    sp.done_value = ++c->fused_seq ? c->fused_seq : ++c->fused_seq;   // never 0
    sp.q_inline = q_inline ? 1 : 0;
    if (q_inline) memcpy(sp.qinline, queries, (size_t)nq * c->d * 4);
    *h_flag = 0;
    std::pair<cudaEvent_t, cudaEvent_t> ev;
    timing_begin(c, s, ev);
    B200_CUDA_OK(launch_flat_scan(sp, qt, blocks_x, s));
    timing_end(c, s, ev);
    c->last_kernel = B200_KERNEL_SCAN; c->last_cg = 0; c->last_mc = 0; c->last_grid = blocks_x;
    c->last_rows_scored = t_last_rows_scored = c->n;
    // wait for the flag; look at the stream now and then so that a failed launch cannot hang the caller
    for (uint64_t spin = 1;; spin++) {
        if (*h_flag == sp.done_value) break;
        if ((spin & 0x3fff) == 0) {
            const cudaError_t qe = cudaStreamQuery(s);
            if (qe == cudaSuccess) {
                if (*h_flag == sp.done_value) break;
                return fail(B200_ERR_CUDA, "fused scan finished without publishing its result");
            }
            if (qe != cudaErrorNotReady) return fail(B200_ERR_CUDA, std::string("fused scan: ") + cudaGetErrorString(qe));
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    memcpy(out_dis, h_dis, (size_t)nq * k * 4);
    memcpy(out_ids, h_ids, (size_t)nq * k * 8);
    *done = true;
    return B200_OK;
}

static int search_host(b200_corpus *c, const void *queries, int64_t nq, int k, const uint8_t *alive_bits, int ip_min_quirk,
                       float *out_dis, int64_t *out_ids) {
    if (!c || (!queries && nq > 0) || !out_dis || !out_ids || nq < 0 || k <= 0)
        return fail(B200_ERR_INVALID, "bad arguments");
    if (nq == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    B200_CUDA_OK(cudaSetDevice(c->device));
    // a selective filter: score only the rows it keeps (the count is taken before the fused path is considered)
    const int64_t limit = alive_bits ? prefilter_limit(c, c->prefilter, nq, k) : -1;
    const int64_t alive = limit >= 0 ? count_alive(alive_bits, c->n, limit) : -1;
    const bool gathered = alive >= 0 && alive <= limit;
    if (!gathered) {
        bool done = false;
        B200_TRY(search_host_fused(c, reinterpret_cast<const float *>(queries), nq, k, alive_bits, ip_min_quirk, out_dis, out_ids, &done));
        if (done) return B200_OK;
    }
    cudaStream_t s = c->stream;
    const size_t q_bytes = c->dtype == B200_DTYPE_BIN ? (size_t)nq * c->d_pad : (size_t)nq * c->d * 4;
    B200_TRY(c->w_stage.reserve(q_bytes));
    B200_TRY(c->w_odis.reserve((size_t)nq * k * 4));
    B200_TRY(c->w_oids.reserve((size_t)nq * k * 8));
    B200_CUDA_OK(cudaMemcpyAsync(c->w_stage.p, queries, q_bytes, cudaMemcpyHostToDevice, s));
    const uint8_t *d_alive = nullptr;
    if (alive_bits) {
        const size_t ab = (size_t)ceil_div(c->n, 8);
        B200_TRY(c->w_alive.reserve(ab + 16));
        B200_CUDA_OK(cudaMemcpyAsync(c->w_alive.p, alive_bits, ab, cudaMemcpyHostToDevice, s));
        d_alive = c->w_alive.as<uint8_t>();
    }
    if (gathered)
        B200_TRY(search_gathered(c, c->w_stage.p, nq, k, d_alive, alive, 0, ip_min_quirk, c->w_odis.as<float>(), c->w_oids.as<int64_t>(), s));
    else
        B200_TRY(search_core(c, full_rows(c), c->w_stage.p, nq, k, d_alive, 0, ip_min_quirk, c->w_odis.as<float>(), c->w_oids.as<int64_t>(), s));
    B200_CUDA_OK(cudaMemcpyAsync(out_dis, c->w_odis.p, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_ids, c->w_oids.p, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

extern "C" int b200_corpus_search(b200_corpus *c, const float *queries, int64_t nq, int k, const uint8_t *alive_bits,
                                  float *out_dis, int64_t *out_ids) {
    return search_host(c, queries, nq, k, alive_bits, 0, out_dis, out_ids);
}

// The host-buffer entry points (b200_flat_knn / b200_binary_knn / b200_part_scan) are called once per part or per
// mark by each ClickHouse worker thread: they reuse one scratch corpus per thread (device buffers, stream and
// workspaces grow-only) instead of paying cudaMalloc / cudaStreamCreate on every call.
static thread_local CorpusPtr t_scratch;

// gives this thread's scratch corpus (device buffers sized for the largest part it has scanned) back to the driver
extern "C" int b200_thread_release(void) {
    t_scratch.reset();
    return B200_OK;
}

static int scratch_corpus(int metric, int dtype, int d, int64_t rows, b200_corpus **out) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (t_scratch && (t_scratch->device != dev || (t_scratch->data && !t_scratch->owned_rows))) t_scratch.reset();
    b200_corpus *c = t_scratch.get();
    if (!c) {
        B200_TRY(b200_corpus_create(metric, dtype, d, rows, &c));
        t_scratch.reset(c);
        *out = c;
        return B200_OK;
    }
    // re-dimension in place; corpus_alloc() keeps the device buffers whenever they are large enough
    c->metric = metric;
    c->dtype = dtype;
    c->d = d;
    c->d_pad = pad_for(dtype, d);
    c->row_bytes = dtype == B200_DTYPE_BIN ? c->d_pad : (int64_t)c->d_pad * (dtype == B200_DTYPE_BF16 ? 2 : 4);
    c->n = 0;
    c->cap = 0;
    c->path = 0;
    c->epoch++;
    (void)rows;
    *out = c;
    return B200_OK;
}

static void fill_empty(int metric, int64_t n, float *dis, int64_t *ids, int quirk) {
    for (int64_t i = 0; i < n; i++) {
        ids[i] = -1;
        dis[i] = quirk ? FLT_MIN : (metric == B200_METRIC_IP ? -FLT_MAX : FLT_MAX);
    }
}

extern "C" int b200_flat_knn(int metric, const float *x, int64_t nx, const float *y, int64_t ny, int d, int k,
                             const uint8_t *alive_bits, float *out_dis, int64_t *out_ids) {
    if (!is_float_metric(metric)) return fail(B200_ERR_INVALID, "b200_flat_knn: metric must be L2, IP or COSINE");
    if (nx < 0 || ny < 0 || d <= 0 || k <= 0 || !out_dis || !out_ids) return fail(B200_ERR_INVALID, "bad arguments");
    B200_TRY(ensure_device());
    if (nx == 0) return B200_OK;
    if (ny == 0) {
        fill_empty(metric, nx * k, out_dis, out_ids, 0);
        return B200_OK;
    }
    b200_corpus *c = nullptr;
    B200_TRY(scratch_corpus(metric, B200_DTYPE_F32, d, ny, &c));
    int rc = b200_corpus_append(c, y, ny);
    if (rc == B200_OK) rc = search_host(c, x, nx, k, alive_bits, 0, out_dis, out_ids);
    return rc;
}

extern "C" int b200_binary_knn(int metric, const uint8_t *x, int64_t nx, const uint8_t *y, int64_t ny, int nbytes, int k,
                               const uint8_t *alive_bits, float *out_dis, int64_t *out_ids) {
    if (!is_bin_metric(metric)) return fail(B200_ERR_INVALID, "b200_binary_knn: metric must be HAMMING or JACCARD");
    if (nx < 0 || ny < 0 || nbytes <= 0 || k <= 0 || !out_dis || !out_ids) return fail(B200_ERR_INVALID, "bad arguments");
    B200_TRY(ensure_device());
    if (nx == 0) return B200_OK;
    if (ny == 0) {
        fill_empty(metric, nx * k, out_dis, out_ids, 0);
        return B200_OK;
    }
    b200_corpus *c = nullptr;
    B200_TRY(scratch_corpus(metric, B200_DTYPE_BIN, nbytes * 8, ny, &c));
    int rc = b200_corpus_append(c, y, ny);
    if (rc == B200_OK) rc = search_host(c, x, nx, k, alive_bits, 0, out_dis, out_ids);
    return rc;
}

extern "C" int b200_part_scan(int metric, const void *x, int64_t nx, const void *y, int64_t ny, int d, int k,
                              int64_t block_rows, const uint8_t *row_exists, const uint8_t *filter_bits, float *out_dis,
                              int64_t *out_ids) {
    (void)block_rows;
    if (nx < 0 || ny < 0 || d <= 0 || k <= 0 || !out_dis || !out_ids) return fail(B200_ERR_INVALID, "bad arguments");
    if (!is_float_metric(metric) && !is_bin_metric(metric)) return fail(B200_ERR_INVALID, "unknown metric");
    B200_TRY(ensure_device());
    if (nx == 0) return B200_OK;
    const int quirk = metric == B200_METRIC_IP;
    if (ny == 0) {
        fill_empty(metric, nx * k, out_dis, out_ids, quirk);
        return B200_OK;
    }
    // alive = filter (which already folds the lightweight-delete mask, MergeTreeVSManager.cpp:1040)
    // or, without filter, the _row_exists column
    std::vector<uint8_t> alive;
    const uint8_t *alive_ptr = filter_bits;
    if (!filter_bits && row_exists) {
        alive.assign((size_t)ceil_div(ny, 8), 0);
        for (int64_t i = 0; i < ny; i++)
            if (row_exists[i]) alive[i >> 3] |= (uint8_t)(1u << (i & 7));
        alive_ptr = alive.data();
    }
    b200_corpus *c = nullptr;
    const bool bin = is_bin_metric(metric);
    B200_TRY(scratch_corpus(metric, bin ? B200_DTYPE_BIN : B200_DTYPE_F32, d, ny, &c));
    int rc = b200_corpus_append(c, y, ny);
    if (rc == B200_OK) rc = search_host(c, x, nx, k, alive_ptr, quirk, out_dis, out_ids);
    return rc;
}

extern "C" int b200_topk_merge_device(const float *d_dis, const int64_t *d_ids, int n_lists, int64_t nq, int k,
                                      int descending, float *d_out_dis, int64_t *d_out_ids, void *stream) {
    return b200_topk_merge_device_strided(d_dis, d_ids, n_lists, nq * k, nq * k, nq, k, descending, d_out_dis, d_out_ids,
                                          stream);
}

extern "C" int b200_topk_merge_device_strided(const float *d_dis, const int64_t *d_ids, int n_lists,
                                              int64_t dis_list_stride, int64_t ids_list_stride, int64_t nq, int k,
                                              int descending, float *d_out_dis, int64_t *d_out_ids, void *stream) {
    return b200_topk_merge_device_ex(d_dis, d_ids, n_lists, dis_list_stride, ids_list_stride, nq, k, k, descending, 0, d_out_dis,
                                     d_out_ids, nullptr, stream);
}

extern "C" int b200_topk_merge_device_ex(const float *d_dis, const int64_t *d_ids, int n_lists, int64_t dis_list_stride,
                                         int64_t ids_list_stride, int64_t nq, int k_in, int k, int descending, int tie_mode,
                                         float *d_out_dis, int64_t *d_out_ids, int32_t *d_out_list, void *stream) {
    if (!d_dis || !d_ids || !d_out_dis || !d_out_ids || n_lists <= 0 || nq < 0 || k <= 0 || k_in <= 0 || tie_mode < 0 || tie_mode > 1)
        return fail(B200_ERR_INVALID, "bad arguments");
    if (k > 2048) return fail(B200_ERR_UNSUPPORTED, "k > 2048 not supported by the merge kernel");
    B200_TRY(ensure_device());
    if (nq == 0) return B200_OK;
    MergeParams mp{};
    mp.in_keys = d_dis;
    mp.in_ids = d_ids;
    mp.list_stride = dis_list_stride;
    mp.id_list_stride = ids_list_stride;
    mp.q_stride = k_in;
    mp.n_lists = n_lists;
    mp.k_in = k_in;
    mp.k = k;
    mp.nq = nq;
    mp.descending = descending;
    mp.tie_mode = tie_mode;
    mp.out_list = d_out_list;
    mp.out_dis = d_out_dis;
    mp.out_ids = d_out_ids;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    B200_CUDA_OK(launch_topk_merge(mp, true, s));
    if (!stream) B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}
