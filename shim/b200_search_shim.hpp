// b200_search_shim.hpp -- header-only C++ adapter that presents the names MyScaleDB's src/VectorIndex and
// src/Storages/MergeTree/TantivyIndexStore.cpp call (namespace Search::, faiss::knn_*, jaccard_knn, TANTIVY::ffi_*) with
// the SIGNATURES OF THEIR CALL SITES, and forwards them to the C ABI of libb200search.so (include/b200_search.h).
//
// The originals live in the un-vendored submodules contrib/search-index and rust/supercrate/libs/tantivy_search; the
// surface below is reconstructed from every call site in the reference (SURVEY.md 8b), each member citing the call site
// it serves (paths relative to /root/reference/src).  tests/cpp/callsite_compile.cpp pastes those call expressions and is
// compiled with -Werror against this header, then run on the GPU.
#pragma once
#include <b200_search.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <ios>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <stdexcept>
#include <string>
#include <vector>

// VectorIndex/Common/VICommon.h:86-91
class SearchIndexException : public std::exception {
    int code_;
    std::string msg_;
public:
    SearchIndexException(int code, std::string msg) : code_(code), msg_(std::move(msg)) {}
    int getCode() const { return code_; }
    const char * what() const noexcept override { return msg_.c_str(); }
};

namespace Search {
inline void b200Check(int rc) { if (rc != B200_OK) throw SearchIndexException(rc, b200_last_error()); }

enum class DataType { FloatVector, BinaryVector };                    // VICommon.h:139-143
enum class Metric { L2, IP, Cosine, Hamming, Jaccard };               // MergeTreeVSManager.cpp:1560-1578
// VICommon.h:178-180 + the type names of tests/queries/2_vector_search (MSTG 111x, HNSWFLAT 45x, IVFFLAT 34x, IVFSQ, IVFPQ, FLAT, BINARYFLAT,
// SCANN, HNSWSQ, BINARYMSTG, HNSWPQ)
enum class IndexType { FLAT, IVFFLAT, IVFSQ, IVFPQ, HNSWFLAT, HNSWSQ, HNSWPQ, SCANN, MSTG, BinaryFLAT, BinaryIVF, BinaryHNSW, BinaryMSTG };
using idx_t = int64_t;

inline int toB200(Metric m) {
    switch (m) {
        case Metric::L2: return B200_METRIC_L2;
        case Metric::IP: return B200_METRIC_IP;
        case Metric::Cosine: return B200_METRIC_COSINE;
        case Metric::Hamming: return B200_METRIC_HAMMING;
        default: return B200_METRIC_JACCARD;
    }
}
inline const char * enumToString(IndexType t) {                       // VIInfo.cpp:45, VIMetadata.cpp:125, VIWithDataPart.cpp:487
    switch (t) {
        case IndexType::FLAT: return "FLAT";
        case IndexType::IVFFLAT: return "IVFFLAT";
        case IndexType::IVFSQ: return "IVFSQ";
        case IndexType::IVFPQ: return "IVFPQ";
        case IndexType::HNSWFLAT: return "HNSWFLAT";
        case IndexType::HNSWSQ: return "HNSWSQ";
        case IndexType::HNSWPQ: return "HNSWPQ";
        case IndexType::SCANN: return "SCANN";
        case IndexType::MSTG: return "MSTG";
        case IndexType::BinaryFLAT: return "BinaryFLAT";
        case IndexType::BinaryIVF: return "BinaryIVF";
        case IndexType::BinaryHNSW: return "BinaryHNSW";
        default: return "BinaryMSTG";
    }
}
inline const char * enumToString(Metric m) {                          // VIMetadata.cpp:129
    switch (m) {
        case Metric::L2: return "L2";
        case Metric::IP: return "IP";
        case Metric::Cosine: return "Cosine";
        case Metric::Hamming: return "Hamming";
        default: return "Jaccard";
    }
}
inline std::string upperOf(std::string s) { for (auto & c : s) c = static_cast<char>(toupper(static_cast<unsigned char>(c))); return s; }
inline bool findEnumByName(const std::string & name, IndexType & out) {   // VIMetadata.cpp:35
    const std::string u = upperOf(name);
    for (int i = 0; i <= static_cast<int>(IndexType::BinaryMSTG); ++i)
        if (upperOf(enumToString(static_cast<IndexType>(i))) == u) { out = static_cast<IndexType>(i); return true; }
    return false;
}
inline bool findEnumByName(const std::string & name, Metric & out) {      // VIMetadata.cpp:41
    const std::string u = upperOf(name);
    for (int i = 0; i <= static_cast<int>(Metric::Jaccard); ++i)
        if (upperOf(enumToString(static_cast<Metric>(i))) == u) { out = static_cast<Metric>(i); return true; }
    return false;
}
inline Metric getMetricType(const std::string & s, DataType dt) {         // VIWithDataPart.cpp:397, :507; MergeTreeVSManager.cpp:397
    Metric m;
    if (!findEnumByName(s, m)) throw SearchIndexException(B200_ERR_INVALID, "unknown metric type " + s);
    const bool binary = m == Metric::Hamming || m == Metric::Jaccard;
    if (binary != (dt == DataType::BinaryVector)) throw SearchIndexException(B200_ERR_INVALID, "metric " + s + " does not fit the vector type");
    return m;
}
inline IndexType getVectorIndexType(const std::string & s, DataType dt) { // VIDescriptions.cpp:137, :318; VIWithDataPart.cpp:173
    IndexType t;
    std::string name = upperOf(s);
    if (dt == DataType::BinaryVector && name.rfind("BINARY", 0) != 0) name = "BINARY" + name;
    if (!findEnumByName(name, t)) throw SearchIndexException(B200_ERR_INVALID, "unknown vector index type " + s);
    const bool binary = t >= IndexType::BinaryFLAT;
    if (binary != (dt == DataType::BinaryVector)) throw SearchIndexException(B200_ERR_INVALID, "index type " + s + " does not fit the vector type");
    return t;
}
inline std::string getDefaultIndexType(const DataType & dt) { return dt == DataType::BinaryVector ? "BinaryFLAT" : "SCANN"; }   // VIDescriptions.cpp:133 (README.md:207)
// VIDescriptions.cpp:172, parseVSParameters.cpp:78: JSON of the parameters every index type accepts (name -> type / range)
static const char * const MYSCALE_VALID_INDEX_PARAMETER = R"({
 "FLAT": {}, "BinaryFLAT": {},
 "IVFFLAT": {"ncentroids": {"type": "int", "range": [1, 1048576]}, "nprobe": {"type": "int", "range": [1, 1048576]}},
 "IVFSQ": {"ncentroids": {"type": "int", "range": [1, 1048576]}, "bit_size": {"type": "string", "candidates": ["8bit"]}, "nprobe": {"type": "int", "range": [1, 1048576]}},
 "IVFPQ": {"ncentroids": {"type": "int", "range": [1, 1048576]}, "M": {"type": "int", "range": [1, 4096]}, "bit_size": {"type": "int", "range": [4, 8]}, "aq_threshold": {"type": "float", "range": [0, 1]}, "opq": {"type": "int", "range": [0, 1]}, "opq_iters": {"type": "int", "range": [0, 1000]}, "nprobe": {"type": "int", "range": [1, 1048576]}},
 "HNSWFLAT": {"m": {"type": "int", "range": [8, 128]}, "ef_c": {"type": "int", "range": [16, 1024]}, "ef_s": {"type": "int", "range": [16, 1024]}, "nprobe": {"type": "int", "range": [1, 1048576]}, "graph_degree": {"type": "int", "range": [0, 64]}, "search_width": {"type": "int", "range": [1, 8]}},
 "HNSWSQ": {"m": {"type": "int", "range": [8, 128]}, "ef_c": {"type": "int", "range": [16, 1024]}, "ef_s": {"type": "int", "range": [16, 1024]}, "nprobe": {"type": "int", "range": [1, 1048576]}},
 "HNSWPQ": {"m": {"type": "int", "range": [8, 128]}, "M": {"type": "int", "range": [1, 4096]}, "aq_threshold": {"type": "float", "range": [0, 1]}, "opq": {"type": "int", "range": [0, 1]}, "opq_iters": {"type": "int", "range": [0, 1000]}, "nprobe": {"type": "int", "range": [1, 1048576]}},
 "SCANN": {"ncentroids": {"type": "int", "range": [1, 1048576]}, "M": {"type": "int", "range": [1, 4096]}, "aq_threshold": {"type": "float", "range": [0, 1]}, "opq": {"type": "int", "range": [0, 1]}, "opq_iters": {"type": "int", "range": [0, 1000]}, "nprobe": {"type": "int", "range": [1, 1048576]}, "reorder_k_factor": {"type": "int", "range": [1, 100]}},
 "MSTG": {"ncentroids": {"type": "int", "range": [1, 1048576]}, "alpha": {"type": "float", "range": [1, 4]}, "nprobe": {"type": "int", "range": [1, 1048576]}, "refine_factor": {"type": "int", "range": [1, 100]}, "disk_mode": {"type": "int", "range": [0, 2]}, "graph_degree": {"type": "int", "range": [0, 64]}, "ef_s": {"type": "int", "range": [16, 1024]}, "search_width": {"type": "int", "range": [1, 8]}},
 "BinaryIVF": {}, "BinaryHNSW": {},
 "BinaryMSTG": {"graph_degree": {"type": "int", "range": [0, 64]}, "ef_s": {"type": "int", "range": [16, 1024]}, "search_width": {"type": "int", "range": [1, 8]}}
})";

// MergeTreeVSManager.cpp:361-366, VIWithDataPart.cpp:405-407 (erase_if over {key, value}), :645
struct Parameters : std::map<std::string, std::string> {
    using std::map<std::string, std::string>::map;
    void setParam(const std::string & k, const std::string & v) { (*this)[k] = v; }
    template <class T> void setParam(const std::string & k, const T & v) { (*this)[k] = std::to_string(v); }
    std::string toString() const {
        std::string s;
        for (auto & kv : *this) s += (s.empty() ? "" : ", ") + kv.first + "=" + kv.second;
        return s;
    }
};

// VectorIndex/Common/VectorIndexIO.h:33-103 / :105-164: the streams ClickHouse hands to serialize() / load()
struct AbstractIStream {
    virtual ~AbstractIStream() = default;
    virtual AbstractIStream & read(char * s, std::streamsize count) = 0;
    virtual bool is_open() const = 0;
    virtual bool fail() const = 0;
    virtual bool eof() const = 0;
    virtual std::streamsize gcount() const = 0;
    virtual explicit operator bool() const = 0;
    virtual AbstractIStream & seekg(std::streampos offset, std::ios_base::seekdir dir) = 0;
};
struct AbstractOStream {
    virtual ~AbstractOStream() = default;
    virtual AbstractOStream & write(const char * s, std::streamsize count) = 0;
    virtual bool good() = 0;
    virtual void close() = 0;
    virtual AbstractOStream & seekp(std::streampos offset, std::ios_base::seekdir dir) = 0;
};
// VIWithDataPart.cpp:461-464, :688-691: (path prefix, factory(name, openmode) -> shared_ptr<stream>)
template <class OS> class IndexDataFileWriter {
    std::string prefix_;
    std::function<std::shared_ptr<OS>(const std::string &, std::ios::openmode)> factory_;
public:
    template <class F> IndexDataFileWriter(const std::string & prefix, F && f) : prefix_(prefix), factory_(std::forward<F>(f)) {}
    std::shared_ptr<OS> open(const std::string & name) { return factory_(prefix_ + name, std::ios::out | std::ios::binary); }
};
template <class IS> class IndexDataFileReader {
    std::string prefix_;
    std::function<std::shared_ptr<IS>(const std::string &, std::ios::openmode)> factory_;
public:
    template <class F> IndexDataFileReader(const std::string & prefix, F && f) : prefix_(prefix), factory_(std::forward<F>(f)) {}
    std::shared_ptr<IS> open(const std::string & name) { return factory_(prefix_ + name, std::ios::in | std::ios::binary); }
};
class DiskIOManager;   // VICommon.h:108 (disk_mode indexes; not used by this engine: everything is HBM resident)

// uses: MergeTreeVSManager.cpp:1060-1062,:1147,:1274,:1456,:1624; VIUtils.cpp:488; MergeTreeTextSearchManager.cpp:191-194
class DenseBitmap {
    size_t n_;
    std::vector<uint8_t> bits_;
public:
    explicit DenseBitmap(size_t n, bool init = false) : n_(n), bits_((n + 7) / 8, init ? 0xff : 0) {
        if (init && (n & 7)) bits_.back() = static_cast<uint8_t>((1u << (n & 7)) - 1);
    }
    size_t get_size() const { return n_; }
    size_t byte_size() const { return bits_.size(); }
    bool test(size_t i) const { return i < n_ && ((bits_[i >> 3] >> (i & 7)) & 1); }
    bool unsafe_test(size_t i) const { return (bits_[i >> 3] >> (i & 7)) & 1; }
    bool is_member(size_t i) const { return test(i); }
    void set(size_t i) { bits_[i >> 3] |= static_cast<uint8_t>(1u << (i & 7)); }
    void unset(size_t i) { bits_[i >> 3] &= static_cast<uint8_t>(~(1u << (i & 7))); }
    size_t count() const { size_t c = 0; for (auto b : bits_) c += static_cast<size_t>(__builtin_popcount(b)); return c; }
    bool any() const { return count() > 0; }
    bool all() const { return count() == n_; }
    uint8_t * get_bitmap() { return bits_.data(); }                    // LSB-first bytes, consumed as-is by the kernels
    const uint8_t * get_bitmap() const { return bits_.data(); }
    std::vector<size_t> to_vector() const { std::vector<size_t> v; for (size_t i = 0; i < n_; ++i) if (unsafe_test(i)) v.push_back(i); return v; }
};
using DenseBitmapPtr = std::shared_ptr<DenseBitmap>;
inline DenseBitmapPtr intersectDenseBitmaps(DenseBitmapPtr a, DenseBitmapPtr b) {   // VIWithDataPart.cpp:908, :560
    if (!a) return b;
    if (!b) return a;
    auto r = std::make_shared<DenseBitmap>(a->get_size());
    b200Check(b200_bitmap_and(a->get_bitmap(), b->get_bitmap(), int64_t(a->get_size()), r->get_bitmap()));
    return r;
}

template <class T> struct DataSet {                                    // VIWithDataPart.cpp:851, :923, :932
    using IndexDatasetType = T;
    T * data; int64_t n, dim;
    DataSet(T * d, int64_t n_, int64_t dim_) : data(d), n(n_), dim(dim_) {}
    T * getData() const { return data; }
    int64_t numData() const { return n; }
    int64_t dimension() const { return dim; }
};

// VIPartReader.h:38-306: the chunked source the index pulls its rows from
template <class T> class IndexSourceDataReader {
public:
    using IndexDatasetType = T;
    class DataChunk {                                                  // VIPartReader.h:164-166, :296-302
        T * data_; size_t n_, dim_; std::function<void()> del_; idx_t * ids_ = nullptr; std::function<void()> del_ids_;
    public:
        DataChunk(T * data, size_t n, size_t dim, std::function<void()> deleter) : data_(data), n_(n), dim_(dim), del_(std::move(deleter)) {}
        ~DataChunk() { if (del_) del_(); if (del_ids_) del_ids_(); }
        DataChunk(const DataChunk &) = delete;
        void setDataID(idx_t * ids, std::function<void()> deleter) { ids_ = ids; del_ids_ = std::move(deleter); }
        T * getData() const { return data_; }
        idx_t * getDataID() const { return ids_; }
        size_t numData() const { return n_; }
        size_t dimension() const { return dim_; }
    };
    virtual ~IndexSourceDataReader() = default;
    virtual size_t numDataRead() const = 0;
    virtual size_t dataDimension() const = 0;
    virtual bool eof() = 0;
    virtual void seekg(std::streamsize offset, std::ios::seekdir dir) = 0;
    virtual std::shared_ptr<DataChunk> sampleData(size_t n) = 0;
    std::shared_ptr<DataChunk> readData(size_t n) { return readDataImpl(n); }
protected:
    virtual std::shared_ptr<DataChunk> readDataImpl(size_t n) = 0;
};

// MergeTreeVSManager.cpp:456-461,:565-567,:604-609; VIWithDataPart.cpp:61-65,:90-95,:114-117
class SearchResult {
    int64_t nq_, k_, ncand_;
    std::vector<idx_t> ids_;
    std::vector<float> dis_;
public:
    struct Span { idx_t * b; idx_t * e; idx_t * begin() const { return b; } idx_t * end() const { return e; } };
    SearchResult(int64_t nq, int64_t k) : nq_(nq), k_(k), ncand_(k), ids_(size_t(nq * k), -1), dis_(size_t(nq * k), 0.f) {}
    static std::shared_ptr<SearchResult> createTopKHolder(int64_t nq, int64_t k) { return std::make_shared<SearchResult>(nq, k); }
    idx_t * getResultIndices() { return ids_.data(); }
    Span getResultIndices(size_t q) { return {ids_.data() + q * size_t(k_), ids_.data() + (q + 1) * size_t(k_)}; }   // VIWithDataPart.cpp:63
    float * getResultDistances() { return dis_.data(); }
    size_t numQueries() const { return size_t(nq_); }
    int64_t getNumCandidates() const { return ncand_; }
    void setNumCandidates(int64_t c) { ncand_ = c; }
    int64_t topK() const { return k_; }
};

struct IndexVersion { std::string toString() const { return b200_version(); } };                 // VIWithDataPart.cpp:475
struct IndexResourceUsage { size_t memory_usage_bytes = 0, disk_usage_bytes = 0, build_memory_usage_bytes = 0; };   // :476-478, VIWithDataPart.h:334

// Search::VectorIndex<IS, OS, Bitmap, DataType> (VICommon.h:142-146) as driven by VIWithColumnInPart
template <class IS, class OS, class Bitmap, DataType DT>
class VectorIndex {
    using T = std::conditional_t<DT == DataType::FloatVector, float, bool>;
    b200_index * h_ = nullptr;      // every type, binary ones too (BINARY*: rows and queries are bytes [n][dim / 8])
    std::string type_, params_;
    int metric_;
    size_t dim_, total_vec_;
    int64_t n_ = 0;
    bool two_stage_;
    size_t train_chunk_ = size_t(100) << 20, add_chunk_ = size_t(10) << 20;   // Settings.h:117-119 (bytes)
    size_t disk_bytes_ = 0;
    std::vector<idx_t> data_ids_;   // only kept when the reader's ids are not 0, 1, 2, ... (rows skipped by the reader)

    void mapIds(SearchResult & r) const {
        if (data_ids_.empty()) return;
        idx_t * p = r.getResultIndices();
        for (size_t i = 0; i < r.numQueries() * size_t(r.topK()); ++i) if (p[i] >= 0 && size_t(p[i]) < data_ids_.size()) p[i] = data_ids_[size_t(p[i])];
    }
    // the C ABI takes row pointers as const float *; binary rows (T = bool) are bytes [n][dim / 8] behind the same pointer
    static const float * rows(const T * p) { return reinterpret_cast<const float *>(p); }
    void noteIds(const idx_t * ids, size_t n) {
        bool identity = data_ids_.empty();
        for (size_t i = 0; identity && ids && i < n; ++i) identity = ids[i] == idx_t(size_t(n_) + i);
        if (identity && ids) return;
        if (data_ids_.empty()) for (int64_t i = 0; i < n_; ++i) data_ids_.push_back(i);
        for (size_t i = 0; i < n; ++i) data_ids_.push_back(ids ? ids[i] : idx_t(size_t(n_) + i));
    }
public:
    VectorIndex(const std::string & /*name*/, IndexType type, Metric metric, size_t dim, size_t total_vec, const Parameters & params)
        : type_(enumToString(type)), params_(params.toString()), metric_(toB200(metric)), dim_(dim), total_vec_(total_vec),
          two_stage_(type == IndexType::MSTG || type == IndexType::SCANN) {
        b200Check(b200_index_create(type_.c_str(), metric_, int(dim), params_.c_str(), &h_));
    }
    ~VectorIndex() { if (h_) b200_index_free(h_); }
    VectorIndex(const VectorIndex &) = delete;

    void setTrainDataChunkSize(size_t bytes) { train_chunk_ = bytes; }                             // VIWithDataPart.h:332
    void setAddDataChunkSize(size_t bytes) { add_chunk_ = bytes; }                                 // VIWithDataPart.h:333
    IndexResourceUsage getResourceUsage() const {                                                  // VIWithDataPart.h:334, .cpp:476
        IndexResourceUsage u;
        uint64_t b = 0;
        if (h_ && b200_index_memory_bytes(h_, &b) == B200_OK) u.memory_usage_bytes = size_t(b);
        u.disk_usage_bytes = disk_bytes_;
        u.build_memory_usage_bytes = std::max(train_chunk_, add_chunk_) * 3;   // pinned staging + device scratch of one chunk
        return u;
    }
    IndexVersion getVersion() const { return {}; }

    // build(part_reader, num_threads, cancel_build_callback) (VIWithDataPart.h:337): train block, then add blocks
    void build(IndexSourceDataReader<T> * reader, int /*num_threads*/, std::function<bool()> cancel = {}) {
        const size_t row_bytes = DT == DataType::BinaryVector ? dim_ / 8 : dim_ * sizeof(float);
        const size_t add_rows = std::max<size_t>(1, add_chunk_ / row_bytes);
        b200Check(b200_index_reserve(h_, int64_t(total_vec_)));
        auto sample = reader->sampleData(std::max<size_t>(1, std::min(total_vec_, train_chunk_ / row_bytes)));
        b200Check(b200_index_train(h_, sample ? rows(sample->getData()) : nullptr, sample ? int64_t(sample->numData()) : 0));
        while (!reader->eof()) {
            if (cancel && cancel()) throw SearchIndexException(B200_ERR_INVALID, "vector index build cancelled");
            auto chunk = reader->readData(add_rows);
            if (!chunk || chunk->numData() == 0) break;
            noteIds(chunk->getDataID(), chunk->numData());
            b200Check(b200_index_add(h_, rows(chunk->getData()), int64_t(chunk->numData())));
            n_ += int64_t(chunk->numData());
        }
        b200Check(b200_index_finalize(h_));
    }
    // search(queries, k, parameters, first_stage_only, filter) (VIWithDataPart.cpp:926, :935)
    std::shared_ptr<SearchResult> search(std::shared_ptr<DataSet<T>> q, int32_t k, Parameters & params, bool first_stage_only = false,
                                         Bitmap * filter = nullptr) {
        auto res = SearchResult::createTopKHolder(q->numData(), k);
        const uint8_t * bits = filter ? filter->get_bitmap() : nullptr;
        int64_t ncand = k;
        b200Check(b200_index_search(h_, rows(q->getData()), q->numData(), k, params.toString().c_str(), first_stage_only ? 1 : 0, bits,
                                    res->getResultDistances(), res->getResultIndices(), &ncand));
        res->setNumCandidates(first_stage_only ? k : ncand);
        mapIds(*res);
        return res;
    }
    // computeTopDistanceSubset(search_queries, first_stage_result, top_k) (VIWithDataPart.cpp:853)
    std::shared_ptr<SearchResult> computeTopDistanceSubset(std::shared_ptr<DataSet<float>> q, std::shared_ptr<SearchResult> first, int32_t top_k) {
        auto res = SearchResult::createTopKHolder(q->numData(), top_k);
        std::vector<idx_t> cand(first->getResultIndices(), first->getResultIndices() + q->numData() * first->topK());
        if (!data_ids_.empty()) {   // candidates come back in the reader's ids: map them to ordinals
            std::map<idx_t, idx_t> inv;
            for (size_t i = 0; i < data_ids_.size(); ++i) inv[data_ids_[i]] = idx_t(i);
            for (auto & c : cand) if (c >= 0) { auto it = inv.find(c); c = it == inv.end() ? -1 : it->second; }
        }
        b200Check(b200_index_refine(h_, q->getData(), q->numData(), cand.data(), first->topK(), top_k, res->getResultDistances(), res->getResultIndices()));
        mapIds(*res);
        return res;
    }
    bool supportTwoStageSearch() const { return two_stage_; }                                       // VIWithDataPart.cpp:878
    bool ready() const { return n_ > 0; }
    size_t numData() const { return size_t(n_); }                                                   // VIWithDataPart.cpp:700

    // serialize(&file_writer) / saveDataID(&file_writer) (VIWithDataPart.cpp:472-473): one stream "data_bin", one "data_id"
    void serialize(IndexDataFileWriter<OS> * writer) {
        auto os = writer->open("data_bin");
        if (!os) throw SearchIndexException(B200_ERR_INVALID, "cannot open the index output stream");
        struct Ctx { OS * os; size_t bytes; } ctx{os.get(), 0};
        auto wr = [](void * c, const void * p, size_t n) -> int { auto * x = static_cast<Ctx *>(c); x->os->write(static_cast<const char *>(p), std::streamsize(n)); x->bytes += n; return 0; };
        b200Check(b200_index_save_cb(h_, wr, &ctx));
        os->close();
        disk_bytes_ = ctx.bytes;
    }
    void saveDataID(IndexDataFileWriter<OS> * writer) {
        auto os = writer->open("data_id");
        if (!os) return;
        const uint64_t n = data_ids_.size();
        os->write(reinterpret_cast<const char *>(&n), sizeof(n));
        if (n) os->write(reinterpret_cast<const char *>(data_ids_.data()), std::streamsize(n * sizeof(idx_t)));
        os->close();
    }
    // load(&file_reader, check_index_expired) / loadDataID(&file_reader) (VIWithDataPart.cpp:698-699)
    void load(IndexDataFileReader<IS> * reader, std::function<bool()> expired = {}) {
        if (expired && expired()) throw SearchIndexException(B200_ERR_INVALID, "vector index expired while loading");
        auto is = reader->open("data_bin");
        if (!is || !is->is_open()) throw SearchIndexException(B200_ERR_INVALID, "cannot open the index input stream");
        auto rd = [](void * c, void * p, size_t n) -> int { auto * s = static_cast<IS *>(c); s->read(static_cast<char *>(p), std::streamsize(n)); return size_t(s->gcount()) == n ? 0 : 1; };
        if (h_) { b200_index_free(h_); h_ = nullptr; }
        b200Check(b200_index_load_cb(rd, is.get(), &h_));
        int64_t n = 0;
        b200Check(b200_index_info(h_, &n, nullptr, nullptr, nullptr));
        n_ = n;
    }
    void loadDataID(IndexDataFileReader<IS> * reader) {
        auto is = reader->open("data_id");
        if (!is || !is->is_open()) return;
        uint64_t n = 0;
        is->read(reinterpret_cast<char *>(&n), sizeof(n));
        data_ids_.assign(size_t(n), 0);
        if (n) is->read(reinterpret_cast<char *>(data_ids_.data()), std::streamsize(n * sizeof(idx_t)));
    }
};

// createVectorIndex<IS, OS, Bitmap, DT>(name, type, metric, dim, total_vec, params, max_threads, cache_prefix, cancel) (VIWithDataPart.cpp:416-430)
template <class IS, class OS, class Bitmap, DataType DT>
std::shared_ptr<VectorIndex<IS, OS, Bitmap, DT>> createVectorIndex(const std::string & name, IndexType type, Metric metric, size_t dim, size_t total_vec,
                                                                   const Parameters & params, size_t /*max_threads*/ = 0,
                                                                   const std::string & /*cache_prefix*/ = "", std::function<bool()> /*cancel*/ = {}) {
    return std::make_shared<VectorIndex<IS, OS, Bitmap, DT>>(name, type, metric, dim, total_vec, params);
}
}  // namespace Search

// ---- faiss entry points used by BruteForceSearch.h:77-105 -------------------------------------
namespace faiss {
struct float_maxheap_array_t { size_t nh, k; int64_t * ids; float * val; };
struct float_minheap_array_t { size_t nh, k; int64_t * ids; float * val; };
inline void knn_L2sqr(const float * x, const float * y, size_t d, size_t nx, size_t ny, float_maxheap_array_t * res, const void * = nullptr) {
    Search::b200Check(b200_flat_knn(B200_METRIC_L2, x, int64_t(nx), y, int64_t(ny), int(d), int(res->k), nullptr, res->val, res->ids));
}
inline void knn_inner_product(const float * x, const float * y, size_t d, size_t nx, size_t ny, float_minheap_array_t * res, const void * = nullptr) {
    Search::b200Check(b200_flat_knn(B200_METRIC_IP, x, int64_t(nx), y, int64_t(ny), int(d), int(res->k), nullptr, res->val, res->ids));
}
inline void hammings_knn_mc(const uint8_t * a, const uint8_t * b, size_t na, size_t nb, size_t k, size_t ncodes, int32_t * distances,
                            int64_t * labels, const void * = nullptr) {
    std::vector<float> d(na * k);
    Search::b200Check(b200_binary_knn(B200_METRIC_HAMMING, a, int64_t(na), b, int64_t(nb), int(ncodes), int(k), nullptr, d.data(), labels));
    for (size_t i = 0; i < na * k; ++i) distances[i] = static_cast<int32_t>(d[i]);   // int32 into the caller's buffer (:99)
}
}  // namespace faiss
inline void jaccard_knn(const uint8_t * a, const uint8_t * b, size_t na, size_t nb, size_t k, size_t ncodes, float * distances,
                        int64_t * labels, const void * = nullptr) {
    Search::b200Check(b200_binary_knn(B200_METRIC_JACCARD, a, int64_t(na), b, int64_t(nb), int(ncodes), int(k), nullptr, distances, labels));
}

// ---- TANTIVY::ffi_* used by Storages/MergeTree/TantivyIndexStore.cpp:654-998 --------------------
namespace TANTIVY {
struct RowIdWithScore { uint64_t row_id; float score; };
struct DocWithFreq { std::string term_str; uint32_t field_id; uint64_t doc_freq; };
struct FieldTokenNums { uint32_t field_id; uint64_t field_total_tokens; };
struct Statistics { std::vector<DocWithFreq> docs_freq; std::vector<FieldTokenNums> total_num_tokens; uint64_t total_num_docs = 0; };
struct FFIError { bool is_error = false; std::string message; };
template <class T> struct FFIResult { T result{}; FFIError error; };
using FFIBoolResult = FFIResult<bool>;
using FFIU64Result = FFIResult<uint64_t>;
using FFIVecRowIdWithScoreResult = FFIResult<std::vector<RowIdWithScore>>;
using FFIVecDocWithFreqResult = FFIResult<std::vector<DocWithFreq>>;
using FFIFieldTokenNumsResult = FFIResult<std::vector<FieldTokenNums>>;

// the Rust side keeps a process-global registry keyed by index directory; so does this adapter.  ClickHouse calls from one
// ThreadPool worker per part: the map is guarded (shared for look-ups, exclusive for create / load / free).
struct Store { b200_bm25 * h = nullptr; std::vector<std::string> columns; };
struct Registry {
    std::shared_mutex mu;
    std::map<std::string, Store> stores;
};
inline Registry & registry() { static Registry r; return r; }
inline bool findStore(const std::string & path, Store & out) {
    std::shared_lock<std::shared_mutex> lk(registry().mu);
    auto it = registry().stores.find(path);
    if (it == registry().stores.end()) return false;
    out = it->second;
    return true;
}
inline std::string indexFile(const std::string & dir) { return dir + (dir.empty() || dir.back() == '/' ? "" : "/") + "b200_bm25.b2tx"; }
inline std::string columnsFile(const std::string & dir) { return dir + (dir.empty() || dir.back() == '/' ? "" : "/") + "b200_bm25.columns"; }
template <class R> inline R failed(R r) { r.error = {true, b200_last_error()}; return r; }
template <class R> inline R noStore(R r, const std::string & path) { r.error = {true, "no text index is open for " + path}; return r; }

// ffi_create_index_with_parameter(path, indexed_columns, index_json_parameter) (:713)
inline FFIBoolResult ffi_create_index_with_parameter(const std::string & path, const std::vector<std::string> & columns, const std::string & /*json*/) {
    FFIBoolResult r; Store s; s.columns = columns;
    if (b200_bm25_create(uint32_t(std::max<size_t>(1, columns.size())), &s.h) != B200_OK) return failed(r);
    std::unique_lock<std::shared_mutex> lk(registry().mu);
    auto it = registry().stores.find(path);
    if (it != registry().stores.end() && it->second.h) b200_bm25_free(it->second.h);
    registry().stores[path] = s;
    r.result = true;
    return r;
}
// ffi_index_multi_column_docs(path, row_id, column_names, docs) (:742)
inline FFIBoolResult ffi_index_multi_column_docs(const std::string & path, uint64_t row_id, const std::vector<std::string> & column_names,
                                                 const std::vector<std::string> & docs) {
    FFIBoolResult r; Store s;
    if (!findStore(path, s)) return noStore(r, path);
    int rc = b200_bm25_add_doc(s.h, row_id);
    for (size_t i = 0; rc == B200_OK && i < docs.size(); ++i) {
        size_t f = i;   // a doc goes to the field of its column name (order of the call may differ from the index definition)
        if (i < column_names.size()) { auto it = std::find(s.columns.begin(), s.columns.end(), column_names[i]); if (it != s.columns.end()) f = size_t(it - s.columns.begin()); }
        rc = b200_bm25_add_text(s.h, uint32_t(f), docs[i].c_str());
    }
    if (rc != B200_OK) return failed(r);
    r.result = true;
    return r;
}
// ffi_index_writer_commit(path) (:824): freeze, upload to HBM, and leave the index file in the part's cache directory
inline FFIBoolResult ffi_index_writer_commit(const std::string & path) {
    FFIBoolResult r; Store s;
    if (!findStore(path, s)) return noStore(r, path);
    if (b200_bm25_commit(s.h) != B200_OK) return failed(r);
    if (b200_bm25_save(s.h, indexFile(path).c_str()) == B200_OK) {   // the directory may not exist in unit tests: then the index is memory-only
        if (FILE * f = fopen(columnsFile(path).c_str(), "w")) { for (auto & c : s.columns) fprintf(f, "%s\n", c.c_str()); fclose(f); }
    }
    r.result = true;
    return r;
}
// ffi_load_index_reader(path) (:654, :668): resident already, or loaded from the directory's index file
inline FFIBoolResult ffi_load_index_reader(const std::string & path) {
    FFIBoolResult r; Store s;
    if (findStore(path, s)) { r.result = true; return r; }
    if (b200_bm25_load(indexFile(path).c_str(), &s.h) != B200_OK) return failed(r);
    if (FILE * f = fopen(columnsFile(path).c_str(), "r")) { char line[4096]; while (fgets(line, sizeof(line), f)) { std::string c(line); while (!c.empty() && (c.back() == '\n' || c.back() == '\r')) c.pop_back(); s.columns.push_back(c); } fclose(f); }
    std::unique_lock<std::shared_mutex> lk(registry().mu);
    auto it = registry().stores.find(path);
    if (it != registry().stores.end()) { b200_bm25_free(s.h); r.result = true; return r; }   // another worker won the race
    registry().stores[path] = s;
    r.result = true;
    return r;
}
inline FFIBoolResult freeStore(const std::string & path) {
    FFIBoolResult r;
    std::unique_lock<std::shared_mutex> lk(registry().mu);
    auto it = registry().stores.find(path);
    if (it != registry().stores.end()) { if (it->second.h) b200_bm25_free(it->second.h); registry().stores.erase(it); }
    r.result = true;
    return r;
}
inline FFIBoolResult ffi_free_index_reader(const std::string & path) { return freeStore(path); }   // :769
inline FFIBoolResult ffi_free_index_writer(const std::string & path) {                              // :792: the reader keeps serving
    FFIBoolResult r; r.result = true; (void)path; return r;
}
inline FFIU64Result ffi_get_total_num_docs(const std::string & path) {                               // :974
    FFIU64Result r; Store s;
    if (!findStore(path, s)) return noStore(r, path);
    if (b200_bm25_total_docs(s.h, &r.result) != B200_OK) return failed(r);
    return r;
}
inline FFIU64Result ffi_get_indexed_doc_counts(const std::string & path) { return ffi_get_total_num_docs(path); }   // :998
inline FFIFieldTokenNumsResult ffi_get_total_num_tokens(const std::string & path) {                  // :986
    FFIFieldTokenNumsResult r; Store s;
    if (!findStore(path, s)) return noStore(r, path);
    for (uint32_t f = 0; f < uint32_t(std::max<size_t>(1, s.columns.size())); ++f) {
        uint64_t t = 0;
        if (b200_bm25_total_tokens(s.h, f, &t) != B200_OK) return failed(r);
        r.result.push_back({f, t});
    }
    return r;
}
inline std::vector<std::string> queryTerms(const std::string & sentence) {
    std::vector<char> buf(sentence.size() + 64); uint32_t n = 0; std::vector<std::string> out;
    if (b200_bm25_query_terms(sentence.c_str(), buf.data(), buf.size(), &n) != B200_OK) return out;
    const char * p = buf.data();
    for (uint32_t i = 0; i < n; ++i) { out.emplace_back(p); p += out.back().size() + 1; }
    return out;
}
inline FFIVecDocWithFreqResult ffi_get_doc_freq(const std::string & path, const std::string & sentence) {   // :962
    FFIVecDocWithFreqResult r; Store s;
    if (!findStore(path, s)) return noStore(r, path);
    for (auto & t : queryTerms(sentence))
        for (uint32_t f = 0; f < uint32_t(std::max<size_t>(1, s.columns.size())); ++f) {
            uint64_t df = 0;
            if (b200_bm25_doc_freq(s.h, f, t.c_str(), &df) != B200_OK) return failed(r);
            r.result.push_back({t, f, df});
        }
    return r;
}
// ffi_bm25_search(path, sentence, column_names, topk, u8_alived_bitmap, use_filter, enable_nlq, operator_or, statistics) (:908-917, :939-948)
// enable_nlq: tantivy's query-language parse of the sentence; plain sentences parse to the same terms, which is what this
// engine evaluates (query operators such as +term / "phrase" are tokenised as words).
inline FFIVecRowIdWithScoreResult ffi_bm25_search(const std::string & path, const std::string & sentence, const std::vector<std::string> & column_names,
                                                  uint32_t topk, const std::vector<uint8_t> & alive_bitmap, bool use_filter, bool /*enable_nlq*/,
                                                  bool operator_or, const Statistics & st) {
    FFIVecRowIdWithScoreResult r; Store s;
    if (!findStore(path, s)) return noStore(r, path);
    const uint32_t n_index_fields = uint32_t(std::max<size_t>(1, s.columns.size()));
    std::vector<uint32_t> fields;
    for (auto & c : column_names) { auto it = std::find(s.columns.begin(), s.columns.end(), c); if (it != s.columns.end()) fields.push_back(uint32_t(it - s.columns.begin())); }
    if (fields.empty()) for (uint32_t f = 0; f < n_index_fields; ++f) fields.push_back(f);   // no column given: every indexed column
    std::vector<uint64_t> rows(topk), tok, df; std::vector<float> sc(topk); uint32_t n = 0;
    const auto terms = queryTerms(sentence);
    if (st.total_num_docs) {
        tok.assign(n_index_fields, 0);   // sized by the INDEX's fields, whatever the statistics mention
        for (auto & t : st.total_num_tokens) if (t.field_id < n_index_fields) tok[t.field_id] = t.field_total_tokens;
        df.assign(fields.size() * 64, 0);
        for (size_t fi = 0; fi < fields.size(); ++fi) for (size_t ti = 0; ti < terms.size() && ti < 64; ++ti)
            for (auto & d : st.docs_freq) if (d.field_id == fields[fi] && d.term_str == terms[ti]) df[fi * 64 + ti] = d.doc_freq;
    }
    if (topk == 0) return r;
    if (b200_bm25_search(s.h, sentence.c_str(), fields.data(), uint32_t(fields.size()), topk, use_filter ? alive_bitmap.data() : nullptr,
                         use_filter, operator_or, st.total_num_docs, tok.data(), df.data(), rows.data(), sc.data(), &n) != B200_OK) return failed(r);
    for (uint32_t i = 0; i < n; ++i) r.result.push_back({rows[i], sc[i]});
    return r;
}
}  // namespace TANTIVY
