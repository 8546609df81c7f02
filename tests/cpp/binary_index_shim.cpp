// binary_index_shim.cpp -- a BinaryIVF index driven through shim/b200_search_shim.hpp the way VIWithColumnInPart drives a
// binary column: createVectorIndex<..., BinaryVector>, build from an IndexSourceDataReader in several add blocks, a filtered
// search, serialize through IndexDataFileWriter, load into a new index through IndexDataFileReader, and the same results
// after the reload.  Compiled with -Wall -Wextra -Werror; prints "BINARY INDEX OK".  Without a GPU the first call fails
// loudly through SearchIndexException (exit 2).
#include <b200_search_shim.hpp>

#include <cstdio>
#include <cstring>

namespace {
using Disk = std::map<std::string, std::string>;

class MemReader : public Search::AbstractIStream {
public:
    MemReader(Disk * disk, const std::string & file) { auto it = disk->find(file); if (it != disk->end()) in_ = &it->second; }
    Search::AbstractIStream & read(char * s, std::streamsize count) override {
        last_ = 0;
        if (in_) { last_ = std::min<size_t>(size_t(count), in_->size() - pos_); memcpy(s, in_->data() + pos_, last_); pos_ += last_; }
        return *this;
    }
    bool is_open() const override { return in_ != nullptr; }
    bool fail() const override { return in_ == nullptr; }
    bool eof() const override { return in_ ? pos_ >= in_->size() : true; }
    std::streamsize gcount() const override { return std::streamsize(last_); }
    explicit operator bool() const override { return in_ != nullptr; }
    Search::AbstractIStream & seekg(std::streampos offset, std::ios_base::seekdir) override { pos_ = size_t(offset); return *this; }
private:
    const std::string * in_ = nullptr;
    size_t pos_ = 0, last_ = 0;
};

class MemWriter : public Search::AbstractOStream {
public:
    MemWriter(Disk * disk, const std::string & file) : out_(&(*disk)[file]) {}
    Search::AbstractOStream & write(const char * s, std::streamsize count) override { out_->append(s, size_t(count)); return *this; }
    bool good() override { return true; }
    void close() override {}
    Search::AbstractOStream & seekp(std::streampos, std::ios_base::seekdir) override { return *this; }
private:
    std::string * out_;
};

// binary rows (bytes [n][dim / 8]) handed out as the part reader hands them: bool * chunks of at most n rows
class ByteReader : public Search::IndexSourceDataReader<bool> {
public:
    using DataChunk = Search::IndexSourceDataReader<bool>::DataChunk;
    ByteReader(const std::vector<uint8_t> & rows, size_t n, size_t dim) : rows_(rows), n_(n), dim_(dim) {}
    size_t numDataRead() const override { return read_; }
    size_t dataDimension() const override { return dim_; }
    bool eof() override { return read_ == n_; }
    void seekg(std::streamsize, std::ios::seekdir) override {}
    std::shared_ptr<DataChunk> sampleData(size_t n) override { return chunk(0, std::min(n, n_)); }
protected:
    std::shared_ptr<DataChunk> readDataImpl(size_t n) override {
        if (n == 0 || read_ == n_) return nullptr;
        const size_t m = std::min(n, n_ - read_);
        auto c = chunk(read_, m);
        read_ += m;
        return c;
    }
private:
    std::shared_ptr<DataChunk> chunk(size_t first, size_t m) {
        const size_t rb = dim_ / 8;
        bool * data = new bool[m * rb];
        memcpy(data, rows_.data() + first * rb, m * rb);
        Search::idx_t * ids = new Search::idx_t[m];
        for (size_t i = 0; i < m; ++i) ids[i] = Search::idx_t(first + i);
        auto c = std::make_shared<DataChunk>(data, m, dim_, [=]() { delete[] data; });
        c->setDataID(ids, [=]() { delete[] ids; });
        return c;
    }
    const std::vector<uint8_t> & rows_;
    size_t n_, dim_, read_ = 0;
};
}  // namespace

#define REQUIRE(cond) do { if (!(cond)) { std::printf("FAILED line %d: %s\n", __LINE__, #cond); return 1; } } while (0)

int main() {
    try {
        const size_t dim = 256, n = 6000, rb = dim / 8;
        std::vector<uint8_t> rows(n * rb);
        uint64_t st = 12345;
        for (auto & b : rows) { st = st * 6364136223846793005ull + 1442695040888963407ull; b = uint8_t(st >> 56); }
        Search::Parameters des;
        des.setParam("ncentroids", 16);
        auto type = Search::getVectorIndexType("BinaryIVF", Search::DataType::BinaryVector);
        auto metric = Search::getMetricType("Hamming", Search::DataType::BinaryVector);
        auto index = Search::createVectorIndex<Search::AbstractIStream, Search::AbstractOStream, Search::DenseBitmap, Search::DataType::BinaryVector>(
            "b1", type, metric, dim, n, des, 8, "store/all_1_1_0/b1/", []() { return false; });
        ByteReader reader(rows, n, dim);
        index->setAddDataChunkSize(2000 * rb);   // three add blocks
        index->build(&reader, 4, []() { return false; });
        REQUIRE(index->numData() == n && index->ready() && !index->supportTwoStageSearch());
        REQUIRE(index->getResourceUsage().memory_usage_bytes > n * rb);

        // queries = rows 7 and 4242; row 7 filtered out
        std::vector<uint8_t> q(2 * rb);
        memcpy(q.data(), rows.data() + 7 * rb, rb);
        memcpy(q.data() + rb, rows.data() + 4242 * rb, rb);
        auto qs = std::make_shared<Search::DataSet<bool>>(reinterpret_cast<bool *>(q.data()), 2, int64_t(dim));
        Search::DenseBitmap filter(n, true);
        filter.unset(7);
        Search::Parameters sp;
        sp.setParam("nprobe", 16);
        auto r1 = index->search(qs, 5, sp, false, &filter);
        REQUIRE(r1->getResultIndices()[0] != 7 && r1->getResultIndices()[5] == 4242 && r1->getResultDistances()[5] == 0.f);

        Disk disk;
        auto writer = Search::IndexDataFileWriter<Search::AbstractOStream>("tmp/b1-", [&](const std::string & name, std::ios::openmode) { return std::make_shared<MemWriter>(&disk, name); });
        index->serialize(&writer);
        index->saveDataID(&writer);
        REQUIRE(disk.count("tmp/b1-data_bin") == 1 && index->getResourceUsage().disk_usage_bytes > 0);

        auto loaded = Search::createVectorIndex<Search::AbstractIStream, Search::AbstractOStream, Search::DenseBitmap, Search::DataType::BinaryVector>(
            "b1", type, metric, dim, n, Search::Parameters{}, 8, "store/all_1_1_0/b1/", []() { return false; });
        auto file_reader = Search::IndexDataFileReader<Search::AbstractIStream>("tmp/b1-", [&](const std::string & name, std::ios::openmode) { return std::make_shared<MemReader>(&disk, name); });
        loaded->load(&file_reader, []() { return false; });
        loaded->loadDataID(&file_reader);
        REQUIRE(loaded->numData() == n);
        auto r2 = loaded->search(qs, 5, sp, false, &filter);
        REQUIRE(memcmp(r1->getResultIndices(), r2->getResultIndices(), 10 * sizeof(Search::idx_t)) == 0);
        REQUIRE(memcmp(r1->getResultDistances(), r2->getResultDistances(), 10 * sizeof(float)) == 0);
        std::printf("BINARY INDEX OK\n");
        return 0;
    } catch (const SearchIndexException & e) {
        std::printf("SearchIndexException %d: %s\n", e.getCode(), e.what());
        return 2;
    } catch (const std::exception & e) {
        std::printf("exception: %s\n", e.what());
        return 3;
    }
}
