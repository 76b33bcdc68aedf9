// tests/cpp/test_knowhere_api.cc — exercises the C++ mirror of the reference interface
// (include/knowhere_b200.hpp) the way the reference's Catch2 tests drive Knowhere:
//   tests/ut/test_search.cc:57-268  (IndexFactory::Create -> Build -> Search, recall vs BruteForce)
//   tests/ut/test_bruteforce.cc:57-77 (self-query KAT)
// Plain asserts instead of Catch2 (not in this image).  Exit code 0 = pass.  Needs an H100.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <set>
#include <vector>

#include "knowhere_b200.hpp"

#define REQUIRE(c)                                                                   \
    do {                                                                             \
        if (!(c)) { fprintf(stderr, "REQUIRE failed: %s @%d (%s)\n", #c, __LINE__, kb2_last_error()); exit(1); } \
    } while (0)

using namespace knowhere;

static std::vector<float>
GenData(int64_t rows, int64_t dim, int seed) {  // tests/ut/utils.h:41-50: mt19937 + uniform_real(0,100)
    std::mt19937 rng(seed);
    std::uniform_real_distribution<float> distrib(0.0, 100.0);
    std::vector<float> v(rows * dim);
    for (auto& x : v) x = distrib(rng);
    return v;
}
static float
GetKNNRecall(const DataSet& gt, const DataSet& res) {  // tests/ut/utils.h:110-133
    const int64_t nq = gt.GetRows(), k = gt.GetDim();
    int64_t hit = 0;
    for (int64_t i = 0; i < nq; i++) {
        std::set<int64_t> s(gt.GetIds() + i * k, gt.GetIds() + (i + 1) * k);
        for (int64_t j = 0; j < k; j++) hit += s.count(res.GetIds()[i * res.GetDim() + j]);
    }
    return hit / (float)(nq * k);
}

int
main() {
    if (kb2_device_count() <= 0) {
        auto e = IndexFactory::Instance().Create<fp32>("FLAT", 0);
        REQUIRE(!e.has_value() && e.error() == Status::cuda_runtime_error);
        printf("no GPU: factory correctly reports cuda_runtime_error\n");
        return 0;
    }
    const int64_t nb = 10000, nq = 100, dim = 128, topk = 10;
    auto xb = GenData(nb, dim, 42), xq = GenData(nq, dim, 43);
    auto train_ds = GenDataSet(nb, dim, xb.data());
    auto query_ds = GenDataSet(nq, dim, xq.data());
    Json base;
    base[meta::DIM] = dim;
    base[meta::METRIC_TYPE] = metric::L2;
    base[meta::TOPK] = topk;
    auto gt = BruteForce::Search<fp32>(train_ds, query_ds, base, nullptr);
    REQUIRE(gt.has_value());

    // self-query KAT
    auto self_ds = GenDataSet(nq, dim, xb.data());
    auto self = BruteForce::Search<fp32>(train_ds, self_ds, base, nullptr);
    REQUIRE(self.has_value());
    for (int64_t i = 0; i < nq; i++) {
        REQUIRE(self.value()->GetIds()[i * topk] == i);
        REQUIRE(self.value()->GetDistance()[i * topk] == 0.0f);
    }

    struct Case { const char* name; float min_recall; };
    for (Case c : {Case{"FLAT", 0.999f}, Case{"IVF_FLAT", 0.6f}, Case{"IVF_PQ", 0.0f}, Case{"HNSW", 0.6f}}) {
        Json json = base;
        json[indexparam::NLIST] = 16;
        json[indexparam::NPROBE] = 8;
        json[indexparam::M] = 4;
        json[indexparam::NBITS] = 8;
        json[indexparam::HNSW_M] = 16;
        json[indexparam::EFCONSTRUCTION] = 100;
        json[indexparam::EF] = 64;
        auto idx_e = IndexFactory::Instance().Create<fp32>(c.name, 0);
        REQUIRE(idx_e.has_value());
        auto idx = idx_e.value();
        REQUIRE(idx.Type() == c.name);
        REQUIRE(idx.Build(train_ds, json) == Status::success);
        REQUIRE(idx.Count() == nb);
        REQUIRE(idx.Dim() == dim);
        auto res = idx.Search(query_ds, json, nullptr);
        REQUIRE(res.has_value());
        const float recall = GetKNNRecall(*gt.value(), *res.value());
        printf("%-8s recall@%ld = %.4f\n", c.name, (long)topk, recall);
        REQUIRE(recall >= c.min_recall);   // test_search.cc:263-268 (IVF_PQ not recall-checked there either)
        // serialize -> deserialize -> identical answers (test_search.cc build->serialize->load->search)
        BinarySet bs;
        REQUIRE(idx.Serialize(bs) == Status::success);
        auto idx2 = IndexFactory::Instance().Create<fp32>(c.name, 0).value();
        REQUIRE(idx2.Deserialize(bs, json) == Status::success);
        auto res2 = idx2.Search(query_ds, json, nullptr);
        REQUIRE(res2.has_value());
        for (int64_t i = 0; i < nq * topk; i++) REQUIRE(res.value()->GetIds()[i] == res2.value()->GetIds()[i]);
    }
    // error behaviour: unknown index, bad metric
    REQUIRE(!IndexFactory::Instance().Create<fp32>("NO_SUCH_INDEX", 0).has_value());
    Json bad = base;
    bad[meta::METRIC_TYPE] = "HAMMING";
    auto idx = IndexFactory::Instance().Create<fp32>("FLAT", 0).value();
    REQUIRE(idx.Build(train_ds, bad) == Status::invalid_metric_type);
    // range search through the facade
    {
        Json json = base;
        json[meta::RADIUS] = gt.value()->GetDistance()[topk - 1];
        auto idx3 = IndexFactory::Instance().Create<fp32>("FLAT", 0).value();
        REQUIRE(idx3.Build(train_ds, json) == Status::success);
        auto rr = idx3.RangeSearch(query_ds, json, nullptr);
        REQUIRE(rr.has_value());
        REQUIRE(rr.value()->GetLims()[1] - rr.value()->GetLims()[0] == (size_t)(topk - 1));
    }
    // AnnIterator, GetIndexMeta, DeserializeFromFile, BitsetView with an id offset, HNSW RangeSearch + filter
    for (const char* name : {"IVF_FLAT", "HNSW"}) {
        Json json = base;
        json[indexparam::NLIST] = 16;
        json[indexparam::NPROBE] = 16;
        json[indexparam::HNSW_M] = 16;
        json[indexparam::EFCONSTRUCTION] = 100;
        json[indexparam::EF] = 64;
        auto ix = IndexFactory::Instance().Create<fp32>(name, 0).value();
        REQUIRE(ix.Build(train_ds, json) == Status::success);
        auto meta_ds = ix.GetIndexMeta(json);
        REQUIRE(meta_ds.has_value() && meta_ds.value()->GetJsonInfo().find(name) != std::string::npos);
        // iterator: the first topk results equal Search's, distances are monotone, and it continues past topk
        auto one = GenDataSet(1, dim, xq.data());
        auto its = ix.AnnIterator(one, json, nullptr);
        REQUIRE(its.has_value() && its.value().size() == 1);
        auto sr = ix.Search(one, json, nullptr);
        REQUIRE(sr.has_value());
        float prev = -1.f;
        int got = 0;
        std::set<int64_t> uniq;
        auto it = its.value()[0];
        const bool exact_scan = std::string(name) == "IVF_FLAT";
        while (got < 100 && it->HasNext().value()) {
            auto nx = it->Next();
            REQUIRE(nx.has_value());
            if (got < (int)topk && exact_scan) REQUIRE(nx.value().first == sr.value()->GetIds()[got]);
            if (exact_scan) REQUIRE(nx.value().second >= prev);
            prev = nx.value().second;
            uniq.insert(nx.value().first);
            got++;
        }
        REQUIRE(got == 100 && (int)uniq.size() == 100);
        // file round trip
        BinarySet bs;
        REQUIRE(ix.Serialize(bs) == Status::success);
        auto bin = bs.GetByName(name);
        REQUIRE(bin != nullptr);
        const char* path = "/tmp/kb2_cpp_test_index.bin";
        FILE* f = fopen(path, "wb");
        REQUIRE(f && fwrite(bin->data.get(), 1, (size_t)bin->size, f) == (size_t)bin->size);
        fclose(f);
        auto ix2 = IndexFactory::Instance().Create<fp32>(name, 0).value();
        REQUIRE(ix2.DeserializeFromFile(path, json) == Status::success);
        auto sr2 = ix2.Search(one, json, nullptr);
        REQUIRE(sr2.has_value());
        for (int64_t i = 0; i < topk; i++) REQUIRE(sr.value()->GetIds()[i] == sr2.value()->GetIds()[i]);
        // bitset over PUBLIC ids with an id offset: public id = internal id + 5 (bitsetview.h:131-175)
        std::vector<uint8_t> bits((nb + 5 + 7) / 8, 0);
        for (int64_t pub = 0; pub < nb + 5; pub += 2) bits[pub >> 3] |= (uint8_t)(1u << (pub & 7));   // even public ids filtered
        BitsetView bv(bits.data(), (size_t)(nb + 5));
        bv.set_id_offset(5);
        bv.set_vector_count((size_t)nb);
        auto fr = ix.Search(query_ds, json, bv);
        REQUIRE(fr.has_value());
        for (int64_t i = 0; i < nq * topk; i++) {
            const int64_t id = fr.value()->GetIds()[i];
            REQUIRE(id < 0 || ((id + 5) % 2) == 1);
        }
        // RangeSearch through the facade (HNSW: ef-bounded beam + closure, HnswSearcher.h:435-553)
        Json rj = json;
        rj[meta::RADIUS] = gt.value()->GetDistance()[topk - 1];
        auto rr = ix.RangeSearch(query_ds, rj, nullptr);
        REQUIRE(rr.has_value());
        REQUIRE(rr.value()->GetLims()[1] - rr.value()->GetLims()[0] >= 1);
    }
    printf("knowhere C++ API tests passed\n");
    return 0;
}
