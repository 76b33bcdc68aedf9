// tests/cpp/test_large_nprobe.cc — AnnIterator on IVF_PQ with nprobe 4096 (compiled and run by
// tests/test_large_nprobe_gpu.py).  The index has 4096 lists, so every list is probed; the iterator draws 500 results:
// ids distinct, distances monotone, the first 100 equal to Search(k = 100) with the same nprobe.  Exit code 0 = pass.
// Needs an H100.
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

int
main() {
    REQUIRE(kb2_device_count() > 0);
    // training takes nlist * 39 rows
    const int64_t nlist = 4096, nb = nlist * 40, dim = 16, want = 500, k_search = 100;
    std::mt19937 rng(11);
    std::uniform_real_distribution<float> u(0.f, 100.f);
    std::vector<float> xb(nb * dim), xq(dim);
    for (auto& x : xb) x = u(rng);
    for (auto& x : xq) x = u(rng);
    auto train_ds = GenDataSet(nb, dim, xb.data());
    auto one = GenDataSet(1, dim, xq.data());
    Json json;
    json[meta::DIM] = dim;
    json[meta::METRIC_TYPE] = metric::L2;
    json[indexparam::NLIST] = nlist;
    json[indexparam::M] = 4;
    json[indexparam::NBITS] = 8;
    json[indexparam::NPROBE] = 4096;
    auto ix = IndexFactory::Instance().Create<fp32>("IVF_PQ", 0).value();
    REQUIRE(ix.Build(train_ds, json) == Status::success);
    Json sj = json;
    sj[meta::TOPK] = k_search;
    auto sr = ix.Search(one, sj, nullptr);
    REQUIRE(sr.has_value());
    auto its = ix.AnnIterator(one, json, nullptr);
    REQUIRE(its.has_value() && its.value().size() == 1);
    auto it = its.value()[0];
    std::set<int64_t> uniq;
    float prev = -1.f;
    int64_t got = 0;
    while (got < want && it->HasNext().value()) {
        auto nx = it->Next();
        REQUIRE(nx.has_value());
        if (got < k_search) REQUIRE(nx.value().first == sr.value()->GetIds()[got]);
        REQUIRE(nx.value().second >= prev);
        prev = nx.value().second;
        uniq.insert(nx.value().first);
        got++;
    }
    REQUIRE(got == want);
    REQUIRE((int64_t)uniq.size() == want);
    printf("iterator ok: %ld results\n", (long)got);
    return 0;
}
