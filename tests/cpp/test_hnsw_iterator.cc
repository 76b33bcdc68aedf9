// tests/cpp/test_hnsw_iterator.cc — AnnIterator on HNSW past the four-queries-per-CTA beam (compiled and run by
// tests/test_hnsw_large_ef_gpu.py).  The iterator doubles k and sets ef = k; on an unfiltered d = 128 index of 40000 rows
// the refills at k = 8192 and 16384 run the one-query-per-CTA beam (k stays below n / 2, so not the exact branch).  It must
// draw 12000 distinct valid ids.  Exit code 0 = pass.  Needs an H100.
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
    const int64_t nb = 40000, dim = 128, want = 12000;
    std::mt19937 rng(11);
    std::uniform_real_distribution<float> u(0.f, 1.f);
    std::vector<float> xb(nb * dim), xq(dim);
    for (auto& x : xb) x = u(rng);
    for (auto& x : xq) x = u(rng);
    auto train_ds = GenDataSet(nb, dim, xb.data());
    auto one = GenDataSet(1, dim, xq.data());
    Json json;
    json[meta::DIM] = dim;
    json[meta::METRIC_TYPE] = metric::L2;
    json[indexparam::HNSW_M] = 16;
    json[indexparam::EFCONSTRUCTION] = 100;
    auto ix = IndexFactory::Instance().Create<fp32>("HNSW", 0).value();
    REQUIRE(ix.Build(train_ds, json) == Status::success);
    auto its = ix.AnnIterator(one, json, nullptr);
    REQUIRE(its.has_value() && its.value().size() == 1);
    auto it = its.value()[0];
    std::set<int64_t> uniq;
    int64_t got = 0;
    while (got < want && it->HasNext().value()) {
        auto nx = it->Next();
        REQUIRE(nx.has_value());
        REQUIRE(nx.value().first >= 0 && nx.value().first < nb);
        uniq.insert(nx.value().first);
        got++;
    }
    printf("drawn %ld results, %ld distinct\n", (long)got, (long)uniq.size());
    REQUIRE(got == want);
    REQUIRE((int64_t)uniq.size() == want);
    printf("iterator ok: %ld results\n", (long)got);
    return 0;
}
