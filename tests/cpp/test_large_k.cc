// tests/cpp/test_large_k.cc — AnnIterator past 1008 results (compiled and run by tests/test_large_k_gpu.py).
// On an IVF_FLAT index that probes every list (an exact scan) the iterator draws 5000 results: ids distinct, distances
// monotone, the first 1008 equal to Search(k = 1008).  Exit code 0 = pass.  Needs an H100.
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
    const int64_t nb = 20000, dim = 64, want = 5000, k_search = 1008;
    std::mt19937 rng(7);
    std::uniform_real_distribution<float> u(0.f, 100.f);
    std::vector<float> xb(nb * dim), xq(dim);
    for (auto& x : xb) x = u(rng);
    for (auto& x : xq) x = u(rng);
    auto train_ds = GenDataSet(nb, dim, xb.data());
    auto one = GenDataSet(1, dim, xq.data());
    Json json;
    json[meta::DIM] = dim;
    json[meta::METRIC_TYPE] = metric::L2;
    json[indexparam::NLIST] = 16;
    json[indexparam::NPROBE] = 16;
    auto ix = IndexFactory::Instance().Create<fp32>("IVF_FLAT", 0).value();
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
