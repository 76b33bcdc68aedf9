// tests/cpp/test_emb_list.cc — BruteForce::Search / SearchWithBuf<fp32> over emb-lists (compiled and run by
// tests/test_emb_list_gpu.py).  EMB_LIST_OFFSET on both DataSets: one result row per query list, the same rows through
// both entry points and the C ABI, trailing empty query lists dropped as EmbListOffset does, and the reference's error
// statuses.  Exit code 0 = pass.  Needs an H100.
#include <cstdio>
#include <cstdlib>
#include <random>
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
    const int64_t dim = 64, k = 7;
    const std::vector<size_t> doc_len = {3, 1, 0, 150, 20, 9, 0, 60, 2, 200, 11, 5};
    std::vector<size_t> xl = {0};
    for (size_t l : doc_len) xl.push_back(xl.back() + l);
    // three query lists, then two trailing empty ones (dropped: the result has three rows)
    const std::vector<size_t> ql = {0, 4, 36, 37, 37, 37};
    const int64_t nb = (int64_t)xl.back(), nq = (int64_t)ql.back(), n_lists = 3;
    std::mt19937 rng(3);
    std::normal_distribution<float> g;
    std::vector<float> xb(nb * dim), xq(nq * dim);
    for (auto& v : xb) v = g(rng);
    for (auto& v : xq) v = g(rng);
    auto base = GenDataSet(nb, dim, xb.data());
    auto query = GenDataSet(nq, dim, xq.data());
    base->Set(meta::EMB_LIST_OFFSET, xl.data());
    query->Set(meta::EMB_LIST_OFFSET, ql.data());
    REQUIRE(query->Get<const size_t*>(meta::EMB_LIST_OFFSET) == ql.data());

    for (const char* m : {metric::MAX_SIM, metric::MAX_SIM_IP, metric::MAX_SIM_L2, "max_sim_cosine"}) {
        Json cfg;
        cfg[meta::METRIC_TYPE] = m;
        cfg[meta::TOPK] = k;
        auto r = BruteForce::Search<fp32>(base, query, cfg, nullptr);
        REQUIRE(r.has_value());
        REQUIRE(r.value()->GetRows() == n_lists && r.value()->GetDim() == k);
        std::vector<int64_t> ids(n_lists * k);
        std::vector<float> dis(n_lists * k);
        REQUIRE(BruteForce::SearchWithBuf<fp32>(base, query, ids.data(), dis.data(), cfg, nullptr) == Status::success);
        // the C ABI with explicit counts gives the same rows
        std::vector<int64_t> xl64(xl.begin(), xl.end()), ql64(ql.begin(), ql.begin() + n_lists + 1);
        int code = 0;
        REQUIRE(kb2_emb_list_metric(m, code) && code > 0);
        std::vector<int64_t> ids2(n_lists * k);
        std::vector<float> dis2(n_lists * k);
        int64_t stats[3];
        REQUIRE(kb2_bruteforce_search_emb_list(xb.data(), xl64.data(), (int64_t)doc_len.size(), dim, code, xq.data(), ql64.data(),
                                               n_lists, k, nullptr, 0, ids2.data(), dis2.data(), stats, 0, nullptr) == 0);
        REQUIRE(stats[0] == n_lists);
        for (int64_t i = 0; i < n_lists * k; i++) {
            REQUIRE(r.value()->GetIds()[i] == ids[i] && r.value()->GetDistance()[i] == dis[i]);
            REQUIRE(ids[i] == ids2[i] && dis[i] == dis2[i]);
            REQUIRE(ids[i] != 2 && ids[i] != 6);   // empty documents are never returned
        }
        // 12 documents, 2 empty: 10 valid >= k, so no padding; rows ordered best first
        const bool l2 = std::string(m) == metric::MAX_SIM_L2;
        for (int64_t q = 0; q < n_lists; q++)
            for (int64_t j = 1; j < k; j++) REQUIRE(l2 ? dis[q * k + j] >= dis[q * k + j - 1] : dis[q * k + j] <= dis[q * k + j - 1]);
    }
    Json cfg;
    cfg[meta::METRIC_TYPE] = metric::MAX_SIM_IP;
    cfg[meta::TOPK] = k;
    std::vector<int64_t> ids(64);
    std::vector<float> dis(64);
    // a missing offset: Search -> invalid_args, SearchWithBuf -> invalid_metric_type (brute_force.cc:272-277, :628-632)
    auto plain = GenDataSet(nq, dim, xq.data());
    auto r1 = BruteForce::Search<fp32>(base, plain, cfg, nullptr);
    REQUIRE(!r1.has_value() && r1.error() == Status::invalid_args);
    REQUIRE(BruteForce::SearchWithBuf<fp32>(base, plain, ids.data(), dis.data(), cfg, nullptr) == Status::invalid_metric_type);
    auto plain_base = GenDataSet(nb, dim, xb.data());
    REQUIRE(!BruteForce::Search<fp32>(plain_base, query, cfg, nullptr).has_value());
    // an emb-list query with a single-vector metric (brute_force.cc:673-676)
    Json l2;
    l2[meta::METRIC_TYPE] = metric::L2;
    l2[meta::TOPK] = k;
    REQUIRE(BruteForce::SearchWithBuf<fp32>(base, query, ids.data(), dis.data(), l2, nullptr) == Status::invalid_metric_type);
    // binary MAX_SIM metrics: no binary vectors in this library
    Json ham = cfg;
    ham[meta::METRIC_TYPE] = metric::MAX_SIM_HAMMING;
    auto r2 = BruteForce::Search<fp32>(base, query, ham, nullptr);
    REQUIRE(!r2.has_value() && r2.error() == Status::invalid_metric_type);
    // range search over emb-lists is not supported (index_node.cc:301-310)
    Json rs = cfg;
    rs[meta::RADIUS] = 1.0f;
    auto r3 = BruteForce::RangeSearch<fp32>(base, query, rs, nullptr);
    REQUIRE(!r3.has_value() && r3.error() == Status::emb_list_inner_error);
    // offsets that never reach the row count
    const std::vector<size_t> short_l = {0, 4, 30, 40};   // jumps past the 37 rows
    auto q_bad = GenDataSet(nq, dim, xq.data());
    q_bad->Set(meta::EMB_LIST_OFFSET, short_l.data());
    REQUIRE(BruteForce::SearchWithBuf<fp32>(base, q_bad, ids.data(), dis.data(), cfg, nullptr) == Status::invalid_args);
    // still usable afterwards
    REQUIRE(BruteForce::Search<fp32>(base, query, cfg, nullptr).has_value());
    printf("emb_list ok\n");
    return 0;
}
