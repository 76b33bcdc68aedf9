// tests/cpp/test_emb_list_muvera.cc — emb-list HNSW / IVF_FLAT with the MUVERA strategy through the C++ mirror (compiled
// and run by tests/test_emb_list_muvera_gpu.py).  Build with EMB_LIST_OFFSET and "emb_list_strategy": "muvera", Search
// with query list offsets (the same rows as the C ABI, emb_list_rerank passed through), and a BinarySet round trip.
// Exit code 0 = pass.  Needs an H100.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "knowhere_b200.hpp"

#define REQUIRE(c)                                                                   \
    do {                                                                             \
        if (!(c)) { fprintf(stderr, "REQUIRE failed: %s @%d (%s)\n", #c, __LINE__, kb2_last_error()); exit(1); } \
    } while (0)

using namespace knowhere;

static bool
same_rows(const DataSetPtr& a, const DataSetPtr& b) {
    const int64_t n = a->GetRows() * a->GetDim();
    if (a->GetRows() != b->GetRows() || a->GetDim() != b->GetDim()) return false;
    return memcmp(a->GetIds(), b->GetIds(), n * 8) == 0 && memcmp(a->GetDistance(), b->GetDistance(), n * 4) == 0;
}

static void
run(const char* type, const char* el_metric, Json extra) {
    const int64_t dim = 16, k = 6;
    std::mt19937 rng(5);
    std::uniform_int_distribution<int> len(0, 12);
    std::vector<size_t> xl = {0};
    for (int i = 0; i < 150; i++) xl.push_back(xl.back() + (i == 149 ? 3 : len(rng)));
    const std::vector<size_t> ql = {0, 5, 5, 17, 30};
    const int64_t nb = (int64_t)xl.back(), nq = (int64_t)ql.back(), n_docs = (int64_t)xl.size() - 1, n_lists = 4;
    std::normal_distribution<float> g;
    std::vector<float> xb(nb * dim), xq(nq * dim);
    for (auto& v : xb) v = g(rng);
    for (auto& v : xq) v = g(rng);
    auto base = GenDataSet(nb, dim, xb.data());
    base->Set(meta::EMB_LIST_OFFSET, xl.data());
    auto query = GenDataSet(nq, dim, xq.data());
    query->Set(meta::EMB_LIST_OFFSET, ql.data());

    Json cfg = extra;
    cfg[meta::METRIC_TYPE] = el_metric;
    cfg[meta::TOPK] = k;
    cfg[meta::EMB_LIST_STRATEGY] = meta::EMB_LIST_STRATEGY_MUVERA;
    cfg["muvera_num_projections"] = 3;
    cfg["muvera_num_repeats"] = 4;
    cfg["muvera_seed"] = 17;
    auto idx = IndexFactory::Instance().Create<fp32>(type, 0).value();
    REQUIRE(idx.Build(base, cfg) == Status::success);
    REQUIRE(idx.Count() == nb);
    auto r = idx.Search(query, cfg, nullptr);
    REQUIRE(r.has_value());
    REQUIRE(r.value()->GetRows() == n_lists && r.value()->GetDim() == k);
    REQUIRE(r.value()->GetIds()[1 * k] == -1);   // the empty query list is a row of padding
    for (int64_t j = 0; j < k; j++) REQUIRE(r.value()->GetIds()[j] >= 0 && r.value()->GetIds()[j] < n_docs);

    // the C ABI gives the same rows
    kb2_index_t h = static_cast<B200IndexNode*>(idx.Node())->handle();
    std::vector<int64_t> qlv(ql.begin(), ql.end()), ids(n_lists * k);
    std::vector<float> dis(n_lists * k);
    REQUIRE(kb2_index_search_emb_list(h, xq.data(), qlv.data(), n_lists, (int)k, cfg.dump().c_str(), nullptr, 0, ids.data(),
                                      dis.data(), nullptr) == 0);
    REQUIRE(memcmp(ids.data(), r.value()->GetIds(), ids.size() * 8) == 0);
    REQUIRE(memcmp(dis.data(), r.value()->GetDistance(), dis.size() * 4) == 0);
    char meta_json[1024];
    REQUIRE(kb2_index_get_meta(h, meta_json, sizeof(meta_json)) == 0);
    REQUIRE(strstr(meta_json, "\"emb_list_strategy\": \"muvera\"") && strstr(meta_json, "\"muvera_encoded_dim\": 512"));

    // emb_list_rerank false: the base's documents, padded with infinities past n_docs
    Json nr = cfg;
    nr[meta::EMB_LIST_RERANK] = false;
    nr[meta::TOPK] = n_docs + 2;
    auto rn = idx.Search(query, nr, nullptr);
    REQUIRE(rn.has_value());
    const bool l2 = std::string(el_metric) == metric::MAX_SIM_L2;
    for (int64_t l = 0; l < n_lists; l++) {
        const int64_t* row = rn.value()->GetIds() + l * (n_docs + 2);
        const float* drow = rn.value()->GetDistance() + l * (n_docs + 2);
        REQUIRE(row[n_docs] == -1 && row[n_docs + 1] == -1);
        REQUIRE(l2 ? drow[n_docs] == INFINITY : drow[n_docs] == -INFINITY);
    }

    // BinarySet: the "KB2I" container under the type name holds everything
    BinarySet bs;
    REQUIRE(idx.Serialize(bs) == Status::success);
    REQUIRE(bs.Contains(type) && !bs.Contains(meta::EMB_LIST_META));
    auto loaded = IndexFactory::Instance().Create<fp32>(type, 0).value();
    REQUIRE(loaded.Deserialize(bs, cfg) == Status::success);
    auto r2 = loaded.Search(query, cfg, nullptr);
    REQUIRE(r2.has_value() && same_rows(r.value(), r2.value()));
    printf("%s %s ok\n", type, el_metric);
}

int
main() {
    REQUIRE(kb2_device_count() > 0);
    Json hnsw;
    hnsw[indexparam::HNSW_M] = 16;
    hnsw[indexparam::EFCONSTRUCTION] = 64;
    hnsw[indexparam::EF] = 160;
    run("HNSW", metric::MAX_SIM_L2, hnsw);
    run("HNSW", metric::MAX_SIM_IP, hnsw);
    Json ivf;
    ivf[indexparam::NLIST] = 4;
    ivf[indexparam::NPROBE] = 2;
    run("IVF_FLAT", metric::MAX_SIM_IP, ivf);
    run("IVF_FLAT", metric::MAX_SIM_COSINE, ivf);
    printf("muvera ok\n");
    return 0;
}
