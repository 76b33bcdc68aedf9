// tests/cpp/test_emb_list_index.cc — emb-list HNSW / IVF_FLAT through the C++ mirror (compiled and run by
// tests/test_emb_list_index_gpu.py).  Build with EMB_LIST_OFFSET and a MAX_SIM metric, Search with query list offsets
// (the same rows as the C ABI), the dispatch errors of index_node.cc:275-324, and BinarySet round trips: EMB_LIST_META
// in the ELMF_V2 / TOKA layout, and a hand-built legacy [count][offsets] one.  Exit code 0 = pass.  Needs an H100.
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

static bool
same_rows(const DataSetPtr& a, const DataSetPtr& b) {
    const int64_t n = a->GetRows() * a->GetDim();
    if (a->GetRows() != b->GetRows() || a->GetDim() != b->GetDim()) return false;
    return memcmp(a->GetIds(), b->GetIds(), n * 8) == 0 && memcmp(a->GetDistance(), b->GetDistance(), n * 4) == 0;
}

static void
run(const char* type, const char* el_metric, Json extra) {
    const int64_t dim = 32, k = 10;
    std::mt19937 rng(11);
    std::uniform_int_distribution<int> len(0, 30);
    std::vector<size_t> xl = {0};
    for (int i = 0; i < 400; i++) xl.push_back(xl.back() + (i == 399 ? 5 : len(rng)));   // the last document is not empty
    const std::vector<size_t> ql = {0, 7, 7, 40, 52};
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
    cfg[meta::RETRIEVAL_ANN_RATIO] = 2.0;
    auto created = IndexFactory::Instance().Create<fp32>(type, 0);
    REQUIRE(created.has_value());
    auto idx = created.value();
    REQUIRE(idx.Build(base, cfg) == Status::success);
    REQUIRE(idx.Count() == nb);
    auto r = idx.Search(query, cfg, nullptr);
    REQUIRE(r.has_value());
    REQUIRE(r.value()->GetRows() == n_lists && r.value()->GetDim() == k);
    REQUIRE(r.value()->GetIds()[1 * k] == -1);   // the empty query list is a row of padding
    REQUIRE(r.value()->GetIds()[0] >= 0 && r.value()->GetIds()[0] < n_docs);

    // the C ABI gives the same rows
    kb2_index_t h = static_cast<B200IndexNode*>(idx.Node())->handle();
    std::vector<int64_t> qlv(ql.begin(), ql.end()), ids(n_lists * k);
    std::vector<float> dis(n_lists * k);
    REQUIRE(kb2_index_search_emb_list(h, xq.data(), qlv.data(), n_lists, (int)k, cfg.dump().c_str(), nullptr, 0, ids.data(),
                                      dis.data(), nullptr) == 0);
    REQUIRE(memcmp(ids.data(), r.value()->GetIds(), ids.size() * 8) == 0);
    REQUIRE(memcmp(dis.data(), r.value()->GetDistance(), dis.size() * 4) == 0);

    // every document filtered out: padding only
    std::vector<uint8_t> all((n_docs + 7) / 8, 0xff);
    auto rf = idx.Search(query, cfg, BitsetView(all.data(), n_docs));
    REQUIRE(rf.has_value());
    for (int64_t i = 0; i < n_lists * k; i++) REQUIRE(rf.value()->GetIds()[i] == -1);

    // dispatch errors (index_node.cc:275-324)
    auto plain_query = GenDataSet(nq, dim, xq.data());
    REQUIRE(idx.Search(plain_query, cfg, nullptr).error() == Status::emb_list_inner_error);
    Json sub = cfg;
    sub[meta::METRIC_TYPE] = std::string(el_metric) == metric::MAX_SIM_L2 ? metric::L2 : metric::IP;
    REQUIRE(idx.Search(query, sub, nullptr).error() == Status::emb_list_inner_error);
    Json rcfg = cfg;
    rcfg[meta::RADIUS] = 1.0;
    REQUIRE(idx.RangeSearch(query, rcfg, nullptr).error() == Status::emb_list_inner_error);
    REQUIRE(idx.AnnIterator(query, cfg, nullptr).error() == Status::emb_list_inner_error);
    REQUIRE(idx.Search(plain_query, sub, nullptr).error() == Status::emb_list_inner_error);   // plain search on an emb-list index

    // BinarySet: the base payload under the type name and EMB_LIST_META in the ELMF_V2 / TOKA layout
    BinarySet bs;
    REQUIRE(idx.Serialize(bs) == Status::success);
    REQUIRE(bs.Contains(type) && bs.Contains(meta::EMB_LIST_META));
    auto mb = bs.GetByName(meta::EMB_LIST_META);
    const uint8_t* p = mb->data.get();
    int64_t magic;
    size_t type_len, count;
    int32_t toka, version;
    memcpy(&magic, p, 8);
    memcpy(&type_len, p + 8, 8);
    REQUIRE(magic == 0x454C4D465F563200LL && type_len == 8 && memcmp(p + 16, "tokenann", 8) == 0);
    memcpy(&toka, p + 24, 4);
    memcpy(&version, p + 28, 4);
    memcpy(&count, p + 32, 8);
    REQUIRE(toka == 0x544F4B41 && version == 1 && count == xl.size() && mb->size == (int64_t)(40 + 8 * count));
    REQUIRE(memcmp(p + 40, xl.data(), 8 * count) == 0);

    auto loaded = IndexFactory::Instance().Create<fp32>(type, 0).value();
    REQUIRE(loaded.Deserialize(bs, cfg) == Status::success);
    auto r2 = loaded.Search(query, cfg, nullptr);
    REQUIRE(r2.has_value() && same_rows(r.value(), r2.value()));
    REQUIRE(loaded.Deserialize(bs, sub) == Status::invalid_metric_type);   // the emb-list metric comes from cfg

    // a legacy EMB_LIST_META: [size_t count][size_t offsets] alone
    BinarySet legacy;
    auto b = bs.GetByName(type);
    legacy.Append(type, b->data, b->size);
    std::shared_ptr<uint8_t[]> lm(new uint8_t[8 + 8 * count]);
    memcpy(lm.get(), &count, 8);
    memcpy(lm.get() + 8, xl.data(), 8 * count);
    legacy.Append(meta::EMB_LIST_META, lm, (int64_t)(8 + 8 * count));
    auto loaded2 = IndexFactory::Instance().Create<fp32>(type, 0).value();
    REQUIRE(loaded2.Deserialize(legacy, cfg) == Status::success);
    auto r3 = loaded2.Search(query, cfg, nullptr);
    REQUIRE(r3.has_value() && same_rows(r.value(), r3.value()));
    // a truncated one is refused
    legacy.Append(meta::EMB_LIST_META, lm, 12);
    REQUIRE(loaded2.Deserialize(legacy, cfg) == Status::emb_list_inner_error);
    printf("%s %s ok\n", type, el_metric);
}

int
main() {
    REQUIRE(kb2_device_count() > 0);
    Json hnsw;
    hnsw[indexparam::HNSW_M] = 16;
    hnsw[indexparam::EFCONSTRUCTION] = 64;
    hnsw[indexparam::EF] = 32;
    run("HNSW", metric::MAX_SIM_L2, hnsw);
    run("HNSW", metric::MAX_SIM_IP, hnsw);
    Json ivf;
    ivf[indexparam::NLIST] = 16;
    ivf[indexparam::NPROBE] = 4;
    run("IVF_FLAT", metric::MAX_SIM_IP, ivf);
    run("IVF_FLAT", metric::MAX_SIM_L2, ivf);

    // FLAT and IVF_PQ have no emb-lists; binary MAX_SIM metrics are refused
    std::vector<float> x(64 * 32, 1.f);
    std::vector<size_t> lims = {0, 30, 64};
    auto ds = GenDataSet(64, 32, x.data());
    ds->Set(meta::EMB_LIST_OFFSET, lims.data());
    Json c;
    c[meta::METRIC_TYPE] = metric::MAX_SIM_L2;
    REQUIRE(IndexFactory::Instance().Create<fp32>("FLAT", 0).value().Build(ds, c) == Status::invalid_metric_type);
    c[meta::METRIC_TYPE] = metric::MAX_SIM_HAMMING;
    REQUIRE(IndexFactory::Instance().Create<fp32>("HNSW", 0).value().Build(ds, c) == Status::invalid_metric_type);
    printf("ok\n");
    return 0;
}
